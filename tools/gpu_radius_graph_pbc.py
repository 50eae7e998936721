"""Periodic radius graph at OC20-IS2RE shape (64 structures of 73 atoms, cutoff 6 A, cap 50): the CUDA kernels
(dig3d_radius_graph_pbc_count / _fill) against the torch restatement of ocpmodels' radius_graph_pbc (oracle/ocp_pbc.py)
on the same GPU, and the ComENet-OCP forward with otf_graph True and False.  Prints one JSON line with the card's name,
power limit and maximum SM clock read in the same process.  Test infrastructure; needs a GPU.

    python tools/gpu_radius_graph_pbc.py [--windows 7] [--iters 20] [--warmup 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import formula_state_dict  # noqa: E402
from oracle import ocp_pbc  # noqa: E402
from dig_b200 import ops  # noqa: E402
from dig_b200.data import Batch, synthetic_pbc_batch  # noqa: E402
from dig_b200.threedgraph.method.comenet_ocp import ComENet  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")] if q.count(",") == 2 else (q, None, None)
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power, "max_sm_clock": clock}


def time_ms(fn, windows, iters, warmup):
    """Median over `windows` of the mean time per call of `iters` back-to-back calls (CUDA events)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    per = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        per.append(a.elapsed_time(b) / iters)
    return {"median_ms": round(statistics.median(per), 4), "min_ms": round(min(per), 4), "max_ms": round(max(per), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    out = card()
    src = synthetic_pbc_batch(64, natoms=73, seed=0)
    inputs = ("atomic_numbers", "pos", "tags", "cell", "natoms", "batch")
    b = Batch(**{k: getattr(src, k) for k in inputs}, num_graphs=src.num_graphs).to(dev)
    kern = ops.radius_graph_pbc(b.pos, b.cell, b.natoms, 6.0, 50)
    ref = ocp_pbc.radius_graph_pbc(b, 6.0, 50)
    reps = ocp_pbc.image_range(b.cell, 6.0).max(dim=0).values.tolist()
    n = b.pos.size(0)
    cand = int((b.natoms ** 2).sum()) * int((2 * torch.tensor(reps) + 1).prod())
    out.update({"shape": "64 x 73 atoms, cutoff 6, cap 50", "image_range": reps, "candidates": cand,
                "edges": kern[0].size(1), "bit_equal_to_restatement": all(torch.equal(x, y) for x, y in zip(kern, ref))})
    out["graph_kernel"] = time_ms(lambda: ops.radius_graph_pbc(b.pos, b.cell, b.natoms, 6.0, 50), args.windows,
                                  args.iters, args.warmup)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out["graph_torch_restated"] = time_ms(lambda: ocp_pbc.radius_graph_pbc(b, 6.0, 50), args.windows,
                                          max(1, args.iters // 4), 2)
    out["graph_torch_restated_peak_mb"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
    out["graph_speedup"] = round(out["graph_torch_restated"]["median_ms"] / out["graph_kernel"]["median_ms"], 1)

    sd = None
    for otf in (True, False):
        model = ComENet(0, 0, hidden_channels=256, num_blocks=4, cutoff=6.0, num_radial=3, num_spherical=2,
                        otf_graph=otf)
        if sd is None:
            sd = formula_state_dict(model.state_dict(), seed=21)
            sd["lin_out.weight"] = sd["lin_out.weight"] + 0.05
        model.load_state_dict(sd)
        model = model.to(dev).eval()
        data = Batch(**vars(b))
        if not otf:
            data.edge_index, data.cell_offsets, data.neighbors = kern
        with torch.no_grad():
            out[f"comenet_ocp_forward_otf_{otf}"] = time_ms(lambda: model(data), args.windows, args.iters // 2,
                                                            args.warmup)
    out["atoms"] = n
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
