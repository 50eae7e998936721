"""Radius graph and triplet geometry at high in-degree: `radius_graph(max_num_neighbors=D)` followed by
`xyz_to_dat(use_torsion=True / False)` on one graph of a few thousand atoms whose in-degree the cap holds at D = 64 /
128 / 256, against the restated reference ops (oracle/restated.py: torch_cluster's radius_graph, xyz_to_dat) run by
ATen on the same GPU.  The restated ops materialise every triplet (about N * D^2) and, for the torsion, every
(triplet, candidate) pair (about N * D^3): they run only where that count fits `--ref-candidates`, and are reported as
skipped elsewhere.  Prints one JSON line with the card's
name, power limit and maximum SM clock read in the same process.  Test infrastructure; needs a GPU.

    python tools/gpu_dense_graph.py [--atoms 2048,256] [--degrees 64,128,256] [--reps 5] [--warmup 2]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import restated  # noqa: E402
from dig_b200.threedgraph.utils import radius_graph, xyz_to_dat  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")] if q.count(",") == 2 else (q, None, None)
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power, "max_sm_clock": clock}


def time_ms(fn, reps, warmup):
    """Per-call CUDA-event times of `reps` calls after `warmup` untimed ones: median / min / max in ms."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    per = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        per.append(a.elapsed_time(b))
    return {"median_ms": round(statistics.median(per), 3), "min_ms": round(min(per), 3), "max_ms": round(max(per), 3)}


def atoms(n, degree, cutoff, seed):
    """n atoms uniform in a cube sized so that an interior atom has about 2 * degree atoms within `cutoff`: the cap
    max_num_neighbors = degree then binds for nearly every atom."""
    side = (n * 4.0 / 3.0 * math.pi * cutoff ** 3 / (2.0 * degree)) ** (1.0 / 3.0)
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, 3, generator=g) * side).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--atoms", default="2048,256")
    ap.add_argument("--degrees", default="64,128,256")
    ap.add_argument("--cutoff", type=float, default=5.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ref-candidates", type=float, default=1e8,
                    help="largest triplet count (no torsion) or (triplet, candidate) count (torsion) for which the "
                         "restated xyz_to_dat is run")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_dense_graph.py needs a CUDA device")
    out = {"tool": "gpu_dense_graph", **card(), "cutoff": args.cutoff, "runs": []}
    for n, d in [(int(a), int(x)) for a in args.atoms.split(",") for x in args.degrees.split(",")]:
        pos = atoms(n, d, args.cutoff, seed=d)
        batch = torch.zeros(n, dtype=torch.long, device=pos.device)
        ei = radius_graph(pos, args.cutoff, batch, max_num_neighbors=d)
        deg = torch.bincount(ei[1], minlength=n).double()
        got = xyz_to_dat(pos, ei, n, use_torsion=True)
        t = got[1].numel()
        per_edge = torch.bincount(got[-1], minlength=ei.size(1)).double()
        candidates = int((per_edge * per_edge).sum())        # an edge's triplets are each other's torsion candidates
        run = {"atoms": n, "degree": d, "edges": int(ei.size(1)), "in_degree_mean": round(float(deg.mean()), 2),
               "in_degree_max": int(deg.max()), "triplets": t, "torsion_candidates": candidates}
        run["radius_graph"] = time_ms(lambda: radius_graph(pos, args.cutoff, batch, max_num_neighbors=d),
                                      args.reps, args.warmup)
        for tors in (False, True):
            key = "torsion" if tors else "no_torsion"
            run[f"radius_graph+xyz_to_dat_{key}"] = time_ms(
                lambda: xyz_to_dat(pos, radius_graph(pos, args.cutoff, batch, max_num_neighbors=d), n, use_torsion=tors),
                args.reps, args.warmup)
        ref_ei = restated.radius_graph(pos, args.cutoff, batch, max_num_neighbors=d)
        run["graph_equal_to_restated"] = bool(torch.equal(ref_ei, ei))
        run["restated_radius_graph"] = time_ms(lambda: restated.radius_graph(pos, args.cutoff, batch,
                                                                             max_num_neighbors=d),
                                               args.reps, args.warmup)
        for tors in (False, True):
            key = "torsion" if tors else "no_torsion"
            size = candidates if tors else t
            if size > args.ref_candidates:
                run[f"restated_{key}"] = f"skipped: {size} {'candidates' if tors else 'triplets'} > --ref-candidates"
                continue
            want = restated.xyz_to_dat(pos, ref_ei, n, use_torsion=tors)
            mine = xyz_to_dat(pos, ei, n, use_torsion=tors)
            run[f"xyz_to_dat_{key}_equal_to_restated"] = all(torch.equal(a, b) for a, b in zip(mine, want))
            del want, mine
            run[f"restated_{key}"] = time_ms(
                lambda: restated.xyz_to_dat(pos, restated.radius_graph(pos, args.cutoff, batch, max_num_neighbors=d),
                                            n, use_torsion=tors), args.reps, args.warmup)
            torch.cuda.empty_cache()
        del got
        torch.cuda.empty_cache()
        out["runs"].append(run)
        print(json.dumps(run), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
