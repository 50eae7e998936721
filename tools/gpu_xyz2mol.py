"""Times xyz2mol on the GPU (csrc/xyz2mol.cu) and RandGenEvaluator end to end, and prints one JSON line with the card
name and its power limit, read in the same run.

  * kernel: ops.xyz2mol by CUDA events at 10,000 and 100,000 molecules, for G-SphereNet output (fixture weights,
    num_max_node=35, one launch per atom count) and for grown geometries (bonded, 20 atoms);
  * end to end: RandGenEvaluator.eval_validity + eval_bond_mmd on 10,000 generated molecules (wall clock, synchronised)
    against the restated reference (oracle/restated_validity.py, numpy + networkx) on this host's CPU, on a subsample.

    python tools/gpu_xyz2mol.py [--reps 5] [--cpu-sample 1000]
"""
import argparse
import contextlib
import io
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def power_limit():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def kernel_ms(groups, reps):
    """ms per pass over the groups [(z, pos) on the device], CUDA events around all launches of one pass."""
    from dig_b200 import ops
    for z, p in groups:
        ops.xyz2mol(z, p)
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for z, p in groups:
            ops.xyz2mol(z, p)
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return sorted(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-sample", type=int, default=1000)
    a = ap.parse_args()
    from dig_b200.ggraph3D.evaluation import RandGenEvaluator
    from oracle import gen_golden_validity as gv
    from oracle import restated_validity as rv
    from test_gpu_xyz2mol import _generated
    if not torch.cuda.is_available():
        raise SystemExit("gpu_xyz2mol needs a CUDA device")
    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}
    gen = _generated(100_000)
    result["generated_sizes"] = {int(n): len(v["_atomic_numbers"]) for n, v in sorted(gen.items())}
    grown = gv.grown(np.random.default_rng(0), 10_000, (20, 21), bonded=True)
    for count in (10_000, 100_000):
        groups, left = [], count
        for n in gen:
            k = min(left, len(gen[n]["_atomic_numbers"]))
            if k:
                groups.append((torch.from_numpy(gen[n]["_atomic_numbers"][:k]).cuda(),
                               torch.from_numpy(gen[n]["_positions"][:k]).cuda()))
            left -= k
        result[f"kernel_ms_gsphere_{count}"] = kernel_ms(groups, a.reps)
        z = torch.from_numpy(np.stack([m[0] for m in grown])).repeat(count // 10_000, 1).cuda()
        p = torch.from_numpy(np.stack([m[1] for m in grown])).repeat(count // 10_000, 1, 1).cuda()
        result[f"kernel_ms_grown20_{count}"] = kernel_ms([(z, p)], a.reps)
    mols10k = {}
    left = 10_000
    for n in gen:
        k = min(left, len(gen[n]["_atomic_numbers"]))
        if k:
            mols10k[n] = {key: gen[n][key][:k] for key in ("_atomic_numbers", "_positions")}
        left -= k
    f = np.load(os.path.join(ROOT, "tests", "golden", "xyz2mol.npz"))
    target = {bt: list(f["target_{}_{}_{}".format(*bt)]) for bt in gv.BOND_TYPES}
    e2e = []
    for _ in range(a.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            ratio = RandGenEvaluator.eval_validity(mols10k)
            mmd = RandGenEvaluator.eval_bond_mmd({"mol_dicts": mols10k, "target_bond_dists": target})
        torch.cuda.synchronize()
        e2e.append(time.perf_counter() - t0)
    result["e2e_s_10000"] = sorted(e2e)
    result["valid_ratio"] = ratio["valid_ratio"]
    result["mmd_types"] = len(mmd)
    sample = [(z, p) for n in mols10k for z, p in zip(mols10k[n]["_atomic_numbers"], mols10k[n]["_positions"])]
    sample = sample[:a.cpu_sample]
    t0 = time.perf_counter()
    for z, p in sample:
        rv.xyz2mol(z, p)
    per_mol = (time.perf_counter() - t0) / len(sample)
    result["cpu_restated_ms_per_molecule"] = per_mol * 1e3
    result["cpu_restated_s_10000_two_calls"] = 2 * per_mol * 10_000       # eval_validity and eval_bond_mmd each call it
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
