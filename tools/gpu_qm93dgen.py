"""Times QM93DGEN's trajectories for QM9-sized synthetic molecules and prints one JSON line with the card name and its
power limit:
  * end_to_end_s: compute_trajectories (host packing, copies, chunked csrc/gen_traj.cu launches, copies back);
  * kernel_s: CUDA events around the dig3d_gen_traj call alone (the launch of one kernel over all molecules);
  * ops_gen_traj_call_s: one ops.gen_traj call until its kernel has finished, including its input checks (one host
    synchronisation), the pointer copy and the allocations.
Where the reference checkout exists (oracle/ref_loader.py), it also times the reference's get() loop on the CPU over
--ref-mols of the molecules; the GPU machines have no reference, so that number comes from a separate run on a host
that has it.

    python tools/gpu_qm93dgen.py [--n-mols 130000] [--reps 3] [--kernel-reps 20] [--ref-mols 2000] [--no-gpu]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def molecules(n_mols, seed=0):
    """QM9-sized molecules: 3 to 29 atoms (mean about 18), grown geometries (as the fixture's), bonds of order 1-3
    between atoms closer than 1.65 A."""
    from oracle.gen_golden_qm93dgen import grown
    rng = np.random.default_rng(seed)
    sizes = np.clip(np.rint(rng.normal(18, 3, n_mols)), 3, 29).astype(int)
    types, pos, con = [], [], []
    for n in sizes:
        p = grown(rng, n)
        d = np.linalg.norm(p[:, None].astype(np.float64) - p[None].astype(np.float64), axis=-1)
        order = np.triu(rng.choice([1, 1, 1, 2, 3], size=(n, n)) * ((d > 0) & (d < 1.65)), 1)
        types.append(torch.from_numpy(rng.integers(0, 5, n).astype(np.int64)))
        pos.append(torch.from_numpy(p))
        con.append(torch.from_numpy((order + order.T).astype(np.int64)))
    return types, pos, con


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-mols", type=int, default=130000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=20)
    ap.add_argument("--ref-mols", type=int, default=2000)
    ap.add_argument("--no-gpu", action="store_true", help="only the reference's CPU loop")
    a = ap.parse_args()
    t0 = time.perf_counter()
    types, pos, con = molecules(a.n_mols)
    result = {"n_mols": a.n_mols, "rows": int(sum(len(t) * (len(t) - 1) // 2 for t in types)),
              "make_molecules_s": round(time.perf_counter() - t0, 1)}
    if not a.no_gpu:
        from dig_b200 import _lib, ops
        from dig_b200.ggraph3D.dataset.ggraph3D_dataset import compute_trajectories
        compute_trajectories(types[:1000], pos[:1000], con[:1000])                       # warm-up
        e2e = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            compute_trajectories(types, pos, con)
            torch.cuda.synchronize()
            e2e.append(time.perf_counter() - t0)
        n_atoms = torch.tensor([len(t) for t in types])
        dev = [torch.cat(types).cuda(), torch.cat(pos).cuda(), torch.cat([c.reshape(-1) for c in con]).cuda()]
        ops.gen_traj(*dev, n_atoms)
        call, launch = [], []
        for _ in range(a.kernel_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _lib.start_timing()            # CUDA events around the dig3d_gen_traj call alone: the launch, no host checks
            ops.gen_traj(*dev, n_atoms)
            launch += [ms / 1e3 for ms in _lib.stop_timing()["dig3d_gen_traj"]]
            call.append(time.perf_counter() - t0)
        stats = lambda v: {"min": min(v), "median": float(np.median(v)), "max": max(v), "n": len(v)}
        result.update(gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), end_to_end_s=sorted(e2e),
                      kernel_s=stats(launch), ops_gen_traj_call_s=stats(call))
    from oracle.ref_loader import reference_available
    if reference_available():
        from oracle.gen_golden_qm93dgen import load_reference_dataset
        ref = load_reference_dataset()
        ds = ref.QM93DGEN.__new__(ref.QM93DGEN)
        k = min(a.ref_mols, a.n_mols)
        ds.atom_type_list, ds.position_list, ds.con_mat_list = types[:k], pos[:k], con[:k]
        import warnings
        warnings.simplefilter("ignore")
        t0 = time.perf_counter()
        for i in range(k):
            ds.get(i)
        per = (time.perf_counter() - t0) / k
        result.update(reference_cpu_get_s_per_mol=per, reference_cpu_threads=torch.get_num_threads(),
                      reference_cpu_projected_s=per * a.n_mols)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
