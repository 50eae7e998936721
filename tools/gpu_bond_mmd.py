"""Times the bond-length MMD (dig_b200.ggraph3D.utils.compute_mmd, csrc/mmd.cu) at the shipped QM9 target sizes of the
six bond types RandGenEvaluator.eval_bond_mmd scores, with seeded synthetic lengths, and the restated reference formula
(oracle/restated_mmd.py: the reference's batched ATen op sequence, fp64 on the same GPU) at the (1, 8, 1) size for
agreement and speed-up.  Prints one JSON line with the card's name and power limit.

    python tools/gpu_bond_mmd.py [--reps 3] [--n-mols 1000]

Rates: `pair_evals` counts the pairs the kernel evaluates (one triangle of S x S and T x T, plus S x T);
`fp64_bound_pairs_per_s` is the instruction-rate bound of the pair loop: the H100 SXM data sheet's 34 TFLOP/s FP64
(non-tensor, an FMA counted as two operations, so 17e12 FP64 instructions/s) over FP64_INSTR_PER_PAIR.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (z1, z2, order) -> number, mean and standard deviation (A) of the lengths in the shipped QM9 table
# examples/ggraph3D/G_SphereNet/target_bond_lengths.dict
BONDS = {(1, 8, 1): (46806, 0.9649, 0.0043), (1, 7, 1): (54283, 1.0119, 0.0051), (6, 7, 1): (145811, 1.4402, 0.056),
         (6, 8, 1): (168672, 1.4144, 0.0312), (6, 6, 1): (609909, 1.5212, 0.0351), (1, 6, 1): (986987, 1.093, 0.0068)}
CH_PER_MOL = 9.0                  # ~9 C-H bonds per QM9-like molecule; the other types in proportion to the target table
# FP64 instructions per pair of the default pair loop (kernel_mul = 2, kernel_num = 5), counted in the SASS of the
# unmasked tile loop of pairs_kernel<true, 5> (cuobjdump -sass): 120 DFMA + 56 DADD + 48 DMUL per 8 pairs
FP64_INSTR_PER_PAIR = 28
FP64_INSTR_PER_S = 34e12 / 2


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def lengths(n, mean, std, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    return (mean + std * torch.randn(n, generator=g, dtype=torch.float64)).to(dtype)


def timed(fn, reps):
    """-> (result of the last call, [ms per call]) by CUDA events; every call ends in its own host read-back."""
    times, out = [], None
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return out, times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n-mols", type=int, default=1000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_bond_mmd.py needs a CUDA device")
    from dig_b200.ggraph3D.utils import compute_mmd
    from oracle import restated_mmd
    dev = torch.device("cuda:0")
    ch_total = BONDS[(1, 6, 1)][0]
    data = {}
    for i, (key, (nt, mean, std)) in enumerate(BONDS.items()):
        ns = max(1, round(CH_PER_MOL * a.n_mols * nt / ch_total))
        src = lengths(ns, mean + 0.01, std * 2, 100 + i, torch.float32).to(dev)    # generated lengths come as float32
        tgt = lengths(nt, mean, std, 200 + i, torch.float64).to(dev)
        data[key] = (src, tgt)
    compute_mmd(*data[(1, 8, 1)])                      # warm-up: module load, allocator
    torch.cuda.synchronize()
    rows, total_ms = [], 0.0
    for key, (src, tgt) in data.items():
        ns, nt = src.numel(), tgt.numel()
        mmd, ms = timed(lambda: compute_mmd(src, tgt), a.reps)
        evals = ns * (ns - 1) // 2 + nt * (nt - 1) // 2 + ns * nt
        best = min(ms)
        total_ms += best
        rows.append(dict(bond=list(key), n_source=ns, n_target=nt, mmd=mmd, ms=[round(t, 3) for t in ms],
                         pair_evals=evals, pair_evals_per_s=evals / (best * 1e-3),
                         reference_pairs=ns * ns + nt * nt + ns * nt))
    bound = FP64_INSTR_PER_S / FP64_INSTR_PER_PAIR
    all_evals = sum(r["pair_evals"] for r in rows)
    src, tgt = data[(1, 8, 1)]
    src64 = src.double()
    restated_mmd.compute_mmd(src64[:100], tgt[:2000])  # warm-up of the ATen kernels
    ref, ref_ms = timed(lambda: restated_mmd.compute_mmd(src64, tgt), max(1, a.reps - 1))
    ours = rows[0]
    out = dict(tool="gpu_bond_mmd", gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), n_mols=a.n_mols,
               per_type=rows, total_ms=round(total_ms, 3), total_pair_evals=all_evals,
               pair_evals_per_s=all_evals / (total_ms * 1e-3), fp64_instr_per_pair=FP64_INSTR_PER_PAIR,
               fp64_bound_pairs_per_s=bound, share_of_fp64_bound=all_evals / (total_ms * 1e-3) / bound,
               restated_reference_1_8_1=dict(ms=[round(t, 3) for t in ref_ms], mmd=ref,
                                             abs_diff=abs(ref - ours["mmd"]), speedup=min(ref_ms) / min(ours["ms"])))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
