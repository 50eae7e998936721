"""Times one G-SphereNet training step (SphGen.forward, the reference loss, backward, Adam) at the config_dict.json
model size on a batch of 64 synthetic QM9-sized molecules, against the restated reference op sequence
(oracle/restated_gsphere_train.py) under ATen autograd in fp32 on the same GPU.  Prints the card name and power limit
of the run.  CUDA events around each step, after warm-up; the batch and noise are fixed.

    python tools/gpu_gsphere_train.py [--steps 20] [--warmup 3] [--mols 64]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or "unknown"


def timed(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2], times[0], times[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mols", type=int, default=64)
    args = ap.parse_args()
    from oracle import restated_gsphere_train as rt
    from test_gpu_gsphere_train import _model, _synthetic_batch, _to
    from test_gsphere_train_cpu import train_sd
    
    print("card (name, power limit):", card())
    batch = _to(_synthetic_batch(args.mols, seed=11))
    n_steps = batch["new_atom_type"].numel()
    print(f"batch: {args.mols} molecules, {n_steps} steps, {batch['atom_type'].numel()} trajectory atoms")
    noise = torch.rand(n_steps, 5, device="cuda")

    model = _model()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)

    def ours():
        opt.zero_grad()
        loss = rt.loss(model(batch, deq_noise=noise), batch["cannot_focus"])
        loss.backward()
        opt.step()

    sd = rt.leaf_state_dict({k: v.cuda() for k, v in train_sd().items()})
    ref_opt = torch.optim.Adam([v for v in sd.values() if v.requires_grad], lr=1e-3)

    def reference():
        ref_opt.zero_grad()
        loss = rt.loss(rt.sphgen_forward(sd, batch, noise), batch["cannot_focus"])
        loss.backward()
        ref_opt.step()

    for name, fn in (("SphGen.forward + backward + Adam (sm_90a kernels)", ours),
                     ("restated reference, ATen autograd fp32", reference)):
        med, lo, hi = timed(fn, args.steps, args.warmup)
        print(f"{name}: median {med:.2f} ms per step (min {lo:.2f}, max {hi:.2f}, {args.steps} steps)")


if __name__ == "__main__":
    main()
