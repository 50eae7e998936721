"""Forces and force training at a generic triplet-branch width against the default SphereNet, on 32 MD17-shaped
(aspirin) molecules, in one process:

  * median ms of a forces forward + backward (E, then -dE/dpos) and of one force-training step (L1(E, y) + p L1(F, f)
    with create_graph=True, backward, Adam), CUDA events around each call after warm-up, at the default SphereNet and at
    int_emb_size=32, basis_emb_size_angle=4, basis_emb_size_torsion=6;
  * the kernel time of dig3d_triplet_basis_bwd from torch.profiler (a separate profiled pass) and the bytes it moves
    over that time against the H100 SXM data-sheet 3.35 TB/s;
  * the card's name and power limit, read in the same run.

    python tools/gpu_generic_forces.py [--steps 20] [--warmup 3] [--mols 32]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BYTES_PER_S = 3.35e12
GENERIC = dict(int_emb_size=32, basis_emb_size_angle=4, basis_emb_size_torsion=6)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or "unknown"


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2], times[0], times[-1]


def bwd_bytes(g, ns, nr, torsion):
    """Bytes dig3d_triplet_basis_bwd has to move: the upstream gradients, geometry and the k->j edges' bases in, the
    three gradients out, and the graph indices it walks (dst, row_ptr, out_ptr, out_list, pos_in, trip_ptr)."""
    T, E, N = g.n_triplets, g.n_edges, g.n_nodes
    nb = ns * nr
    f = 4 * (T * nb + (T * ns * ns * nr if torsion else 0) + T * (2 if torsion else 1) + 2 * E * nb)
    f += 4 * (T * (2 if torsion else 1) + E)
    i = 4 * (E + 2 * (N + 1) + 3 * E)
    return f + i


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mols", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from dig_b200 import ops
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph.method import SphereNet
    print("card (name, power limit):", card())
    dev = torch.device("cuda:0")
    data = synthetic_batch(args.mols, "md17-aspirin", seed=5).to(dev)
    gen = torch.Generator().manual_seed(1)
    y = torch.randn(args.mols, 1, generator=gen).to(dev)
    f_t = torch.randn(data.pos.size(0), 3, generator=gen).to(dev)
    print(f"batch: {args.mols} molecules, {data.pos.size(0)} atoms")

    class B:
        pass

    def batch_with(pos):
        b = B()
        b.z, b.pos, b.batch, b.num_graphs = data.z, pos, data.batch, args.mols
        return b

    for label, kw in (("default SphereNet", {}), ("generic " + ", ".join(f"{k}={v}" for k, v in GENERIC.items()), GENERIC)):
        torch.manual_seed(0)
        model = SphereNet(energy_and_force=True, cutoff=5.0, **kw).to(dev)
        opt = torch.optim.Adam(model.parameters(), lr=1e-4)

        def forces():
            b = batch_with(data.pos.clone())
            out = model(b)
            return -torch.autograd.grad(out, b.pos, grad_outputs=torch.ones_like(out))[0]

        def train_step():
            opt.zero_grad()
            b = batch_with(data.pos.clone())
            out = model(b)
            force = -torch.autograd.grad(out, b.pos, grad_outputs=torch.ones_like(out), create_graph=True,
                                         retain_graph=True)[0]
            loss = torch.nn.functional.l1_loss(out, y) + 100.0 * torch.nn.functional.l1_loss(force, f_t)
            loss.backward()
            opt.step()

        model.eval()
        med, lo, hi = timed(forces, args.steps, args.warmup)
        print(f"{label}: forces forward + backward: median {med:.2f} ms (min {lo:.2f}, max {hi:.2f}, {args.steps} calls)")
        model.train()
        med, lo, hi = timed(train_step, args.steps, args.warmup)
        print(f"{label}: force-training step: median {med:.2f} ms (min {lo:.2f}, max {hi:.2f}, {args.steps} steps)")

        if kw:
            from torch.profiler import ProfilerActivity, profile
            model.eval()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    forces()
                torch.cuda.synchronize()
            evs = [e for e in prof.events() if "triplet_basis_bwd_kernel" in e.name]
            if not evs:
                raise SystemExit("no dig3d_triplet_basis_bwd launch in the profile")
            us = sum(e.device_time for e in evs) / len(evs)
            g = ops.build_graph(data.pos, data.batch, 5.0, num_graphs=args.mols)
            nbytes = bwd_bytes(g, model.num_spherical, model.num_radial, True)
            print(f"dig3d_triplet_basis_bwd: {us:.1f} us per launch ({len(evs)} launches), E={g.n_edges} "
                  f"T={g.n_triplets}, {nbytes / 1e6:.1f} MB -> {nbytes / (us * 1e-6) / 1e12:.3f} TB/s = "
                  f"{100 * nbytes / (us * 1e-6) / HBM_BYTES_PER_S:.1f}% of 3.35 TB/s")


if __name__ == "__main__":
    main()
