"""ComENet forces and force training on the GPU, in one process:

  * median ms of a forces forward + backward (E, then -dE/dpos) and of one force-training step (L1(E, y) + p L1(F, f)
    with create_graph=True, backward, Adam), CUDA events around each call after warm-up, default ComENet widths, on 32
    MD17-shaped (aspirin) molecules at cutoff 5 and on one batch of 16 OC20-shaped structures at cutoff 6;
  * the time of each new entry point from CUDA events around its call (dig_b200._lib timing: dig3d_comenet_features_bwd
    is its three passes), with the compulsory bytes it moves (every input read once, every output and intermediate
    written once, intermediates read back once) and the achieved share of the H100 SXM data-sheet 3.35 TB/s;
  * how far apart two evaluations of plain torch.autograd over oracle/restated.py land on this GPU (the noise of the
    aliased cross products, csrc/comenet.cu), next to the same for the kernels;
  * the card's name and power limit, read in the same run.

    python tools/gpu_comenet_forces.py [--steps 20] [--warmup 3]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BYTES_PER_S = 3.35e12
ENTRY_POINTS = ("dig3d_comenet_features_bwd", "dig3d_comenet_features_tangent", "dig3d_graphnorm_tangent",
                "dig3d_graphnorm_tangent_bwd")


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


def entry_bytes(name, n, e, n_graphs, width=256):
    """Compulsory traffic of one call (see the module docstring)."""
    if name == "dig3d_comenet_features_bwd":
        # pos, dist, src / dst / out_list, row_ptr / out_ptr, refs, df1 + df2 in; work (15 E) + dvec (3 E) out and back;
        # dpos out
        return 12 * n + 4 * e + 12 * e + 8 * (n + 1) + 16 * n + 72 * e + 2 * 72 * e + 12 * n
    if name == "dig3d_comenet_features_tangent":
        return 12 * n + 12 * n + 4 * e + 8 * e + 16 * n + 72 * e            # pos, cvec, dist, src / dst, refs, f1d + f2d
    if name == "dig3d_graphnorm_tangent":
        return 3 * 4 * n * width + 4 * n_graphs * width * 2                 # h, h_dot in; y_dot out; shift / std
    return 5 * 4 * n * width + 4 * n_graphs * width * 2                     # h, h_dot, dy_dot in; dh, dh_dot out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from dig_b200 import _lib, ops
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph.method import ComENet
    from oracle import restated
    from oracle.weights import formula_state_dict
    print("card (name, power limit):", card())
    dev = torch.device("cuda:0")

    class B:
        pass

    for label, nmol, shape, cutoff in (("32 aspirin-shaped molecules", 32, "md17-aspirin", 5.0),
                                       ("16 OC20-shaped structures", 16, "oc20-is2re", 6.0)):
        data = synthetic_batch(nmol, shape, seed=5).to(dev)
        gen = torch.Generator().manual_seed(1)
        y = torch.randn(nmol, 1, generator=gen).to(dev)
        f_t = torch.randn(data.pos.size(0), 3, generator=gen).to(dev)
        g = ops.build_graph(data.pos, data.batch, cutoff, num_graphs=nmol)
        print(f"{label}: {data.pos.size(0)} atoms, {g.n_edges} edges, cutoff {cutoff}")
        torch.manual_seed(0)
        model = ComENet(energy_and_force=True, cutoff=cutoff)
        sd = formula_state_dict(model.state_dict(), seed=4)
        model.load_state_dict(sd)
        model = model.to(dev)
        opt = torch.optim.Adam(model.parameters(), lr=1e-4)

        def batch_with(pos):
            b = B()
            b.z, b.pos, b.batch, b.num_graphs = data.z, pos, data.batch, nmol
            return b

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
        print(f"  forces forward + backward: median {med:.2f} ms (min {lo:.2f}, max {hi:.2f}, {args.steps} calls)")
        f0, f1 = forces(), forces()
        sd_dev = {k: v.to(dev) for k, v in sd.items()}
        ref = []
        for _ in range(2):
            p = data.pos.clone().requires_grad_(True)
            u = restated.comenet_forward(sd_dev, data.z, p, data.batch, cutoff=cutoff)
            ref.append(torch.autograd.grad(u.sum(), p)[0])
        scale = float(f0.abs().max())
        print(f"  kernels, two runs: max |dF| / max |F| = {float((f0 - f1).abs().max()) / scale:.2e}; plain autograd "
              f"over oracle/restated.py, two runs: {float((ref[0] - ref[1]).abs().max()) / scale:.2e}")
        model.train()
        med, lo, hi = timed(train_step, args.steps, args.warmup)
        print(f"  force-training step: median {med:.2f} ms (min {lo:.2f}, max {hi:.2f}, {args.steps} steps)")
        _lib.start_timing()
        for _ in range(args.steps):
            train_step()
        times = _lib.stop_timing()
        for name in ENTRY_POINTS:
            ts = sorted(times.get(name, []))
            if not ts:
                raise SystemExit(f"no {name} call in a force-training step")
            ms = ts[len(ts) // 2]
            nbytes = entry_bytes(name, g.n_nodes, g.n_edges, nmol)
            print(f"  {name}: median {1e3 * ms:.1f} us per call ({len(ts)} calls), {nbytes / 1e6:.2f} MB -> "
                  f"{nbytes / (ms * 1e-3) / 1e12:.3f} TB/s = {100 * nbytes / (ms * 1e-3) / HBM_BYTES_PER_S:.1f}% of "
                  f"3.35 TB/s")


if __name__ == "__main__":
    main()
