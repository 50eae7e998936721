"""ComENet-OCP forces, cell gradients and force training on the GPU, in one process:

  * median ms of the energy-only forward, of a forces + cell-gradient forward + backward (E, then dE/dpos and dE/dcell
    from pos / cell leaves) and of one force-training step (L1(E, y) + p L1(F, f) with create_graph=True, backward, Adam),
    CUDA events around each call after warm-up, on one OC20-sized batch (synthetic_pbc_batch: 24 slabs of 70 atoms,
    cutoff 6, 50-neighbour cap) with the shipped widths (ocp/comenet.yml: hidden 256, 4 blocks, 3 output layers);
  * the time of each new entry point from CUDA events around its call (dig_b200._lib timing), with the compulsory bytes
    it moves (every input read once, every output and intermediate written once, intermediates read back once) and the
    achieved share of the H100 SXM data-sheet 3.35 TB/s;
  * the card's name and power limit, read in the same run.

    python tools/gpu_comenet_ocp_forces.py [--steps 20] [--warmup 3] [--structures 24] [--atoms 70]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BYTES_PER_S = 3.35e12
ENTRY_POINTS = ("dig3d_comenet_features_bwd_vec", "dig3d_pbc_cell_bwd", "dig3d_comenet_features_tangent_vec")


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


def entry_bytes(name, n, e, n_graphs):
    """Compulsory traffic of one call (see the module docstring)."""
    if name == "dig3d_comenet_features_bwd_vec":
        # vec, dist, src / dst / out_list, row_ptr / out_ptr, refs, df1 + df2 in; work (15 E) + dvec (3 E) out and back;
        # dpos out
        return 12 * e + 4 * e + 12 * e + 8 * (n + 1) + 16 * n + 72 * e + 2 * 72 * e + 12 * n
    if name == "dig3d_comenet_features_tangent_vec":
        return 12 * e + 4 * e + 8 * e + 16 * n + 12 * n + 72 * e           # vec, dist, src / dst, refs, cvec, f1d + f2d
    return 12 * e + 12 * e + 4 * (n + 1) + 4 * (n_graphs + 1) + 36 * n_graphs   # dvec, offsets, ptrs in; dcell out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--structures", type=int, default=24)
    ap.add_argument("--atoms", type=int, default=70)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from dig_b200 import _lib
    from dig_b200.data import synthetic_pbc_batch
    from dig_b200.threedgraph.method.comenet_ocp import ComENet
    from oracle.weights import formula_state_dict
    print("card (name, power limit):", card())
    dev = torch.device("cuda:0")
    nb = args.structures
    data = synthetic_pbc_batch(nb, natoms=args.atoms, seed=5).to(dev)
    n, e = data.pos.size(0), data.edge_index.size(1)
    print(f"{nb} OC20-shaped structures: {n} atoms, {e} edges, cutoff 6, cap 50")
    torch.manual_seed(0)
    model = ComENet(0, 0, hidden_channels=256, num_blocks=4, cutoff=6.0, num_radial=3, num_spherical=2,
                    num_output_layers=3)
    sd = formula_state_dict(model.state_dict(), seed=21)
    sd["lin_out.weight"] = sd["lin_out.weight"] + 0.05
    model.load_state_dict(sd)
    model = model.to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=1e-4)
    gen = torch.Generator().manual_seed(1)
    y = torch.randn(nb, 1, generator=gen).to(dev)
    f_t = torch.randn(n, 3, generator=gen).to(dev)
    pos0, cell0 = data.pos.clone(), data.cell.clone()

    def energy():
        with torch.no_grad():
            return model(data)

    def forces_and_cell():
        data.pos, data.cell = pos0.clone().requires_grad_(True), cell0.clone().requires_grad_(True)
        out = model(data)
        return torch.autograd.grad(out, [data.pos, data.cell], grad_outputs=torch.ones_like(out))

    def train_step():
        opt.zero_grad()
        data.pos, data.cell = pos0.clone().requires_grad_(True), cell0
        out = model(data)
        force = -torch.autograd.grad(out, data.pos, grad_outputs=torch.ones_like(out), create_graph=True,
                                     retain_graph=True)[0]
        loss = torch.nn.functional.l1_loss(out, y) + 100.0 * torch.nn.functional.l1_loss(force, f_t)
        loss.backward()
        opt.step()

    model.eval()
    for label, fn in (("energy-only forward", energy), ("forces + cell gradient forward + backward", forces_and_cell)):
        med, lo, hi = timed(fn, args.steps, args.warmup)
        print(f"  {label}: median {med:.2f} ms (min {lo:.2f}, max {hi:.2f}, {args.steps} calls)")
    (d0, c0), (d1, c1) = forces_and_cell(), forces_and_cell()
    print(f"  two runs: max |d dpos| / max |dpos| = {float((d0 - d1).abs().max() / d0.abs().max()):.2e}, "
          f"max |d dcell| / max |dcell| = {float((c0 - c1).abs().max() / c0.abs().max()):.2e}")
    _lib.start_timing()
    for _ in range(args.steps):
        forces_and_cell()
    times = _lib.stop_timing()
    model.train()
    med, lo, hi = timed(train_step, args.steps, args.warmup)
    print(f"  force-training step: median {med:.2f} ms (min {lo:.2f}, max {hi:.2f}, {args.steps} steps)")
    _lib.start_timing()
    for _ in range(args.steps):
        train_step()
    for k, v in _lib.stop_timing().items():
        times.setdefault(k, []).extend(v)
    for name in ENTRY_POINTS:
        ts = sorted(times.get(name, []))
        if not ts:
            raise SystemExit(f"no {name} call")
        ms = ts[len(ts) // 2]
        nbytes = entry_bytes(name, n, e, nb)
        print(f"  {name}: median {1e3 * ms:.1f} us per call ({len(ts)} calls), {nbytes / 1e6:.2f} MB -> "
              f"{nbytes / (ms * 1e-3) / 1e12:.3f} TB/s = {100 * nbytes / (ms * 1e-3) / HBM_BYTES_PER_S:.1f}% of "
              f"3.35 TB/s")


if __name__ == "__main__":
    main()
