"""Derivatives of `xyz_to_dat` in pos, timed: the forward with and without the recorded torsion candidates (tors_arg),
the first-order backward (forces), the second-order backward (force training), the derivative kernels alone, and one
force-training step of a small model built on xyz_to_dat; against the restated reference ops (oracle/restated.py) run
by ATen on the same GPU where their (triplet, candidate) sets fit `--ref-candidates`.

Shapes: 128 QM9-like molecules of about 18 atoms (cutoff 5, 32 neighbours), and one graph of 2,048 atoms at cutoff 5
whose in-degree the cap holds at D = 64 / 128 / 256 (tools/gpu_dense_graph.py's shapes).  use_torsion=True throughout.
Medians of `--reps` calls by CUDA events after `--warmup` untimed ones.  Prints one JSON line with the card's name,
power limit and maximum SM clock read in the same process.  Test infrastructure; needs a GPU.

    python tools/gpu_xyz_to_dat_grad.py [--degrees 64,128,256] [--reps 5] [--warmup 2]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gpu_dense_graph import atoms, card, time_ms  # noqa: E402
from oracle import restated  # noqa: E402
from dig_b200 import ops  # noqa: E402
from dig_b200.threedgraph.utils import geometric_computing as gc  # noqa: E402
from dig_b200.threedgraph.utils import radius_graph, xyz_to_dat  # noqa: E402


class Tiny(torch.nn.Module):
    """Gaussian distance features, (cos, sin) of angle and torsion, one triplet interaction, node and graph sums."""

    def __init__(self, geometry, cutoff=5.0, hidden=64):
        super().__init__()
        self.geometry, self.cutoff = geometry, cutoff
        self.register_buffer("mu", torch.linspace(0.0, cutoff, 16))
        self.lin_e = torch.nn.Linear(16, hidden)
        self.lin_t = torch.nn.Linear(4, hidden)
        self.lin_m = torch.nn.Linear(hidden, hidden)
        self.out = torch.nn.Linear(hidden, 1)

    def forward(self, pos, batch, n_graphs):
        ei = radius_graph(pos, self.cutoff, batch, max_num_neighbors=32)
        dist, angle, torsion, i, j, idx_kj, idx_ji = self.geometry(pos, ei, pos.size(0), use_torsion=True)
        h_e = torch.nn.functional.silu(self.lin_e(torch.exp(-(dist[:, None] - self.mu) ** 2 / 0.5)))
        tf = torch.stack([torch.cos(angle), torch.sin(angle), torch.cos(torsion), torch.sin(torsion)], dim=1)
        m = h_e + torch.zeros_like(h_e).index_add(0, idx_ji, torch.nn.functional.silu(self.lin_t(tf)) * h_e[idx_kj])
        node = torch.zeros(pos.size(0), m.size(1), device=pos.device).index_add(0, i, self.lin_m(m))
        e = self.out(torch.nn.functional.silu(node)).squeeze(-1)
        return torch.zeros(n_graphs, device=pos.device).index_add(0, batch, e)


def qm9_shape(n_mol=128, seed=0):
    from dig_b200.data import collate, synthetic_molecules
    b = collate(synthetic_molecules(n_mol, "qm9", seed=seed, variable=True)).to("cuda")
    return b.pos.contiguous(), b.batch, n_mol


def derivative_timings(pos, ei, n, reps, warmup, fn=xyz_to_dat):
    """forward (no grad), forward (grad, tors_arg), backward, double backward of sum(w * geometry) for `fn`."""
    gen = torch.Generator().manual_seed(0)
    p = pos.clone().requires_grad_()
    out = fn(p, ei, n, use_torsion=True)
    w = [torch.randn(x.numel(), generator=gen).cuda() for x in out[:3]]
    G = torch.randn(n, 3, generator=gen).cuda()
    loss = sum((a * b).sum() for a, b in zip(w, out[:3]))
    res = {}
    with torch.no_grad():
        res["forward"] = time_ms(lambda: fn(pos, ei, n, use_torsion=True), reps, warmup)
    res["forward_with_grad"] = time_ms(lambda: fn(p, ei, n, use_torsion=True), reps, warmup)
    res["backward"] = time_ms(lambda: torch.autograd.grad(loss, p, retain_graph=True), reps, warmup)
    (dpos,) = torch.autograd.grad(loss, p, create_graph=True)
    l2 = (G * dpos).sum()
    res["double_backward"] = time_ms(lambda: torch.autograd.grad(l2, p, retain_graph=True), reps, warmup)
    return res, w, G


def kernel_timings(pos, ei, n, w, G, reps, warmup):
    """The derivative kernels alone on the graph xyz_to_dat builds (the forward recording tors_arg, included)."""
    g = gc._xyz_to_dat_sorted(pos, ei, n, True, None, want_grad=True)
    n_heavy = int((torch.bincount(ei[1], minlength=n)[ei[0]] > 64).sum())
    res = {"n_heavy_edges": n_heavy}
    res["kernel_forward_any_degree"] = time_ms(lambda: ops.triplet_geometry_any_degree(g, pos, 1, n_heavy), reps, warmup)
    res["kernel_forward_any_degree_arg"] = time_ms(lambda: ops.triplet_geometry_any_degree_arg(g, pos, n_heavy),
                                                   reps, warmup)
    dpos = torch.zeros_like(pos)
    res["kernel_edge_dist_bwd"] = time_ms(lambda: ops.edge_dist_bwd(pos, g, w[0], dpos), reps, warmup)
    res["kernel_triplet_angle_bwd"] = time_ms(lambda: ops.triplet_angle_bwd(pos, g, w[1], dpos), reps, warmup)
    res["kernel_triplet_torsion_bwd_arg"] = time_ms(lambda: ops.triplet_torsion_bwd_arg(pos, g, w[2], dpos), reps,
                                                    warmup)
    res["kernel_edge_dist_bwd2"] = time_ms(lambda: ops.edge_dist_bwd2(pos, g, w[0], G), reps, warmup)
    res["kernel_triplet_geometry_bwd2"] = time_ms(lambda: ops.triplet_geometry_bwd2(pos, g, w[1], w[2], G, dpos),
                                                  reps, warmup)
    return res


def force_step(pos, batch, n_graphs, geometry, reps, warmup):
    torch.manual_seed(0)
    model = Tiny(geometry).cuda()
    gen = torch.Generator().manual_seed(1)
    te = torch.randn(n_graphs, generator=gen).cuda()
    tf = torch.randn(pos.size(0), 3, generator=gen).cuda()

    def step():
        model.zero_grad()
        p = pos.clone().requires_grad_()
        e = model(p, batch, n_graphs)
        f = -torch.autograd.grad(e, p, torch.ones_like(e), create_graph=True)[0]
        ((e - te).abs().mean() + 100 * (f - tf).abs().mean()).backward()

    return time_ms(step, reps, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--atoms", type=int, default=2048)
    ap.add_argument("--degrees", default="64,128,256")
    ap.add_argument("--cutoff", type=float, default=5.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ref-candidates", type=float, default=1e8,
                    help="largest (triplet, candidate) count for which the restated ops are run")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_xyz_to_dat_grad.py needs a CUDA device")
    out = {"tool": "gpu_xyz_to_dat_grad", **card(), "cutoff": args.cutoff, "runs": []}
    shapes = [("qm9", *qm9_shape())]
    for d in [int(x) for x in args.degrees.split(",")]:
        pos = atoms(args.atoms, d, args.cutoff, seed=d)
        shapes.append((f"dense_D{d}", pos, torch.zeros(args.atoms, dtype=torch.long, device=pos.device), 1, d))
    for shape in shapes:
        name, pos, batch, n_graphs = shape[:4]
        d = shape[4] if len(shape) > 4 else 32
        n = pos.size(0)
        ei = radius_graph(pos, args.cutoff, batch, max_num_neighbors=d)
        got = xyz_to_dat(pos, ei, n, use_torsion=True)
        per_edge = torch.bincount(got[-1], minlength=ei.size(1)).double()
        candidates = int((per_edge * per_edge).sum())
        run = {"shape": name, "atoms": n, "graphs": n_graphs, "max_num_neighbors": d, "edges": int(ei.size(1)),
               "triplets": int(got[1].numel()), "torsion_candidates": candidates}
        del got
        t, w, G = derivative_timings(pos, ei, n, args.reps, args.warmup)
        run["xyz_to_dat"] = t
        run.update(kernel_timings(pos, ei, n, w, G, args.reps, args.warmup))
        if name == "qm9":
            run["force_training_step_tiny_model"] = force_step(pos, batch, n_graphs, xyz_to_dat, args.reps,
                                                               args.warmup)
        if candidates <= args.ref_candidates:
            run["restated"], _, _ = derivative_timings(pos, ei, n, args.reps, args.warmup, fn=restated.xyz_to_dat)
            if name == "qm9":
                run["restated_force_training_step_tiny_model"] = force_step(pos, batch, n_graphs, restated.xyz_to_dat,
                                                                            args.reps, args.warmup)
        else:
            run["restated"] = f"skipped: {candidates} candidates > --ref-candidates"
        torch.cuda.empty_cache()
        out["runs"].append(run)
        print(json.dumps(run), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
