"""Cost of forces and of second derivatives in the positions with ComENet (default widths) on --mols MD17-aspirin-shaped
molecules and with ComENet-OCP on the 24-slab OC20 batch of tests/golden/comenet_ocp_otf.npz (otf_graph=True):

  * first-order steps (run on any tree of the project with --root, so two trees can be compared): a force evaluation
    through `E.sum().backward()` in eval mode, and one force-training step (train mode, L1(E) + 100 L1(F), backward
    restricted to the parameters as `run.train` does, Adam);
  * unless --steps-only: a force evaluation through `grad(E, pos, create_graph=True)` plus one Hessian-vector product,
    `threedgraph.utils.molecular_hessians` (ComENet) against the same block-diagonal scheme over the comparator
    (tests/comenet_hessian_ref.py, fp32 on the same GPU) with the largest difference of the two Hessians, the new
    kernel `dig3d_comenet_features_tangent_bwd` per call with its compulsory bytes and their share of the H100's
    3.35 TB/s, the run-to-run spread of one HVP here and over the comparator, and a torch.profiler breakdown of one
    force + HVP (kernel time by group, launches, wall time).

Median / min / max ms over --steps runs after --warmup, by CUDA events; one JSON line per measurement, the first line
names the card and its power limit.

    python tools/gpu_comenet_hessian.py [--steps 10] [--warmup 3] [--mols 32] [--steps-only] [--root TREE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "unknown"


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return {"median_ms": round(statistics.median(ts), 3), "min_ms": round(min(ts), 3), "max_ms": round(max(ts), 3),
            "runs": steps}


class _B:
    pass


def mol_batch(z, pos, batch):
    b = _B()
    b.z, b.pos, b.batch = z, pos, batch
    b.num_graphs = int(batch.max().item()) + 1
    return b


def ocp_batch(root):
    from dig_b200.data import Batch
    g = np.load(os.path.join(root, "tests", "golden", "comenet_ocp_otf.npz"))
    b = Batch(**{k: torch.from_numpy(g[k]).cuda() for k in ("atomic_numbers", "pos", "tags", "cell", "natoms",
                                                            "batch")})
    b.num_graphs = int(g["natoms"].size)
    return b


def first_order(name, model, make, n_graphs, steps, warmup, tag):
    """Eval-mode force by E.sum().backward() and one force-training step."""
    def force():
        b = make()
        b.pos = b.pos.detach().clone().requires_grad_(True)
        model(b).sum().backward()
    model.eval()
    out = {"force_backward": timed(force, steps, warmup)}
    model.train()
    params = [p for p in model.parameters() if p.requires_grad]
    opt = torch.optim.Adam(params, lr=1e-6)
    b0 = make()
    y = torch.zeros(n_graphs, 1, device="cuda")
    ft = torch.zeros(b0.pos.shape, device="cuda")

    def train_step():
        b = make()
        b.pos = b.pos.detach().clone().requires_grad_(True)
        e = model(b)
        f = -torch.autograd.grad(e.sum(), b.pos, create_graph=True)[0]
        loss = torch.nn.functional.l1_loss(e, y) + 100.0 * torch.nn.functional.l1_loss(f, ft)
        opt.zero_grad()
        loss.backward(inputs=params)
        opt.step()
    out["train_step"] = timed(train_step, steps, warmup)
    print(json.dumps({"model": name, "tree": tag, **out}), flush=True)


def second_order(name, model, make, steps, warmup):
    model.eval()
    gen = torch.Generator().manual_seed(1)

    def hvp():
        b = make()
        b.pos = b.pos.detach().clone().requires_grad_(True)
        f = torch.autograd.grad(model(b).sum(), b.pos, create_graph=True)[0]
        v = torch.randn(b.pos.shape, generator=gen).cuda()
        torch.autograd.grad(f, b.pos, v)

    def force():
        b = make()
        b.pos = b.pos.detach().clone().requires_grad_(True)
        torch.autograd.grad(model(b).sum(), b.pos, create_graph=True)
    print(json.dumps({"model": name, "force_create_graph": timed(force, steps, warmup),
                      "force_plus_one_hvp": timed(hvp, steps, warmup)}), flush=True)


def comparator_hvp(model, z, pos, batch, steps, warmup):
    import comenet_hessian_ref as chr_
    sd = {k: v.detach() for k, v in model.state_dict().items()}
    gen = torch.Generator().manual_seed(1)

    def hvp():
        p = pos.clone().requires_grad_(True)
        f = torch.autograd.grad(chr_.comenet_forward(sd, z, p, batch, cutoff=model.cutoff,
                                                     num_layers=model.num_layers).sum(), p, create_graph=True)[0]
        torch.autograd.grad(f, p, torch.randn(pos.shape, generator=gen).cuda())
    return timed(hvp, steps, warmup), sd


def block_hessians(fn, pos, batch):
    """The block-diagonal scheme of molecular_hessians over a plain differentiable energy fn(pos)."""
    p = pos.clone().requires_grad_(True)
    force = torch.autograd.grad(fn(p).sum(), p, create_graph=True)[0]
    counts = torch.bincount(batch)
    start = torch.cumsum(counts, 0) - counts
    local = torch.arange(pos.size(0), device=pos.device) - start[batch]
    n_max = int(counts.max())
    full = pos.new_zeros(counts.numel(), n_max, 3, 3 * n_max)
    for k in range(n_max):
        for d in range(3):
            v = torch.zeros_like(pos)
            v[local == k, d] = 1.0
            full[batch, local, :, 3 * k + d] = torch.autograd.grad(force, p, v, retain_graph=True)[0]
    return [full[g, :n].reshape(3 * n, 3 * n_max)[:, :3 * n] for g, n in enumerate(counts.tolist())]


def kernel(model, z, pos, batch, steps):
    from dig_b200 import ops
    g = ops.build_graph(pos, batch, model.cutoff, num_graphs=int(batch.max()) + 1)
    ops.comenet_geometry(g, pos, model.cutoff)
    gen = torch.Generator().manual_seed(2)
    e, n = g.n_edges, g.n_nodes
    c = torch.randn(n, 3, generator=gen).cuda()
    u1, u2 = torch.randn(e, 12, generator=gen).cuda(), torch.randn(e, 6, generator=gen).cuda()
    t = timed(lambda: ops.comenet_features_tangent_bwd(g, pos, model.cutoff, c, u1, u2), steps * 10, 5)
    # compulsory traffic: pos and cvec [N,3]; per edge dist, src, dst, g1 [12], g2 [6]; refs [4N]; the [15E] work and
    # [3E] dvec written once and read once; the CSR / out lists; dpos [N,3]
    nbytes = 4 * (3 * n + 3 * n + e * (1 + 2 + 12 + 6) + 4 * n + 2 * 18 * e + 2 * (n + 1) + e + 3 * n)
    return {"edges": e, "nodes": n, "tangent_bwd_ms": t, "compulsory_bytes": nbytes,
            "hbm_share": round(nbytes / (t["median_ms"] * 1e-3) / HBM_BYTES_PER_S, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mols", type=int, default=32)
    ap.add_argument("--steps-only", action="store_true")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--tag", default="this")
    a = ap.parse_args()
    root = os.path.abspath(a.root)
    sys.path.insert(0, root)
    sys.path.insert(0, os.path.join(root, "tests"))
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph.method import ComENet
    from dig_b200.threedgraph.method.comenet_ocp import ComENet as ComENetOCP
    from oracle.weights import formula_state_dict
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    torch.manual_seed(0)
    model = ComENet(cutoff=5.0)
    model.load_state_dict(formula_state_dict(model.state_dict(), seed=41))
    model = model.cuda()
    b = synthetic_batch(a.mols, "md17-aspirin", seed=17)
    z, pos, batch = b.z.cuda(), b.pos.float().cuda(), b.batch.cuda()
    mk = lambda: mol_batch(z, pos, batch)                       # noqa: E731
    ocp = ComENetOCP(num_atoms=0, bond_feat_dim=0, num_radial=3, num_spherical=2, otf_graph=True).cuda()
    ob = ocp_batch(root)

    def mk_ocp():
        c = _B()
        for k in ("atomic_numbers", "pos", "tags", "cell", "natoms", "batch", "num_graphs"):
            setattr(c, k, getattr(ob, k))
        return c
    first_order("comenet", model, mk, a.mols, a.steps, a.warmup, a.tag)
    first_order("comenet_ocp", ocp, mk_ocp, ob.num_graphs, a.steps, a.warmup, a.tag)
    if a.steps_only:
        return
    second_order("comenet", model, mk, a.steps, a.warmup)
    second_order("comenet_ocp", ocp, mk_ocp, a.steps, a.warmup)
    ref_t, sd = comparator_hvp(model, z, pos, batch, a.steps, a.warmup)
    print(json.dumps({"model": "comenet", "comparator_force_plus_one_hvp": ref_t}), flush=True)
    from dig_b200.threedgraph.utils import molecular_hessians
    model.eval()
    holder = {}

    def ours():
        holder["h"] = molecular_hessians(model, mk())

    def theirs():
        import comenet_hessian_ref as chr_
        holder["r"] = block_hessians(lambda p: chr_.comenet_forward(sd, z, p, batch, cutoff=model.cutoff,
                                                                     num_layers=model.num_layers), pos, batch)
    t_ours, t_ref = timed(ours, 3, 1), timed(theirs, 3, 1)
    err = max(float((h - r).abs().max()) / float(r.abs().max()) for h, r in zip(holder["h"], holder["r"]))
    print(json.dumps({"model": "comenet", "molecular_hessians": t_ours, "comparator_blocks": t_ref,
                      "max_rel_diff": err}), flush=True)
    print(json.dumps({"model": "comenet", "kernel": kernel(model, z, pos, batch, a.steps)}), flush=True)
    print(json.dumps({"model": "comenet", "spread": spread(model, sd, z, pos, batch)}), flush=True)
    print(json.dumps({"model": "comenet", "hvp_profile": profile_hvp(model, mk)}), flush=True)


def spread(model, sd, z, pos, batch):
    """Run-to-run spread of one HVP (same v), two runs each of this path and of the comparator (fp32, same GPU), and
    their difference, relative to the largest component of this path's product; the comparator's rows where plain fp32
    autograd returns NaN are counted and left out."""
    import comenet_hessian_ref as chr_
    v = torch.randn(pos.shape, generator=torch.Generator().manual_seed(5)).cuda()

    def ours():
        p = pos.clone().requires_grad_(True)
        f = torch.autograd.grad(model(mol_batch(z, p, batch)).sum(), p, create_graph=True)[0]
        return torch.autograd.grad(f, p, v)[0]

    def theirs():
        p = pos.clone().requires_grad_(True)
        f = torch.autograd.grad(chr_.comenet_forward(sd, z, p, batch, cutoff=model.cutoff,
                                                     num_layers=model.num_layers).sum(), p, create_graph=True)[0]
        return torch.autograd.grad(f, p, v)[0]
    o1, o2, r1, r2 = ours(), ours(), theirs(), theirs()
    scale = float(o1.abs().max())
    rows = torch.isfinite(r1).all(1) & torch.isfinite(r2).all(1)   # plain fp32 autograd is NaN at some exact zeros

    def rel(x, y):
        return float((x[rows] - y[rows]).abs().max()) / scale
    return {"ours_run_to_run": float((o1 - o2).abs().max()) / scale, "comparator_run_to_run": rel(r1, r2),
            "ours_vs_comparator": rel(o1, r1), "comparator_nonfinite_rows": int((~rows).sum()), "rows": rows.numel()}


def profile_hvp(model, make):
    """Where the time of one force + HVP goes (eval mode): CUDA kernel time by kernel group, the number of launches,
    and the wall time of the profiled call."""
    import time
    from torch.profiler import ProfilerActivity, profile
    model.eval()
    v = None

    def hvp():
        nonlocal v
        b = make()
        b.pos = b.pos.detach().clone().requires_grad_(True)
        f = torch.autograd.grad(model(b).sum(), b.pos, create_graph=True)[0]
        v = torch.ones_like(b.pos) if v is None else v
        torch.autograd.grad(f, b.pos, v)
    for _ in range(3):
        hvp()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        hvp()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
    groups, n, total = {}, 0, 0.0
    for ev in prof.key_averages():
        t = ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
        if t <= 0:
            continue
        k = ev.key
        grp = ("comenet_features" if "comenet_features" in k else "linear_gemm" if ("gemm" in k or "linear" in k)
               else "graph_build" if ("radius" in k or "graph" in k or "scan" in k or "refs" in k)
               else "other")
        groups[grp] = round(groups.get(grp, 0.0) + t, 3)
        n += ev.count
        total += t
    return {"wall_ms": round(wall, 3), "kernel_ms": round(total, 3), "launches": n, "kernel_ms_by_group": groups}


if __name__ == "__main__":
    main()
