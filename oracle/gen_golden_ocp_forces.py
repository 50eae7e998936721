"""Writes tests/golden/comenet_ocp_forces.npz and tests/golden/comenet_ocp_forces_shapes.json from the UNMODIFIED
reference ComENet-OCP (dig/threedgraph/method/comenet/ocp/comenet-ocp.py, run on the CPU over oracle/shim.py and
oracle/ocp_stub.py, whose get_pbc_distances is plain torch and so differentiable in pos and cell).  Per case (array
names prefixed "<case>/"): the inputs, the energies, the forces -dE/dpos and the cell gradient dE/dcell in fp32 from
formula_state_dict weights, seeded energy / force targets, and the fp32 parameter gradients of the force-training loss
L1(E, y) + P * L1(F, f) with F = -grad(E, pos, create_graph=True): in full ("grad/<name>") for tensors of at most
FULL_GRAD_NUMEL entries, as seeded projections ("grad_proj/<name>", gen_golden_comenet_forces.projection) for larger
ones.

It checks, before writing anything, that oracle/restated.comenet_ocp_forward reproduces the reference: energies bit for
bit, forces, cell gradients and parameter gradients at fp32 rounding level.  Everything runs on ONE thread, for the
reason gen_golden_comenet_forces.py gives (the aliased cross products' derivative terms cancel only to their own last
bits, so the reference's position gradient depends on the order of the CPU's sums).

    python -m oracle.gen_golden_ocp_forces          (needs the reference checkout, see oracle/ref_loader.py)
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.gen_golden_comenet_forces import (FIXTURE_THREADS, FORCE_TOL, GRAD_TOL, force_loss,  # noqa: E402
                                              gradient_record)
from oracle.weights import formula_state_dict  # noqa: E402
from dig_b200.data import Batch, synthetic_pbc_batch  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
warnings.filterwarnings("ignore")

CTOR = dict(num_atoms=0, bond_feat_dim=0, hidden_channels=128, num_blocks=3, cutoff=6.0, num_radial=3,
            num_spherical=2, hetero=False, num_output_layers=2)
# name: (synthetic_pbc_batch kwargs, or "bulk" for BULK_CELLS, weight seed, index of a zero-length edge to insert into
# structure 0 or None)
CASES = {
    # three OC20-shaped slabs, shuffled edge lists, 50-neighbour cap
    "oc20": (dict(nsys=3, natoms=24, seed=31), 23, None),
    # a 4.5 x 4.5 cell at cutoff 6: every atom sees its own periodic images (row == col edges), plus one zero-length
    # edge (an atom to itself, offset 0), which get_pbc_distances drops
    "small_cell": (dict(nsys=2, natoms=5, cell=(4.5, 4.5, 6.0), seed=3), 29, 7),
    # primitive cells smaller than twice the nearest-neighbour distance, periodic in all three axes: an atom's nearest
    # in-neighbours are its own images at +a and -a
    "tiny_cell": ("bulk", 31, None),
}
# (cell rows, fractional positions) of the "bulk" case: a one-atom triclinic cell and a two-atom cell
BULK_CELLS = (
    ([[2.9, 0.0, 0.0], [0.4, 2.8, 0.0], [0.3, 0.2, 3.0]], [[0.0, 0.0, 0.0]]),
    ([[3.1, 0.0, 0.0], [0.2, 3.0, 0.0], [0.1, 0.3, 3.2]], [[0.05, 0.0, 0.02], [0.5, 0.45, 0.55]]),
)
KEYS = ("atomic_numbers", "pos", "tags", "cell", "edge_index", "cell_offsets", "neighbors", "batch")
TARGET_SEED = 5


def bulk_batch(cutoff=6.0, max_neighbors=50, seed=11):
    """BULK_CELLS as one batch with every periodic image within `cutoff` (shifts -3..3 on all three axes), at most
    `max_neighbors` nearest per target atom, edges in a seeded shuffled order."""
    gen = torch.Generator().manual_seed(seed)
    shifts = torch.tensor([[i, j, k] for i in range(-3, 4) for j in range(-3, 4) for k in range(-3, 4)],
                          dtype=torch.float32)
    out = {k: [] for k in ("atomic_numbers", "pos", "cell", "edge_index", "cell_offsets", "neighbors")}
    sizes, base = [], 0
    for rows, frac in BULK_CELLS:
        box, frac = torch.tensor(rows), torch.tensor(frac)
        n, ns = frac.size(0), shifts.size(0)
        pos = frac @ box
        d = (pos[None, :, None, :] + (shifts @ box)[None, None, :, :] - pos[:, None, None, :]).norm(dim=-1)
        d = d.reshape(n, n * ns)
        dd = torch.where((d < cutoff) & (d > 1e-6), d, torch.full_like(d, float("inf")))
        order = torch.argsort(dd, dim=1, stable=True)[:, :max_neighbors]
        valid = torch.gather(dd, 1, order) < float("inf")
        tgt = torch.arange(n)[:, None].expand_as(order)[valid]
        flat = order[valid]
        src, sh = flat // ns, flat % ns
        p = torch.randperm(tgt.numel(), generator=gen)
        tgt, src, sh = tgt[p], src[p], sh[p]
        out["edge_index"].append(torch.stack([src, tgt]) + base)
        out["cell_offsets"].append(shifts[sh])
        out["neighbors"].append(torch.tensor([tgt.numel()]))
        out["atomic_numbers"].append(torch.randint(1, 84, (n,), generator=gen))
        out["pos"].append(pos)
        out["cell"].append(box[None])
        sizes.append(n)
        base += n
    b = Batch(**{k: torch.cat(v, 1 if k == "edge_index" else 0) for k, v in out.items()})
    b.tags = torch.ones(base, dtype=torch.long)
    b.batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    b.natoms = torch.tensor(sizes)
    b.num_graphs = len(sizes)
    return b


def make_batch(name):
    """The case's batch (CPU, fp32), built the same way by the generator and the tests."""
    data, _, zero_at = CASES[name]
    b = bulk_batch() if data == "bulk" else synthetic_pbc_batch(**data)
    if zero_at is not None:
        a = int(b.edge_index[1, zero_at])
        b.edge_index = torch.cat([b.edge_index[:, :zero_at], torch.tensor([[a], [a]]), b.edge_index[:, zero_at:]], 1)
        b.cell_offsets = torch.cat([b.cell_offsets[:zero_at], torch.zeros(1, 3), b.cell_offsets[zero_at:]])
        b.neighbors = b.neighbors.clone()
        b.neighbors[0] += 1
    return b


def batch_from(g, device="cpu"):
    """A Batch of the fixture's stored inputs."""
    b = Batch(**{k: torch.from_numpy(g[k]).to(device) for k in KEYS})
    b.num_graphs = int(g["cell"].shape[0])
    return b


def state_dict(shapes_or_sd, wseed):
    sd = formula_state_dict(shapes_or_sd, seed=wseed)
    sd["lin_out.weight"] = sd["lin_out.weight"] + 0.05          # the class initialises lin_out to zeros
    return sd


def targets(n_graphs, n_atoms):
    gen = torch.Generator().manual_seed(TARGET_SEED)
    return torch.randn(n_graphs, 1, generator=gen), torch.randn(n_atoms, 3, generator=gen)


def restated_kwargs():
    return dict(cutoff=CTOR["cutoff"], num_blocks=CTOR["num_blocks"], num_output_layers=CTOR["num_output_layers"])


def _np(t):
    return t.detach().cpu().numpy()


def _leaves(b):
    b.pos = b.pos.clone().requires_grad_(True)
    b.cell = b.cell.clone().requires_grad_(True)
    return b


def run_case(mod, name):
    from oracle import restated
    _, wseed, _ = CASES[name]
    torch.manual_seed(0)
    model = mod.ComENet(**CTOR)
    sd = state_dict(model.state_dict(), wseed)
    model.load_state_dict(sd)
    model.eval()
    b = make_batch(name)
    out = {k: _np(getattr(b, k)) for k in KEYS}
    y, ft = targets(b.num_graphs, b.pos.size(0))
    out.update(y=_np(y), force_target=_np(ft))
    b = _leaves(b)
    e = model(b)
    dpos, dcell = torch.autograd.grad(e.sum(), [b.pos, b.cell])
    out.update(energy=_np(e), force=_np(-dpos), dcell=_np(dcell))
    # force training (cell held constant): the double backward of the reference
    b = make_batch(name)
    b.pos = b.pos.clone().requires_grad_(True)
    e = model(b)
    f = -torch.autograd.grad(e.sum(), b.pos, create_graph=True)[0]
    names = [k for k, _ in model.named_parameters()]
    grads = torch.autograd.grad(force_loss(e, f, y, ft), [p for _, p in model.named_parameters()])
    out.update(gradient_record(names, grads))
    # the restatement: energies bit for bit, forces / cell gradients / parameter gradients at fp32 level
    b = _leaves(make_batch(name))
    sd_r = {k: v.clone().requires_grad_(k in names) for k, v in sd.items()}
    u = restated.comenet_ocp_forward(sd_r, b, **restated_kwargs())
    assert np.array_equal(_np(u), out["energy"]), (name, _np(u), out["energy"])
    rp, rc = torch.autograd.grad(u.sum(), [b.pos, b.cell])
    ferr = float(np.abs(-_np(rp) - out["force"]).max() / np.abs(out["force"]).max())
    cerr = float(np.abs(_np(rc) - out["dcell"]).max() / np.abs(out["dcell"]).max())
    assert ferr < FORCE_TOL and cerr < FORCE_TOL, (name, ferr, cerr)
    b = make_batch(name)
    b.pos = b.pos.clone().requires_grad_(True)
    u = restated.comenet_ocp_forward(sd_r, b, **restated_kwargs())
    fr = -torch.autograd.grad(u.sum(), b.pos, create_graph=True)[0]
    grads_r = torch.autograd.grad(force_loss(u, fr, y, ft), [sd_r[k] for k in names])
    gerr = max(float(np.abs(_np(a) - _np(c)).max() / max(float(c.abs().max()), 1e-30)) for a, c in zip(grads_r, grads))
    assert gerr < GRAD_TOL, (name, gerr)
    n_self = int((b.edge_index[0] == b.edge_index[1]).sum())
    print(name, "E", out["energy"].ravel(), f"edges {b.edge_index.size(1)} (row == col: {n_self}),",
          f"restated force rel-err {ferr:.2e}, dcell {cerr:.2e}, grad {gerr:.2e}")
    shapes = {k: list(v.shape) for k, v in model.state_dict().items()}
    return out, shapes


def main():
    from oracle.ocp_stub import load_comenet_ocp
    torch.set_num_threads(FIXTURE_THREADS)
    mod = load_comenet_ocp()
    arrays, shapes = {}, {}
    for name in CASES:
        out, shapes[name] = run_case(mod, name)
        arrays.update({f"{name}/{k}": v for k, v in out.items()})
    np.savez_compressed(os.path.join(GOLD, "comenet_ocp_forces.npz"), **arrays)
    with open(os.path.join(GOLD, "comenet_ocp_forces_shapes.json"), "w") as fh:
        json.dump(shapes, fh)


if __name__ == "__main__":
    main()
