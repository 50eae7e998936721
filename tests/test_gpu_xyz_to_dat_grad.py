"""GPU tests: xyz_to_dat's dist / angle / torsion differentiated in pos, first and second order, at any in-degree.

Graphs: a QM9-like batch, a ragged batch, hubs of in-degree 65 / 128 / 300 / 1000, a 100-atom cluster at cutoff 6, the
corners (coincident atoms, collinear triplets, isolated atoms, edges without triplets, an empty graph) and an unsorted
edge list.  Comparators (tests/xyz_to_dat_grad_ref.py): autograd over the restated op sequence with the torsion's
gradient sent to the first minimal candidate, run by ATen on this GPU, and fp64 autograd of the geometry at the kernels'
candidates.
"""
import numpy as np
import pytest
import torch

import xyz_to_dat_grad_ref as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
U = 2.0 ** -24


def _api():
    from dig_b200.threedgraph.utils import geometric_computing as gc
    return gc


# ------------------------------------------------------------------------------------------------- graphs
def _batch(sizes, seed, cutoff=5.0, spread=1.6):
    gen = torch.Generator().manual_seed(seed)
    pos = torch.cat([torch.randn(s, 3, generator=gen) * spread + 40.0 * g for g, s in enumerate(sizes)])
    batch = torch.cat([torch.full((s,), g, dtype=torch.long) for g, s in enumerate(sizes)])
    pos, batch = pos.to(DEV), batch.to(DEV)
    ei = _api().radius_graph(pos, cutoff, batch, max_num_neighbors=32)
    return pos, ei, batch


def _hub(d, seed):
    """Atom 0 with d in-neighbours (and d out-edges) on a shell, plus a ring among the leaves."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(d, 3, generator=gen)
    x = x / x.norm(dim=1, keepdim=True) * (1.0 + torch.rand(d, 1, generator=gen))
    pos = torch.cat([torch.zeros(1, 3), x]).to(DEV)
    leaves = torch.arange(1, d + 1)
    nxt = leaves % d + 1
    src = torch.cat([leaves, torch.zeros(d, dtype=torch.long), leaves, nxt])
    dst = torch.cat([torch.zeros(d, dtype=torch.long), leaves, nxt, leaves])
    return _sorted(pos, torch.stack([src, dst]).to(DEV)), torch.zeros(d + 1, dtype=torch.long, device=DEV)


def _sorted(pos, ei):
    order = torch.argsort(ei[1] * pos.size(0) + ei[0], stable=True)
    return pos, ei[:, order].contiguous()


def _cluster(seed=3):
    gen = torch.Generator().manual_seed(seed)
    pos = (torch.rand(100, 3, generator=gen) * 7.0).to(DEV)
    batch = torch.zeros(100, dtype=torch.long, device=DEV)
    return pos, _api().radius_graph(pos, 6.0, batch, max_num_neighbors=128), batch


def _corners():
    """Coincident atoms (1, 2), a collinear chain (3, 4, 5), an isolated atom (6), a pair whose edges have no triplets
    (7, 8), and a generic atom (9); graph id 1 holds no atom (an empty graph inside the batch)."""
    pos = torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.2, 0.1], [1.0, 0.2, 0.1], [0.0, 1.5, 0.0], [0.0, 2.5, 0.0],
                        [0.0, 3.5, 0.0], [30.0, 0.0, 0.0], [60.0, 0.0, 0.0], [61.0, 0.3, 0.0],
                        [-0.6, 0.7, 0.8]], device=DEV)
    batch = torch.tensor([0, 0, 0, 0, 0, 0, 2, 3, 3, 0], device=DEV)
    order = torch.argsort(batch, stable=True)
    pos, batch = pos[order].contiguous(), batch[order].contiguous()
    return pos, _api().radius_graph(pos, 2.2, batch, max_num_neighbors=32), batch


def _graph(name):
    if name == "qm9":
        return _batch([18] * 16, 0)
    if name == "ragged":
        return _batch([3, 25, 7, 1, 14, 2, 19, 9], 1)
    if name.startswith("hub"):
        (pos, ei), batch = _hub(int(name[3:]), 2)
        return pos, ei, batch
    if name == "cluster":
        return _cluster()
    if name == "corners":
        return _corners()
    raise KeyError(name)


GRAPHS = ["qm9", "ragged", "hub65", "hub128", "hub300", "hub1000", "cluster", "corners"]
ATEN_GRAPHS = ["qm9", "ragged", "hub65", "hub128", "hub300", "cluster"]      # where the candidate sets fit in memory


def _kernel_graph(pos, ei, heavy_all=False):
    gc = _api()
    old = gc._HEAVY_KERNEL_FOR_ALL_EDGES
    gc._HEAVY_KERNEL_FOR_ALL_EDGES = heavy_all
    try:
        return gc._xyz_to_dat_sorted(pos, ei, pos.size(0), True, None, want_grad=True)
    finally:
        gc._HEAVY_KERNEL_FOR_ALL_EDGES = old


def _bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _weights(ne, nt, seed):
    gen = torch.Generator().manual_seed(seed)
    return [torch.randn(m, generator=gen).to(DEV) for m in (ne, nt, nt)]


# ------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("name", GRAPHS)
def test_tors_arg_and_values(name):
    """tors_arg has the same bits on the warp-per-edge and heavy kernels; the outputs with and without grad have the
    same bits; without grad nothing requires grad; tors_arg equals the first-argmin comparator's slots."""
    gc = _api()
    pos, ei, _ = _graph(name)
    n = pos.size(0)
    g0 = _kernel_graph(pos, ei)
    g1 = _kernel_graph(pos, ei, heavy_all=True)
    assert torch.equal(g0.tors_arg, g1.tors_arg)
    assert _bits(g0.torsion, g1.torsion) and _bits(g0.angle, g1.angle)
    plain = gc.xyz_to_dat(pos, ei, n, use_torsion=True)
    assert not any(t.requires_grad for t in plain)
    p = pos.clone().requires_grad_()
    withg = gc.xyz_to_dat(p, ei, n, use_torsion=True)
    assert withg[0].requires_grad and withg[1].requires_grad and withg[2].requires_grad
    for a, b in zip(withg[:3], plain[:3]):
        assert _bits(a.detach(), b)
    for a, b in zip(withg[3:], plain[3:]):
        assert torch.equal(a, b)
    with torch.no_grad():
        assert not any(t.requires_grad for t in gc.xyz_to_dat(p, ei, n, use_torsion=True))
    assert _bits(g0.torsion, plain[2])
    if name in ATEN_GRAPHS or name == "corners":
        (ref, slots) = R.first_argmin_xyz_to_dat(pos, ei, n, use_torsion=True, return_slots=True)
        assert torch.equal(g0.tors_arg.long(), slots)
        if name != "corners":                 # a zero-length ji: the kernels' torsion is inf, ATen's min is NaN
            assert _bits(ref[2], plain[2])


# ------------------------------------------------------------------------------------------------- first order
def _dpos(fn, pos, ei, w, create_graph=False):
    p = pos.clone().requires_grad_()
    out = fn(p, ei, pos.size(0), use_torsion=True)
    loss = (w[0] * out[0]).sum() + (w[1] * out[1]).sum() + (w[2] * out[2]).sum()
    return torch.autograd.grad(loss, p, create_graph=create_graph)[0]


@pytest.mark.parametrize("name", GRAPHS)
def test_first_order_against_aten_and_fp64(name):
    pos, ei, _ = _graph(name)
    n = pos.size(0)
    g = _kernel_graph(pos, ei)
    tors_c = R.candidate_atoms(ei, n, g.tors_arg)
    e_bad, a_bad, t_bad = R.degenerate(pos, ei, tors_c)
    w = _weights(ei.size(1), g.n_triplets, 5)
    w = [w[0] * ~e_bad, w[1] * ~a_bad, w[2] * ~t_bad]
    got = _dpos(_api().xyz_to_dat, pos, ei, w)
    assert bool(torch.isfinite(got).all())
    # Float atomics: the last bits vary from run to run.  The in-degree-1000 hub sums about 10^6 triplet terms per atom
    # in an order that changes from run to run; on an H100 its spread was 1.6e-6, 1.08e-5 and 1.22e-5 of the largest
    # component in three runs (every other graph: at most 1.9e-6), so its bounds here and against fp64 below are 5e-5,
    # about 4 times the largest spread seen.
    tol = 5e-5 if name == "hub1000" else 1e-5
    again = _dpos(_api().xyz_to_dat, pos, ei, w)
    spread = float((got - again).abs().max()) / max(float(got.abs().max()), 1e-30)
    print(f"{name}: run-to-run spread of dpos / max = {spread:.2e}")
    assert spread <= tol
    if name in ATEN_GRAPHS:
        ref = _dpos(R.first_argmin_xyz_to_dat, pos, ei, w)
        scale = float(ref.abs().max())
        err = float((got - ref).abs().max())
        print(f"{name}: |dpos - ATen comparator| / max = {err / scale:.2e}")
        assert err <= 1e-5 * scale, (err, scale)
    ref64 = _dpos(lambda p, e, m, use_torsion: R.geometry_at(p, e, m, tors_c), pos.double(), ei,
                  [x.double() for x in w])
    scale = float(ref64.abs().max())
    err = float((got.double() - ref64).abs().max())
    print(f"{name}: |dpos - fp64 at the kernels' candidates| / max = {err / scale:.2e}")
    assert err <= tol * scale, (err, scale)


def test_degenerate_elements_pass_convention_conformant_gradients():
    """Nonzero upstream gradients on every element of the corner graph give a finite dpos, and each degenerate class
    passes exactly nothing on its own: zero-length edges, the exactly collinear chain's angles (fp32 cross product 0),
    and torsions with |ji| = 0, atan2(0, 0), no candidate or the self candidate.  The self-candidate torsions of a
    generic molecule get rounding residues only from autograd over the ATen comparator."""
    from dig_b200 import ops
    pos, ei, _ = _corners()
    n = pos.size(0)
    g = _kernel_graph(pos, ei)
    tors_c = R.candidate_atoms(ei, n, g.tors_arg)
    e_bad, a_bad, t_bad = R.degenerate(pos, ei, tors_c)
    assert bool(e_bad.any()) and bool(a_bad.any()) and bool(t_bad.any())
    w = [torch.ones(ei.size(1), device=DEV), torch.ones(g.n_triplets, device=DEV), torch.ones(g.n_triplets, device=DEV)]
    assert bool(torch.isfinite(_dpos(_api().xyz_to_dat, pos, ei, w)).all())
    G = torch.randn(n, 3, generator=torch.Generator().manual_seed(3)).to(DEV)
    assert all(x is None or bool(torch.isfinite(x).all()) for x in _second(_api().xyz_to_dat, pos, ei, w, G))
    idx_i, idx_j, idx_k, _, _ = R.triplets(ei, n)
    u, v = pos[idx_i] - pos[idx_j], pos[idx_k] - pos[idx_j]
    chain = a_bad & (u.norm(dim=1) > 0) & (v.norm(dim=1) > 0) & ((u - v).norm(dim=1) > 0)
    assert bool(chain.any())
    for ddist, dangle, dtors in ((e_bad.float(), None, None), (None, chain.float(), None), (None, None, t_bad.float())):
        dpos = torch.zeros_like(pos)
        if ddist is not None:
            ops.edge_dist_bwd(pos, g, ddist, dpos)
        if dangle is not None:
            ops.triplet_angle_bwd(pos, g, dangle, dpos)
        if dtors is not None:
            ops.triplet_torsion_bwd_arg(pos, g, dtors, dpos)
        ops.triplet_geometry_bwd2(pos, g, dangle, dtors, G, dpos, want_dangle=False, want_dtorsion=False)
        assert float(dpos.abs().max()) == 0.0
    d_da, d_dt = ops.triplet_geometry_bwd2(pos, g, None, None, G, torch.zeros_like(pos))
    assert float(d_da[chain].abs().max()) == 0.0 and float(d_dt[t_bad].abs().max()) == 0.0
    # self-candidate winners on a generic molecule: zero in the kernels, rounding residue in the ATen comparator
    pos, ei, _ = _graph("qm9")
    n = pos.size(0)
    g = _kernel_graph(pos, ei)
    tors_c = R.candidate_atoms(ei, n, g.tors_arg)
    self_c = tors_c == R.triplets(ei, n)[2]
    assert int(self_c.sum()) > 0
    wt = self_c.float()
    zero_e, zero_t = torch.zeros(ei.size(1), device=DEV), torch.zeros(g.n_triplets, device=DEV)
    got = _dpos(_api().xyz_to_dat, pos, ei, [zero_e, zero_t, wt])
    ref = _dpos(R.first_argmin_xyz_to_dat, pos, ei, [zero_e, zero_t, wt])
    full = _dpos(R.first_argmin_xyz_to_dat, pos, ei, [zero_e, zero_t, torch.ones_like(wt)])
    print(f"self candidate: {int(self_c.sum())} of {g.n_triplets} torsions; ATen comparator's gradient through them "
          f"{float(ref.abs().max()):.2e} against {float(full.abs().max()):.2e} through all torsions")
    assert float(got.abs().max()) == 0.0
    assert float(ref.abs().max()) <= 1e-5 * float(full.abs().max())


# ------------------------------------------------------------------------------------------------- identities
def _abs_terms(pos, ei, tors_c, w, G=None):
    """Per atom: sum_t |w_t| |term_t| of the fp64 derivation (first order, or the HVP with G)."""
    n = pos.size(0)
    p = pos.double()
    terms = R.triplet_terms(p, ei, n, tors_c, G=None if G is None else G.double())
    return (R.scatter_terms(terms["angle"], w[1].double(), n, absolute=True)
            + R.scatter_terms(terms["torsion"], w[2].double(), n, absolute=True))


@pytest.mark.parametrize("name", GRAPHS)
def test_identities(name):
    """<J c, w> = <c, J^T w>, <c1, H c2> = <c2, H c1>, and per graph sum dpos = 0 and sum pos x dpos = 0, each to fp32
    rounding of the terms involved (256 roundings of the largest sum of |terms|)."""
    from dig_b200 import ops
    pos, ei, batch = _graph(name)
    n = pos.size(0)
    g = _kernel_graph(pos, ei)
    tors_c = R.candidate_atoms(ei, n, g.tors_arg)
    e_bad, a_bad, t_bad = R.degenerate(pos, ei, tors_c)
    w = _weights(ei.size(1), g.n_triplets, 9)
    w = [w[0] * 0, w[1] * ~a_bad, w[2] * ~t_bad]
    gen = torch.Generator().manual_seed(10)
    c1, c2 = (torch.randn(n, 3, generator=gen).to(DEV) for _ in range(2))
    # J^T w
    vjp = torch.zeros_like(pos)
    ops.triplet_angle_bwd(pos, g, w[1], vjp)
    ops.triplet_torsion_bwd_arg(pos, g, w[2], vjp)
    # J c (the value part of bwd2)
    scratch = torch.zeros_like(pos)
    ja, jt = ops.triplet_geometry_bwd2(pos, g, None, None, c1, scratch)
    assert float(scratch.abs().max()) == 0.0
    m_vjp = _abs_terms(pos, ei, tors_c, w)
    M = float((m_vjp * c1.double().abs()).sum())
    lhs = float((ja.double() * w[1].double()).sum() + (jt.double() * w[2].double()).sum())
    rhs = float((c1.double() * vjp.double()).sum())
    assert abs(lhs - rhs) <= 256 * U * M + 1e-30, (lhs, rhs, M)
    # H c symmetric
    h1, h2 = torch.zeros_like(pos), torch.zeros_like(pos)
    ops.triplet_geometry_bwd2(pos, g, w[1], w[2], c1, h1, want_dangle=False, want_dtorsion=False)
    ops.triplet_geometry_bwd2(pos, g, w[1], w[2], c2, h2, want_dangle=False, want_dtorsion=False)
    M = float((_abs_terms(pos, ei, tors_c, w, c2) * c1.double().abs()).sum()
              + (_abs_terms(pos, ei, tors_c, w, c1) * c2.double().abs()).sum())
    a12, a21 = float((c1.double() * h2.double()).sum()), float((c2.double() * h1.double()).sum())
    assert abs(a12 - a21) <= 256 * U * M + 1e-30, (a12, a21, M)
    # rigid-motion invariance, per graph
    ng = int(batch.max()) + 1 if n else 0
    for gi in range(ng):
        sel = batch == gi
        if not bool(sel.any()):
            continue
        Mg = float(m_vjp[sel].sum())
        s = vjp[sel].double().sum(0)
        assert float(s.abs().max()) <= 256 * U * Mg + 1e-30, (gi, s, Mg)
        p = pos[sel].double()
        torque = torch.linalg.cross(p, vjp[sel].double(), dim=-1).sum(0)
        Mt = float((p.abs().sum(1, keepdim=True) * m_vjp[sel]).sum())
        assert float(torque.abs().max()) <= 256 * U * Mt + 1e-30, (gi, torque, Mt)


# ------------------------------------------------------------------------------------------------- second order
def _second(fn, pos, ei, w, G):
    p = pos.clone().requires_grad_()
    w = [x.clone().requires_grad_() for x in w]
    out = fn(p, ei, pos.size(0), use_torsion=True)
    loss = (w[0] * out[0]).sum() + (w[1] * out[1]).sum() + (w[2] * out[2]).sum()
    (dpos,) = torch.autograd.grad(loss, p, create_graph=True)
    return torch.autograd.grad((G * dpos).sum(), [p] + w, allow_unused=True)


@pytest.mark.parametrize("name", GRAPHS)
def test_second_order_against_fp64_double_backward(name):
    """d/dpos and d/dw of <G, dpos> through xyz_to_dat (the HVPs and the JVPs of triplet_geometry_bwd2 and
    edge_dist_bwd2) within 1e-4 of the largest component of torch's double backward over the fp64 comparator at the
    kernels' candidates, non-degenerate elements only."""
    pos, ei, _ = _graph(name)
    n = pos.size(0)
    g = _kernel_graph(pos, ei)
    tors_c = R.candidate_atoms(ei, n, g.tors_arg)
    e_bad, a_bad, t_bad = R.degenerate(pos, ei, tors_c)
    w = _weights(ei.size(1), g.n_triplets, 21)
    w = [w[0] * ~e_bad, w[1] * ~a_bad, w[2] * ~t_bad]
    G = torch.randn(n, 3, generator=torch.Generator().manual_seed(22)).to(DEV)
    got = _second(_api().xyz_to_dat, pos, ei, w, G)
    ref = _second(lambda p, e, m, use_torsion: R.geometry_at(p, e, m, tors_c), pos.double(), ei,
                  [x.double() for x in w], G.double())
    masks = [None, ~e_bad, ~a_bad, ~t_bad]
    for what, a, b, m in zip(("d_pos", "d_ddist", "d_dangle", "d_dtorsion"), got, ref, masks):
        if b is None or b.numel() == 0:
            continue
        a = torch.zeros_like(b) if a is None else a.double()
        if m is not None:
            a, b = a[m], b[m]
        scale = float(b.abs().max()) if b.numel() else 0.0
        err = float((a - b).abs().max()) if b.numel() else 0.0
        print(f"{name} {what}: |got - fp64| / max = {err / max(scale, 1e-300):.2e}")
        assert err <= 1e-4 * scale, (what, err, scale)


# ------------------------------------------------------------------------------------------------- unsorted edges
def test_unsorted_edge_list():
    """A shuffled edge list: values, first- and second-order results equal those of the sorted list mapped through the
    permutation (the torch index plumbing carries the gradient)."""
    gc = _api()
    pos, ei, _ = _graph("qm9")
    n = pos.size(0)
    perm = torch.randperm(ei.size(1), generator=torch.Generator().manual_seed(4)).to(DEV)
    eu = ei[:, perm].contiguous()
    ps = pos.clone().requires_grad_()
    pu = pos.clone().requires_grad_()
    s = gc.xyz_to_dat(ps, ei, n, use_torsion=True)
    u = gc.xyz_to_dat(pu, eu, n, use_torsion=True)
    assert _bits(u[0].detach(), s[0].detach()[perm])
    # triplets: match by (caller's idx_ji, idx_kj) -> sorted ids
    key_s = s[6] * ei.size(1) + s[5]
    key_u = perm[u[6]] * ei.size(1) + perm[u[5]]
    order_s = torch.argsort(key_s)
    order_u = torch.argsort(key_u)
    assert torch.equal(key_s[order_s], key_u[order_u])
    assert _bits(u[1].detach()[order_u], s[1].detach()[order_s])
    assert _bits(u[2].detach()[order_u], s[2].detach()[order_s])
    w = _weights(ei.size(1), s[1].numel(), 30)
    ws = [w[0], w[1], w[2]]
    wu = [w[0][perm], torch.empty_like(w[1]), torch.empty_like(w[2])]
    wu[1][order_u] = w[1][order_s]
    wu[2][order_u] = w[2][order_s]
    G = torch.randn(n, 3, generator=torch.Generator().manual_seed(31)).to(DEV)
    loss_s = sum((a * b).sum() for a, b in zip(ws, s[:3]))
    loss_u = sum((a * b).sum() for a, b in zip(wu, u[:3]))
    (ds,) = torch.autograd.grad(loss_s, ps, create_graph=True)
    (du,) = torch.autograd.grad(loss_u, pu, create_graph=True)
    scale = float(ds.abs().max())
    assert float((ds - du).abs().max()) <= 1e-5 * scale
    (hs,) = torch.autograd.grad((G * ds).sum(), ps)
    (hu,) = torch.autograd.grad((G * du).sum(), pu)
    assert float((hs - hu).abs().max()) <= 1e-5 * float(hs.abs().max())


# ------------------------------------------------------------------------------------------------- end to end
class TinyModel(torch.nn.Module):
    """A small 3D model on xyz_to_dat: Gaussian distance features, (cos, sin) of angle and torsion, one triplet
    interaction, a node sum and a graph sum."""

    def __init__(self, geometry, cutoff=5.0, hidden=16, energy_and_force=True):
        super().__init__()
        self.geometry, self.cutoff, self.energy_and_force = geometry, cutoff, energy_and_force
        self.register_buffer("mu", torch.linspace(0.0, cutoff, 8))
        self.lin_e = torch.nn.Linear(8, hidden)
        self.lin_t = torch.nn.Linear(4, hidden)
        self.lin_m = torch.nn.Linear(hidden, hidden)
        self.out = torch.nn.Linear(hidden, 1)

    def forward(self, data):
        pos, batch = data.pos, data.batch
        if self.energy_and_force:
            pos.requires_grad_()
        ei = _api().radius_graph(pos, self.cutoff, batch, max_num_neighbors=32)
        dist, angle, torsion, i, j, idx_kj, idx_ji = self.geometry(pos, ei, pos.size(0), use_torsion=True)
        rbf = torch.exp(-(dist[:, None] - self.mu) ** 2 / 0.5)
        h_e = torch.nn.functional.silu(self.lin_e(rbf))
        tf = torch.stack([torch.cos(angle), torch.sin(angle), torch.cos(torsion), torch.sin(torsion)], dim=1)
        h_t = torch.nn.functional.silu(self.lin_t(tf)) * h_e[idx_kj]
        m = h_e + torch.zeros_like(h_e).index_add(0, idx_ji, h_t)
        node = torch.zeros(pos.size(0), m.size(1), device=pos.device).index_add(0, i, self.lin_m(m))
        e = self.out(torch.nn.functional.silu(node)).squeeze(-1)
        n_graphs = int(batch.max()) + 1
        return torch.zeros(n_graphs, device=pos.device).index_add(0, batch, e).unsqueeze(1)


def _data(n_mol, seed):
    from dig_b200.data import collate, synthetic_molecules
    return collate(synthetic_molecules(n_mol, "qm9", seed=seed, variable=True)).to(DEV)


def _energy_force_grads(model, data, target_e, target_f):
    data.pos = data.pos.detach().clone()
    model.zero_grad()
    e = model(data)
    f = -torch.autograd.grad(e, data.pos, torch.ones_like(e), create_graph=True)[0]
    loss = (e - target_e).abs().mean() + 100 * (f - target_f).abs().mean()
    loss.backward()
    return e.detach(), f.detach(), {k: p.grad.detach().clone() for k, p in model.named_parameters()}


def test_model_energies_forces_and_force_training_gradients():
    torch.manual_seed(0)
    ours = TinyModel(_api().xyz_to_dat).to(DEV)
    ref = TinyModel(R.first_argmin_xyz_to_dat).to(DEV)
    ref.load_state_dict(ours.state_dict())
    data = _data(16, 3)
    gen = torch.Generator().manual_seed(5)
    target_e = torch.randn(int(data.batch.max()) + 1, 1, generator=gen).to(DEV)
    target_f = torch.randn(data.pos.size(0), 3, generator=gen).to(DEV)
    e1, f1, g1 = _energy_force_grads(ours, data, target_e, target_f)
    e0, f0, g0 = _energy_force_grads(ref, data, target_e, target_f)
    assert float((e1 - e0).abs().max()) <= 1e-5 * float(e0.abs().max())
    ferr = float((f1 - f0).abs().max()) / float(f0.abs().max())
    print(f"model forces: {ferr:.2e} of the largest")
    assert ferr <= 1e-5
    worst = max(float((g1[k] - g0[k]).abs().max()) / max(float(g0[k].abs().max()), 1e-30) for k in g0)
    print(f"model force-training gradients: worst {worst:.2e}")
    assert worst <= 2e-4


def test_run_train_step_on_forces():
    from dig_b200.data import DataLoader, synthetic_molecules
    from dig_b200.threedgraph.method import run
    torch.manual_seed(1)
    model = TinyModel(_api().xyz_to_dat).to(DEV)
    mols = synthetic_molecules(8, "qm9", seed=9, variable=True)
    for m in mols:
        if not hasattr(m, "force") or m.force is None:
            m.force = torch.zeros_like(m.pos)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    before = {k: p.detach().clone() for k, p in model.named_parameters()}
    loss = run().train(model, opt, DataLoader(mols, 4, shuffle=False), True, 100, torch.nn.L1Loss(), DEV)
    assert np.isfinite(loss)
    assert any(not torch.equal(before[k], p.detach()) for k, p in model.named_parameters())
