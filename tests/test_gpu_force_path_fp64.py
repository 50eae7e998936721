"""The first-order force path of SphereNet / DimeNet++ at their default widths, kernel by kernel against fp64.

    ops.edge_basis_bwd                   ddist from d rbf0, and bess_dx          ag.edge_basis, ag.basis_project
    ops.triplet_basis_project_bwd_geom   d dist_kj, d angle, d torsion of the fused lin_sbf1 / lin_t1 projection
    ops.triplet_torsion_bwd              d pos of the model graph's torsion, re-searching the minimising candidate

References, magnitudes and rounding counts: tests/triplet_backward_ref.py (its module docstring derives every bound;
the CPU side is checked by tests/test_force_path_ref_cpu.py).  Every per-element check is

    |got - fp64| <= gamma(c) M + (closed-form term) + c ETA

edge_basis_bwd: a sorted distance sweep from 1e-3 cutoff to the float below the cutoff (the envelope cancels there) and
the real edges of the graphs below, basis (7, 6) and (3, 6), envelope on / off, envelope exponents 5, 2 and 4 (powf(x,
p - 2) changes form).  Below X_MIN only finiteness is asserted.
triplet_basis_project_bwd_geom: a QM9-like batch, a molecule on which the neighbour cap binds (> 32 atoms: the candidate
loop runs two and three 32-lane chunks; in- and out-lists asymmetric), a ragged batch, a three-atom batch with fewer
edges than one CTA has warps, a collinear chain (sin theta = 0) and the golden SphereNet inputs; 4, 3, 2, 1 layer slots,
None slots and zero slots, the autograd Function with non-contiguous upstream gradients, six layers in two launches,
and the adjoint identity with the tangent kernels.  The `i_in` guard of the candidate's triplet index cannot be reached
by a graph of the radius-graph build (tests/test_triplet_backward_reference_cpu.py asserts why); the capped molecule
covers its reachable side.
triplet_torsion_bwd: against triplet_torsion_bwd_arg at the forward's recorded winners (a different candidate is an O(1)
difference), on a geometry built with exact ties between two candidates, and against fp64 autograd of the geometry at
the winners.  Its bound is the measured-tolerance policy of test_gpu_xyz_to_dat_grad.py (1e-5 of the largest
component): the torsion's gradient is a ratio whose conditioning has no closed-form count here.
End to end: default-width SphereNet (ns 7 and 3) and DimeNet++ forces against autograd over the fp32 restatement on
the same GPU, on the ragged batch, a six-layer model and (ns 3 only) the capped batch.  With the seven-order bases the
capped batch's forces differ from the restatement's by 4.9e-2 (SphereNet) and 4.2e-4 (DimeNet++) of the largest
component on an H100, while every kernel above holds its per-element bound on the same graph; the dense box puts
atom pairs at x ~ 1e-3, where the (7, 6) closed forms and their autograd in the restatement cancel in fp32.  That
comparison is left out until the comparator is evaluated in fp64 there.

Run with -s to see the largest |got - exact| / bound per output.
"""
import math

import pytest
import torch

import triplet_backward_ref as ref
import xyz_to_dat_grad_ref as R
from helpers import case_inputs, formula_state_dict, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NR = 6
FTOL = 1e-5
WORST = {}
_CACHE = {}
BASES = [(0, False), (0, True), (1, False), (1, True)]          # (basis_id, torsion)


def _note(name, ratio):
    WORST[name] = max(WORST.get(name, 0.0), ratio)


def _rand(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(DEV)


def _positions(name):
    """(pos, batch, cutoff, num_graphs) on the host."""
    from dig_b200.data import synthetic_batch
    if name == "qm9":
        b = synthetic_batch(32, "qm9", seed=5, variable=True)
        return b.pos, b.batch, 5.0, None
    if name == "capped":
        return (*ref.capped_batch(), None)
    if name == "ragged":
        return ref.ragged_batch()
    if name == "tiny":
        return (*ref.tiny_batch(), None)
    if name == "collinear":
        return (*ref.collinear_batch(), None)
    if name == "tie":
        return (*_tie_batch(), None)
    _, _, pos, batch = case_inputs({"golden_qm9": "spherenet_qm9", "golden_ns3": "spherenet_ns3"}[name])
    return pos, batch, 5.0, None


def _graph(name):
    from dig_b200 import ops
    if name not in _CACHE:
        pos, batch, cutoff, num_graphs = _positions(name)
        pos, batch = pos.float().contiguous().to(DEV), batch.long().to(DEV)
        g = ops.build_graph(pos, batch, cutoff, num_graphs=num_graphs)
        ops.triplet_geometry(g, pos, use_torsion=True, want_idx=True, want_idx64=True)
        _CACHE[name] = (g, pos, cutoff)
    return _CACHE[name]


# ------------------------------------------------------------------------------------------------ A. edge_basis_bwd
def _sweep(cutoff, n=4097):
    last = float(torch.nextafter(torch.tensor(cutoff, dtype=torch.float32), torch.tensor(0.0)))
    dist = torch.linspace(1e-3 * cutoff, cutoff, n, dtype=torch.float64).float().clamp(max=last)
    assert float(dist.max()) == last < cutoff
    return dist.to(DEV)


def _edge_dists(name):
    if name == "sweep":
        return _sweep(5.0), 5.0
    g, _, cutoff = _graph(name)
    return g.dist, cutoff


@pytest.mark.parametrize("exponent", [5, 2, 4])
@pytest.mark.parametrize("basis_id,env_on", [(0, True), (0, False), (1, True), (1, False)])
@pytest.mark.parametrize("dists", ["sweep", "capped", "qm9"])
def test_edge_basis_bwd_matches_fp64(dists, basis_id, env_on, exponent):
    from dig_b200 import ops
    dist, cutoff = _edge_dists(dists)
    ns = 7 if basis_id == 0 else 3
    e = dist.numel()
    freq = (torch.arange(1, NR + 1, dtype=torch.float32) * math.pi
            + 0.01 * torch.randn(NR, generator=torch.Generator().manual_seed(5))).to(DEV)
    drbf0 = _rand(90 + exponent, e, NR)                                    # mixed signs: the sum over n cancels
    args = (dist, cutoff, exponent, freq, basis_id, env_on, drbf0, ns * NR)
    ddist, bdx = ops.edge_basis_bwd(*args, want_ddist=True, want_bess_dx=True)
    ddist2, bdx2 = ops.edge_basis_bwd(*args, want_ddist=True, want_bess_dx=True)
    only_d, none_b = ops.edge_basis_bwd(*args, want_ddist=True, want_bess_dx=False)
    none_d, only_b = ops.edge_basis_bwd(*args[:6], None, ns * NR, want_ddist=False, want_bess_dx=True)
    torch.cuda.synchronize()
    # plain stores: the same bits every launch, and one output does not depend on whether the other was asked for
    assert torch.equal(ddist, ddist2) and torch.equal(bdx, bdx2)
    assert none_b is None and none_d is None
    assert torch.equal(only_d, ddist) and torch.equal(only_b, bdx)
    x = ref.kernel_x(dist, cutoff)
    tag = f"{dists} basis {basis_id} env {env_on} p-1 {exponent}"
    v, m1, m2 = ref.edge_bwd_reference(x, freq, cutoff, exponent, drbf0)
    c1, c2 = ref.edge_bwd_count(NR)
    limit = ref.U * (c1 * m1 + c2 * m2) / (1 - c1 * ref.U) + c1 * ref.ETA
    _note("edge_basis_bwd.ddist", ref.check(ddist, v, limit, tag + " ddist"))
    if e > 1:
        assert float((v.abs() / m1).min()) < 0.5                           # the sum did cancel
    exact, lim = ref.bess_dx_reference(x, ns, NR, exponent, env_on)
    live = x >= ref.X_MIN[basis_id]
    assert bool(torch.isfinite(bdx[~live]).all())
    _note("edge_basis_bwd.bess_dx", ref.check(bdx[live], exact[live], lim[live], tag + " bess_dx"))


def test_edge_basis_bwd_without_edges():
    """E = 0 returns before any launch: outputs passed to the C entry point keep their contents."""
    from dig_b200 import ops
    freq = torch.ones(NR, device=DEV)
    dist, drbf0 = torch.ones(4, device=DEV), torch.ones(4, NR, device=DEV)
    ddist, bdx = torch.full((4,), 7.0, device=DEV), torch.full((4, 42), 7.0, device=DEV)
    ops.call("dig3d_edge_basis_bwd", ops._p(dist), 0, 5.0, 5, ops._p(freq), 0, 1, ops._p(drbf0), ops._p(ddist),
             ops._p(bdx), ops._stream())
    torch.cuda.synchronize()
    assert bool((ddist == 7.0).all() and (bdx == 7.0).all())


# ------------------------------------------------------------------------------------------------ B. the projection
def _bases(name, basis_id, tors):
    """bess / bess_dx of the graph's edges from the kernels, made finite as in the generic-width test."""
    from dig_b200 import ops
    key = ("bases", name, basis_id, tors)
    if key not in _CACHE:
        g, _, cutoff = _graph(name)
        ns = 7 if basis_id == 0 else 3
        freq = (torch.arange(1, NR + 1, dtype=torch.float32) * math.pi).to(DEV)
        _, bess = ops.edge_basis(g.dist, cutoff, 5, freq, basis_id, not tors, NR, ns * NR)
        _, bess_dx = ops.edge_basis_bwd(g.dist, cutoff, 5, None, basis_id, not tors, None, ns * NR, want_ddist=False,
                                        want_bess_dx=True)
        # atoms of the dense box closer than the closed forms can be evaluated in fp32 at: keep the inputs finite
        bess = torch.nan_to_num(bess, nan=0.0, posinf=0.0, neginf=0.0).clamp_(-100.0, 100.0)
        bess_dx = torch.nan_to_num(bess_dx, nan=0.0, posinf=0.0, neginf=0.0).clamp_(-1e3, 1e3)
        _CACHE[key] = (bess, bess_dx, ns)
    return _CACHE[key]


def _layer_grads(t, seed, n=4):
    scale = torch.logspace(-6, 0, 8, device=DEV)                  # small channels are really checked
    return [(_rand(seed + l, t, 8) * scale).contiguous() for l in range(n)]


def _weights(ns, tors, seed, rows=32):
    w_s = _rand(seed, rows, ns * NR) * 0.3
    w_t = _rand(seed + 1, rows, ns * ns * NR) * 0.1 if tors else None
    return w_s, w_t


def _contract(ds, w, mag):
    """sum_l d[l] W[8 l : 8 l + 8] in fp64 (|d| |W| with mag); None slots contribute nothing."""
    out = 0.0
    for l, d in enumerate(ds):
        if d is None:
            continue
        a, b = d.double(), w[8 * l:8 * l + 8].double()
        out = out + ((a.abs() @ b.abs()) if mag else (a @ b))
    return out


def _geom_reference(name, basis_id, tors, d_s, d_t, w_s, w_t, extra=0):
    """{output: (exact, bound)} of triplet_basis_project_bwd_geom; `extra` roundings for a sum of launches."""
    g, _, cutoff = _graph(name)
    bess, bess_dx, ns = _bases(name, basis_id, tors)
    tor = g.torsion if tors else None
    ds_v, ds_m = _contract(d_s, w_s, False), _contract(d_s, w_s, True)
    dt_v = _contract(d_t, w_t, False) if tors else None
    dt_m = _contract(d_t, w_t, True) if tors else None
    v = ref.basis_bwd_reference(g, cutoff, ns, bess, bess_dx, g.angle, tor, ds_v, dt_v)["v"]
    r = ref.basis_bwd_reference(g, cutoff, ns, bess, bess_dx, g.angle, tor, ds_m, dt_m)
    c_t = NR + 32 + ns + (ns * ns if tors else 0) + extra
    atoms = (g.graph_ptr[1:] - g.graph_ptr[:-1]).long()[g.batch[g.dst.long()]]
    c_e = c_t + torch.ceil(atoms.double() / 32) + 5 + 2
    out = {}
    for i, name_ in enumerate(("ddist", "dangle", "dtorsion")):
        if v[i] is None:
            continue
        c = c_e if name_ == "ddist" else float(c_t)
        out[name_] = (v[i], ref.gamma(c) * r["m"][i] + ref.CLOSED_FORM_TOL * r["h"][i] + c * ref.ETA)
    return out


def _check_geom(got, exact, tag):
    for name, out in zip(("ddist", "dangle", "dtorsion"), got):
        if name not in exact:
            assert out is None, name
            continue
        _note("project_bwd_geom." + name, ref.check(out, exact[name][0], exact[name][1], f"{tag} {name}"))


GEOM_GRAPHS = ["qm9", "capped", "ragged", "tiny", "collinear", "golden_qm9", "golden_ns3"]


@pytest.mark.parametrize("basis_id,tors", BASES)
@pytest.mark.parametrize("graph", GEOM_GRAPHS)
def test_project_bwd_geom_matches_fp64(graph, basis_id, tors):
    from dig_b200 import ops
    name = graph
    g, _, cutoff = _graph(name)
    bess, bess_dx, ns = _bases(name, basis_id, tors)
    if graph == "capped":
        per_mol = g.graph_ptr[1:] - g.graph_ptr[:-1]
        assert int(per_mol.min()) > 32 and int(per_mol.max()) > 64          # two and three candidate chunks
    if graph == "collinear":
        a = g.angle.double()
        assert bool((a == 0).any()) and bool((a - math.pi).abs().lt(1e-6).any())
    t = g.n_triplets
    d_s = _layer_grads(t, 30)
    d_t = _layer_grads(t, 40) if tors else None
    w_s, w_t = _weights(ns, tors, 50)
    run = lambda s, tt: ops.triplet_basis_project_bwd_geom(g, bess, bess_dx, basis_id, s, tt, w_s, w_t, cutoff)
    cut = lambda lst, n: None if lst is None else lst[:n]
    for n in (4, 3, 2, 1):
        got = run(cut(d_s, n), cut(d_t, n))
        _check_geom(got, _geom_reference(name, basis_id, tors, cut(d_s, n), cut(d_t, n), w_s, w_t),
                    f"{graph} basis {basis_id} torsion {tors} {n} slots")
        if n == 4:
            again = run(d_s, d_t)
            torch.cuda.synchronize()
            for a, b in zip(got, again):
                assert (a is None and b is None) or torch.equal(a, b), "plain stores: two runs must agree bit for bit"
            counts = torch.bincount(g.idx_kj.long(), minlength=g.n_edges)
            assert bool((got[0][counts == 0] == 0).all())                  # no triplet reads the edge: exactly 0
            if graph == "ragged":
                assert bool((counts == 0).any())
    # slots 1 and 3 without a gradient: None and explicit zeros give the same bits, and match the reference
    skip = lambda lst: None if lst is None else [lst[0], None, lst[2], None]
    zero = lambda lst: None if lst is None else [lst[0], torch.zeros_like(lst[1]), lst[2], torch.zeros_like(lst[3])]
    a, b = run(skip(d_s), skip(d_t)), run(zero(d_s), zero(d_t))
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert (x is None and y is None) or torch.equal(x, y), "a None slot must equal an explicit zero slot"
    _check_geom(a, _geom_reference(name, basis_id, tors, skip(d_s), skip(d_t), w_s, w_t),
                f"{graph} basis {basis_id} torsion {tors} slots 1, 3 None")


@pytest.mark.parametrize("basis_id,tors", BASES)
@pytest.mark.parametrize("graph", ["qm9", "tiny", "golden_ns3"])
def test_basis_project_function_geometry_grads(graph, basis_id, tors):
    """ag.basis_project with dist / angle / torsion requiring grad and non-contiguous upstream gradients: dist.grad,
    angle.grad and the torsion's grad meet the kernel's bounds (bess_dx is recomputed inside the backward)."""
    from dig_b200 import autograd as ag
    g, _, cutoff = _graph(graph)
    bess, bess_dx, ns = _bases(graph, basis_id, tors)
    assert bool(torch.isfinite(bess).all() and torch.isfinite(bess_dx).all() and bess_dx.abs().max() < 1e3)
    w_s, w_t = _weights(ns, tors, 60)
    ws_l = [w_s[8 * l:8 * l + 8].clone().requires_grad_(True) for l in range(4)]
    wt_l = [w_t[8 * l:8 * l + 8].clone().requires_grad_(True) for l in range(4)] if tors else None
    dist = g.dist.clone().requires_grad_(True)
    angle = g.angle.clone().requires_grad_(True)
    tor = g.torsion.clone().requires_grad_(True) if tors else None
    geo_cfg = (cutoff, 5, not tors, dist)
    s_l, t_l = ag.basis_project(g, bess, dist, angle, tor, geo_cfg, basis_id, ns, NR, ws_l, wt_l)
    d_s = _layer_grads(g.n_triplets, 70)
    d_t = _layer_grads(g.n_triplets, 80) if tors else None
    outs, ups = list(s_l), list(d_s)
    if tors:
        outs, ups = outs + list(t_l), ups + list(d_t)
    strided = []
    for d in ups:
        wide = torch.zeros(d.size(0), 16, device=DEV)
        wide[:, 1::2] = d
        strided.append(wide[:, 1::2])
    assert not strided[0].is_contiguous()
    torch.autograd.backward(outs, strided)
    exact = _geom_reference(graph, basis_id, tors, d_s, d_t, w_s, w_t)
    _check_geom((dist.grad, angle.grad, None if tor is None else tor.grad), exact,
                f"{graph} Function basis {basis_id} torsion {tors}")


@pytest.mark.parametrize("basis_id,tors", [(0, True), (0, False)])
def test_basis_project_six_layers(basis_id, tors):
    """Six layers as dimenet_family splits them (slots 0-3, then 4-5): the summed geometry gradients against one fp64
    reference over all six layers (one more rounding for the sum of the two launches)."""
    from dig_b200 import autograd as ag
    graph = "qm9"
    g, _, cutoff = _graph(graph)
    bess, _, ns = _bases(graph, basis_id, tors)
    w_s6, w_t6 = _weights(ns, tors, 100, rows=48)
    dist = g.dist.clone().requires_grad_(True)
    angle = g.angle.clone().requires_grad_(True)
    tor = g.torsion.clone().requires_grad_(True) if tors else None
    d_s = _layer_grads(g.n_triplets, 110, 6)
    d_t = _layer_grads(g.n_triplets, 120, 6) if tors else None
    outs, ups = [], []
    for first in (0, 4):
        last = min(first + 4, 6)
        ws = [w_s6[8 * l:8 * l + 8] for l in range(first, last)]
        wt = [w_t6[8 * l:8 * l + 8] for l in range(first, last)] if tors else None
        s_l, t_l = ag.basis_project(g, bess, dist, angle, tor, (cutoff, 5, not tors, dist), basis_id, ns, NR, ws, wt)
        outs += s_l
        ups += d_s[first:last]
        if tors:
            outs += t_l
            ups += d_t[first:last]
    torch.autograd.backward(outs, ups)
    exact = _geom_reference(graph, basis_id, tors, d_s, d_t, w_s6, w_t6, extra=1)
    _check_geom((dist.grad, angle.grad, None if tor is None else tor.grad), exact,
                f"six layers basis {basis_id} torsion {tors}")


@pytest.mark.parametrize("basis_id,tors", BASES)
def test_project_bwd_geom_is_the_adjoint_of_the_tangent(basis_id, tors):
    """<d_s, W_s sbf_dot> + <d_t, W_t tbf_dot> == <ddist, dist_dot> + <dangle, angle_dot> + <dtorsion, torsion_dot>, with
    sbf_dot / tbf_dot from the tangent kernels along random geometry tangents; fp64 sums, relative to the magnitude."""
    from dig_b200 import ops
    graph = "qm9"
    g, _, cutoff = _graph(graph)
    bess, bess_dx, ns = _bases(graph, basis_id, tors)
    d_s = _layer_grads(g.n_triplets, 130)
    d_t = _layer_grads(g.n_triplets, 140) if tors else None
    w_s, w_t = _weights(ns, tors, 150)
    d_dot, a_dot = _rand(161, g.n_edges), _rand(162, g.n_triplets)
    t_dot = _rand(163, g.n_triplets) if tors else None
    _, bess_d = ops.edge_basis_tangent(g.dist, d_dot, cutoff, 5, None, basis_id, not tors, NR, ns * NR,
                                       want_rbf0=False, want_bess=True)
    sbf_d, tbf_d = ops.triplet_basis_tangent(bess, bess_d, g.angle, a_dot, g.torsion if tors else None, t_dot, g.idx_kj,
                                             basis_id, ns, NR, want_tbf=tors)
    ddist, dangle, dtors = ops.triplet_basis_project_bwd_geom(g, bess, bess_dx, basis_id, d_s, d_t, w_s, w_t, cutoff)
    dot = lambda a, b: float((a.double() * b.double()).sum())
    lhs = dot(_contract(d_s, w_s, False), sbf_d) + (dot(_contract(d_t, w_t, False), tbf_d) if tors else 0.0)
    rhs = dot(ddist, d_dot) + dot(dangle, a_dot) + (dot(dtors, t_dot) if tors else 0.0)
    tor = g.torsion if tors else None
    m = ref.basis_bwd_reference(g, cutoff, ns, bess, bess_dx, g.angle, tor, _contract(d_s, w_s, True),
                                _contract(d_t, w_t, True) if tors else None)["m"]
    mag = dot(m[0], d_dot.abs()) + dot(m[1], a_dot.abs()) + (dot(m[2], t_dot.abs()) if tors else 0.0)
    assert abs(lhs - rhs) <= 1e-5 * mag, (lhs, rhs, mag)


# ------------------------------------------------------------------------------------------------ C. torsion backward
def _tie_batch():
    """(pos, batch, cutoff): centre j = atom 0, i = atom 1 on the z axis, k = atom 2, and candidates c1 = atom 3 and
    c2 = atom 4 = c1 + (0, 0, 1): vc2 - vc1 is parallel to u = pos_i - pos_j, so u x vc1 == u x vc2 bit for bit
    (exactly representable coordinates, exact products) and the two candidates of triplet (k, j, i) give equal
    (ta, tb).  The forward takes the first one in slot order."""
    pos = torch.tensor([[0.0, 0.0, 0.0], [0.0, 0.0, 1.5], [0.5, 1.0, 0.25], [1.0, 0.0, 0.0], [1.0, 0.0, 1.0]])
    return pos, torch.zeros(5, dtype=torch.long), 5.0


def _model_graph(name):
    """The model graph, with the forward's winners g.tors_arg from the _arg variant of the geometry kernel."""
    from dig_b200 import ops
    g, pos, cutoff = _graph(name)
    key = ("arg", name)
    if key not in _CACHE:
        torsion = g.torsion.clone()
        ops.triplet_geometry_any_degree_arg(g, pos, 0)
        assert torch.equal(g.torsion, torsion), "the _arg geometry must give the model graph's torsion bits"
        _CACHE[key] = True
    return g, pos


TORSION_GRAPHS = ["qm9", "capped", "ragged", "collinear", "tie"]


@pytest.mark.parametrize("graph", TORSION_GRAPHS)
def test_torsion_bwd_search_matches_recorded_candidate_and_fp64(graph):
    from dig_b200 import ops
    g, pos = _model_graph(graph)
    n = pos.size(0)
    ei = torch.stack([g.src, g.dst]).long()
    tors_c = R.candidate_atoms(ei, n, g.tors_arg)
    _, _, t_bad = R.degenerate(pos, ei, tors_c)
    w = (_rand(7, g.n_triplets) * ~t_bad).contiguous()
    search, arg = torch.zeros_like(pos), torch.zeros_like(pos)
    ops.triplet_torsion_bwd(pos, g, w, search)
    ops.triplet_torsion_bwd_arg(pos, g, w, arg)
    torch.cuda.synchronize()
    p64 = pos.double().requires_grad_(True)
    _, _, t64 = R.geometry_at(p64, ei, n, tors_c)
    (ref64,) = torch.autograd.grad((t64 * w.double()).sum(), p64)
    scale = max(float(ref64.abs().max()), 1e-30)
    d_arg = float((search - arg).abs().max()) / scale
    d_64 = float((search.double() - ref64).abs().max()) / scale
    print(f"{graph}: |search - arg| / max {d_arg:.2e}, |search - fp64| / max {d_64:.2e}")
    # the capped molecule packs 90 atoms into a 3 A box (pairs a few hundredths of an A apart): on an H100 its dpos was
    # 8.8e-6 of max from the recorded candidates' and 1.4e-5 from fp64, so its bound is 5e-5 as for the in-degree-1000
    # hub of test_gpu_xyz_to_dat_grad.py; a different candidate is an O(1) difference either way
    tol = 5e-5 if graph == "capped" else FTOL
    _note("torsion_bwd.vs_arg (tol of max)", d_arg / tol)
    _note("torsion_bwd.vs_fp64 (tol of max)", d_64 / tol)
    assert bool(torch.isfinite(search).all())
    assert d_arg <= tol, f"{graph}: the search kernel's dpos is {d_arg:.2e} of max from the recorded candidates'"
    assert d_64 <= tol, f"{graph}: dpos is {d_64:.2e} of max from fp64 at the recorded candidates"
    if graph == "capped":
        assert int((g.row_ptr[1:] - g.row_ptr[:-1]).max()) > 32


def test_torsion_bwd_search_breaks_exact_ties_like_the_forward():
    """On the tie geometry, triplet (k = 2, j = 0, i = 1) has two candidates with bit-equal (ta, tb): the forward records
    the first (atom 3), and the search backward sends the gradient there, not to atom 4."""
    from dig_b200 import ops
    g, pos = _model_graph("tie")
    n = pos.size(0)
    ei = torch.stack([g.src, g.dst]).long()
    idx_i, idx_j, idx_k, _, _ = R.triplets(ei, n)
    t = int(((idx_i == 1) & (idx_j == 0) & (idx_k == 2)).nonzero()[0])
    u = pos[1] - pos[0]
    p3 = torch.linalg.cross(u, pos[3] - pos[0], dim=-1)
    p4 = torch.linalg.cross(u, pos[4] - pos[0], dim=-1)
    assert torch.equal(p3, p4), "the two candidates' planes must be bit-equal"
    tors_c = R.candidate_atoms(ei, n, g.tors_arg)
    assert int(tors_c[t]) == 3, "the forward records the first minimal candidate"
    w = torch.zeros(g.n_triplets, device=DEV)
    w[t] = 1.0
    search = torch.zeros_like(pos)
    ops.triplet_torsion_bwd(pos, g, w, search)
    other = g.tors_arg.clone()
    other[t] += 1                                                         # atom 4 sits in the next slot of j
    assert int(R.candidate_atoms(ei, n, other)[t]) == 4
    p64 = pos.double().requires_grad_(True)
    grads = []
    for cand in (tors_c, R.candidate_atoms(ei, n, other)):
        _, _, t64 = R.geometry_at(p64, ei, n, cand)
        grads.append(torch.autograd.grad((t64 * w.double()).sum(), p64)[0])
    scale = float(grads[0].abs().max())
    assert float((grads[0] - grads[1]).abs().max()) > 0.1 * scale             # the candidates are distinguishable
    err = float((search.double() - grads[0]).abs().max()) / scale
    _note("torsion_bwd.vs_fp64 (tol of max)", err / FTOL)
    assert err <= FTOL, err


# ------------------------------------------------------------------------------------------------ D. end to end
class _B:
    pass


def _model_case(model_name, ns, num_layers, graph):
    from dig_b200.threedgraph import method
    pos, batch, cutoff, num_graphs = _positions(graph)
    ctor = dict(energy_and_force=True, cutoff=cutoff, num_layers=num_layers)
    if model_name == "SphereNet":
        ctor["num_spherical"] = ns
    model = getattr(method, model_name)(**ctor)
    sd = formula_state_dict(model.state_dict(), seed=3)
    model.load_state_dict(sd)
    model = model.to(DEV).eval()
    z = torch.tensor([1, 6, 7, 8])[torch.arange(pos.size(0)) % 4].to(DEV)
    b = _B()
    b.z, b.pos, b.batch = z, pos.float().to(DEV), batch.long().to(DEV)
    b.num_graphs = num_graphs if num_graphs is not None else int(batch.max()) + 1
    return model, {k: v.to(DEV) for k, v in sd.items()}, b, cutoff


@pytest.mark.parametrize("model_name,ns,num_layers,graph", [
    ("SphereNet", 3, 4, "capped"),
    ("SphereNet", 7, 4, "ragged"), ("SphereNet", 3, 4, "ragged"), ("DimeNetPP", 7, 4, "ragged"),
    ("SphereNet", 7, 6, "qm9"), ("DimeNetPP", 7, 6, "qm9")])
def test_model_forces_on_graphs_the_golden_cases_miss(model_name, ns, num_layers, graph):
    """Default-width forces in eval mode against autograd over the fp32 restatement on the same GPU (the fixed CPU
    comparator differs in the torsion's self-candidate ties), and per-molecule force sums zero to the atomics spread."""
    from oracle import restated
    model, sd, b, cutoff = _model_case(model_name, ns, num_layers, graph)
    assert not model._triplet_generic
    pos = b.pos.clone().requires_grad_(True)
    b.pos = pos
    out = model(b)
    force = -torch.autograd.grad(out, pos, grad_outputs=torch.ones_like(out))[0]
    pos2 = b.pos.detach().clone().requires_grad_(True)
    kw = dict(cutoff=cutoff, num_layers=num_layers, num_graphs=b.num_graphs)
    if model_name == "SphereNet":
        kw["num_spherical"] = ns
    fwd = restated.spherenet_forward if model_name == "SphereNet" else restated.dimenetpp_forward
    r = fwd(sd, b.z, pos2, b.batch, **kw)
    f_ref = -torch.autograd.grad(r.sum(), pos2)[0]
    assert bool(torch.isfinite(force).all())
    e_err = rel_err(out.detach().cpu().numpy(), r.detach().cpu().numpy())
    f_err = rel_err(force.cpu().numpy(), f_ref.cpu().numpy())
    print(f"{model_name} ns {ns} L {num_layers} {graph}: energy {e_err:.2e}, force {f_err:.2e} of max")
    _note("model.forces (FTOL of max)", f_err / FTOL)
    assert e_err < 1e-5 and f_err < FTOL, (e_err, f_err)
    net = torch.zeros(b.num_graphs, 3, dtype=torch.float64, device=DEV).index_add_(0, b.batch, force.double())
    absum = torch.zeros(b.num_graphs, 3, dtype=torch.float64, device=DEV).index_add_(0, b.batch, force.double().abs())
    assert bool((net.abs() <= 1e-5 * absum.clamp_min(1e-30) + 1e-30).all()), (net, absum)


def test_report_worst_ratios():
    """Largest |got - exact| / bound per kernel output over everything above (shown with -s)."""
    for name in sorted(WORST):
        print(f"worst |got - exact| / bound  {name:36s} {WORST[name]:.4f}")
    assert all(r <= 1.0 for r in WORST.values())
