"""SchNet's kernels and the force-path kernels it uses, element by element against an fp64 restatement.

    dig3d_schnet_block (through ops.call, with buffers the test owns)   vlin = lin(v), agg = cfconv, v_out = update_v
    ops.schnet_readout + ops.segment_sum                                update_u and the per-graph sum
    ops.schnet_edge_features / _bwd / _bwd2                             Gaussians and cosine cutoff, first / second order
    ops.edge_dist_bwd / edge_dist_bwd2 / geometry_jvp's dist_dot        the edge length, reverse / second / forward order
    ops.rowdot

Every boundary is restated in fp64 from the KERNEL'S OWN fp32 inputs (schnet.py:24-103 of the reference, the op
sequence of oracle/restated.py's schnet_forward), and each output y must satisfy |y - y64| <= e for every element, e
being the running bound of tests/fp64_bound.py (the rounding model of each op is that module's docstring).

Graphs (SchNet's radius graph keeps 32 neighbours per target, 33 when the atom itself is not among the first 33
candidates, as the reference's radius_graph counts it): a 6-edge batch, one of exactly 64 and 128 edges,
a ragged batch (an isolated atom, an empty graph slot, two coincident atoms, pairs at 0.99 - 1.0 x cutoff), the
benchmark's first batch (16 x 12 atoms, cutoff 10: 33 tiles of 64 edges) and a 48-atom cluster in a 3 A box behind a
diatomic, so every target of the cluster has 32 or 33 in-edges and its segments start two edges into a tile (many
cross a tile boundary).  Weights: the formula weights, and mlp.0 scaled by 300 so that ssp's pre-activations cross 20
and go below -88.  Far Gaussians underflow into subnormals.  Run with -s to see the largest |y - y64| / e per output."""
import ctypes
import math

import pytest
import torch

from fp64_bound import ETA, PI_F, U, Bounded, add, cutoff_fn, f32, gauss, index_add, linear, mul, ssp
from helpers import case_inputs, formula_state_dict

pytestmark = pytest.mark.gpu
CUTOFF = 10.0
WORST = {}
_CACHE = {}


def _note(name, ratio):
    WORST[name] = max(WORST.get(name, 0.0), ratio)


def _b(v, e):
    return Bounded(v, v.abs(), e)


def _graph(name):
    """(pos, batch, num_graphs, graph) on cuda:0, built by the model's own radius graph."""
    from dig_b200 import ops
    if name in _CACHE:
        return _CACHE[name]
    gen = torch.Generator().manual_seed(5)
    mols = []                                        # (atoms [n, 3]) per graph slot; None = empty slot
    if name == "small":                              # 3 atoms: 6 edges
        mols = [torch.rand(3, 3, generator=gen) * 2]
    elif name in ("e64", "e128"):                    # 8 + 2 + 3 atoms, all within the cutoff: 56 + 2 + 6 = 64 edges
        mols = [torch.rand(k, 3, generator=gen) * 3 for k in (8, 2, 3)] * (1 if name == "e64" else 2)
    elif name == "ragged":
        mols = [torch.zeros(1, 3),                                       # isolated atom
                None,                                                    # empty graph slot
                torch.tensor([[1.0, 2.0, 3.0], [1.0, 2.0, 3.0]]),         # coincident atoms: d = 0
                torch.tensor([[0.0, 0.0, 0.0], [0.995 * CUTOFF, 0.0, 0.0]]),
                torch.tensor([[0.0, 0.0, 0.0], [0.0, 0.9999 * CUTOFF, 0.0], [0.0, 0.0, 0.99 * CUTOFF]]),
                torch.rand(7, 3, generator=gen) * 12]                   # some pairs beyond the cutoff
    elif name == "dense":                            # diatomic, then 48 atoms in a 3 A box: the cap binds everywhere
        mols = [torch.tensor([[0.0, 0.0, 0.0], [1.1, 0.0, 0.0]]), torch.rand(48, 3, generator=gen) * 3]
    if name == "cfg1":
        _, z, pos, batch = case_inputs("schnet_cfg1", "cuda:0")
        ng = int(batch.max()) + 1
    else:
        pos = torch.cat([m for m in mols if m is not None]).float()
        batch = torch.cat([torch.full((m.size(0),), i) for i, m in enumerate(mols) if m is not None])
        ng = len(mols)
        z = torch.randint(1, 10, (pos.size(0),), generator=gen)
        pos, batch, z = pos.to("cuda:0"), batch.to("cuda:0"), z.to("cuda:0")
    g = ops.build_graph(pos, batch, CUTOFF, num_graphs=ng, want_edge_index=False)
    _CACHE[name] = (z, pos, batch, ng, g)
    return _CACHE[name]


GRAPHS = ["small", "e64", "e128", "ragged", "cfg1", "dense"]


def test_graphs_cover_the_regimes():
    sizes = {n: _graph(n)[4].n_edges for n in GRAPHS}
    assert sizes["small"] == 6 and sizes["e64"] == 64 and sizes["e128"] == 128 and sizes["cfg1"] % 64 == 0, sizes
    g = _graph("ragged")[4]
    d = g.dist.cpu()
    assert (d == 0).sum() == 2 and ((d > 0.99 * CUTOFF) & (d <= CUTOFF)).sum() >= 4
    g = _graph("dense")[4]
    deg = (g.row_ptr[1:] - g.row_ptr[:-1]).cpu()
    assert deg[2:].min() >= 32 and deg.max() <= 33                    # the cap binds on every atom of the cluster
    start = g.row_ptr[2:-1].cpu()
    assert ((start % 64) + deg[2:] > 64).sum() >= 20                    # segments split across two tiles


# ------------------------------------------------------------------------------------------------ the fused block
def _model(hidden, n_gauss, scaled):
    from dig_b200.threedgraph.method import SchNet
    model = SchNet(num_layers=1, hidden_channels=hidden, num_filters=hidden, num_gaussians=n_gauss, cutoff=CUTOFF)
    sd = formula_state_dict(model.state_dict(), seed=hidden + n_gauss)
    if scaled:
        sd["update_es.0.mlp.0.weight"] = sd["update_es.0.mlp.0.weight"] * 300.0
    model.load_state_dict(sd)
    return model.to("cuda:0").eval()


def _block(model, v, g):
    """dig3d_schnet_block with buffers the test owns: (vlin, agg, v_out).  NaN-filled outputs catch unwritten rows."""
    from dig_b200 import ops
    n, h = v.shape
    ue, uv = model.update_es[0], model.update_vs[0]
    w, padded = ops.pack_schnet_block(ue, uv)
    vlin = torch.full((n, h), float("nan"), device=v.device)
    agg = torch.zeros(n, h, device=v.device)
    v_out = torch.full((n, h), float("nan"), device=v.device)
    off = model.dist_emb.offset
    ops.call("dig3d_schnet_block", ops._p(v, torch.float32, "v", 16), n, ops._p(g.dist), ops._p(g.src), ops._p(g.dst),
             g.n_edges, ops._p(off, torch.float32), off.numel(), float(model.dist_emb.coeff), float(CUTOFF), h, h,
             ctypes.byref(w), ops._p(vlin), ops._p(agg), ops._p(v_out), ops._stream())
    torch.cuda.synchronize()
    del padded
    return vlin, agg, v_out


def _block64(model, v, g, vlin_k, agg_k):
    """vlin = v W^T;  agg_i = sum_{j -> i} vlin_k[j] * (lin2(ssp(lin0(gauss(d)))) * C(d));
    v_out = v + lin2(ssp(lin1(agg_k)))."""
    ue, uv = model.update_es[0], model.update_vs[0]
    n = v.size(0)
    vlin = linear(Bounded.exact(v), ue.lin.weight, None, "fp32")
    dist = g.dist
    pre = linear(gauss(dist, model.dist_emb.offset, model.dist_emb.coeff), ue.mlp[0].weight, ue.mlp[0].bias, "fp32")
    filt = mul(linear(ssp(pre), ue.mlp[2].weight, ue.mlp[2].bias, "fp32"), cutoff_fn(dist, CUTOFF)[:, None])
    agg = index_add(mul(Bounded.exact(vlin_k)[g.src.long()], filt), g.dst, n)
    t = ssp(linear(Bounded.exact(agg_k), uv.lin1.weight, uv.lin1.bias, "fp32"))
    v_out = add(Bounded.exact(v), linear(t, uv.lin2.weight, uv.lin2.bias, "fp32"))
    return vlin, agg, v_out, pre


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("n_gauss", [2, 50, 64])
@pytest.mark.parametrize("hidden", [32, 64, 128])
@pytest.mark.parametrize("graph", GRAPHS)
def test_schnet_block_matches_fp64(graph, hidden, n_gauss, scaled):
    z, pos, batch, ng, g = _graph(graph)
    model = _model(hidden, n_gauss, scaled)
    v = model.init_v.weight.detach()[z].contiguous()
    vlin, agg, v_out = _block(model, v, g)
    r_vlin, r_agg, r_out, pre = _block64(model, v, g, vlin, agg)
    if scaled and graph == "cfg1":
        assert (pre.v > 20).any() and (pre.v < -88).any()
    tag = f"{graph} H={hidden} G={n_gauss}{' scaled' if scaled else ''}"
    _note("schnet_block.vlin", r_vlin.check(vlin, f"vlin {tag}"))
    _note("schnet_block.agg", r_agg.check(agg, f"agg {tag}"))
    _note("schnet_block.v_out", r_out.check(v_out, f"v_out {tag}"))


@pytest.mark.parametrize("hidden", [32, 64, 128])
def test_schnet_block_is_deterministic_at_the_cap(hidden):
    """Segments split across two tiles take two atomics onto a zeroed row: the first is exact, so the order does not
    matter and v_out has the same bits on every run (dense.cuh, tile_segment_accumulate)."""
    z, pos, batch, ng, g = _graph("dense")
    model = _model(hidden, 50, True)
    v = model.init_v.weight.detach()[z].contiguous()
    runs = [_block(model, v, g) for _ in range(3)]
    for r in runs[1:]:
        assert torch.equal(r[1], runs[0][1]) and torch.equal(r[2], runs[0][2])


# ------------------------------------------------------------------------------------------------ readout
@pytest.mark.parametrize("scale", [1.0, 100.0])
@pytest.mark.parametrize("out_channels", [1, 3])
@pytest.mark.parametrize("hidden", [32, 64, 128])
def test_schnet_readout_and_graph_sum_match_fp64(hidden, out_channels, scale):
    from dig_b200 import ops
    from dig_b200.threedgraph.method.schnet import update_u
    uu = update_u(hidden, out_channels)
    sd = formula_state_dict(uu.state_dict(), seed=hidden + out_channels)
    uu.load_state_dict(sd)
    uu = uu.to("cuda:0")
    gen = torch.Generator().manual_seed(hidden)
    sizes = [3, 0, 1, 40, 7, 0, 12]                  # empty graph slots in the middle and at the end
    ptr = torch.tensor([0] + sizes).cumsum(0).to(torch.int32)
    n = int(ptr[-1])
    v = (torch.randn(n, hidden, generator=gen) * 10.0 ** (torch.rand(n, 1, generator=gen) * 3 - 2) * scale).float()
    v, ptr = v.to("cuda:0"), ptr.to("cuda:0")
    node = ops.schnet_readout(v, uu.lin1, uu.lin2, out_channels)
    energy = ops.segment_sum(node, ptr)
    torch.cuda.synchronize()
    pre = linear(Bounded.exact(v), uu.lin1.weight, uu.lin1.bias, "fp32")
    if scale > 1:
        assert (pre.v > 20).any() and (pre.v < -88).any()
    r_node = linear(ssp(pre), uu.lin2.weight, uu.lin2.bias, "fp32")
    tag = f"H={hidden} out={out_channels} scale={scale}"
    _note("schnet_readout", r_node.check(node, f"readout {tag}"))
    gid = torch.repeat_interleave(torch.arange(len(sizes), device="cuda:0"), (ptr[1:] - ptr[:-1]).long())
    r_e = index_add(Bounded.exact(node), gid, len(sizes))
    _note("segment_sum(graph_ptr)", r_e.check(energy, f"graph sum {tag}"))
    assert (energy[1] == 0).all() and (energy[-2] == 0).all()


# ------------------------------------------------------------------------------------------------ edge features
def _dists(cutoff, seed=3):
    """Coincident atoms, tiny, random and 0.99 - 1.0 x cutoff distances; 1000 + ragged many."""
    gen = torch.Generator().manual_seed(seed)
    d = torch.cat([torch.zeros(3), torch.tensor([1e-30, 1e-7, 1e-3]), torch.rand(1000, generator=gen) * cutoff,
                   cutoff * (0.99 + 0.01 * torch.rand(77, generator=gen)), torch.tensor([cutoff])]).float()
    return d.to("cuda:0"), gen


def _gauss_d1(dist, offset, coeff):
    """gauss' = 2 c t expf(c t^2) as (expf(.) * 2 c) * t: value and bound [E, G]."""
    ga = gauss(dist, offset, coeff)
    c = f32(coeff)
    t = dist.double()[:, None] - offset.double()[None, :]
    v = 2 * c * t * ga.v
    rel = (ga.e - 4 * ETA) / ga.v.clamp_min(1e-300) + 4 * U
    return v, v.abs() * rel + 2 * abs(c * t) * 4 * ETA + 3 * ETA


def _gauss_d2(dist, offset, coeff):
    """gauss'' = (2c + 4 c^2 t^2) expf(c t^2): the sum can cancel, so its error is relative to 2|c| + 4 c^2 t^2."""
    ga = gauss(dist, offset, coeff)
    c = f32(coeff)
    t = dist.double()[:, None] - offset.double()[None, :]
    q = 2 * c + 4 * c * c * t * t
    mag = 2 * abs(c) + 4 * c * c * t * t
    v = q * ga.v
    e = q.abs() * ga.e + 7 * U * mag * (ga.v + ga.e) + 2 * ETA
    return v, e


def _cut_d(dist, cutoff, order):
    """cut' = -0.5 w sin(d w), cut'' = -0.5 w^2 cos(d w), w = fp32(pi_f inv_f): value and bound [E]."""
    w = PI_F * f32(1.0 / cutoff)
    x = dist.double() * w
    ex = 3 * U * x.abs()
    f, fd = (torch.sin(x), torch.cos(x)) if order == 1 else (torch.cos(x), torch.sin(x))
    k = -0.5 * w ** order
    v = k * f
    return v, abs(k) * (fd.abs() * ex + ex * ex / 2 + 4 * U * f.abs() + (order + 2) * U * (f.abs() + ex)) + 2 * ETA


@pytest.mark.parametrize("n_gauss", [2, 50, 64, 70])
def test_schnet_edge_features_and_their_derivatives_match_fp64(n_gauss):
    from dig_b200 import ops
    d, gen = _dists(CUTOFF, seed=n_gauss)
    offset = torch.linspace(0.0, CUTOFF, n_gauss).to("cuda:0")
    coeff = -0.5 / (offset[1] - offset[0]).item() ** 2
    e_, tag = d.numel(), f"G={n_gauss}"
    gs, cut = ops.schnet_edge_features(d, offset, coeff, CUTOFF)
    torch.cuda.synchronize()
    r_g = gauss(d, offset, coeff)
    assert ((r_g.v > 0) & (r_g.v < 2.0 ** -126)).any() or n_gauss == 2
    _note("schnet_edge_features.gauss", r_g.check(gs, f"gauss {tag}"))
    _note("schnet_edge_features.cut", cutoff_fn(d, CUTOFF).check(cut, f"cut {tag}"))

    dg = torch.randn(e_, n_gauss, generator=gen).float().to("cuda:0")
    dc = torch.randn(e_, generator=gen).float().to("cuda:0")
    gg = (torch.randn(e_, generator=gen) * 10.0 ** (torch.rand(e_, generator=gen) * 4 - 2)).float().to("cuda:0")
    ddist = ops.schnet_edge_features_bwd(d, offset, coeff, CUTOFF, dg, dc)
    d_dg, d_dc, d_d = ops.schnet_edge_features_bwd2(d, offset, coeff, CUTOFF, dg, dc, gg)
    torch.cuda.synchronize()
    dg64, dc64, gg64 = dg.double(), dc.double(), gg.double()
    n_terms = n_gauss + 1                                    # fmas from zero: one rounding each of sum |terms|
    # first order: ddist = sum_k dgauss gauss_k' + dcut cut'
    g1, e1 = _gauss_d1(d, offset, coeff)
    c1, ec1 = _cut_d(d, CUTOFF, 1)
    terms = (dg64 * g1).abs().sum(1) + (dc64 * c1).abs()
    v = (dg64 * g1).sum(1) + dc64 * c1
    e = (dg64.abs() * e1).sum(1) + dc64.abs() * ec1 + n_terms * (U * (terms + (dg64.abs() * e1).sum(1)) + ETA)
    _note("schnet_edge_features_bwd", _b(v, e).check(ddist, f"ddist {tag}"))
    # second order: d_dgauss = g gauss', d_dcut = g cut', d_dist = g (sum_k dgauss gauss'' + dcut cut'')
    _note("schnet_edge_features_bwd2.d_dgauss",
          _b(gg64[:, None] * g1, gg64.abs()[:, None] * e1 * (1 + U) + U * (gg64[:, None] * g1).abs() + ETA)
          .check(d_dg, f"d_dgauss {tag}"))
    _note("schnet_edge_features_bwd2.d_dcut",
          _b(gg64 * c1, gg64.abs() * ec1 * (1 + U) + U * (gg64 * c1).abs() + ETA).check(d_dc, f"d_dcut {tag}"))
    g2, e2 = _gauss_d2(d, offset, coeff)
    c2, ec2 = _cut_d(d, CUTOFF, 2)
    terms2 = (dg64 * g2).abs().sum(1) + (dc64 * c2).abs()
    acc_e = (dg64.abs() * e2).sum(1) + dc64.abs() * ec2
    acc_e = acc_e + n_terms * (U * (terms2 + acc_e) + ETA)
    v2 = gg64 * ((dg64 * g2).sum(1) + dc64 * c2)
    e2t = gg64.abs() * acc_e + U * gg64.abs() * (terms2 + acc_e) + ETA
    _note("schnet_edge_features_bwd2.d_dist", _b(v2, e2t).check(d_d, f"d_dist {tag}"))


# ------------------------------------------------------------------------------------------------ edge length
def _edge_terms(pos, g):
    """Per edge: delta = pos_i - pos_j [E, 3] (fp64 of fp32 positions), the kernel's d [E], and the d > 0 mask."""
    p = pos.double()
    delta = p[g.dst.long()] - p[g.src.long()]
    d = g.dist.double()
    return delta, d, d > 0


def _scatter_pm(t, te, g, n):
    """sum over the edges of +t at the target, -t at the source, by atomics in any order (index_add's model)."""
    idx = torch.cat([g.dst.long(), g.src.long()])
    return index_add(Bounded(torch.cat([t, -t]), torch.cat([t.abs(), t.abs()]), torch.cat([te, te])), idx, n)


@pytest.mark.parametrize("graph", GRAPHS)
def test_edge_length_derivatives_match_fp64(graph):
    from dig_b200 import ops
    z, pos, batch, ng, g = _graph(graph)
    n, e_ = pos.size(0), g.n_edges
    gen = torch.Generator().manual_seed(e_)
    ddist = (torch.randn(e_, generator=gen) * 10.0 ** (torch.rand(e_, generator=gen) * 4 - 2)).float().to("cuda:0")
    gpos = torch.randn(n, 3, generator=gen).float().to("cuda:0")
    cvec = torch.randn(n, 3, generator=gen).float().to("cuda:0")
    dpos = torch.zeros(n, 3, device="cuda:0")
    ops.edge_dist_bwd(pos, g, ddist, dpos)
    d_ddist, d_pos = ops.edge_dist_bwd2(pos, g, ddist, gpos)
    dist_dot = ops.geometry_jvp(pos, cvec, g, want_angle=False)[0]
    torch.cuda.synchronize()
    delta, d, ok = _edge_terms(pos, g)
    dsafe = torch.where(ok, d, torch.ones_like(d))[:, None]
    okc = ok[:, None].double()
    dd = ddist.double()[:, None]
    # edge_dist_bwd: +- ddist * delta / d per edge (sub, division, product: 3u), atomics
    t = okc * dd * delta / dsafe
    r_dpos = _scatter_pm(t, 3 * U * t.abs() + ETA, g, n)
    _note("edge_dist_bwd", r_dpos.check(dpos, f"dpos {graph}"))
    # edge_dist_bwd2: u = delta * fp32(1/d) (3u), w = G_i - G_j (1u), uw = u . w (three roundings)
    u = okc * delta / dsafe
    gp = gpos.double()
    w = gp[g.dst.long()] - gp[g.src.long()]
    uw = (u * w).sum(1, keepdim=True)
    muw = (u * w).abs().sum(1, keepdim=True)
    e_uw = 7 * U * muw + 3 * ETA
    _note("edge_dist_bwd2.d_ddist", _b(uw[:, 0], e_uw[:, 0]).check(d_ddist, f"d_ddist {graph}"))
    # h = (w - u uw) * (ddist / d): magnitude |w| + |u| |uw|
    s = okc * dd / dsafe
    mag = w.abs() + u.abs() * uw.abs()
    e_in = U * w.abs() + u.abs() * e_uw + 5 * U * u.abs() * (uw.abs() + e_uw) + U * (mag + u.abs() * e_uw)
    h = s * (w - u * uw)
    r_dp = _scatter_pm(h, s.abs() * (e_in + 2 * U * (mag + e_in)) + 2 * ETA, g, n)
    _note("edge_dist_bwd2.d_pos", r_dp.check(d_pos, f"d_pos {graph}"))
    # dist_dot = (delta . dc) / d  (two subtractions, three roundings of the dot, the division)
    cv = cvec.double()
    dc = cv[g.dst.long()] - cv[g.src.long()]
    jd = okc[:, 0] * (delta * dc).sum(1) / dsafe[:, 0]
    e_jd = okc[:, 0] * (7 * U * (delta * dc).abs().sum(1) / dsafe[:, 0]) + 4 * ETA
    _note("geometry_jvp.dist_dot", _b(jd, e_jd).check(dist_dot, f"dist_dot {graph}"))
    # d = 0 (coincident atoms): exactly zero, as torch's norm subgradient
    zero = ~ok
    if zero.any():
        assert (dist_dot[zero] == 0).all() and (d_ddist[zero] == 0).all()
        atoms = torch.cat([g.src[zero], g.dst[zero]]).long()
        assert (dpos[atoms] == 0).all() and (d_pos[atoms] == 0).all()
    # adjoint: <J c, w> = <c, J^T w>, with J^T w = edge_dist_bwd(ddist = w), both sides from the kernels' outputs
    wv = ddist.double()
    lhs = float((dist_dot.double() * wv).sum())
    rhs = float((cv * dpos.double()).sum())
    slack = float((wv.abs() * e_jd).sum() + (cv.abs() * r_dpos.e).sum()
                  + 1e-12 * ((dist_dot.double() * wv).abs().sum() + (cv * dpos.double()).abs().sum()))
    assert abs(lhs - rhs) <= slack, (lhs, rhs, slack)


# ------------------------------------------------------------------------------------------------ rowdot
@pytest.mark.parametrize("rows", [1, 63, 64, 65, 10007])
@pytest.mark.parametrize("width", [1, 31, 32, 33, 128, 200])
def test_rowdot_matches_fp64(width, rows):
    """One warp per row: ceil(width / 32) fmas per lane, then five butterfly additions."""
    from dig_b200 import ops
    gen = torch.Generator().manual_seed(rows * 1000 + width)
    a = (torch.randn(rows, width, generator=gen) * 10.0 ** (torch.rand(rows, 1, generator=gen) * 6 - 3)).float()
    b = torch.randn(rows, width, generator=gen).float()
    out = ops.rowdot(a.to("cuda:0"), b.to("cuda:0"))
    torch.cuda.synchronize()
    p = a.double() * b.double()
    k = math.ceil(width / 32) + 5
    r = Bounded(p.sum(1), p.abs().sum(1), k * U * p.abs().sum(1) + k * ETA)
    _note("rowdot", r.check(out.cpu(), f"rowdot {rows}x{width}"))


def test_report_worst_ratios():
    """Largest |got - exact| / bound per kernel output over everything above (shown with -s)."""
    for name in sorted(WORST):
        print(f"worst |got - exact| / bound  {name:40s} {WORST[name]:.4f}")
    assert all(r <= 1.0 for r in WORST.values())
