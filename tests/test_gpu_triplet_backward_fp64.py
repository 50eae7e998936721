"""The triplet-stage backward kernels of SphereNet / DimeNet++ training, one by one and element by element against fp64.

    ops.sphere_triplet_gather (warp and edge kernels) / ops.sphere_triplet_gather_bwd  ag.triplet_gather
    ops.triplet_basis_project_bwd                                                      ag.basis_project
    ops.rbf_freq_grad                                                                  ag.edge_basis

References, magnitudes (sum |terms|) and the rounding counts of every output: tests/triplet_backward_ref.py (checked
without a device by tests/test_triplet_backward_reference_cpu.py).  Graphs: A the benchmark shape (128 QM9-like molecules:
the persistent grid-stride loops run many times), B a molecule on which the neighbour cap binds (in-degree 33, the
target of an edge absent from its source's in-list, > 32 atoms per molecule) next to a 40-atom one, C a ragged batch
(isolated atoms, a single atom, a diatomic without triplets, an empty graph slot, a quadruple), a three-atom batch with
fewer edges than one CTA has warps, and D the two golden SphereNet cases (bases (7, 6) and (3, 6)).
On B the gather backward's `p_i == d` side (i absent from j's in-list) and its second 32-lane chunk are taken; the
projection backward's `i_in` guard cannot be decided by any graph of the radius-graph build (a cut i sorts after every
kept in-neighbour of j -- asserted in test_triplet_backward_reference_cpu.py), so B pins its index arithmetic only on
the reachable side.
Run with -s to see the largest |got - exact| / bound per output."""
import math

import pytest
import torch

import triplet_backward_ref as ref
from helpers import case_inputs

pytestmark = pytest.mark.gpu
GRAPHS = ["A", "B", "C", "tiny", "qm9", "ns3"]
WORST = {}
_CACHE = {}


def _note(name, ratio):
    WORST[name] = max(WORST.get(name, 0.0), ratio)


def _graph(name):
    """Graph + triplet geometry + materialised bases, built once per module."""
    from dig_b200 import ops
    if name in _CACHE:
        return _CACHE[name]
    from dig_b200.data import synthetic_batch
    dev = torch.device("cuda:0")
    ns, basis_id, num_graphs = 7, 0, None
    if name == "A":
        b = synthetic_batch(128, "qm9", seed=3)
        pos, batch, cutoff = b.pos, b.batch, 5.0
    elif name == "B":
        pos, batch, cutoff = ref.capped_batch()
    elif name == "C":
        pos, batch, cutoff, num_graphs = ref.ragged_batch()
    elif name == "tiny":
        pos, batch, cutoff = ref.tiny_batch()
    else:
        _, _, pos, batch = case_inputs("spherenet_" + name)
        cutoff = 5.0
        if name == "ns3":
            ns, basis_id = 3, 1
    pos, batch = pos.float().contiguous().to(dev), batch.long().to(dev)
    g = ops.build_graph(pos, batch, cutoff, num_graphs=num_graphs)
    ops.triplet_geometry(g, pos, use_torsion=True, want_idx=True, want_idx64=True)
    freq = (torch.arange(1, 7, dtype=torch.float32) * math.pi).to(dev)
    out = dict(g=g, ns=ns, basis_id=basis_id, cutoff=cutoff, freq=freq, name=name)
    for tors in (True, False):
        # SphereNet keeps the envelope off the Bessel basis, DimeNet++ folds it in (the values are inputs here)
        _, bess = ops.edge_basis(g.dist, cutoff, 5, freq, basis_id, not tors, 6, ns * 6)
        # near-coincident atoms of the dense box: the closed-form Bessel values of high order cancel catastrophically
        # in fp32 there; keep the inputs finite and moderate
        bess = torch.nan_to_num(bess, nan=0.0, posinf=0.0, neginf=0.0).clamp_(-100.0, 100.0)
        sbf, tbf = ops.triplet_basis(bess, g.angle, g.torsion, g.idx_kj, basis_id, ns, 6, tors)
        out[tors] = (bess, sbf, tbf)
    torch.cuda.synchronize()
    _CACHE[name] = out
    return out


def _rand(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to("cuda:0")


def _gather_inputs(G, tors):
    g = G["g"]
    e, t = g.n_edges, g.n_triplets
    x, s = _rand(11, e, 64), _rand(12, t, 8)
    tp = _rand(13, t, 8) if tors else None
    ws = _rand(14, 64, 8) * 0.35
    wt = _rand(15, 64, 8) * 0.35 if tors else None
    dm = _rand(16, e, 64) * torch.logspace(-9, 0, 64, device="cuda:0")     # small channels are really checked
    return x, s, tp, ws, wt, dm.contiguous()


def _gather_ref(G, tors):
    key = ("gather", G["name"], tors)
    if key not in _CACHE:
        g = G["g"]
        x, s, tp, ws, wt, dm = _gather_inputs(G, tors)
        _CACHE[key] = (ref.gather_reference(x, s, tp, ws, wt, g.idx_kj64, g.idx_ji64, g.n_edges, dm),
                       ref.gather_counts(g.idx_kj64, g.idx_ji64, g.n_edges, tors))
    return _CACHE[key]


def _check_gather_bwd(outs, exact, counts, tors, tag):
    names = ["dx", "d_sbf_p", "d_t_p", "dw_sbf2", "dw_t2"]
    for name, got in zip(names, outs):
        if exact[name] is None:
            assert got is None, name
            continue
        v, m = exact[name]
        _note("gather_bwd." + name, ref.check(got, v, ref.bound(m, counts[name]), f"{tag} {name}"))


# ------------------------------------------------------------------------------------------------ the gather
@pytest.mark.parametrize("tors", [True, False], ids=["torsion", "no_torsion"])
@pytest.mark.parametrize("graph", GRAPHS)
def test_triplet_gather_forward_warp_and_edge_kernels(graph, tors):
    from dig_b200 import ops
    G = _graph(graph)
    x, s, tp, ws, wt, _ = _gather_inputs(G, tors)
    exact, counts = _gather_ref(G, tors)
    v, m = exact["m"]
    g = G["g"]
    got = {"warp": ops.sphere_triplet_gather(x, s, tp, g, ws, wt), "edge": torch.empty(g.n_edges, 64, device="cuda:0")}
    ops.call("dig3d_sphere_triplet_gather", ops._p(x), ops._p(s), ops._p(tp), 8, ops._p(g.src), ops._p(g.dst),
             ops._p(g.row_ptr), ops._p(g.trip_ptr), g.n_edges, ops._p(ws), ops._p(wt), ops._p(got["edge"]),
             ops._stream())
    for mode in ("warp", "edge"):
        _note("gather_fwd.m", ref.check(got[mode], v, ref.bound(m, counts["m"]), f"{graph} m ({mode})"))
    assert torch.equal(got["warp"], got["edge"])
    torch.cuda.synchronize()
    assert ops.tc_timeouts() == 0


@pytest.mark.parametrize("tors", [True, False], ids=["torsion", "no_torsion"])
@pytest.mark.parametrize("graph", GRAPHS)
def test_triplet_gather_backward_all_outputs(graph, tors):
    from dig_b200 import ops
    G = _graph(graph)
    x, s, tp, ws, wt, dm = _gather_inputs(G, tors)
    exact, counts = _gather_ref(G, tors)
    first = ops.sphere_triplet_gather_bwd(dm, x, s, tp, G["g"], ws, wt)
    _check_gather_bwd(first, exact, counts, tors, graph)
    # d sbf_p / d t_p are written, not accumulated: the same bits every run; the atomic outputs stay within the bound
    again = ops.sphere_triplet_gather_bwd(dm, x, s, tp, G["g"], ws, wt)
    _check_gather_bwd(again, exact, counts, tors, graph + " (second run)")
    assert torch.equal(first[1], again[1])
    if tors:
        assert torch.equal(first[2], again[2])
    torch.cuda.synchronize()


@pytest.mark.parametrize("tors", [True, False], ids=["torsion", "no_torsion"])
@pytest.mark.parametrize("graph", ["B", "C", "qm9"])
def test_triplet_gather_function(graph, tors):
    """ag.triplet_gather: forward value, x_down.grad and the parameter gradients, with a non-contiguous upstream."""
    from dig_b200 import autograd as ag, ops
    G = _graph(graph)
    x, s, tp, ws, wt, dm = _gather_inputs(G, tors)
    exact, counts = _gather_ref(G, tors)
    leaves = [t if t is None else t.clone().requires_grad_(True) for t in (x, s, tp, ws, wt)]
    out = ag.triplet_gather(*leaves, G["g"])
    _note("gather_fwd.m", ref.check(out, exact["m"][0], ref.bound(exact["m"][1], counts["m"]), f"{graph} Function m"))
    wide = torch.zeros(dm.size(0), 128, device=dm.device)
    wide[:, ::2] = dm
    up = wide[:, ::2]
    assert not up.is_contiguous() and torch.equal(up, dm)
    torch.autograd.backward([out], [up])
    _check_gather_bwd([None if t is None else t.grad for t in leaves], exact, counts, tors, f"{graph} Function")
    torch.cuda.synchronize()
    assert ops.tc_timeouts() == 0


# ------------------------------------------------------------------------------------------------ the projection
def _project_grads(G, tors):
    t = G["g"].n_triplets
    scale = torch.logspace(-6, 0, 8, device="cuda:0")
    d_s = [(_rand(30 + l, t, 8) * scale).contiguous() for l in range(4)]
    d_t = [(_rand(40 + l, t, 8) * scale).contiguous() for l in range(4)] if tors else None
    return d_s, d_t


def _run_project_bwd(G, tors, d_s, d_t):
    from dig_b200 import ops
    ns = G["ns"]
    bess = G[tors][0]
    return ops.triplet_basis_project_bwd(G["g"], bess, G["basis_id"], d_s, d_t, ns * 6, ns * ns * 6)


def _check_project(G, tors, got, d_s, d_t, tag):
    g = G["g"]
    _, sbf, tbf = G[tors]
    exact = ref.project_reference(sbf, tbf, d_s, d_t)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    c = ref.project_count(g.idx_kj64, g.n_edges, n_sm)
    for name, out in zip(("dw_sbf1", "dw_t1"), got):
        if exact[name] is None:
            assert out is None, name
            continue
        v, m = exact[name]
        _note("project_bwd." + name, ref.check(out, v, ref.bound(m, c), f"{tag} {name}"))
    return exact


@pytest.mark.parametrize("tors", [True, False], ids=["torsion", "no_torsion"])
@pytest.mark.parametrize("graph", GRAPHS)
def test_basis_project_backward_layer_configurations(graph, tors):
    G = _graph(graph)
    d_s, d_t = _project_grads(G, tors)
    sub = lambda lst, idx: None if lst is None else [lst[i] if i in idx else None for i in range(max(idx) + 1)]
    for n_layers in (4, 2, 1):                      # a shorter list leaves the remaining slots of the kernel NULL
        keep = range(n_layers)
        got = _run_project_bwd(G, tors, sub(d_s, keep), sub(d_t, keep))
        _check_project(G, tors, got, sub(d_s, keep), sub(d_t, keep), f"{graph} {n_layers} layers")
        for out in got:
            if out is not None and n_layers < 4:
                assert float(out[8 * n_layers:].abs().max()) == 0.0
    # layers 1 and 3 without a gradient: their rows are exactly zero, the others as with explicit zero tensors
    skipped = _run_project_bwd(G, tors, sub(d_s, (0, 2)) + [None], None if d_t is None else sub(d_t, (0, 2)) + [None])
    _check_project(G, tors, skipped, sub(d_s, (0, 2)), sub(d_t, (0, 2)), f"{graph} layers 1, 3 skipped")
    zero = lambda lst: None if lst is None else [lst[0], torch.zeros_like(lst[1]), lst[2], torch.zeros_like(lst[3])]
    zeroed = _run_project_bwd(G, tors, zero(d_s), zero(d_t))
    exact = _check_project(G, tors, zeroed, zero(d_s), zero(d_t), f"{graph} layers 1, 3 zero")
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    c = ref.project_count(G["g"].idx_kj64, G["g"].n_edges, n_sm)
    for name, a, b in zip(("dw_sbf1", "dw_t1"), skipped, zeroed):
        if a is None:
            continue
        for l in (1, 3):
            assert float(a[8 * l:8 * l + 8].abs().max()) == 0.0 and float(b[8 * l:8 * l + 8].abs().max()) == 0.0, (name, l)
        # the live rows are accumulated by atomics in an order that varies from run to run, so two runs agree to the
        # rounding of the sums (twice the bound between them), not bit for bit
        assert ((a.double() - b.double()).abs() <= 2 * ref.bound(exact[name][1], c)).all(), name
    torch.cuda.synchronize()


@pytest.mark.parametrize("tors", [True, False], ids=["torsion", "no_torsion"])
@pytest.mark.parametrize("graph", ["B", "tiny", "ns3"])
def test_basis_project_function(graph, tors):
    """ag.basis_project with separate requires_grad weights per layer: the forward against the materialised basis (with
    the harmonic-recurrence term), then weight.grad per layer; layer 1 of sbf and layers 1, 3 of t get no gradient."""
    from dig_b200 import autograd as ag, ops
    G = _graph(graph)
    g, ns = G["g"], G["ns"]
    bess, sbf, tbf = G[tors]
    w_s = [(_rand(50 + l, 8, ns * 6) * 0.3).requires_grad_(True) for l in range(4)]
    w_t = [(_rand(60 + l, 8, ns * ns * 6) * 0.1).requires_grad_(True) for l in range(4)] if tors else None
    geo_cfg = (G["cutoff"], 5, not tors, g.dist)
    s_l, t_l = ag.basis_project(g, bess, g.dist, g.angle, g.torsion if tors else None, geo_cfg, G["basis_id"], ns, 6,
                                w_s, w_t)
    bess_kj = bess[g.idx_kj64]
    for name, outs, basis, ws in (("sbf_p", s_l, sbf, w_s), ("t_p", t_l, tbf, w_t)):
        if outs is None:
            continue
        v, lim = ref.project_forward_bound(basis, bess_kj, torch.cat([w.detach() for w in ws], 0), 6)
        _note("project_fwd." + name, ref.check(torch.cat(outs, 1), v, lim, f"{graph} Function {name}"))
    d_s, d_t = _project_grads(G, tors)
    d_s[1] = None
    if tors:
        d_t[1] = d_t[3] = None
    loss_terms = [(o, d) for o, d in zip(s_l, d_s) if d is not None]
    if tors:
        loss_terms += [(o, d) for o, d in zip(t_l, d_t) if d is not None]
    # upstream gradients as non-contiguous column slices of a wider buffer
    ups = []
    for _, d in loss_terms:
        wide = torch.zeros(d.size(0), 16, device=d.device)
        wide[:, 1::2] = d
        ups.append(wide[:, 1::2])
    torch.autograd.backward([o for o, _ in loss_terms], ups)
    exact = ref.project_reference(sbf, tbf, d_s, d_t)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    c = ref.project_count(g.idx_kj64, g.n_edges, n_sm)
    for name, ws, ds in (("dw_sbf1", w_s, d_s), ("dw_t1", w_t, d_t)):
        if ws is None:
            continue
        v, m = exact[name]
        for l, (w, d) in enumerate(zip(ws, ds)):
            if d is None:
                assert w.grad is None, (name, l)
                continue
            _note("project_bwd." + name, ref.check(w.grad, v[8 * l:8 * l + 8], ref.bound(m[8 * l:8 * l + 8], c),
                                                   f"{graph} Function {name} layer {l}"))
    torch.cuda.synchronize()
    assert ops.tc_timeouts() == 0


# ------------------------------------------------------------------------------------------------ d freq
def _freq_inputs(n_edges, cutoff):
    last = float(torch.nextafter(torch.tensor(cutoff, dtype=torch.float32), torch.tensor(0.0)))
    dist = torch.linspace(1e-3 * cutoff, cutoff, n_edges, dtype=torch.float64).float() if n_edges > 1 else torch.tensor([last])
    dist = dist.clamp(max=last)[torch.randperm(n_edges, generator=torch.Generator().manual_seed(n_edges))]
    assert float(dist.max()) == last < cutoff
    freq = torch.arange(1, 7, dtype=torch.float32) * math.pi + 0.01 * torch.randn(6, generator=torch.Generator().manual_seed(5))
    return dist.to("cuda:0"), freq.to("cuda:0"), _rand(70 + n_edges % 97, n_edges, 6)      # mixed signs: the sum cancels


@pytest.mark.parametrize("exponent", [5, 2, 4])
@pytest.mark.parametrize("n_edges", [1, 31, 257, 592 * 256 + 1000])
def test_rbf_freq_grad(n_edges, exponent):
    from dig_b200 import ops
    cutoff = 5.0
    dist, freq, drbf0 = _freq_inputs(n_edges, cutoff)
    got = ops.rbf_freq_grad(dist, cutoff, exponent, freq, drbf0)
    v, m1, m2 = ref.freq_reference(dist, freq, cutoff, exponent, drbf0)
    c1, c2 = ref.freq_counts(n_edges, exponent)
    limit = ref.U * (c1 * m1 + c2 * m2) / (1 - c1 * ref.U) + c1 * ref.ETA
    _note("rbf_freq_grad.dfreq", ref.check(got, v, limit, f"dfreq E={n_edges} exponent={exponent}"))
    if n_edges > 1:
        assert float((v.abs() / m1).min()) < 0.5                           # the sum did cancel
    torch.cuda.synchronize()


@pytest.mark.parametrize("tors", [True, False], ids=["torsion", "no_torsion"])
def test_edge_basis_function(tors):
    """ag.edge_basis: freq.grad from a non-contiguous d rbf0, on the edges of the capped graph."""
    from dig_b200 import autograd as ag
    G = _graph("B")
    g = G["g"]
    freq = G["freq"].clone().requires_grad_(True)
    rbf0, bess = ag.edge_basis(freq, g.dist, G["cutoff"], 5, G["basis_id"], not tors, 6, 42)
    assert not bess.requires_grad
    wide = _rand(81, g.n_edges, 12)
    up = wide[:, ::2]
    assert not up.is_contiguous()
    rbf0.backward(gradient=up)
    v, m1, m2 = ref.freq_reference(g.dist, freq, G["cutoff"], 5, up)
    c1, c2 = ref.freq_counts(g.n_edges, 5)
    limit = ref.U * (c1 * m1 + c2 * m2) / (1 - c1 * ref.U) + c1 * ref.ETA
    _note("rbf_freq_grad.dfreq", ref.check(freq.grad, v, limit, "Function dfreq"))
    torch.cuda.synchronize()


def test_report_worst_ratios():
    """Largest |got - exact| / bound per kernel output over everything above (shown with -s)."""
    for name in sorted(WORST):
        print(f"worst |got - exact| / bound  {name:24s} {WORST[name]:.4f}")
    assert all(r <= 1.0 for r in WORST.values())
