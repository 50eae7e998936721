"""The SphereNet / DimeNet++ inference dense chains, element by element against an fp64 restatement.

Every kernel boundary -- init_e (three-panel and table form), update_e part A, the triplet gather (warp per source
node, at the graph's split and at pinned ones, and warp per edge), part B, part B + next part A, update_v, linear_h16
-- is restated in fp64 from the KERNEL'S OWN fp32 inputs (spherenet.py:79-91, 150-182, 209-216; the op sequence of
oracle/restated.py:229-262), so only the kernel's arithmetic is under test.  Each output element y must satisfy
|y - y64| <= e, the running error bound of tests/fp64_bound.py: TOL * M + FLOOR per layer, with M the magnitude chain
and TOL / FLOOR derived from the operand split (11-bit hi, fp16 subnormal spacing 2^-24 / H_SA and / H_SW), the
truncating wgmma accumulation of the K = 64 chunks and their fp32 sums -- the derivation is that module's docstring.
The same bound is checked for the 3xTF32 chains and the exact-fp32 FFMA twins (their own constants), so the references
the older parity tests lean on are pinned too.

Regimes: formula weights; molecules stretched so that many edges lie at 0.9-1.0 x cutoff (rbf0 -> 0: tiny rbf gates
and e2 rows); inputs scaled until the largest operand a 3xFP16 layer splits is ~4000, then ~8100 (4000 / 8100 x 1.005 at most) (the flag must stay
clear); activations ~1e-4 (the absolute floor); the dense weight matrices scaled by 2^-8, 2^-4 and 4; the exact
(libdevice) swish as well as the default MUFU form; the 3xTF32 chain at ~3e4.  Last, one operand placed exactly at
the range edge for every 3xFP16 entry point: 8189 splits, 8191 must raise the overflow flag in that launch."""
import ctypes
import re

import pytest
import torch

from fp64_bound import Bounded, add, cat, index_add, linear, mul, swish
from helpers import formula_state_dict

pytestmark = pytest.mark.gpu
CUTOFF = 5.0


# ------------------------------------------------------------------------------------------------ fp64 restatements
def _init_e(z, src, dst, rbf0, ie, n_nodes, eng, tables=False):
    """e1 = act(lin(cat[x_i, x_j, act(lin_rbf_0(rbf))])), v_in = sum over dst of lin_rbf_1(rbf) * e1."""
    x = Bounded.exact(ie.emb.weight)[z.long()]
    xi, xj = x[dst.long()], x[src.long()]
    r = Bounded.exact(rbf0)
    r0 = swish(linear(r, ie.lin_rbf_0.weight, ie.lin_rbf_0.bias, "fp32"))
    w = ie.lin.weight
    if tables:      # tab_i[z_i] + tab_j[z_j] (exact-fp32 GEMMs over the embedding) + the rbf panel on the tensor cores
        t = add(linear(xi, w[:, :128], None, "fp32"), linear(xj, w[:, 128:256], None, "fp32"))
        pre = add(add(t, linear(r0, w[:, 256:], None, eng)), Bounded.exact(ie.lin.bias))
    else:
        pre = linear(cat([xi, xj, r0]), w, ie.lin.bias, eng)
    e1 = swish(pre)
    e2 = mul(linear(r, ie.lin_rbf_1.weight, None, "fp32"), e1)
    return e1, index_add(e2, dst, n_nodes)


def _part_a(x, r, ue, eng):
    """x_ji = act(lin_ji(e1)); x_down = act(lin_down(act(lin_kj(e1)) * lin_rbf2(lin_rbf1(rbf0))))."""
    x_ji = swish(linear(x, ue.lin_ji.weight, ue.lin_ji.bias, eng))
    gate = linear(linear(r, ue.lin_rbf1.weight, None, "fp32"), ue.lin_rbf2.weight, None, "fp32")
    x_kj = mul(swish(linear(x, ue.lin_kj.weight, ue.lin_kj.bias, eng)), gate)
    return x_ji, swish(linear(x_kj, ue.lin_down.weight, None, eng))


def _gather(x_down, sbf, tp, idx_kj, idx_ji, n_edges, ue, eng):
    """m[e] = sum over the triplets t of e of x_down[kj(t)] * lin_sbf2(sbf_p[t]) (* lin_t2(t_p[t]))."""
    y = mul(Bounded.exact(x_down)[idx_kj], linear(Bounded.exact(sbf), ue.lin_sbf2.weight, None, eng))
    if tp is not None:
        y = mul(y, linear(Bounded.exact(tp), ue.lin_t2.weight, None, eng))
    return index_add(y, idx_ji, n_edges)


def _residual(h, layer, eng):
    t = swish(linear(h, layer.lin1.weight, layer.lin1.bias, eng))
    return add(h, swish(linear(t, layer.lin2.weight, layer.lin2.bias, eng)))


def _part_b(m, e1, x_ji, r, dst, n_nodes, ue, eng):
    """h = x_ji + act(lin_up(m)); residual stack; e1_out; v_in = sum over dst of lin_rbf(rbf0) * e1_out."""
    h = add(x_ji, swish(linear(m, ue.lin_up.weight, None, eng)))
    for layer in ue.layers_before_skip:
        h = _residual(h, layer, eng)
    h = add(swish(linear(h, ue.lin.weight, ue.lin.bias, eng)), e1)
    for layer in ue.layers_after_skip:
        h = _residual(h, layer, eng)
    return h, index_add(mul(linear(r, ue.lin_rbf.weight, None, "fp32"), h), dst, n_nodes)


def _update_v(v_in, holder, eng):
    v = linear(Bounded.exact(v_in), holder.lin_up.weight, holder.lin_up.bias, eng)
    for lin in holder.lins:
        v = swish(linear(v, lin.weight, lin.bias, eng))
    return linear(v, holder.lin.weight, None, "fp32")


# ------------------------------------------------------------------------------------------------ models, inputs
_DENSE = re.compile(r"^(update_es\.\d+\.(lin_ji|lin_kj|lin_down|lin_up|lin|layers_\w+_skip\.\d+\.lin[12])"
                    r"|init_e\.lin|(init_v|update_vs\.\d+)\.(lin_up|lins\.\d+))\.(weight|bias)$")


def _model(cls_name, ws=1.0, bs=1.0, edit=None, **kw):
    """Formula weights; the matrices the 3xFP16 chains split scaled by ws, their biases by bs."""
    from dig_b200.threedgraph import method
    model = getattr(method, cls_name)(**kw)
    sd = formula_state_dict(model.state_dict(), seed=2)
    for k in sd:
        if _DENSE.match(k):
            sd[k] = sd[k] * (ws if k.endswith("weight") else bs)
    if edit:
        edit(sd)
    model.load_state_dict(sd)
    return model.to("cuda:0").eval()


_GEOM = {}


def _geom(cls_name, stretch=1.0):
    """The first benchmark batch (128 QM9-shape molecules, seed 0), optionally stretched: graph, rbf0, sbf_p / t_p."""
    from dig_b200 import ops
    from dig_b200.data import synthetic_batch
    key = (cls_name, stretch)
    if key not in _GEOM:
        tors = cls_name == "SphereNet"
        model = _model(cls_name)
        b = synthetic_batch(128, "qm9", seed=0).to("cuda:0")
        pos = (b.pos * stretch).contiguous()
        g = ops.build_graph(pos, b.batch, CUTOFF, num_graphs=128)
        ops.triplet_geometry(g, pos, use_torsion=tors, want_idx=False, want_idx64=True)
        rbf0, bess = ops.edge_basis(g.dist, CUTOFF, 5, model.emb.dist_emb.freq, 0, not tors, 6, 42)
        sbf_p, t_p = ops.triplet_basis_project(g, bess, 0, *model._projection_rows(0, 4))
        _GEOM[key] = dict(z=b.z, g=g, rbf0=rbf0, sbf=sbf_p[1].contiguous(),
                          tp=t_p[1].contiguous() if t_p is not None else None, pos=pos)
    return _GEOM[key]


def _fit(run, target):
    """Input scale s at which the largest operand any split layer of run(s) multiplies is ~target: the chains are close
    to positively homogeneous in their inputs (small biases), so a few fixed-point steps converge."""
    s = 1.0
    for _ in range(8):
        Bounded.split_max = []
        run(s)
        s *= target / max(Bounded.split_max)
    Bounded.split_max = []
    run(s)
    assert abs(max(Bounded.split_max) / target - 1) < 5e-3, (max(Bounded.split_max), target)
    return s


class _Swish:
    """The exact (libdevice) swish in the 3xFP16 epilogues for the duration of a with-block."""

    def __init__(self, fast):
        self.fast = fast

    def __enter__(self):
        from dig_b200 import ops
        ops.h16_set_fast_swish(self.fast)

    def __exit__(self, *exc):
        from dig_b200 import ops
        ops.h16_set_fast_swish(True)


# ------------------------------------------------------------------------------------------------ kernel launches
def _p(t):
    from dig_b200 import ops
    return ops._p(t)


def _call(name, *args):
    from dig_b200._lib import call
    call(name, *args)


def _st():
    from dig_b200 import ops
    return ops._stream()


def _h16_part_a(e1, rbf0, n, w):
    x_ji = torch.empty(n, 128, device=e1.device)
    x_down = torch.empty(n, 64, device=e1.device)
    _call("dig3d_sphere_update_e_a_h16", _p(e1), _p(rbf0), n, ctypes.byref(w), _p(x_ji), _p(x_down), _st())
    return x_ji, x_down


def _h16_part_b(m, e1, x_ji, rbf0, dst, n, n_nodes, w, w_next=None):
    dev = m.device
    e1_out, v_in = torch.empty(n, 128, device=dev), torch.zeros(n_nodes, 128, device=dev)
    if w_next is None:
        _call("dig3d_sphere_update_e_b_h16", _p(m), _p(e1), _p(x_ji), _p(rbf0), _p(dst), n, ctypes.byref(w),
              _p(e1_out), _p(v_in), _st())
        return e1_out, v_in
    x_ji2, x_down2 = torch.empty(n, 128, device=dev), torch.empty(n, 64, device=dev)
    _call("dig3d_sphere_update_e_ba_h16", _p(m), _p(e1), _p(x_ji), _p(rbf0), _p(dst), n, ctypes.byref(w),
          ctypes.byref(w_next), _p(e1_out), _p(v_in), _p(x_ji2), _p(x_down2), _st())
    return e1_out, v_in, x_ji2, x_down2


def _gather_kernel(x_down, geo, w, mode):
    """mode: "warp" (the inference gather, split by the graph), "warp_split<n>" (the same kernel at split n) or "edge"
    (dig3d_sphere_triplet_gather, one warp per edge)."""
    from dig_b200 import ops
    g = geo["g"]
    m = torch.zeros(g.n_edges, 64, device=x_down.device)
    sp = ctypes.c_void_p(geo["sbf"].data_ptr())
    tp = ctypes.c_void_p(geo["tp"].data_ptr()) if geo["tp"] is not None else None
    if mode == "edge":
        _call("dig3d_sphere_triplet_gather", _p(x_down), sp, tp, 8, _p(g.src), _p(g.dst), _p(g.row_ptr),
              _p(g.trip_ptr), g.n_edges, w.w_sbf2, w.w_t2, _p(m), _st())
    else:
        split = int(mode[len("warp_split"):]) if mode.startswith("warp_split") else None
        ops.triplet_gather(x_down, sp, tp, g, w.w_sbf2, w.w_t2, m, _st(), split=split)
    return m


def _init_e_h16(model, geo, cache, tables):
    from dig_b200 import ops
    packed = ops.tc_pack_matrix(model.init_e.lin.weight, cache, "init_e", kind="h16")
    tab = ops.init_e_tables(model.init_e, cache) if tables else None
    return ops.sphere_init_e_h16(geo["z"], geo["g"], geo["rbf0"], ops.pack_init_e(model.init_e), packed, 128, tables=tab)


def _clear_flag():
    from dig_b200 import ops
    ops.h16_overflow(clear=True)


def _flag_clear():
    from dig_b200 import ops
    return ops.tc_timeouts() == 0 and not ops.h16_overflow(clear=True)


# ------------------------------------------------------------------------------------------------ update_e
REGIMES = {
    "formula": dict(),
    "near_cutoff": dict(stretch=1.3),
    "large_4000": dict(target=4000.0),
    "large_8100": dict(target=8100.0),
    "tiny_1e-4": dict(target=3e-4, bs=1e-4),
    "weights_2^-8": dict(ws=2.0 ** -8),
    "weights_2^-4": dict(ws=2.0 ** -4),
    "weights_4": dict(ws=4.0, bs=2.0 ** -12, target=1000.0),    # 4^8 through part B: inputs and biases scaled down
    "exact_swish": dict(fast=False),
}


def _update_e_inputs(cls_name, regime):
    """Model, geometry and the real e1 of the batch (init_e on the 3xFP16 engine), scaled by the regime."""
    r = REGIMES[regime]
    model = _model(cls_name, ws=r.get("ws", 1.0), bs=r.get("bs", 1.0))
    geo = _geom(cls_name, r.get("stretch", 1.0))
    e1, _ = _init_e_h16(_model(cls_name), geo, {}, tables=False)
    torch.cuda.synchronize()
    return model, geo, e1, r


@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("cls_name", ["SphereNet", "DimeNetPP"])
def test_update_e_register_engine_and_gather_against_fp64(cls_name, regime):
    """Part A, the default triplet gather, part B and the fused part B + next part A on the 128-molecule batch."""
    from dig_b200 import ops
    model, geo, e1_base, r = _update_e_inputs(cls_name, regime)
    g, rbf0 = geo["g"], geo["rbf0"]
    E, N = g.n_edges, g.n_nodes
    ue, ue2 = model.update_es[1], model.update_es[2]
    R = Bounded.exact(rbf0)
    idx_kj, idx_ji = g.idx_kj64, g.idx_ji64
    sbf, tp = geo["sbf"], geo["tp"]

    def chain(s):        # the whole block in fp64: the largest operand split anywhere in it sets the scale
        x_ji, x_down = _part_a(Bounded.exact(e1_base * s), R, ue, "h16")
        m = _gather(x_down.v.float(), sbf, tp, idx_kj, idx_ji, E, ue, "fp32")
        e1_out, _ = _part_b(Bounded.exact(m.v.float()), Bounded.exact(e1_base * s), Bounded.exact(x_ji.v.float()),
                            R, g.dst, N, ue, "h16")
        _part_a(e1_out, R, ue2, "h16")

    s = _fit(chain, r["target"]) if "target" in r else 1.0
    e1 = (e1_base * s).contiguous()
    if regime == "near_cutoff":
        assert int((g.dist >= 0.9 * CUTOFF).sum()) > 2000          # rbf0 -> 0 on these rows: tiny gates and e2 rows
    cache = {}
    w = ops.tc_pack_update_e(ue, cls_name == "SphereNet", cache, kind="h16")
    w2 = ops.tc_pack_update_e(ue2, cls_name == "SphereNet", cache, kind="h16")
    _clear_flag()
    with _Swish(r.get("fast", True)):
        x_ji, x_down = _h16_part_a(e1, rbf0, E, w)
        m = _gather_kernel(x_down, geo, w, "warp")
        e1_out, v_in = _h16_part_b(m, e1, x_ji, rbf0, g.dst, E, N, w)
        e1_f, v_f, x_ji2, x_down2 = _h16_part_b(m, e1, x_ji, rbf0, g.dst, E, N, w, w2)
    torch.cuda.synchronize()
    assert _flag_clear(), regime
    X = Bounded.exact(e1)
    ref_ji, ref_down = _part_a(X, R, ue, "h16")
    ref_ji.check(x_ji, "part A x_ji")
    ref_down.check(x_down, "part A x_down")
    _gather(x_down, sbf, tp, idx_kj, idx_ji, E, ue, "fp32").check(m, "gather m")
    ref_e1, ref_v = _part_b(Bounded.exact(m), X, Bounded.exact(x_ji), R, g.dst, N, ue, "h16")
    ref_e1.check(e1_out, "part B e1_out")
    ref_v.check(v_in, "part B v_in")
    ref_e1.check(e1_f, "fused e1_out")
    ref_v.check(v_f, "fused v_in")
    ref_ji2, ref_down2 = _part_a(ref_e1, R, ue2, "h16")     # the fused part A reads e1_out from its registers
    ref_ji2.check(x_ji2, "fused x_ji")
    ref_down2.check(x_down2, "fused x_down")


@pytest.mark.parametrize("n_edges", [1, 63, 64, 65, 129])
@pytest.mark.parametrize("cls_name", ["SphereNet", "DimeNetPP"])
def test_update_e_partial_units_against_fp64(cls_name, n_edges):
    """Single partial unit, one full unit, one past it, two units and one edge: the first n_edges edges of the batch."""
    from dig_b200 import ops
    model, geo, e1, _ = _update_e_inputs(cls_name, "formula")
    g, rbf0, n = geo["g"], geo["rbf0"], n_edges
    ue, ue2 = model.update_es[1], model.update_es[2]
    cache = {}
    w = ops.tc_pack_update_e(ue, cls_name == "SphereNet", cache, kind="h16")
    w2 = ops.tc_pack_update_e(ue2, cls_name == "SphereNet", cache, kind="h16")
    _clear_flag()
    x_ji_full, x_down_full = _h16_part_a(e1, rbf0, g.n_edges, w)
    m = _gather_kernel(x_down_full, geo, w, "warp")
    x_ji, x_down = _h16_part_a(e1, rbf0, n, w)
    e1_out, v_in = _h16_part_b(m, e1, x_ji_full, rbf0, g.dst, n, g.n_nodes, w)
    e1_f, v_f, x_ji2, x_down2 = _h16_part_b(m, e1, x_ji_full, rbf0, g.dst, n, g.n_nodes, w, w2)
    torch.cuda.synchronize()
    assert _flag_clear()
    R, X = Bounded.exact(rbf0[:n]), Bounded.exact(e1[:n])
    ref_ji, ref_down = _part_a(X, R, ue, "h16")
    ref_ji.check(x_ji, "x_ji")
    ref_down.check(x_down, "x_down")
    ref_e1, ref_v = _part_b(Bounded.exact(m[:n]), X, Bounded.exact(x_ji_full[:n]), R, g.dst[:n], g.n_nodes, ue, "h16")
    for got, ref, what in ((e1_out, ref_e1, "e1_out"), (v_in, ref_v, "v_in"), (e1_f, ref_e1, "fused e1_out"),
                           (v_f, ref_v, "fused v_in")):
        ref.check(got, what)
    ref_ji2, ref_down2 = _part_a(ref_e1, R, ue2, "h16")
    ref_ji2.check(x_ji2, "fused x_ji")
    ref_down2.check(x_down2, "fused x_down")


@pytest.mark.parametrize("mode", ["warp", "warp_split1", "warp_split2", "warp_split3", "edge"])
@pytest.mark.parametrize("stretch", [1.0, 1.3])
@pytest.mark.parametrize("cls_name", ["SphereNet", "DimeNetPP"])
def test_triplet_gather_kernels_against_fp64(cls_name, stretch, mode):
    from dig_b200 import ops
    model = _model(cls_name)
    geo = _geom(cls_name, stretch)
    g = geo["g"]
    ue = model.update_es[1]
    w = ops.tc_pack_update_e(ue, cls_name == "SphereNet", {}, kind="h16")
    gen = torch.Generator(device="cuda:0").manual_seed(3)
    x_down = torch.randn(g.n_edges, 64, device="cuda:0", generator=gen) * 10.0 ** (
        torch.rand(g.n_edges, 1, device="cuda:0", generator=gen) * 4 - 3)      # rows over four decades
    m = _gather_kernel(x_down, geo, w, mode)
    torch.cuda.synchronize()
    _gather(x_down, geo["sbf"], geo["tp"], g.idx_kj64, g.idx_ji64, g.n_edges, ue, "fp32").check(m, f"gather {mode}")


# ------------------------------------------------------------------------------------------------ init_e
INIT_REGIMES = {
    "formula": dict(),
    "near_cutoff": dict(stretch=1.3),
    "large_4000": dict(target=4000.0),
    "large_8100": dict(target=8100.0),
    "tiny_1e-4": dict(target=3e-4, bs=1e-4),
    "weights_2^-8": dict(ws=2.0 ** -8),
    "weights_4": dict(ws=4.0),
    "exact_swish": dict(fast=False),
}


@pytest.mark.parametrize("tables", [False, True], ids=["panels", "tables"])
@pytest.mark.parametrize("regime", list(INIT_REGIMES))
def test_init_e_against_fp64(regime, tables):
    """The embedding rows (and, at ~1e-4, lin_rbf_0 too) carry the activation scale of the regime."""
    r = INIT_REGIMES[regime]
    geo = _geom("SphereNet", r.get("stretch", 1.0))
    g = geo["g"]
    tiny = regime.startswith("tiny")

    def scaled(s):
        def edit(sd):
            sd["init_e.emb.weight"] = sd["init_e.emb.weight"] * s
            if tiny:
                sd["init_e.lin_rbf_0.weight"] = sd["init_e.lin_rbf_0.weight"] * s
                sd["init_e.lin_rbf_0.bias"] = sd["init_e.lin_rbf_0.bias"] * s
        return _model("SphereNet", ws=r.get("ws", 1.0), bs=r.get("bs", 1.0), edit=edit)

    s = 1.0
    if "target" in r:
        base = scaled(1.0).init_e
        emb0, w0, b0 = (t.detach().clone() for t in (base.emb.weight, base.lin_rbf_0.weight, base.lin_rbf_0.bias))

        def run(sc):
            with torch.no_grad():
                base.emb.weight.copy_(emb0 * sc)
                if tiny:
                    base.lin_rbf_0.weight.copy_(w0 * sc)
                    base.lin_rbf_0.bias.copy_(b0 * sc)
            _init_e(geo["z"], g.src, g.dst, geo["rbf0"], base, g.n_nodes, "h16")
        s = _fit(run, r["target"])
    model = scaled(s)
    _clear_flag()
    with _Swish(r.get("fast", True)):
        e1, v_in = _init_e_h16(model, geo, {}, tables)
    torch.cuda.synchronize()
    assert _flag_clear()
    ref_e1, ref_v = _init_e(geo["z"], g.src, g.dst, geo["rbf0"], model.init_e, g.n_nodes, "h16", tables)
    ref_e1.check(e1, "init_e e1")
    ref_v.check(v_in, "init_e v_in")


# ------------------------------------------------------------------------------------------------ update_v
V_REGIMES = {"formula": dict(), "large_4000": dict(target=4000.0), "large_8100": dict(target=8100.0),
             "tiny_1e-4": dict(target=3e-4, bs=1e-4), "weights_2^-8": dict(ws=2.0 ** -8),
             "weights_2^-4": dict(ws=2.0 ** -4), "weights_4": dict(ws=4.0, bs=2.0 ** -12, target=1000.0),
             "exact_swish": dict(fast=False)}


@pytest.mark.parametrize("regime", list(V_REGIMES))
@pytest.mark.parametrize("out_channels", [1, 3])
@pytest.mark.parametrize("layers", [1, 3, 5])
def test_update_v_against_fp64(layers, out_channels, regime):
    """All node MLPs of a forward in one launch; node rows spread over four decades, 2304 nodes (the benchmark batch)
    and 129 (one tile + one row)."""
    from dig_b200 import ops
    r = V_REGIMES[regime]
    model = _model("SphereNet", ws=r.get("ws", 1.0), bs=r.get("bs", 1.0), num_output_layers=layers,
                   out_channels=out_channels)
    holders = [model.init_v] + list(model.update_vs)
    gen = torch.Generator(device="cuda:0").manual_seed(layers * 10 + out_channels)
    for n in (2304, 129):
        v0 = torch.randn(len(holders), n, 128, device="cuda:0", generator=gen) * 10.0 ** (
            torch.rand(len(holders), n, 1, device="cuda:0", generator=gen) * 4 - 3)
        if "target" in r:
            v0 = v0 * _fit(lambda sc: [_update_v(v0[b] * sc, h, "h16") for b, h in enumerate(holders)], r["target"])
        out = torch.full((len(holders), n, out_channels), float("nan"), device="cuda:0")
        _clear_flag()
        with _Swish(r.get("fast", True)):
            ops.sphere_update_v_h16(v0.contiguous(), holders, out_channels, out, {})
        torch.cuda.synchronize()
        assert _flag_clear()
        for b, h in enumerate(holders):
            _update_v(v0[b], h, "h16").check(out[b], f"update_v block {b} n={n}")


# ------------------------------------------------------------------------------------------------ 3xTF32 and fp32 twins
@pytest.mark.parametrize("target", [None, 3.0e4], ids=["formula", "act_3e4"])
@pytest.mark.parametrize("cls_name", ["SphereNet", "DimeNetPP"])
def test_tf32_fallback_chain_against_fp64(cls_name, target):
    """The 3xTF32 chain (init_e, part A, part B) is the fallback with fp32 operand range: it holds the bound at
    activations ~3e4, where the 3xFP16 split would overflow."""
    from dig_b200 import ops
    tors = cls_name == "SphereNet"
    model, geo, e1_base, _ = _update_e_inputs(cls_name, "formula")
    g, rbf0 = geo["g"], geo["rbf0"]
    E, N = g.n_edges, g.n_nodes
    ue = model.update_es[1]
    R = Bounded.exact(rbf0)

    def chain(s):
        x_ji, x_down = _part_a(Bounded.exact(e1_base * s), R, ue, "tf32")
        m = _gather(x_down.v.float(), geo["sbf"], geo["tp"], g.idx_kj64, g.idx_ji64, E, ue, "fp32")
        _part_b(Bounded.exact(m.v.float()), Bounded.exact(e1_base * s), Bounded.exact(x_ji.v.float()),
                R, g.dst, N, ue, "tf32")

    s = _fit(chain, target) if target else 1.0
    e1 = (e1_base * s).contiguous()
    cache = {}
    w = ops.tc_pack_update_e(ue, tors, cache)
    x_ji, x_down = torch.empty(E, 128, device="cuda:0"), torch.empty(E, 64, device="cuda:0")
    _call("dig3d_sphere_update_e_a_tc", _p(e1), _p(rbf0), E, ctypes.byref(w), _p(x_ji), _p(x_down), _st())
    m = _gather_kernel(x_down, geo, w, "warp")
    e1_out, v_in = torch.empty(E, 128, device="cuda:0"), torch.zeros(N, 128, device="cuda:0")
    _call("dig3d_sphere_update_e_b_tc", _p(m), _p(e1), _p(x_ji), _p(rbf0), _p(g.dst), E, ctypes.byref(w),
          _p(e1_out), _p(v_in), _st())
    packed = ops.tc_pack_matrix(model.init_e.lin.weight, cache, "init_e")
    e1_i, v_i = ops.sphere_init_e_tc(geo["z"], g, rbf0, ops.pack_init_e(model.init_e), packed, 128)
    torch.cuda.synchronize()
    assert ops.tc_timeouts() == 0
    X = Bounded.exact(e1)
    ref_ji, ref_down = _part_a(X, R, ue, "tf32")
    ref_ji.check(x_ji, "tf32 x_ji")
    ref_down.check(x_down, "tf32 x_down")
    ref_e1, ref_v = _part_b(Bounded.exact(m), X, Bounded.exact(x_ji), R, g.dst, N, ue, "tf32")
    ref_e1.check(e1_out, "tf32 e1_out")
    ref_v.check(v_in, "tf32 v_in")
    ref_i, ref_iv = _init_e(geo["z"], g.src, g.dst, rbf0, model.init_e, N, "tf32")
    ref_i.check(e1_i, "tf32 init_e e1")
    ref_iv.check(v_i, "tf32 init_e v_in")


@pytest.mark.parametrize("stretch", [1.0, 1.3])
@pytest.mark.parametrize("cls_name", ["SphereNet", "DimeNetPP"])
def test_fp32_twins_against_fp64(cls_name, stretch):
    """The exact-fp32 FFMA kernels (init_e, part A, gather + part B, update_v): the references of the parity tests."""
    from dig_b200 import ops
    tors = cls_name == "SphereNet"
    model = _model(cls_name)
    geo = _geom(cls_name, stretch)
    g, rbf0 = geo["g"], geo["rbf0"]
    E, N = g.n_edges, g.n_nodes
    ue = model.update_es[1]
    e1, v0 = ops.sphere_init_e(geo["z"], g, rbf0, ops.pack_init_e(model.init_e), 128)
    w = ops.pack_update_e(ue, tors)
    x_ji, x_down = torch.empty(E, 128, device="cuda:0"), torch.empty(E, 64, device="cuda:0")
    _call("dig3d_sphere_update_e_a", _p(e1), _p(rbf0), E, ctypes.byref(w), _p(x_ji), _p(x_down), _st())
    e1_out, v_in = torch.empty(E, 128, device="cuda:0"), torch.zeros(N, 128, device="cuda:0")
    tp = ctypes.c_void_p(geo["tp"].data_ptr()) if tors else None
    _call("dig3d_sphere_update_e_b", _p(e1), _p(x_ji), _p(x_down), _p(rbf0), ctypes.c_void_p(geo["sbf"].data_ptr()),
          tp, 8, _p(g.src), _p(g.dst), _p(g.row_ptr), _p(g.trip_ptr), E, ctypes.byref(w), _p(e1_out), _p(v_in), _st())
    holders = [model.init_v] + list(model.update_vs)
    v_all = torch.stack([v0] * len(holders)).contiguous()
    out = torch.empty(len(holders), N, 1, device="cuda:0")
    ops.sphere_update_v_batched(v_all, holders, 1, out)
    torch.cuda.synchronize()
    R = Bounded.exact(rbf0)
    ref_e1, ref_v0 = _init_e(geo["z"], g.src, g.dst, rbf0, model.init_e, N, "fp32")
    ref_e1.check(e1, "twin init_e e1")
    ref_v0.check(v0, "twin init_e v_in")
    ref_ji, ref_down = _part_a(Bounded.exact(e1), R, ue, "fp32")
    ref_ji.check(x_ji, "twin x_ji")
    ref_down.check(x_down, "twin x_down")
    m = _gather(x_down, geo["sbf"], geo["tp"], g.idx_kj64, g.idx_ji64, E, ue, "fp32")
    ref_e1o, ref_v = _part_b(m, Bounded.exact(e1), Bounded.exact(x_ji), R, g.dst, N, ue, "fp32")
    ref_e1o.check(e1_out, "twin e1_out")
    ref_v.check(v_in, "twin v_in")
    for b, h in enumerate(holders):
        _update_v(v0, h, "fp32").check(out[b], f"twin update_v block {b}")


# ------------------------------------------------------------------------------------------------ range edge
# One operand of each 3xFP16 entry point placed at the edge of the split's range: 8189 * 8 = 65512 rounds to 65504,
# 8191 * 8 = 65528 overflows.  The dense weights are scaled by 2^-4 so that no operand further down the same launch
# reaches the limit on its own: a flag raised at 8189 would otherwise not say which split overflowed.
EDGE_ENTRIES = ["part_a_e1", "part_b_m", "part_b_e1_in", "update_v_v_in", "init_e_emb", "init_e_tables_r0",
                "linear_h16_x"]
EDGE_ROW, EDGE_COL = 77, 5


@pytest.mark.parametrize("value", [8189.0, 8191.0])
@pytest.mark.parametrize("entry", EDGE_ENTRIES)
def test_split_range_edge_and_overflow_flag(entry, value):
    from dig_b200 import ops
    cls_name = "SphereNet"
    geo = _geom(cls_name)
    g, rbf0 = geo["g"], geo["rbf0"]
    E, N = g.n_edges, g.n_nodes
    R = Bounded.exact(rbf0)
    ws = 2.0 ** -4
    c = EDGE_COL

    def edit(sd):
        if entry == "part_b_e1_in":       # act(lin(h)) ~ 0 in column c of every split after q = 3: h stays at e1_in
            for k in ("update_es.1.lin.bias", "update_es.1.layers_after_skip.0.lin2.bias",
                      "update_es.1.layers_after_skip.1.lin2.bias"):
                sd[k][c] = -60.0
        if entry == "init_e_emb":
            sd["init_e.emb.weight"][6, c] = value             # carbon: x_i and x_j of many edges
        if entry == "init_e_tables_r0":   # r0[:, c] = swish(0 * rbf0 + value) = value on every edge
            sd["init_e.lin_rbf_0.weight"][c] = 0.0
            sd["init_e.lin_rbf_0.bias"][c] = value

    model = _model(cls_name, ws=ws, edit=edit)
    ue = model.update_es[1]
    cache = {}
    w = ops.tc_pack_update_e(ue, True, cache, kind="h16")
    e1, _ = _init_e_h16(_model(cls_name), geo, {}, tables=False)
    torch.cuda.synchronize()
    _clear_flag()
    if entry == "part_a_e1":
        e1[EDGE_ROW, c] = value
        x_ji, x_down = _h16_part_a(e1, rbf0, E, w)
        outs = (x_ji, x_down)
        refs = lambda: _part_a(Bounded.exact(e1), R, ue, "h16")
    elif entry in ("part_b_m", "part_b_e1_in"):
        x_ji, _ = _h16_part_a(e1, rbf0, E, w)
        gen = torch.Generator(device="cuda:0").manual_seed(5)
        m = 0.5 * torch.randn(E, 64, device="cuda:0", generator=gen)
        (m if entry == "part_b_m" else e1)[EDGE_ROW, c] = value
        torch.cuda.synchronize()
        _clear_flag()
        outs = _h16_part_b(m, e1, x_ji, rbf0, g.dst, E, N, w)
        refs = lambda: _part_b(Bounded.exact(m), Bounded.exact(e1), Bounded.exact(x_ji), R, g.dst, N, ue, "h16")
    elif entry == "update_v_v_in":
        holders = [model.init_v] + list(model.update_vs)
        gen = torch.Generator(device="cuda:0").manual_seed(6)
        v = torch.randn(len(holders), N, 128, device="cuda:0", generator=gen)
        v[2, EDGE_ROW, c] = value
        out = torch.empty(len(holders), N, 1, device="cuda:0")
        ops.sphere_update_v_h16(v, holders, 1, out, cache)
        outs = (out,)
        refs = lambda: (Bounded(*(torch.stack([getattr(_update_v(v[b], h, "h16"), f) for b, h in enumerate(holders)])
                                  for f in ("v", "m", "e"))),)
    elif entry.startswith("init_e"):
        tables = entry == "init_e_tables_r0"
        outs = _init_e_h16(model, geo, cache, tables)
        refs = lambda: _init_e(geo["z"], g.src, g.dst, rbf0, model.init_e, N, "h16", tables)
    else:
        x = e1[:4096].clone()
        x[EDGE_ROW, c] = value
        lin = ue.lin
        outs = (ops.linear_h16(x, lin.weight, lin.bias),)
        refs = lambda: (linear(Bounded.exact(x), lin.weight, lin.bias, "h16"),)
    torch.cuda.synchronize()
    raised = ops.h16_overflow(clear=True)
    assert ops.tc_timeouts() == 0
    if value == 8191.0:
        assert raised, f"{entry}: an operand of 8191 overflowed the split without raising the flag"
        return
    assert not raised, f"{entry}: the flag was raised for an operand of 8189"
    for got, ref in zip(outs, refs()):
        ref.check(got, entry)
