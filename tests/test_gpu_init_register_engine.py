"""init_e on the register-accumulator engine (dig3d_sphere_init_e_h16 / _tab) and the fused init_e + part A of block 0
(dig3d_sphere_init_update_e_a_h16): bit-identity with the separate launches, independence of a row from the rest of
the batch, determinism of the edge -> node sums across 64-edge unit boundaries, and the overflow flag at the split's
range edge."""
import ctypes

import pytest
import torch

from helpers import formula_state_dict

pytestmark = pytest.mark.gpu
CUTOFF = 5.0
_GEO = {}


def _model(cls_name, edit=None):
    from dig_b200.threedgraph import method
    model = getattr(method, cls_name)()
    sd = formula_state_dict(model.state_dict(), seed=2)
    if edit:
        edit(sd)
    model.load_state_dict(sd)
    return model.to("cuda:0").eval()


def _geo(cls_name):
    """The first benchmark batch (128 QM9-shape molecules, seed 0): graph and rbf0."""
    from dig_b200 import ops
    from dig_b200.data import synthetic_batch
    if cls_name not in _GEO:
        tors = cls_name == "SphereNet"
        model = _model(cls_name)
        b = synthetic_batch(128, "qm9", seed=0).to("cuda:0")
        g = ops.build_graph(b.pos, b.batch, CUTOFF, num_graphs=128)
        ops.triplet_geometry(g, b.pos, use_torsion=tors, want_idx=False)
        rbf0, _ = ops.edge_basis(g.dist, CUTOFF, 5, model.emb.dist_emb.freq, 0, not tors, 6, 42)
        _GEO[cls_name] = dict(z=b.z.to(torch.int64).contiguous(), g=g, rbf0=rbf0)
    return _GEO[cls_name]


class _Launch:
    """The init_e / part A entry points of one model on the first n edges of the benchmark graph."""

    def __init__(self, model, geo, tables):
        from dig_b200 import ops
        # the model stays referenced: the weight structs below hold raw pointers to its parameters
        self.model, self.ops, self.geo, self.tables, self.cache = model, ops, geo, tables, {}
        ie = model.init_e
        self.w_init = ops.pack_init_e(ie)
        if tables:
            tab_i, tab_j, packed = ops.init_e_tables(ie, self.cache)
            self.init_args = (packed.data_ptr(), tab_i.data_ptr(), tab_j.data_ptr())
        else:
            packed = ops.tc_pack_matrix(ie.lin.weight, self.cache, "init_e", kind="h16")
            self.init_args = (packed.data_ptr(), None, None)
        self.w = ops.tc_pack_update_e(model.update_es[0], type(model).__name__ == "SphereNet", self.cache,
                                        kind="h16")

    def _common(self, n):
        g, ops = self.geo["g"], self.ops
        return (ops._p(self.geo["z"], torch.int64, "z"), g.src.data_ptr(), g.dst.data_ptr(),
                self.geo["rbf0"].data_ptr(), n, ctypes.byref(self.w_init))

    def init_e(self, n):
        from dig_b200._lib import call
        g = self.geo["g"]
        e1 = torch.full((max(n, 1), 128), float("nan"), device="cuda:0")
        v_in = torch.zeros(g.n_nodes, 128, device="cuda:0")
        if self.tables:
            call("dig3d_sphere_init_e_h16_tab", *self._common(n), *self.init_args, e1.data_ptr(), v_in.data_ptr(),
                 self.ops._stream())
        else:
            call("dig3d_sphere_init_e_h16", *self._common(n), self.init_args[0], e1.data_ptr(), v_in.data_ptr(),
                 self.ops._stream())
        return e1[:n], v_in

    def part_a(self, e1, n):
        from dig_b200._lib import call
        x_ji, x_down = torch.empty(n, 128, device="cuda:0"), torch.empty(n, 64, device="cuda:0")
        call("dig3d_sphere_update_e_a_h16", e1.data_ptr(), self.geo["rbf0"].data_ptr(), n, ctypes.byref(self.w),
             x_ji.data_ptr(), x_down.data_ptr(), self.ops._stream())
        return x_ji, x_down

    def fused(self, n):
        from dig_b200._lib import call
        g = self.geo["g"]
        e1 = torch.full((n, 128), float("nan"), device="cuda:0")
        v_in = torch.zeros(g.n_nodes, 128, device="cuda:0")
        x_ji, x_down = torch.empty(n, 128, device="cuda:0"), torch.empty(n, 64, device="cuda:0")
        call("dig3d_sphere_init_update_e_a_h16", *self._common(n), *self.init_args, ctypes.byref(self.w),
             e1.data_ptr(), v_in.data_ptr(), x_ji.data_ptr(), x_down.data_ptr(), self.ops._stream())
        return e1, v_in, x_ji, x_down


def _flag_clear():
    from dig_b200 import ops
    return ops.tc_timeouts() == 0 and not ops.h16_overflow(clear=True)


@pytest.mark.parametrize("tables", [True, False], ids=["table", "panel"])
@pytest.mark.parametrize("cls_name", ["SphereNet", "DimeNetPP"])
def test_fused_init_part_a_is_bit_identical(cls_name, tables):
    geo = _geo(cls_name)
    run = _Launch(_model(cls_name), geo, tables)
    E = geo["g"].n_edges
    e1, v_in = run.init_e(E)
    x_ji, x_down = run.part_a(e1, E)
    f_e1, f_v_in, f_x_ji, f_x_down = run.fused(E)
    torch.cuda.synchronize()
    assert _flag_clear()
    for name, a, b in (("e1", e1, f_e1), ("v_in", v_in, f_v_in), ("x_ji", x_ji, f_x_ji), ("x_down", x_down, f_x_down)):
        assert torch.isfinite(a).all(), name
        assert torch.equal(a, b), f"{name}: fused init_e + part A differs from the two launches"


@pytest.mark.parametrize("tables", [True, False], ids=["table", "panel"])
@pytest.mark.parametrize("cls_name", ["SphereNet", "DimeNetPP"])
def test_init_e_prefix_rows_are_bit_equal(cls_name, tables):
    """A row of e1 depends on its own edge only: the first n rows of a launch over n edges equal those of the full
    graph, across the 64-edge unit boundaries (and the fused kernel's x_ji / x_down rows likewise)."""
    geo = _geo(cls_name)
    run = _Launch(_model(cls_name), geo, tables)
    E = geo["g"].n_edges
    full, _ = run.init_e(E)
    f_full = run.fused(E)
    for n in (1, 63, 64, 65, 127, 128, 129):
        e1, _ = run.init_e(n)
        f_e1, _, f_x_ji, f_x_down = run.fused(n)
        torch.cuda.synchronize()
        assert torch.equal(e1, full[:n]), f"init_e rows of an {n}-edge prefix differ from the full graph's"
        assert torch.equal(f_e1, full[:n]), n
        assert torch.equal(f_x_ji, f_full[2][:n]) and torch.equal(f_x_down, f_full[3][:n]), n
    assert _flag_clear()


@pytest.mark.parametrize("tables", [True, False], ids=["table", "panel"])
def test_init_e_node_sums_are_deterministic(tables):
    """v_in is summed per 64-edge unit; a node whose in-edges straddle a unit boundary gets two atomic adds onto zero,
    which commute: two runs are bit-identical, and such nodes exist in the benchmark graph."""
    geo = _geo("SphereNet")
    g = geo["g"]
    dst = g.dst.long()
    E = g.n_edges
    first = torch.arange(64, E, 64, device=dst.device)
    straddle = dst[first] == dst[first - 1]
    assert int(straddle.sum()) > 0, "no node's in-edges straddle a unit boundary in the benchmark graph"
    run = _Launch(_model("SphereNet"), geo, tables)
    _, a = run.init_e(E)
    _, b = run.init_e(E)
    _, c, _, _ = run.fused(E)
    torch.cuda.synchronize()
    assert torch.isfinite(a).all()
    assert torch.equal(a, b) and torch.equal(a, c)


@pytest.mark.parametrize("value", [8189.0, 8191.0])
@pytest.mark.parametrize("tables", [True, False], ids=["table", "panel"])
def test_fused_entry_overflow_flag(tables, value):
    """One operand of the fused launch at the split's range edge: 8189 * 8 = 65512 rounds to 65504, 8191 * 8 overflows
    and must raise the flag; the dense weights are scaled by 2^-4 so that no later operand reaches the limit itself."""
    from dig_b200 import ops
    c = 5

    def edit(sd):
        for k in list(sd):
            if k.endswith(".weight") and (k.startswith("init_e.lin.") or k.startswith("update_es.0.lin_")):
                sd[k] = sd[k] * 2.0 ** -4
        if tables:        # r0[:, c] = swish(0 * rbf0 + value) = value on every edge
            sd["init_e.lin_rbf_0.weight"][c] = 0.0
            sd["init_e.lin_rbf_0.bias"][c] = value
        else:             # carbon: x_i and x_j of many edges
            sd["init_e.emb.weight"][6, c] = value

    geo = _geo("SphereNet")
    run = _Launch(_model("SphereNet", edit), geo, tables)
    torch.cuda.synchronize()
    ops.h16_overflow(clear=True)
    e1, _, x_ji, x_down = run.fused(geo["g"].n_edges)
    torch.cuda.synchronize()
    raised = ops.h16_overflow(clear=True)
    assert ops.tc_timeouts() == 0
    if value == 8191.0:
        assert raised, "an operand of 8191 overflowed the split without raising the flag"
    else:
        assert not raised, "the flag was raised for an operand of 8189"
        assert torch.isfinite(e1).all() and torch.isfinite(x_ji).all() and torch.isfinite(x_down).all()


@pytest.mark.parametrize("n_blocks", [1, 5])
def test_update_v_prefix_rows_are_bit_equal(n_blocks):
    """update_v on the register engine: a node's outputs depend on its own row only, so the rows of a launch over the
    first n nodes equal those of the full input, across the 64-node unit boundaries and for every block."""
    from dig_b200 import ops
    model = _model("SphereNet")
    holders = ([model.init_v] + list(model.update_vs))[:n_blocks]
    gen = torch.Generator(device="cuda:0").manual_seed(9)
    N = 2304
    v = torch.randn(n_blocks, N, 128, device="cuda:0", generator=gen)
    cache = {}
    full = ops.sphere_update_v_h16(v, holders, 1, torch.empty(n_blocks, N, 1, device="cuda:0"), cache)
    for n in (1, 63, 64, 65, 129, 2304):
        out = ops.sphere_update_v_h16(v[:, :n].contiguous(), holders, 1, torch.empty(n_blocks, n, 1, device="cuda:0"),
                                      cache)
        torch.cuda.synchronize()
        assert torch.isfinite(out).all()
        assert torch.equal(out, full[:, :n]), f"update_v rows of a {n}-node prefix differ from the full input's"
    assert _flag_clear()
