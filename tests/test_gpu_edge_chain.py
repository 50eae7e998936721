"""update_e's dense chain on the register-accumulator engine (dig3d_sphere_update_e_{a,b,ba}_h16): parity with the
exact-fp32 twin, edge counts on and around the 64-edge unit boundaries, deterministic edge -> node sums, and fused part
A bit-identical to the separate launch."""
import ctypes

import pytest
import torch

from helpers import formula_state_dict, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-5
UNIT = 64          # edges per consumer unit of the engine


def _block(nmol, seed):
    """SphereNet with formula weights, a seeded QM9-shape batch of nmol molecules, its graph and the inputs of block 1."""
    from dig_b200 import ops
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph.method import SphereNet
    dev = torch.device("cuda:0")
    model = SphereNet()
    model.load_state_dict(formula_state_dict(model.state_dict(), seed=2))
    model = model.to(dev)
    b = synthetic_batch(nmol, "qm9", seed=seed).to(dev)
    g = ops.build_graph(b.pos, b.batch, 5.0, num_graphs=nmol)
    ops.triplet_geometry(g, b.pos, use_torsion=True, want_idx=False)
    rbf0, bess = ops.edge_basis(g.dist, 5.0, 5, model.emb.dist_emb.freq, 0, False, 6, 42)
    w_s, w_t = model._projection_rows(0, 4)
    sbf_p, t_p = ops.triplet_basis_project(g, bess, 0, w_s, w_t)
    e1, _ = ops.sphere_init_e(b.z, g, rbf0, ops.pack_init_e(model.init_e), 128)
    return model, g, rbf0, sbf_p, t_p, e1


@pytest.mark.parametrize("nmol,seed", [(1, 0), (2, 0), (5, 1), (11, 2), (24, 2), (128, 0)])
def test_register_chain_matches_fp32_twin(nmol, seed):
    """One interaction block (part A, triplet gather, part B) against the exact-fp32 FFMA kernels; 128 molecules with
    seed 0 is the first benchmark batch.  The sizes cover a single partial unit, odd and even unit counts and more
    units than two per SM."""
    from dig_b200 import ops
    model, g, rbf0, sbf_p, t_p, e1 = _block(nmol, seed)
    ue = model.update_es[1]
    cache = {}     # owns the packed weight buffers: must outlive the kernels that read them
    e_ref, v_ref = ops.sphere_update_e(e1, g, rbf0, sbf_p, t_p, 8, ops.pack_update_e(ue, True), 128, 64)
    e_h, v_h, _, _ = ops.sphere_update_e_h16(e1, g, rbf0, sbf_p, t_p, 8,
                                             ops.tc_pack_update_e(ue, True, cache, kind="h16"), 128, 64)
    torch.cuda.synchronize()
    assert rel_err(e_h.cpu().numpy(), e_ref.cpu().numpy()) < TOL, g.n_edges
    assert rel_err(v_h.cpu().numpy(), v_ref.cpu().numpy()) < TOL, g.n_edges
    assert ops.tc_timeouts() == 0 and not ops.h16_overflow()


def _chain(g, e1, rbf0, m, w, w_next, n):
    """Parts A, B and B + next A on the first n edges of g (every input row beyond n is ignored)."""
    from dig_b200 import ops
    from dig_b200._lib import call
    dev, byref, p = e1.device, ctypes.byref, ops._p
    st = ops._stream()

    def part_a(e1_src):
        x_ji, x_down = torch.empty(n, 128, device=dev), torch.empty(n, 64, device=dev)
        call("dig3d_sphere_update_e_a_h16", p(e1_src), p(rbf0), n, byref(w_next), p(x_ji), p(x_down), st)
        return x_ji, x_down

    x_ji = torch.empty(n, 128, device=dev)
    x_down = torch.empty(n, 64, device=dev)
    call("dig3d_sphere_update_e_a_h16", p(e1), p(rbf0), n, byref(w), p(x_ji), p(x_down), st)
    out = {"x_ji": x_ji, "x_down": x_down}
    for fused in (False, True):
        e1_out = torch.empty(n, 128, device=dev)
        v_in = torch.zeros(g.n_nodes, 128, device=dev)
        if fused:
            x_ji2, x_down2 = torch.empty(n, 128, device=dev), torch.empty(n, 64, device=dev)
            call("dig3d_sphere_update_e_ba_h16", p(m), p(e1), p(x_ji), p(rbf0), p(g.dst), n, byref(w), byref(w_next),
                 p(e1_out), p(v_in), p(x_ji2), p(x_down2), st)
            out.update(e1_f=e1_out, v_f=v_in, x_ji_f=x_ji2, x_down_f=x_down2)
        else:
            call("dig3d_sphere_update_e_b_h16", p(m), p(e1), p(x_ji), p(rbf0), p(g.dst), n, byref(w),
                 p(e1_out), p(v_in), st)
            out.update(e1_out=e1_out, v_in=v_in)
            out["x_ji_next"], out["x_down_next"] = part_a(e1_out)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("n_edges", [1, 63, 64, 65, 127, 128, 129])
def test_unit_boundaries_on_edge_prefixes(n_edges):
    """A symmetric radius graph has an even edge count, so the odd sizes around the unit boundaries run the kernels on
    the first n_edges edges of a larger graph.  Every chain output is row-local, so each row equals the full run's
    row bit for bit; so does the edge -> node sum of every node whose in-edges all lie in the prefix (the 64-row units
    are the same).  Fused part A equals part B followed by part A, bit for bit."""
    from dig_b200 import ops
    model, g, rbf0, sbf_p, t_p, e1 = _block(3, 1)
    E = g.n_edges
    assert E > 129 + UNIT
    cache = {}
    w = ops.tc_pack_update_e(model.update_es[1], True, cache, kind="h16")
    w_next = ops.tc_pack_update_e(model.update_es[2], True, cache, kind="h16")
    gen = torch.Generator(device=e1.device).manual_seed(5)
    m = 0.5 * torch.randn(E, 64, device=e1.device, generator=gen)   # stands in for the triplet gather's output
    full = _chain(g, e1, rbf0, m, w, w_next, E)
    pre = _chain(g, e1, rbf0, m, w, w_next, n_edges)
    for k in ("x_ji", "x_down", "e1_out", "e1_f", "x_ji_f", "x_down_f", "x_ji_next", "x_down_next"):
        assert torch.equal(pre[k], full[k][:n_edges]), k
    for r in (pre, full):
        assert torch.equal(r["e1_f"], r["e1_out"]) and torch.equal(r["v_f"], r["v_in"])
        assert torch.equal(r["x_ji_f"], r["x_ji_next"]) and torch.equal(r["x_down_f"], r["x_down_next"])
    row_ptr = g.row_ptr.long()
    complete = row_ptr[1:] <= n_edges                    # nodes whose in-edge segment lies inside the prefix
    untouched = row_ptr[:-1] >= n_edges
    assert torch.equal(pre["v_in"][complete], full["v_in"][complete])
    assert not pre["v_in"][untouched].any()
    assert ops.tc_timeouts() == 0 and not ops.h16_overflow()


def test_edge_to_node_sums_are_deterministic_across_unit_boundaries():
    """A node whose in-edges straddle a 64-edge unit boundary receives one atomic partial sum from each of the two
    units; two atomics onto zero commute, so repeated calls agree bit for bit."""
    from dig_b200 import ops
    model, g, rbf0, sbf_p, t_p, e1 = _block(24, 2)
    row_ptr = g.row_ptr.long()
    lo, hi = row_ptr[:-1], row_ptr[1:]
    straddles = ((lo // UNIT) != ((hi - 1) // UNIT)) & (hi > lo)
    assert straddles.any()
    cache = {}
    w = ops.tc_pack_update_e(model.update_es[1], True, cache, kind="h16")
    runs = [ops.sphere_update_e_h16(e1, g, rbf0, sbf_p, t_p, 8, w, 128, 64) for _ in range(2)]
    torch.cuda.synchronize()
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)
    assert ops.tc_timeouts() == 0 and not ops.h16_overflow()


@pytest.mark.parametrize("nmol", [1, 5, 24, 128])
def test_fused_part_a_is_bit_identical_in_the_model(nmol):
    """The model forward, with part A of block l + 1 fused into part B of block l, gives the same energies bit for bit as
    the chain with separate launches."""
    from dig_b200 import ops
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph.method import SphereNet
    from helpers import sphere_forward_op_by_op
    dev = torch.device("cuda:0")
    model = SphereNet()
    model.load_state_dict(formula_state_dict(model.state_dict(), seed=4))
    model = model.to(dev).eval()
    b = synthetic_batch(nmol, "qm9", seed=0).to(dev)
    with torch.no_grad():
        fused = model(b)
        apart = sphere_forward_op_by_op(model, b)
    torch.cuda.synchronize()
    assert torch.isfinite(fused).all()
    assert torch.equal(apart, fused)
    assert ops.tc_timeouts() == 0 and not ops.h16_overflow()
