"""Second derivatives of ComENet's and ComENet-OCP's energy in the positions: the kernels
`dig3d_comenet_features_tangent_bwd` / `_vec` (the reverse of the feature tangent in pos), Hessian-vector products
`grad(force, pos, v)`, `threedgraph.utils.molecular_hessians` and the position term of a plain `loss.backward()` in
force training.

Comparators (tests/comenet_hessian_ref.py), every row compared:
  * the kernels and the molecular model: fp64 double backward at the kernel's fp32 inputs.  An aliased a x a is exactly
    zero in fp64 but an FMA residue in fp32, and phi / tau of those edges are angles of that residue, so the fp64
    comparator holds every value the kernel reads -- edge vectors, cross products, the length, the angles -- at the
    kernel's fp32 value and takes fp64 derivatives; an aliased product is a constant.  Its fp32 features equal the
    kernel's bit for bit.
  * ComENet-OCP's model: the same for the OCP restatement, whose fp64 distance vectors carry the derivative in pos (the
    cell constant).
Bound: TOL of the largest component of the comparator's product, as for the other models (tests/test_gpu_hessians.py).
An exactly collinear triplet (theta = 0) is not covered: there the reference's d/dtheta of Y_l^m (cos / sin) is 0 / 0
already in the first-order forces."""
import pytest
import torch

import comenet_hessian_ref as chr_
from helpers import case_inputs

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = 1e-4
KTOL = 1e-4                # kernel level, relative to the largest component of the comparator's product


def _rel(a, b):
    return float((a.double() - b.double()).abs().max()) / max(float(b.abs().max()), 1e-30)


# ----------------------------------------------------------------------------- the kernel
def _graph(name):
    from dig_b200.data import synthetic_batch
    if name == "qm9":
        b = synthetic_batch(4, "qm9", seed=4, variable=True)
        return b.pos.float(), b.batch, 5.0
    if name == "aspirin":
        b = synthetic_batch(3, "md17-aspirin", seed=17)
        return b.pos.float(), b.batch, 5.0
    if name == "oc20":
        _, _, pos, batch = case_inputs("comenet_oc20")
        return pos, batch, 6.0
    if name == "single_in_edge":   # atom 3 sees only atom 1 (e0i == e1i for its one in-edge)
        pos = torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.1, 0.0], [0.2, 1.1, 0.3], [4.5, 0.2, 0.1]])
        return pos, torch.zeros(4, dtype=torch.long), 4.0
    if name == "no_out_edge":      # atom 0 has no out-edge in molecule 0's 5-atom cluster under the 32-neighbour cap
        gen = torch.Generator().manual_seed(5)
        mol0 = torch.tensor([[0.03, 1.5, 0.07], [0.0, 0.0, 0.0], [1.0, 0.02, -0.05], [0.04, -0.03, 2.2],
                             [2.0, 2.0, 0.3]])
        pos = torch.cat([mol0, 20.0 + torch.rand(70, 3, generator=gen) * 3.0])
        return pos, torch.cat([torch.zeros(5, dtype=torch.long), torch.ones(70, dtype=torch.long)]), 6.0
    if name == "near_collinear":   # atoms 0, 1, 2 nearly on one line
        pos = torch.tensor([[0.0, 0.0, 0.0], [1.1, 0.002, 0.0], [2.3, 0.0, 0.003], [0.6, 1.2, 0.4], [1.4, -0.9, 0.8]])
        return pos, torch.zeros(5, dtype=torch.long), 5.0
    raise KeyError(name)


KERNEL_GRAPHS = ["qm9", "aspirin", "oc20", "single_in_edge", "no_out_edge", "near_collinear"]


def _kernel_setup(name):
    from dig_b200 import ops
    pos, batch, cutoff = _graph(name)
    pos, batch = pos.to(DEV).contiguous(), batch.to(DEV)
    g = ops.build_graph(pos, batch, cutoff, num_graphs=int(batch.max()) + 1)
    f1, f2, ang = ops.comenet_geometry(g, pos, cutoff, want_angles=True)
    gen = torch.Generator().manual_seed(11)
    u1 = torch.randn(g.n_edges, 12, generator=gen).to(DEV)
    u2 = torch.randn(g.n_edges, 6, generator=gen).to(DEV)
    cs = [torch.randn(pos.shape, generator=gen).to(DEV) for _ in range(2)]
    return g, pos, batch, cutoff, f1, f2, ang, u1, u2, cs


def _fp64_products(pos, vec, dist, src, dst, refs, cutoff, periodic, angles, f1, f2, u1, u2, cs):
    """d/dpos <u, J(pos) c> for each c by fp64 double backward of chr_.features_at_kernel_inputs (the kernel's fp32
    values held, fp64 derivatives), after checking that those values give the kernel's features bit for bit."""
    p = pos.double().requires_grad_(True)
    r1, r2, f32 = chr_.features_at_kernel_inputs(p, vec, dist, src, dst, refs, cutoff, periodic, angles)
    assert torch.equal(f32[0], f1) and torch.equal(f32[1], f2)
    (gp,) = torch.autograd.grad((r1 * u1.double()).sum() + (r2 * u2.double()).sum(), p, create_graph=True)
    out = []
    for c in cs:
        (w,) = torch.autograd.grad((gp * c.double()).sum(), p, retain_graph=True)
        assert torch.isfinite(w).all()
        out.append(w)
    return out


@pytest.mark.parametrize("name", KERNEL_GRAPHS)
def test_tangent_bwd_matches_fp64_double_backward(name):
    """dig3d_comenet_features_tangent_bwd = d/dpos <u, J(pos) c> (c constant) against the fp64 double backward of the
    comparator's features at the kernel's fp32 inputs (aliased products and angles held at the kernel's fp32 values) for
    random u and c, every row within KTOL of the largest component; two runs give the same bits."""
    from dig_b200 import ops
    g, pos, batch, cutoff, f1, f2, ang, u1, u2, cs = _kernel_setup(name)
    vec = pos[g.src.long()] - pos[g.dst.long()]
    wants = _fp64_products(pos, vec, g.dist, g.src, g.dst, g.comenet_refs, cutoff, False, ang, f1, f2, u1, u2, cs)
    for c, want in zip(cs, wants):
        got = ops.comenet_features_tangent_bwd(g, pos, cutoff, c, u1, u2)
        assert torch.isfinite(got).all()
        assert torch.equal(got, ops.comenet_features_tangent_bwd(g, pos, cutoff, c, u1, u2))
        assert _rel(got, want) <= KTOL, (name, _rel(got, want))


@pytest.mark.parametrize("name", KERNEL_GRAPHS)
def test_tangent_bwd_is_a_symmetric_form(name):
    """<c', K(c)> = <c, K(c')> with K(c) = sum_k u_k (d2 f_k / dpos2) c, in fp64 sums."""
    from dig_b200 import ops
    g, pos, _, cutoff, _, _, _, u1, u2, (c, c2) = _kernel_setup(name)
    k1 = ops.comenet_features_tangent_bwd(g, pos, cutoff, c, u1, u2).double()
    k2 = ops.comenet_features_tangent_bwd(g, pos, cutoff, c2, u1, u2).double()
    lhs, rhs = (c2.double() * k1).sum(), (c.double() * k2).sum()
    scale = float((c2.double() * k1).abs().sum() + (c.double() * k2).abs().sum()) + 1e-30
    assert abs(float(lhs - rhs)) <= 1e-5 * scale, (name, float(lhs), float(rhs))


OCP_KERNEL_CASES = ["oc20", "small_cell", "tiny_cell", "otf"]


def _ocp_kernel_setup(name):
    """(model, batch, graph view with the force-path fields, f1, f2, u1, u2) on the sorted periodic edges."""
    from test_gpu_comenet_ocp_forces import _kernel_setup as ocp_setup, _model, _otf_batch
    if name != "otf":
        return ocp_setup(name)
    model, _, _ = _model("oc20", otf_graph=True)
    b = _otf_batch()
    with torch.no_grad():
        model(b)                                      # writes the graph it builds onto b
    gv, f1, f2 = model._edge_geometry(b, forces=True)
    gen = torch.Generator().manual_seed(11)
    u1 = torch.randn(gv.n_edges, 12, generator=gen).to(DEV)
    u2 = torch.randn(gv.n_edges, 6, generator=gen).to(DEV)
    return model, b, gv, f1, f2, u1, u2


@pytest.mark.parametrize("name", OCP_KERNEL_CASES)
def test_tangent_bwd_vec_matches_fp64_double_backward(name):
    """The OCP kernel on the sorted periodic edges (tiny_cell holds the periodic line pairs, otf the graph built on the
    GPU) against the fp64 double backward at its fp32 inputs, every row within KTOL; the same bits on two runs; a
    symmetric form; a rigid translation of every atom (the cell held fixed) moves no edge vector: K(t) = 0 exactly."""
    from dig_b200 import ops
    model, b, gv, f1, f2, u1, u2 = _ocp_kernel_setup(name)
    gen = torch.Generator().manual_seed(3)
    cs = [torch.randn(b.pos.shape, generator=gen).to(DEV) for _ in range(2)]
    wants = _fp64_products(b.pos.detach(), gv.vec, gv.dist, gv.src, gv.dst, gv.refs, model.cutoff, True, None, f1, f2,
                           u1, u2, cs)
    ks = []
    for c, want in zip(cs, wants):
        got = ops.comenet_ocp_features_tangent_bwd(gv, model.cutoff, c, u1, u2)
        assert torch.isfinite(got).all()
        assert torch.equal(got, ops.comenet_ocp_features_tangent_bwd(gv, model.cutoff, c, u1, u2))
        assert _rel(got, want) <= KTOL, (name, _rel(got, want))
        ks.append(got.double())
    (c, c2), (k1, k2) = cs, ks
    lhs, rhs = (c2.double() * k1).sum(), (c.double() * k2).sum()
    scale = float((c2.double() * k1).abs().sum() + (c.double() * k2).abs().sum()) + 1e-30
    assert abs(float(lhs - rhs)) <= 1e-5 * scale
    t = torch.zeros_like(c)
    t[:] = torch.tensor([0.3, -0.5, 0.8], device=DEV)
    kt = ops.comenet_ocp_features_tangent_bwd(gv, model.cutoff, t, u1, u2)
    assert torch.equal(kt, torch.zeros_like(kt))


# ----------------------------------------------------------------------------- the molecular model
MODEL_CASES = {
    "default": dict(cutoff=5.0, num_layers=2),
    "generic": dict(cutoff=5.0, num_layers=2, hidden_channels=128, middle_channels=32, num_output_layers=2),
}
_MODELS = {}


class _B:
    pass


def _batch(z, pos, batch):
    b = _B()
    b.z, b.pos, b.batch = z, pos, batch
    b.num_graphs = int(batch.max().item()) + 1
    return b


def _setup(case):
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph.method import ComENet
    from oracle.weights import formula_state_dict
    if case not in _MODELS:
        model = ComENet(energy_and_force=True, **MODEL_CASES[case])
        model.load_state_dict(formula_state_dict(model.state_dict(), seed=41))
        model = model.to(DEV)
        b = synthetic_batch(3, "md17-aspirin", seed=17)
        _MODELS[case] = (model, b.z.to(DEV), b.pos.float().to(DEV), b.batch.to(DEV))
    return _MODELS[case]


def _comparator(case, model, z, pos, batch):
    """The restated model in fp64 over chr_.geometry_at_kernel_inputs on the graph the model builds for the same fp32
    positions; pos is an fp64 leaf."""
    from dig_b200 import ops
    sd = {k: (v.detach().double() if v.is_floating_point() else v) for k, v in model.state_dict().items()}
    kw = {k: v for k, v in MODEL_CASES[case].items() if k in ("cutoff", "num_layers", "num_output_layers")}
    p32 = pos.detach().float()
    g = ops.build_graph(p32, batch, model.cutoff, num_graphs=int(batch.max()) + 1)
    _, _, ang = ops.comenet_geometry(g, p32, model.cutoff, want_angles=True)
    return chr_.comenet_forward_at_kernel_inputs(sd, z, pos, batch, g, ang, **kw)


def _hvps(model, z, pos, batch, vs):
    p = pos.clone().requires_grad_(True)
    f = torch.autograd.grad(model(_batch(z, p, batch)).sum(), p, create_graph=True)[0]
    return [torch.autograd.grad(f, p, v, retain_graph=True)[0] for v in vs]


def _hvps_ref(case, model, z, pos, batch, vs):
    p = pos.double().requires_grad_(True)
    f = torch.autograd.grad(_comparator(case, model, z, p, batch).sum(), p, create_graph=True)[0]
    return [torch.autograd.grad(f, p, v.double(), retain_graph=True)[0] for v in vs]


def _mode(model, mode):
    model.train(mode == "train")
    for p in model.parameters():
        p.requires_grad_(mode != "frozen")


@pytest.mark.parametrize("mode", ["train", "eval", "frozen"])
@pytest.mark.parametrize("case", list(MODEL_CASES))
def test_hvp_matches_double_backward_of_the_comparator(case, mode):
    model, z, pos, batch = _setup(case)
    _mode(model, mode)
    try:
        gen = torch.Generator().manual_seed(1)
        vs = [torch.randn(pos.shape, generator=gen).to(DEV) for _ in range(2)]
        got = _hvps(model, z, pos, batch, vs)
        want = _hvps_ref(case, model, z, pos, batch, vs)
        for a, b in zip(got, want):
            assert torch.isfinite(a).all() and torch.isfinite(b).all()
            assert _rel(a, b) < TOL, f"{_rel(a, b):.3e}"
        s1, s2 = float((vs[0] * got[1]).sum()), float((vs[1] * got[0]).sum())
        assert abs(s1 - s2) <= TOL * float(vs[0].abs().sum()) * float(got[1].abs().max())
        t = torch.zeros_like(pos)
        t[:] = torch.tensor([0.3, -0.5, 0.8], device=DEV)
        (ht,) = _hvps(model, z, pos, batch, [t])
        assert float(ht.abs().max()) <= TOL * float(got[0].abs().max()) * 3
    finally:
        _mode(model, "train")


@pytest.mark.parametrize("case", list(MODEL_CASES))
def test_molecular_hessians_match_functional_hessian(case):
    from dig_b200.threedgraph.utils import molecular_hessians
    model, z, pos, batch = _setup(case)
    model.eval()
    try:
        blocks = molecular_hessians(model, _batch(z, pos, batch))
        n = pos.size(0)
        full = torch.autograd.functional.hessian(lambda p: _comparator(case, model, z, p, batch).sum(),
                                                 pos.double()).reshape(3 * n, 3 * n)
        start = 0
        for blk in blocks:
            m = blk.size(0) // 3
            want = full[3 * start:3 * (start + m), 3 * start:3 * (start + m)]
            assert _rel(blk, want) < TOL, f"{_rel(blk, want):.3e}"
            assert float((blk - blk.T).abs().max()) <= TOL * float(blk.abs().max())
            start += m
        assert start == n
    finally:
        model.train()


def test_plain_backward_fills_pos_grad_with_the_double_backward():
    """Force training with a plain loss.backward(): pos.grad is the comparator's double backward (the H c term), and the
    parameter gradients are those of the parameter-only pass."""
    model, z, pos, batch = _setup("default")
    model.train()
    gen = torch.Generator().manual_seed(2)
    ft = torch.randn(pos.shape, generator=gen).to(DEV)

    def loss_of(e, f):
        return e.sum() * 0.01 + ((f - ft) ** 2).sum()
    p = pos.clone().requires_grad_(True)
    e = model(_batch(z, p, batch))
    f = -torch.autograd.grad(e.sum(), p, create_graph=True)[0]
    params = [q for q in model.parameters() if q.requires_grad]
    loss = loss_of(e, f)
    g_params = torch.autograd.grad(loss, params, retain_graph=True)
    model.zero_grad()
    loss.backward()
    pr = pos.double().requires_grad_(True)
    er = _comparator("default", model, z, pr, batch)
    fr = -torch.autograd.grad(er.sum(), pr, create_graph=True)[0]
    (want,) = torch.autograd.grad(loss_of(er, fr), pr)
    assert torch.isfinite(p.grad).all()
    assert _rel(p.grad, want) < TOL, f"{_rel(p.grad, want):.3e}"
    for a, q in zip(g_params, params):
        assert _rel(q.grad, a) < 1e-5
    model.zero_grad()


def test_energies_bit_equal_and_the_parameter_pass_builds_no_pos_dual():
    """Energies equal the energy-only training path bit for bit in train and eval mode; forces agree between the modes
    (to the float atomics of the backward);
    autograd.grad(loss, params) and backward(inputs=params) build the dual with pos as data."""
    model, z, pos, batch = _setup("default")
    model.train()
    saved = model.energy_and_force
    model.energy_and_force = False
    try:
        e_plain = model(_batch(z, pos.clone(), batch))            # the energy-only differentiable path
    finally:
        model.energy_and_force = saved
    forces = []
    for mode in ("train", "eval"):
        model.train(mode == "train")
        p = pos.clone().requires_grad_(True)
        e = model(_batch(z, p, batch))
        assert torch.equal(e.detach(), e_plain.detach())
        forces.append(torch.autograd.grad(e.sum(), p)[0])
    assert _rel(forces[1], forces[0]) < 1e-6
    model.train()
    seen = []
    orig = model._forward_dual

    def spy(z_, g_, p_, c_, f1_, f2_):
        seen.append(bool(p_.requires_grad))
        return orig(z_, g_, p_, c_, f1_, f2_)
    model._forward_dual = spy
    try:
        params = [q for q in model.parameters() if q.requires_grad]
        p = pos.clone().requires_grad_(True)
        e = model(_batch(z, p, batch))
        f = torch.autograd.grad(e.sum(), p, create_graph=True)[0]
        loss = (f ** 2).sum()
        torch.autograd.grad(loss, params, retain_graph=True, allow_unused=True)
        loss.backward(inputs=params, retain_graph=True)
        assert seen == [False, False]
        torch.autograd.grad(loss, [p])
        assert seen == [False, False, True]
    finally:
        del model._forward_dual
        model.zero_grad()


# ----------------------------------------------------------------------------- ComENet-OCP
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("case", ["oc20", "small_cell", "otf"])
def test_ocp_hvp_matches_double_backward_of_the_comparator(case, mode):
    """HVPs in pos with the cell constant on the OC20 slabs, the small cell and an otf_graph batch, against the fp64
    double backward of the OCP restatement at the kernel's fp32 inputs, every row; symmetric; a rigid translation gives
    H t ~ 0."""
    from oracle.gen_golden_ocp_forces import restated_kwargs
    from test_gpu_comenet_ocp_forces import _leaves, _model_case
    model, sd, b, ref = _model_case(case)
    model.train(mode == "train")
    gen = torch.Generator().manual_seed(1)
    vs = [torch.randn(b.pos.shape, generator=gen).to(DEV) for _ in range(2)]
    b = _leaves(b, cell=False)
    f = torch.autograd.grad(model(b).sum(), b.pos, create_graph=True)[0]
    got = [torch.autograd.grad(f, b.pos, v, retain_graph=True)[0] for v in vs]
    gv, _, _ = model._edge_geometry(b, forces=True)          # the graph the model read (otf: built and written onto b)
    ref = _leaves(ref, cell=False)
    ref.pos = ref.pos.detach().double().requires_grad_(True)
    ref.cell, ref.cell_offsets = ref.cell.double(), ref.cell_offsets.double()
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    e64 = chr_.comenet_ocp_forward_at_kernel_inputs(sd64, ref, gv, **restated_kwargs())
    fr = torch.autograd.grad(e64.sum(), ref.pos, create_graph=True)[0]
    want = [torch.autograd.grad(fr, ref.pos, v.double(), retain_graph=True)[0] for v in vs]
    for a, w in zip(got, want):
        assert torch.isfinite(a).all() and torch.isfinite(w).all()
        assert _rel(a, w) < TOL, f"{_rel(a, w):.3e}"
    s1, s2 = float((vs[0] * got[1]).sum()), float((vs[1] * got[0]).sum())
    assert abs(s1 - s2) <= TOL * float(vs[0].abs().sum()) * float(got[1].abs().max())
    t = torch.zeros_like(b.pos)
    t[:] = torch.tensor([0.3, -0.5, 0.8], device=DEV)
    (ht,) = torch.autograd.grad(f, b.pos, t, retain_graph=True)
    assert float(ht.abs().max()) <= TOL * float(got[0].abs().max()) * 3
    model.train()


def test_ocp_second_backward_through_the_cell_gradient_raises():
    """Eval mode with a cell that requires grad keeps the first-order path: a second backward raises instead of
    returning a partial Hessian."""
    from test_gpu_comenet_ocp_forces import _leaves, _model_case
    model, _, b, _ = _model_case("oc20")
    model.eval()
    b = _leaves(b)
    gp, gc = torch.autograd.grad(model(b).sum(), [b.pos, b.cell], create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(gp.sum(), b.pos)
    model.train()
