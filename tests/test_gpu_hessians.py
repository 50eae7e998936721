"""Second derivatives of the energy in the positions: Hessian-vector products `grad(force, pos, v)` and
`threedgraph.utils.molecular_hessians` with SphereNet and DimeNet++ (fused default widths and the generic triplet
branch) and SchNet, in training and eval mode, against torch.autograd's double backward over the restated models
(oracle/restated.py) on the same GPU.

Bound: 1e-4 of the largest component of the comparator's product.  The first-order forces of these models already sit
within ~1e-5 of the restatement (tests/test_gpu_generic_triplet_forces.py), and the products add one more reverse pass
in fp32 over the same network.  SphereNet is compared with the restatement in fp32 on the same GPU: its torsion is a min
over candidates that includes the self candidate (torsion ~0 or 2 pi by the sign of a rounding), so fp64 and fp32 pick
different candidates for some triplets, as in the first-order force tests."""
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-4
CASES = {
    "spherenet": ("SphereNet", dict(num_layers=2)),
    "spherenet_generic": ("SphereNet", dict(num_layers=2, int_emb_size=32, basis_emb_size_angle=4,
                                            basis_emb_size_torsion=4)),
    "dimenetpp": ("DimeNetPP", dict(num_layers=2)),
    "dimenetpp_generic": ("DimeNetPP", dict(num_layers=2, int_emb_size=32, basis_emb_size=4)),
    "schnet": ("SchNet", dict(num_layers=3)),
}
_MODELS = {}


class _B:
    pass


def _batch(z, pos, batch):
    b = _B()
    b.z, b.pos, b.batch = z, pos, batch
    b.num_graphs = int(batch.max().item()) + 1
    return b


def _setup(case, n_mol=3):
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph import method
    key = (case, n_mol)
    if key not in _MODELS:
        name, kw = CASES[case]
        torch.manual_seed(7)
        model = getattr(method, name)(energy_and_force=True, **kw).cuda()
        with torch.no_grad():                 # non-zero output layers, so every block reaches the energy
            for n, p in model.named_parameters():
                if n.endswith(".lin.weight") and ("update_vs" in n or "init_v" in n):
                    p.normal_(0, 0.1)
        if hasattr(model, "invalidate_packed"):
            model.invalidate_packed()
        b = synthetic_batch(n_mol, "qm9", seed=4, variable=True)
        _MODELS[key] = (model, b.z.cuda(), b.pos.float().cuda(), b.batch.cuda())
    return _MODELS[key]


def _restated(case, model, z, pos, batch):
    from oracle import restated
    name, kw = CASES[case]
    sd = {k: (v.detach().to(pos.dtype) if v.is_floating_point() else v) for k, v in model.state_dict().items()}
    if name == "SchNet":
        return restated.schnet_forward(sd, z, pos, batch, cutoff=model.cutoff, num_layers=kw["num_layers"],
                                       num_gaussians=model.dist_emb.offset.numel())
    return restated.dimenet_family_forward(sd, z, pos, batch, torsion=(name == "SphereNet"), cutoff=model.cutoff,
                                           num_layers=kw["num_layers"], num_spherical=model.num_spherical)


def _hvps(model, z, pos, batch, vs):
    p = pos.clone().requires_grad_(True)
    out = model(_batch(z, p, batch))
    f = torch.autograd.grad(out.sum(), p, create_graph=True)[0]
    return [torch.autograd.grad(f, p, v, retain_graph=True)[0] for v in vs]


def _ref_dtype(case):
    return torch.float32 if CASES[case][0] == "SphereNet" else torch.float64


def _hvps_ref(case, model, z, pos, batch, vs):
    dt = _ref_dtype(case)
    p = pos.detach().to(dt, copy=True).requires_grad_(True)
    out = _restated(case, model, z, p, batch)
    f = torch.autograd.grad(out.sum(), p, create_graph=True)[0]
    return [torch.autograd.grad(f, p, v.to(dt), retain_graph=True)[0] for v in vs]


def _rel(a, b):
    return float((a.double() - b.double()).abs().max()) / max(float(b.abs().max()), 1e-30)


def _mode(model, mode):
    model.train(mode == "train")
    for p in model.parameters():
        p.requires_grad_(mode != "frozen")


@pytest.mark.parametrize("mode", ["train", "eval", "frozen"])
@pytest.mark.parametrize("case", list(CASES))
def test_hvp_matches_double_backward_of_the_restatement(case, mode):
    model, z, pos, batch = _setup(case)
    _mode(model, mode)
    try:
        gen = torch.Generator().manual_seed(1)
        vs = [torch.randn(pos.shape, generator=gen).cuda() for _ in range(2)]
        got = _hvps(model, z, pos, batch, vs)
        want = _hvps_ref(case, model, z, pos, batch, vs)
        for a, b in zip(got, want):
            assert _rel(a, b) < TOL, f"{_rel(a, b):.3e}"
        # symmetry: v^T H w = w^T H v
        s1, s2 = float((vs[0] * got[1]).sum()), float((vs[1] * got[0]).sum())
        scale = float(vs[0].abs().sum()) * float(got[1].abs().max())
        assert abs(s1 - s2) <= TOL * scale
        # a rigid translation of every atom leaves the energy unchanged: H t = 0
        t = torch.zeros_like(pos)
        t[:] = torch.tensor([0.3, -0.5, 0.8], device=pos.device)
        (ht,) = _hvps(model, z, pos, batch, [t])
        assert float(ht.abs().max()) <= TOL * float(got[0].abs().max()) * 3
    finally:
        _mode(model, "train")


@pytest.mark.parametrize("case", list(CASES))
def test_molecular_hessians_match_functional_hessian(case):
    from dig_b200.threedgraph.utils import molecular_hessians
    model, z, pos, batch = _setup(case, n_mol=2)
    model.eval()
    try:
        hs = molecular_hessians(model, _batch(z, pos, batch))
        counts = torch.bincount(batch).tolist()
        o = 0
        for g, n in enumerate(counts):
            sl = slice(o, o + n)

            def energy(p, g=g, sl=sl):
                full = pos.to(p.dtype).clone()
                full[sl] = p
                return _restated(case, model, z, full, batch)[g].sum()
            ref = torch.autograd.functional.hessian(energy, pos[sl].to(_ref_dtype(case), copy=True))
            ref = ref.reshape(3 * n, 3 * n)
            assert hs[g].shape == (3 * n, 3 * n)
            assert _rel(hs[g], ref) < TOL, f"{_rel(hs[g], ref):.3e}"
            o += n
    finally:
        model.train()


@pytest.mark.parametrize("mode", ["train", "eval", "frozen"])
@pytest.mark.parametrize("case", [c for c in CASES if c != "schnet"])
def test_energies_and_forces_bit_equal_first_order_path(case, mode):
    """The forward with forces (energy_with_force) gives the energy bits of the first-order forward it wraps, and its
    forces up to the run-to-run spread of the float-atomic position scatter (~2e-6 of the largest component)."""
    from dig_b200 import ops
    model, z, pos, batch = _setup(case)
    _mode(model, mode)
    try:
        p = pos.clone().requires_grad_(True)
        out = model(_batch(z, p, batch))
        f = torch.autograd.grad(out, p, torch.ones_like(out), create_graph=True)[0]
        p2 = pos.clone().requires_grad_(True)
        g = ops.build_graph(p2, batch, model.cutoff, num_graphs=int(batch.max()) + 1, z=z,
                            z_rows=model.init_e.emb.num_embeddings)
        out2 = model._exact(model._forward_train, z, p2, g, None)
        f2 = torch.autograd.grad(out2, p2, torch.ones_like(out2))[0]
        assert torch.equal(out.detach(), out2.detach())
        assert _rel(f.detach(), f2) < 1e-5
    finally:
        _mode(model, "train")


@pytest.mark.parametrize("case", [c for c in CASES if c != "schnet"])
def test_force_training_parameter_gradients_unaffected_by_the_position_term(case):
    """Force training: `autograd.grad(loss, params)` (and `backward(inputs=params)`) runs the parameter pass on the dual
    with pos as data, the path force training always took; `loss.backward()` also reaches pos (H c) and builds the dual
    differentiable in pos.  The parameter gradients agree (up to the float-atomic spread of the force kernels), only
    the pos-differentiable pass fills pos.grad, and the parameter-only pass never builds the pos-differentiable dual."""
    from dig_b200.threedgraph.method import dimenet_family
    model, z, pos, batch = _setup(case)
    gen = torch.Generator().manual_seed(2)
    f_t = torch.randn(pos.shape, generator=gen).cuda()
    params = [p for p in model.parameters()]
    seen = []
    orig = dimenet_family._DimeNetFamily._forward_dual

    def spy(self, z_, p_, *a, **k):
        seen.append(bool(p_.requires_grad))
        return orig(self, z_, p_, *a, **k)

    def loss_of(p):
        out = model(_batch(z, p, batch))
        f = -torch.autograd.grad(out, p, torch.ones_like(out), create_graph=True)[0]
        return out.sum() + 10.0 * torch.nn.functional.l1_loss(f, f_t)
    dimenet_family._DimeNetFamily._forward_dual = spy
    try:
        ref = torch.autograd.grad(loss_of(pos.clone().requires_grad_(True)), params, allow_unused=True)
        assert seen == [False]
        model.zero_grad(set_to_none=True)
        p = pos.clone().requires_grad_(True)
        loss_of(p).backward(inputs=params)
        assert seen == [False, False] and p.grad is None
        inputs_grads = [q.grad for q in params]
        model.zero_grad(set_to_none=True)
        p = pos.clone().requires_grad_(True)
        loss_of(p).backward()
        assert seen == [False, False, True]
        assert p.grad is not None and float(p.grad.abs().max()) > 0
    finally:
        dimenet_family._DimeNetFamily._forward_dual = orig
    for prm, r, r2 in zip(params, ref, inputs_grads):
        if r is None:
            assert prm.grad is None and r2 is None
        else:
            assert torch.equal(r2, r) or _rel(r2, r) < 1e-5
            assert _rel(prm.grad, r) < 1e-5
    model.zero_grad(set_to_none=True)
