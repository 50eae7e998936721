"""GPU tests of the training path: every backward kernel against torch.autograd over the oracle restatement
(same inputs, same weights), and run.train end to end.

Tolerances: the backward is a different summation order from ATen's (tiled GEMMs, atomics for the weight
gradients), so gradients are compared at 1e-4 of the gradient tensor's max magnitude (fp32)."""
import numpy as np
import pytest
import torch

from helpers import case_inputs, formula_state_dict, rel_err

pytestmark = pytest.mark.gpu
GTOL = 1e-4


class _B:
    pass


def _batch(z, pos, batch, y=None):
    b = _B()
    b.z, b.pos, b.batch = z, pos, batch
    b.num_graphs = int(batch.max().item()) + 1
    b.y = y
    return b


@pytest.mark.parametrize("rows,k,nout", [(1000, 128, 128), (777, 128, 64), (300, 256, 128), (513, 50, 32),
                                         (64, 6, 128), (129, 42, 8), (5, 128, 1), (2000, 384, 128)])
def test_linear_fwd_bwd(rows, k, nout):
    from dig_b200 import autograd as ag
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(rows + k)
    x = torch.randn(rows, k, generator=gen).to(dev).requires_grad_(True)
    w = (torch.randn(nout, k, generator=gen) / k ** 0.5).to(dev).requires_grad_(True)
    b = torch.randn(nout, generator=gen).to(dev).requires_grad_(True)
    dy = torch.randn(rows, nout, generator=gen).to(dev)
    y = ag.linear(x, w, b)
    y.backward(dy)
    got = [y.detach(), x.grad, w.grad, b.grad]
    x2, w2, b2 = (t.detach().double().requires_grad_(True) for t in (x, w, b))
    y2 = torch.nn.functional.linear(x2, w2, b2)
    y2.backward(dy.double())
    for a, r in zip(got, [y2.detach(), x2.grad, w2.grad, b2.grad]):
        assert rel_err(a.cpu().numpy(), r.cpu().numpy()) < 2e-5


def _placed(x, aligned):
    """x in a 16-byte aligned buffer (the float4 kernels) or in the misaligned view buf[1:] of one (the scalar ones)."""
    buf = torch.empty(x.numel() + 4, device="cuda:0")
    view = buf[:x.numel()] if aligned else buf[1:x.numel() + 1]
    return view.copy_(x.to("cuda:0"))


@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_activations_fwd_bwd(mode, aligned):
    """act / act_bwd against the fp64 bound per element (tests/fp64_bound.py: swish, ssp, act'), on n = 4000 in an
    aligned buffer (float4 kernels) and in a misaligned view (scalar kernels); both paths give the same bits."""
    from dig_b200 import autograd as ag
    from dig_b200 import ops
    from fp64_bound import Bounded, act_d1, mul, ssp, swish
    gen = torch.Generator().manual_seed(mode)
    x_c = (torch.rand(4000, generator=gen, dtype=torch.float64) * 60 - 30).float()
    dy_c = torch.randn(4000, generator=gen).float()
    x, dy = _placed(x_c, aligned).requires_grad_(True), _placed(dy_c, aligned)
    y = [ag.swish, ag.ssp, ag.relu][mode](x)
    y.backward(dy)
    xb = Bounded.exact(x_c)
    ref_y = [swish(xb), ssp(xb), Bounded(xb.v.clamp_min(0), xb.m, xb.e)][mode]
    ref_y.check(y.detach().cpu(), f"act mode {mode}")
    mul(Bounded.exact(dy_c), act_d1(x_c, mode)).check(x.grad.cpu(), f"act_bwd mode {mode}")
    x_o, dy_o = _placed(x_c, not aligned), _placed(dy_c, not aligned)
    assert torch.equal(ops.act(x_o, mode), y.detach())
    assert torch.equal(ops.act_bwd(x_o, dy_o, mode), x.grad)


def _act_bwd2_x():
    """[-100, 100]: dense around 0, dense over [8, 20] and around the ssp threshold at 20."""
    return torch.cat([torch.linspace(-100, 100, 20001), torch.linspace(-4, 4, 8001), torch.linspace(8, 20, 12001),
                      torch.linspace(19.9, 20.1, 2001), torch.tensor([20.0, -88.0, 88.0, 0.0])]).float()


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_act_bwd2_matches_fp64_double_backward(mode):
    """out = g * dy * act''(x) against torch.autograd's double backward in fp64 (swish, softplus with threshold 20 - ln 2,
    relu), element by element: a few ulp of the magnitude s (1 - s) (2 + |x| |1 - 2s|) of act'' plus a subnormal floor
    (tests/fp64_bound.py, act_d2).  1 - s evaluated as 1.0f - s loses every digit of it as s -> 1 (from x ~ 8).
    fp64's own 1 - s cancels too (beyond x ~ 25 at fp32's precision), so the reference is act_d2's closed form with
    sigmoid(-x), held to torch's double backward within fp64's 1e-14."""
    from dig_b200 import ops
    from fp64_bound import Bounded, act_d2, mul
    x = _act_bwd2_x()
    gen = torch.Generator().manual_seed(11)
    dy = (torch.rand(x.numel(), generator=gen) + 0.5).float()
    g = (torch.rand(x.numel(), generator=gen) * 2 - 1).float()
    out = ops.act_bwd2(x.to("cuda:0"), dy.to("cuda:0"), g.to("cuda:0"), mode).cpu()
    x2 = x.double().requires_grad_(True)
    y2 = [lambda t: t * torch.sigmoid(t), lambda t: torch.nn.functional.softplus(t, threshold=20.0) - np.log(2.0),
          torch.relu][mode](x2)
    (gx,) = torch.autograd.grad(y2, x2, dy.double(), create_graph=True)
    (ref,) = torch.autograd.grad(gx, x2, g.double(), allow_unused=True) if mode != 2 else (torch.zeros_like(x2),)
    bound = mul(mul(Bounded.exact(g), Bounded.exact(dy)), act_d2(x, mode))
    # act_d2's closed form is torch's act''.  Except at x = 20 itself for softplus: torch's forward and first backward
    # switch to the identity at x > 20 but its double backward masks x >= 20; the kernel follows the forward.
    keep = x != 20.0 if mode == 1 else torch.ones_like(x, dtype=torch.bool)
    assert torch.allclose(bound.v[keep], ref.detach()[keep], rtol=1e-9, atol=1e-14)
    bound.check(out, f"act_bwd2 mode {mode}")


def test_gather_scatter_segment_bwd():
    from dig_b200 import autograd as ag
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(3)
    n, e, w = 50, 400, 16
    idx = torch.sort(torch.randint(0, n, (e,), generator=gen)).values.to(dev)
    ptr = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    ptr[1:] = torch.cumsum(torch.bincount(idx, minlength=n), 0).to(torch.int32)
    perm = torch.randperm(e, generator=gen).to(dev)
    x = torch.randn(n, w, generator=gen).to(dev).requires_grad_(True)
    ye = torch.randn(e, w, generator=gen).to(dev).requires_grad_(True)
    up = torch.randn(e, w, generator=gen).to(dev)
    un = torch.randn(n, w, generator=gen).to(dev)
    # sorted gather (segment-sum backward), unsorted gather (atomic backward), segment sum, scatter add
    loss = (ag.gather_rows(x, idx.to(torch.int32), ptr) * up).sum() + (ag.gather_rows(x, idx[perm]) * up).sum() \
        + (ag.segment_sum(ye, ptr, idx) * un).sum() + (ag.scatter_add_rows(ye, idx[perm], n) * un).sum()
    loss.backward()
    x2 = x.detach().double().requires_grad_(True)
    y2 = ye.detach().double().requires_grad_(True)
    ref = (x2[idx] * up.double()).sum() + (x2[idx[perm]] * up.double()).sum() \
        + (torch.zeros(n, w, dtype=torch.float64, device=dev).index_add_(0, idx, y2) * un.double()).sum() \
        + (torch.zeros(n, w, dtype=torch.float64, device=dev).index_add_(0, idx[perm], y2) * un.double()).sum()
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-3
    assert rel_err(x.grad.cpu().numpy(), x2.grad.cpu().numpy()) < 1e-5
    assert rel_err(ye.grad.cpu().numpy(), y2.grad.cpu().numpy()) < 1e-5


def _grad_compare(model, sd, ref_forward, z, pos, batch, target):
    """Param grads of L1(model(batch), target) from the product's backward kernels vs torch.autograd on the oracle."""
    model.zero_grad()
    out = model(_batch(z, pos, batch))
    assert out.requires_grad
    loss = torch.nn.functional.l1_loss(out, target)
    loss.backward()
    sd_ref = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    ref = ref_forward(sd_ref, z, pos, batch)
    ref_loss = torch.nn.functional.l1_loss(ref, target)
    ref_loss.backward()
    assert rel_err(out.detach().cpu().numpy(), ref.detach().cpu().numpy()) < 1e-5
    worst = {}
    for name, p in model.named_parameters():
        r = sd_ref[name].grad
        assert r is not None, name
        assert p.grad is not None, f"no gradient for {name}"
        worst[name] = rel_err(p.grad.cpu().numpy(), r.cpu().numpy()) if r.abs().max() > 0 else \
            float(p.grad.abs().max())
    bad = {k: v for k, v in worst.items() if v > GTOL}
    assert not bad, f"gradient mismatch: {bad}"
    return worst


def test_schnet_gradients_match_oracle_autograd():
    from dig_b200.threedgraph.method import SchNet
    from oracle import restated
    dev = torch.device("cuda:0")
    _, z, pos, batch = case_inputs("schnet_cfg1", dev)
    model = SchNet(num_layers=2, hidden_channels=32, num_filters=32, cutoff=10.0)
    sd = formula_state_dict(model.state_dict(), seed=1)
    model.load_state_dict(sd)
    model = model.to(dev)
    sd = {k: v.to(dev) for k, v in sd.items()}
    target = torch.linspace(-1, 1, 16, device=dev).view(16, 1)
    _grad_compare(model, sd, lambda s, *a: restated.schnet_forward(s, *a, cutoff=10.0, num_layers=2),
                  z, pos, batch, target)


def test_schnet_train_path_equals_inference_path():
    from dig_b200.threedgraph.method import SchNet
    dev = torch.device("cuda:0")
    _, z, pos, batch = case_inputs("schnet_cfg1", dev)
    model = SchNet(num_layers=3, hidden_channels=128, num_filters=128, cutoff=10.0).to(dev)
    with torch.no_grad():
        u_inf = model(_batch(z, pos, batch))
    u_tr = model(_batch(z, pos, batch))
    assert u_tr.requires_grad and not u_inf.requires_grad
    assert rel_err(u_tr.detach().cpu().numpy(), u_inf.cpu().numpy()) < 1e-5


def test_run_train_schnet_loss_decreases():
    """run.train (reference run.py:103-135) on synthetic molecules: the mean loss falls over a few epochs of Adam."""
    from dig_b200.data import DataLoader, synthetic_molecules
    from dig_b200.threedgraph.method import SchNet, run
    dev = torch.device("cuda:0")
    mols = synthetic_molecules(32, natoms=10, seed=5)
    for m in mols:
        m.y = torch.tensor([float(m.z.sum()) * 0.02])
    torch.manual_seed(0)
    model = SchNet(num_layers=2, hidden_channels=32, num_filters=32, cutoff=6.0).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=2e-3)
    loader = DataLoader(mols, 8, shuffle=True)
    r = run()
    losses = [r.train(model, opt, loader, False, 100, torch.nn.L1Loss(), dev) for _ in range(5)]
    assert losses[-1] < losses[0], losses


@pytest.mark.parametrize("name", ["spherenet_qm9", "dimenetpp_md17", "spherenet_ns3"])
def test_dimenet_family_gradients_match_oracle_autograd(name):
    """Every parameter gradient of SphereNet / DimeNet++ (incl. dist_emb.freq and the basis projections) vs
    torch.autograd over the oracle restatement, on the golden cases."""
    from dig_b200.threedgraph import method
    from helpers import CASES
    from oracle import restated
    dev = torch.device("cuda:0")
    model_name, ctor, _, wseed = CASES[name]
    _, z, pos, batch = case_inputs(name, dev)
    model = getattr(method, model_name)(**ctor)
    sd = formula_state_dict(model.state_dict(), seed=wseed)
    model.load_state_dict(sd)
    model = model.to(dev)
    sd = {k: v.to(dev) for k, v in sd.items()}
    nb = int(batch.max().item()) + 1
    target = torch.linspace(-1, 1, nb, device=dev).view(nb, 1)
    kw = {k: v for k, v in ctor.items() if k in ("cutoff", "num_spherical")}
    fwd = restated.spherenet_forward if model_name == "SphereNet" else restated.dimenetpp_forward
    worst = _grad_compare(model, sd, lambda s, *a: fwd(s, *a, **kw), z, pos, batch, target)
    assert "emb.dist_emb.freq" in worst and len(worst) == len(list(model.parameters()))


def test_spherenet_train_path_equals_inference_path():
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph.method import SphereNet
    dev = torch.device("cuda:0")
    torch.manual_seed(1)
    model = SphereNet().to(dev)
    b = synthetic_batch(8, "qm9", seed=11).to(dev)
    with torch.no_grad():
        u_inf = model(b)
    u_tr = model(b)
    assert u_tr.requires_grad
    assert rel_err(u_tr.detach().cpu().numpy(), u_inf.cpu().numpy()) < 1e-5


def test_run_train_spherenet_step():
    """One epoch of run.train on SphereNet: finite loss, every parameter receives a gradient and moves."""
    from dig_b200.data import DataLoader, synthetic_molecules
    from dig_b200.threedgraph.method import SphereNet, run
    dev = torch.device("cuda:0")
    mols = synthetic_molecules(16, "qm9", seed=7)
    torch.manual_seed(0)
    model = SphereNet().to(dev)
    before = {k: v.detach().clone() for k, v in model.named_parameters()}
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    loss = run().train(model, opt, DataLoader(mols, 8, shuffle=False), False, 100, torch.nn.L1Loss(), dev)
    assert np.isfinite(loss)
    moved = {k: bool((v.detach() != before[k]).any()) for k, v in model.named_parameters()}
    assert all(moved.values()), [k for k, m in moved.items() if not m]


def test_graphnorm_fwd_bwd():
    from dig_b200 import autograd as ag
    from dig_b200.threedgraph.method.comenet import GraphNorm
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(8)
    sizes = [5, 1, 17, 9]
    n, wd = sum(sizes), 256
    ptr = torch.tensor([0] + list(np.cumsum(sizes)), dtype=torch.int32, device=dev)
    batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes)).to(dev)
    norm = GraphNorm(wd).to(dev)
    with torch.no_grad():
        norm.weight.copy_(torch.rand(wd, generator=gen) + 0.5)
        norm.bias.copy_(torch.randn(wd, generator=gen))
        norm.mean_scale.copy_(torch.rand(wd, generator=gen) + 0.3)
    h = torch.randn(n, wd, generator=gen).to(dev).requires_grad_(True)
    dy = torch.randn(n, wd, generator=gen).to(dev)
    y = ag.graphnorm(h, norm, ptr)
    y.backward(dy)
    h2 = h.detach().double().requires_grad_(True)
    w2, b2, s2 = (p.detach().double().requires_grad_(True) for p in (norm.weight, norm.bias, norm.mean_scale))
    cnt = torch.tensor(sizes, dtype=torch.float64, device=dev).unsqueeze(1)
    mean = torch.zeros(len(sizes), wd, dtype=torch.float64, device=dev).index_add_(0, batch, h2) / cnt
    out = h2 - mean[batch] * s2
    var = torch.zeros(len(sizes), wd, dtype=torch.float64, device=dev).index_add_(0, batch, out * out) / cnt
    y2 = w2 * out / (var + 1e-5).sqrt()[batch] + b2
    y2.backward(dy.double())
    assert rel_err(y.detach().cpu().numpy(), y2.detach().cpu().numpy()) < 2e-6
    for a, r in ((h.grad, h2.grad), (norm.weight.grad, w2.grad), (norm.bias.grad, b2.grad),
                 (norm.mean_scale.grad, s2.grad)):
        assert rel_err(a.cpu().numpy(), r.cpu().numpy()) < 2e-5


def test_comenet_gradients_match_oracle_autograd():
    from dig_b200.threedgraph.method import ComENet
    from oracle import restated
    dev = torch.device("cuda:0")
    _, z, pos, batch = case_inputs("comenet_oc20", dev)
    model = ComENet(cutoff=6.0)
    sd = formula_state_dict(model.state_dict(), seed=4)
    model.load_state_dict(sd)
    model = model.to(dev)
    sd = {k: v.to(dev) for k, v in sd.items()}
    target = torch.tensor([[0.3], [-0.7]], device=dev)
    _grad_compare(model, sd, lambda s, *a: restated.comenet_forward(s, *a, cutoff=6.0), z, pos, batch, target)


def test_comenet_train_step_moves_every_parameter():
    from dig_b200.data import DataLoader, synthetic_molecules
    from dig_b200.threedgraph.method import ComENet, run
    dev = torch.device("cuda:0")
    mols = synthetic_molecules(4, "oc20-is2re", seed=9)
    torch.manual_seed(0)
    model = ComENet(cutoff=6.0).to(dev)
    before = {k: v.detach().clone() for k, v in model.named_parameters()}
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    loss = run().train(model, opt, DataLoader(mols, 2, shuffle=False), False, 100, torch.nn.L1Loss(), dev)
    assert np.isfinite(loss)
    assert all(bool((v.detach() != before[k]).any()) for k, v in model.named_parameters())


# ------------------------------------------------------------------------------------------------ forces
FTOL = 1e-5      # north_star: forces within 1e-5 (relative to the largest force component)


@pytest.mark.parametrize("name", ["schnet_cfg1", "dimenetpp_md17"])
def test_forces_match_reference(name):
    """forces = -dE/dpos through the geometry / basis backward kernels vs (a) the real reference's fp32 and fp64
    forces (golden fixture) and (b) torch.autograd over the oracle restatement on the same GPU."""
    from dig_b200.threedgraph import method
    from helpers import CASES
    from oracle import restated
    dev = torch.device("cuda:0")
    model_name, ctor, _, wseed = CASES[name]
    gold, z, pos, batch = case_inputs(name, dev)
    model = getattr(method, model_name)(energy_and_force=True, **ctor)
    sd = formula_state_dict(model.state_dict(), seed=wseed)
    model.load_state_dict(sd)
    model = model.to(dev)
    b = _batch(z, pos.clone(), batch)
    out = model(b)
    assert b.pos.requires_grad
    force = -torch.autograd.grad(out, b.pos, grad_outputs=torch.ones_like(out), create_graph=True, retain_graph=True)[0]
    force = force.detach()
    assert rel_err(out.detach().cpu().numpy(), gold["energy_f32"]) < 1e-5
    assert rel_err(force.cpu().numpy(), gold["force_f64"]) < FTOL
    assert rel_err(force.cpu().numpy(), gold["force_f32"]) < FTOL
    pos2 = pos.clone().requires_grad_(True)
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    kw = {k: v for k, v in ctor.items() if k in ("cutoff", "num_layers")}
    fwd = restated.schnet_forward if model_name == "SchNet" else restated.dimenetpp_forward
    ref = fwd(sd_dev, z, pos2, batch, **kw)
    f_ref = -torch.autograd.grad(ref.sum(), pos2)[0]
    assert rel_err(force.cpu().numpy(), f_ref.cpu().numpy()) < FTOL


def test_force_path_parameter_gradients_still_match():
    """energy_and_force=True changes the graph (dist / angle become functions of pos); parameter gradients must not move."""
    from dig_b200.threedgraph.method import DimeNetPP
    from oracle import restated
    dev = torch.device("cuda:0")
    _, z, pos, batch = case_inputs("dimenetpp_md17", dev)
    model = DimeNetPP(energy_and_force=True, cutoff=5.0)
    sd = formula_state_dict(model.state_dict(), seed=3)
    model.load_state_dict(sd)
    model = model.to(dev)
    sd = {k: v.to(dev) for k, v in sd.items()}
    target = torch.linspace(-1, 1, 4, device=dev).view(4, 1)
    _grad_compare(model, sd, lambda s, *a: restated.dimenetpp_forward(s, *a, cutoff=5.0), z, pos.clone(), batch, target)


def test_run_val_energy_and_force_and_force_training():
    """run.val with forces; run.train ON forces (run.py:110-123) lowers the loss for SchNet (twice-differentiable
    Functions, autograd_dd.py) and for DimeNet++ (tangent network, autograd_jvp.py)."""
    from dig_b200.data import DataLoader, synthetic_molecules
    from dig_b200.threedgraph.evaluation import ThreeDEvaluator
    from dig_b200.threedgraph.method import DimeNetPP, SchNet, run
    dev = torch.device("cuda:0")
    mols = synthetic_molecules(8, "md17-aspirin", seed=3)
    torch.manual_seed(0)
    model = SchNet(energy_and_force=True, num_layers=2, hidden_channels=32, num_filters=32, cutoff=5.0).to(dev)
    mae = run().val(model, DataLoader(mols, 4, shuffle=False), True, 100, ThreeDEvaluator(), dev)
    assert np.isfinite(mae)
    opt = torch.optim.Adam(model.parameters(), lr=2e-3)
    losses = [run().train(model, opt, DataLoader(mols, 4, shuffle=False), True, 100, torch.nn.L1Loss(), dev)
              for _ in range(6)]
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    # DimeNet++ trains on forces too (round 2: tangent network, dig_b200/autograd_jvp.py)
    torch.manual_seed(0)
    dpp = DimeNetPP(energy_and_force=True, num_layers=2, hidden_channels=64, out_emb_channels=64).to(dev)
    opt = torch.optim.Adam(dpp.parameters(), lr=1e-3)
    losses = [run().train(dpp, opt, DataLoader(mols, 4, shuffle=False), True, 100, torch.nn.L1Loss(), dev)
              for _ in range(6)]
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    mae = run().val(dpp, DataLoader(mols, 4, shuffle=False), True, 100, ThreeDEvaluator(), dev)
    assert np.isfinite(mae)


def test_schnet_force_training_gradients_match_oracle():
    """d/d(parameters) of  L1(E, y) + p * L1(F, f)  with F = -dE/dpos taken with create_graph=True (run.py:110-123):
    the second backward through the twice-differentiable Functions (dig_b200/autograd_dd.py) vs torch.autograd over the
    oracle restatement."""
    from dig_b200.threedgraph.method import SchNet
    from oracle import restated
    dev = torch.device("cuda:0")
    _, z, pos, batch = case_inputs("schnet_cfg1", dev)
    model = SchNet(energy_and_force=True, num_layers=2, hidden_channels=32, num_filters=32, cutoff=10.0)
    sd = formula_state_dict(model.state_dict(), seed=1)
    model.load_state_dict(sd)
    model = model.to(dev)
    gen = torch.Generator().manual_seed(12)
    y = torch.randn(16, 1, generator=gen).to(dev)
    f_t = torch.randn(pos.size(0), 3, generator=gen).to(dev)
    p_w = 100.0

    def total_loss(energy, position):
        force = -torch.autograd.grad(energy, position, grad_outputs=torch.ones_like(energy), create_graph=True,
                                     retain_graph=True)[0]
        return torch.nn.functional.l1_loss(energy, y) + p_w * torch.nn.functional.l1_loss(force, f_t), force

    b = _batch(z, pos.clone(), batch)
    out = model(b)
    loss, force = total_loss(out, b.pos)
    assert force.requires_grad
    loss.backward()
    sd_ref = {k: v.to(dev).clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    pos2 = pos.clone().requires_grad_(True)
    ref = restated.schnet_forward(sd_ref, z, pos2, batch, cutoff=10.0, num_layers=2)
    ref_loss, ref_force = total_loss(ref, pos2)
    ref_loss.backward()
    assert rel_err(force.detach().cpu().numpy(), ref_force.detach().cpu().numpy()) < FTOL
    assert abs(loss.item() - ref_loss.item()) < 1e-5 * abs(ref_loss.item())
    bad = {}
    for name, prm in model.named_parameters():
        r = sd_ref[name].grad
        assert prm.grad is not None and r is not None, name
        err = rel_err(prm.grad.cpu().numpy(), r.cpu().numpy())
        if err > 2e-4:
            bad[name] = err
    assert not bad, bad


@pytest.mark.parametrize("name", ["dimenetpp_md17", "spherenet_qm9", "spherenet_ns3"])
def test_dimenet_family_force_training_gradients_match_oracle(name):
    """VERDICT r1 item 7: d/d(parameters) of  L1(E, y) + 100 * L1(F, f),  F = -dE/dpos under create_graph=True
    (reference run.py:110-123), for DimeNet++ and SphereNet.  The product differentiates the directional derivative of E
    along c = dL/dF (reverse over forward mode, dig_b200/autograd_jvp.py: geometry_jvp, edge_basis_tangent,
    triplet_basis_tangent, act''); the comparator is torch.autograd's double backward over the oracle restatement on the
    same GPU.  Every parameter tensor is compared (2e-4 of its largest entry)."""
    from dig_b200.threedgraph import method
    from helpers import CASES
    from oracle import restated
    dev = torch.device("cuda:0")
    model_name, ctor, _, wseed = CASES[name]
    _, z, pos, batch = case_inputs(name, dev)
    model = getattr(method, model_name)(energy_and_force=True, **ctor)
    sd = formula_state_dict(model.state_dict(), seed=wseed)
    model.load_state_dict(sd)
    model = model.to(dev)
    n_mol = int(batch.max()) + 1
    gen = torch.Generator().manual_seed(21)
    y = torch.randn(n_mol, 1, generator=gen).to(dev)
    f_t = torch.randn(pos.size(0), 3, generator=gen).to(dev)

    def total_loss(energy, position):
        force = -torch.autograd.grad(energy, position, grad_outputs=torch.ones_like(energy), create_graph=True,
                                     retain_graph=True)[0]
        return torch.nn.functional.l1_loss(energy, y) + 100.0 * torch.nn.functional.l1_loss(force, f_t), force

    b = _batch(z, pos.clone(), batch)
    out = model(b)
    loss, force = total_loss(out, b.pos)
    assert force.requires_grad, "the force must stay differentiable in the parameters"
    loss.backward()
    sd_ref = {k: v.to(dev).clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    pos2 = pos.clone().requires_grad_(True)
    kw = {k: v for k, v in ctor.items() if k in ("cutoff", "num_layers", "num_spherical", "num_radial")}
    ref = restated.dimenet_family_forward(sd_ref, z, pos2, batch, torsion=(model_name == "SphereNet"), **kw)
    ref_loss, ref_force = total_loss(ref, pos2)
    ref_loss.backward()
    assert rel_err(force.detach().cpu().numpy(), ref_force.detach().cpu().numpy()) < FTOL
    assert abs(loss.item() - ref_loss.item()) < 1e-5 * abs(ref_loss.item())
    bad, checked = {}, 0
    for pname, prm in model.named_parameters():
        r = sd_ref[pname].grad
        if r is None:
            continue
        assert prm.grad is not None, pname
        checked += 1
        err = rel_err(prm.grad.cpu().numpy(), r.cpu().numpy())
        if err > 2e-4:
            bad[pname] = err
    assert checked > 50 and not bad, (checked, bad)


@pytest.mark.parametrize("name", ["spherenet_qm9", "spherenet_ns3"])
def test_spherenet_forces_match_oracle_autograd(name):
    """SphereNet forces (torsion basis + torsion-angle backward through the minimising candidate) vs torch.autograd over
    the oracle restatement on the same GPU (the real reference's CPU forces differ in the self-candidate coin flips of
    the torsion, SURVEY.md 5.9b, so the comparator must share the device arithmetic)."""
    from dig_b200.threedgraph.method import SphereNet
    from helpers import CASES
    from oracle import restated
    dev = torch.device("cuda:0")
    _, ctor, _, wseed = CASES[name]
    _, z, pos, batch = case_inputs(name, dev)
    model = SphereNet(energy_and_force=True, **ctor)
    sd = formula_state_dict(model.state_dict(), seed=wseed)
    model.load_state_dict(sd)
    model = model.to(dev)
    b = _batch(z, pos.clone(), batch)
    out = model(b)
    force = -torch.autograd.grad(out, b.pos, grad_outputs=torch.ones_like(out), create_graph=True)[0].detach()
    pos2 = pos.clone().requires_grad_(True)
    kw = {k: v for k, v in ctor.items() if k in ("cutoff", "num_spherical")}
    ref = restated.spherenet_forward({k: v.to(dev) for k, v in sd.items()}, z, pos2, batch, **kw)
    f_ref = -torch.autograd.grad(ref.sum(), pos2)[0]
    assert rel_err(out.detach().cpu().numpy(), ref.detach().cpu().numpy()) < 1e-5
    assert rel_err(force.cpu().numpy(), f_ref.cpu().numpy()) < FTOL


@pytest.mark.parametrize("k,nout", [(128, 128), (64, 128), (128, 64), (256, 128), (384, 128)])
def test_linear_tc_matches_fp64(k, nout):
    """wgmma 3xTF32 linear of the training path (forward, fused swish, and the W^T orientation used for dX)."""
    from dig_b200 import ops
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(k + nout)
    rows = 1000
    x = torch.randn(rows, k, generator=gen).to(dev)
    w = (torch.randn(nout, k, generator=gen) / k ** 0.5).to(dev)
    b = torch.randn(nout, generator=gen).to(dev)
    y, a = ops.linear_tc(x, w, b, want_act=True)
    ref = torch.nn.functional.linear(x.double(), w.double(), b.double())
    assert rel_err(y.cpu().numpy(), ref.cpu().numpy()) < 2e-6
    assert rel_err(a.cpu().numpy(), (ref * torch.sigmoid(ref)).cpu().numpy()) < 2e-6
    if ops.linear_tc_supported(nout, k):
        dy = torch.randn(rows, nout, generator=gen).to(dev)
        dx = ops.linear_tc(dy, w, None, transposed=True)
        assert rel_err(dx.cpu().numpy(), (dy.double() @ w.double()).cpu().numpy()) < 2e-6
    w2 = w.clone()
    w2.mul_(2.0)                                       # new storage: packed separately
    y2 = ops.linear_tc(x, w2, b)
    assert rel_err(y2.cpu().numpy(), torch.nn.functional.linear(x.double(), w2.double(), b.double()).cpu().numpy()) < 2e-6
    w.mul_(0.5)                                        # in-place update bumps _version: the cache must re-pack
    y3 = ops.linear_tc(x, w, b)
    assert rel_err(y3.cpu().numpy(), torch.nn.functional.linear(x.double(), w.double(), b.double()).cpu().numpy()) < 2e-6
    assert ops.tc_timeouts() == 0


def test_training_path_on_tensor_cores_opt_in(monkeypatch):
    """DIG3D_TRAIN_DENSE=tc: the 128-wide linears (forward and input-gradient GEMMs) on wgmma 3xTF32; two different
    models back to back (freed parameters' addresses get reused: the packed-weight copies must not be)."""
    from dig_b200.threedgraph import method
    from helpers import CASES
    from oracle import restated
    from dig_b200 import ops
    monkeypatch.setenv("DIG3D_TRAIN_DENSE", "tc")
    dev = torch.device("cuda:0")
    for name in ("spherenet_qm9", "dimenetpp_md17", "spherenet_qm9"):
        model_name, ctor, _, wseed = CASES[name]
        _, z, pos, batch = case_inputs(name, dev)
        model = getattr(method, model_name)(**ctor)
        sd = formula_state_dict(model.state_dict(), seed=wseed)
        model.load_state_dict(sd)
        model = model.to(dev)
        sd = {k: v.to(dev) for k, v in sd.items()}
        nb = int(batch.max().item()) + 1
        target = torch.linspace(-1, 1, nb, device=dev).view(nb, 1)
        fwd = restated.spherenet_forward if model_name == "SphereNet" else restated.dimenetpp_forward
        _grad_compare(model, sd, lambda s_, *a: fwd(s_, *a, cutoff=5.0), z, pos, batch, target)
        assert any("_dig3d_packed" in p.__dict__ for p in model.parameters())      # the tensor path really ran
        del model
    assert ops.tc_timeouts() == 0


def test_run_run_end_to_end(tmp_path, capsys):
    """run().run(...) as in the reference notebook (threedgraph.ipynb cell 11 / run.py:20-101): two epochs on synthetic
    molecules, checkpoint written with the reference's keys, printed summary lines."""
    from dig_b200.data import synthetic_molecules
    from dig_b200.threedgraph.evaluation import ThreeDEvaluator
    from dig_b200.threedgraph.method import SchNet, run
    dev = torch.device("cuda:0")
    mols = synthetic_molecules(24, natoms=8, seed=2)
    for m in mols:
        m.y = torch.tensor([float(m.z.sum()) * 0.05])
    torch.manual_seed(0)
    model = SchNet(num_layers=2, hidden_channels=32, num_filters=32, cutoff=5.0)
    run().run(dev, mols[:16], mols[16:20], mols[20:], model, loss_func=torch.nn.L1Loss(), evaluation=ThreeDEvaluator(),
              epochs=2, batch_size=8, vt_batch_size=4, lr=1e-3, lr_decay_factor=0.5, lr_decay_step_size=1,
              save_dir=str(tmp_path / "ckpt"), log_dir='')
    out = capsys.readouterr().out
    assert "#Params: 15393" in out and "=====Epoch 2" in out and "Best validation MAE so far" in out
    ckpt = torch.load(str(tmp_path / "ckpt" / "valid_checkpoint.pt"), weights_only=False)
    assert set(ckpt) == {'epoch', 'model_state_dict', 'optimizer_state_dict', 'scheduler_state_dict', 'best_valid_mae',
                         'num_params'}
    fresh = SchNet(num_layers=2, hidden_channels=32, num_filters=32, cutoff=5.0)
    fresh.load_state_dict(ckpt['model_state_dict'])


@pytest.mark.parametrize("k,nout,act", [(128, 256, False), (256, 256, True), (256, 1, False), (48, 80, True)])
def test_grouped_linear_fwd_bwd(k, nout, act):
    """G independent linears in one launch (the node MLPs of all interaction blocks) vs a loop of fp64 linears."""
    from dig_b200 import autograd as ag
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(k + nout)
    G, rows = 5, 300
    mods = [torch.nn.Linear(k, nout, bias=(nout != 1)).to(dev) for _ in range(G)]
    x = torch.randn(G, rows, k, generator=gen).to(dev).requires_grad_(True)
    dy = torch.randn(G, rows, nout, generator=gen).to(dev)
    y = ag.grouped_lin(mods, x, act=act)
    y.backward(dy)
    x2 = x.detach().double().requires_grad_(True)
    ys, refs = [], []
    for g_, m in enumerate(mods):
        w2 = m.weight.detach().double().requires_grad_(True)
        b2 = m.bias.detach().double().requires_grad_(True) if m.bias is not None else None
        o = torch.nn.functional.linear(x2[g_], w2, b2)
        ys.append(o * torch.sigmoid(o) if act else o)
        refs.append((w2, b2))
    y2 = torch.stack(ys)
    y2.backward(dy.double())
    assert rel_err(y.detach().cpu().numpy(), y2.detach().cpu().numpy()) < 2e-5
    assert rel_err(x.grad.cpu().numpy(), x2.grad.cpu().numpy()) < 2e-5
    for m, (w2, b2) in zip(mods, refs):
        assert rel_err(m.weight.grad.cpu().numpy(), w2.grad.cpu().numpy()) < 2e-5
        if b2 is not None:
            assert rel_err(m.bias.grad.cpu().numpy(), b2.grad.cpu().numpy()) < 2e-5


def test_flat_adam_matches_torch_adam():
    """parallel.FlatAdam (one fused kernel over the flat parameter / gradient / moment buffers) vs torch.optim.Adam
    on the same gradients: 5 steps with weight decay and a StepLR schedule, then the state_dict round trip."""
    from dig_b200 import parallel
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    mk = lambda: torch.nn.Sequential(torch.nn.Linear(37, 19), torch.nn.Linear(19, 3), torch.nn.Linear(3, 1)).to(dev)
    a, b = mk(), mk()
    b.load_state_dict(a.state_dict())
    flat = parallel.FlatParameters(a)
    assert all(p.data_ptr() % 16 == 0 for p in a.parameters())
    opt_a = parallel.FlatAdam(flat, lr=1e-2, weight_decay=1e-3)
    opt_b = torch.optim.Adam(b.parameters(), lr=1e-2, weight_decay=1e-3)
    sch_a = torch.optim.lr_scheduler.StepLR(opt_a, step_size=2, gamma=0.5)
    sch_b = torch.optim.lr_scheduler.StepLR(opt_b, step_size=2, gamma=0.5)
    for step in range(5):
        x = torch.randn(11, 37, device=dev)
        opt_a.zero_grad()
        opt_b.zero_grad()
        a(x).square().mean().backward()
        b(x).square().mean().backward()
        for p, q in zip(a.parameters(), b.parameters()):
            assert p.grad.data_ptr() >= flat.grad.data_ptr()          # autograd accumulated into the flat views
            # (cuBLAS may pick another algorithm for the differently aligned views: equal to fp32 rounding)
            assert rel_err(p.grad.cpu().numpy(), q.grad.cpu().numpy()) < 1e-5
            q.grad.copy_(p.grad)                                      # same gradients into both optimizers
        opt_a.step()
        opt_b.step()
        sch_a.step()
        sch_b.step()
        for p, q in zip(a.parameters(), b.parameters()):
            assert rel_err(p.detach().cpu().numpy(), q.detach().cpu().numpy()) < 2e-6, step
    sd = opt_a.state_dict()
    assert set(sd["state"][0]) == {"step", "exp_avg", "exp_avg_sq"} and float(sd["state"][0]["step"]) == 5.0
    ref = opt_b.state_dict()
    for k in sd["state"]:
        assert rel_err(sd["state"][k]["exp_avg_sq"].cpu().numpy(), ref["state"][k]["exp_avg_sq"].cpu().numpy()) < 1e-5
    opt_c = parallel.FlatAdam(flat, lr=1e-2, weight_decay=1e-3)
    opt_c.load_state_dict(sd)
    assert opt_c.steps == 5 and torch.equal(opt_c.exp_avg, opt_a.exp_avg)


def test_warp_triplet_gather_splits_equal_edge_centred():
    """The warp-per-source-node gather (x_down rows staged in the warp's shared memory) sums the same triplets in the
    same order as the one-warp-per-edge kernel: m is BITWISE equal at splits 1, 2, 3 and the graph's own split, with
    and without the torsion factor, incl. isolated atoms."""
    import ctypes
    from dig_b200 import ops
    from dig_b200.data import synthetic_batch, collate, Molecule
    dev = torch.device("cuda:0")
    mols = synthetic_batch(9, "qm9", seed=4, variable=True)
    far = torch.tensor([[50.0, 50.0, 50.0]])
    b = collate([Molecule(mols.z[:7], mols.pos[:7]), Molecule(torch.tensor([6]), far),
                 Molecule(mols.z[7:40], mols.pos[7:40])]).to(dev)
    g = ops.build_graph(b.pos, b.batch, 5.0, num_graphs=3)
    ops.triplet_geometry(g, b.pos, use_torsion=True, want_idx=False)
    e, t = g.n_edges, g.n_triplets
    torch.manual_seed(1)
    x_down = torch.randn(e, 64, device=dev)
    sbf_p, t_p = torch.randn(t, 8, device=dev), torch.randn(t, 8, device=dev)
    w_s, w_t = torch.randn(64, 8, device=dev), torch.randn(64, 8, device=dev)
    for tors in (True, False):
        sp, tp = ctypes.c_void_p(sbf_p.data_ptr()), ctypes.c_void_p(t_p.data_ptr()) if tors else None
        ws, wt = w_s.data_ptr(), w_t.data_ptr() if tors else None
        edge = torch.full((e, 64), float("nan"), device=dev)
        ops.call("dig3d_sphere_triplet_gather", ops._p(x_down), sp, tp, 8, ops._p(g.src), ops._p(g.dst),
                 ops._p(g.row_ptr), ops._p(g.trip_ptr), e, ws, wt, ops._p(edge), ops._stream())
        assert torch.isfinite(edge).all(), tors
        for split in (1, 2, 3, None):
            m = torch.full((e, 64), float("nan"), device=dev)
            ops.triplet_gather(x_down, sp, tp, g, ws, wt, m, ops._stream(), split=split)
            assert torch.equal(edge, m), (tors, split)


def test_training_step_parity_at_the_headline_size():
    """BASELINE configs[1] / [4] per-GPU size (SphereNet defaults, 128 QM9-shape molecules): loss and EVERY parameter
    gradient of one training step vs torch.autograd over the oracle on the same GPU (VERDICT r1 item 1c asked for the
    loss + 5 tensors; _grad_compare checks all of them)."""
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph.method import SphereNet
    from oracle import restated
    dev = torch.device("cuda:0")
    model = SphereNet()
    sd = formula_state_dict(model.state_dict(), seed=2)
    model.load_state_dict(sd)
    model = model.to(dev)
    sd = {k: v.to(dev) for k, v in sd.items()}
    b = synthetic_batch(128, "qm9", seed=2).to(dev)
    target = torch.linspace(-1, 1, 128, device=dev).view(128, 1)
    worst = _grad_compare(model, sd, restated.spherenet_forward, b.z, b.pos, b.batch, target)
    for name in ("init_e.lin.weight", "update_es.0.lin_t1.weight", "update_es.3.lin_kj.weight",
                 "update_vs.3.lin.weight", "emb.dist_emb.freq"):
        assert worst[name] < GTOL, (name, worst[name])


def test_config5_global_batch_1024_shards_reproduce_the_single_batch():
    """BASELINE configs[4]: a global batch of 1024 QM9-shape molecules split into contiguous per-rank shards
    (parallel.shard_molecules, world = 2 / 4 / 8; each shard evaluated here in turn) gives the energies of the
    unsplit batch in rank order -- the path has no cross-molecule term.  Tile boundaries fall differently in a shard,
    so the comparison is to fp32 rounding, and the unsplit batch is checked against the oracle."""
    from dig_b200 import parallel
    from dig_b200.data import collate, synthetic_molecules
    from dig_b200.threedgraph.method import SphereNet
    from oracle import restated
    dev = torch.device("cuda:0")
    model = SphereNet()
    sd = formula_state_dict(model.state_dict(), seed=2)
    model.load_state_dict(sd)
    model = model.to(dev)
    mols = synthetic_molecules(1024, "qm9", seed=2)
    with torch.no_grad():
        full = model(collate(mols).to(dev))
        for world in (2, 4, 8):
            parts = [model(collate(parallel.shard_molecules(mols, r, world)).to(dev)) for r in range(world)]
            got = torch.cat(parts, 0)
            assert got.shape == full.shape == (1024, 1)
            assert rel_err(got.cpu().numpy(), full.cpu().numpy()) < 2e-6, world
        b = collate(mols[:256]).to(dev)
        ref = restated.spherenet_forward({k: v.to(dev) for k, v in sd.items()}, b.z, b.pos, b.batch)
    assert rel_err(full[:256].cpu().numpy(), ref.cpu().numpy()) < 1e-5


@pytest.mark.parametrize("k,nout", [(128, 128), (64, 128), (128, 64), (256, 256), (384, 128), (128, 256), (256, 64)])
def test_linear_on_the_two_tile_engine_matches_fp64(k, nout):
    """dig3d_linear_h16 (3xFP16 operands on wgmma): y = x W^T + b, its fused swish output and the input-gradient GEMM
    (packed W^T, column slices) vs fp64, ragged row count, odd tile count."""
    from dig_b200 import ops
    dev = torch.device("cuda:0")
    torch.manual_seed(k * 7 + nout)
    for rows in (1300, 129):
        x = torch.randn(rows, k, device=dev)
        w = torch.nn.Parameter(torch.randn(nout, k, device=dev) / k ** 0.5)
        b = torch.randn(nout, device=dev)
        y, a = ops.linear_h16(x, w, b, want_act=True)
        wd = w.detach().double()
        ref = x.double() @ wd.t() + b.double()
        assert rel_err(y.cpu().numpy(), ref.cpu().numpy()) < 2e-6
        assert rel_err(a.cpu().numpy(), (ref * torch.sigmoid(ref)).cpu().numpy()) < 2e-6
        res = torch.randn(rows, nout, device=dev)
        a_r = ops.linear_h16(x, w, b, want_act=True, act_only=True, residual=res)      # swish(y) + r, y not written
        assert rel_err(a_r.cpu().numpy(), (ref * torch.sigmoid(ref) + res.double()).cpu().numpy()) < 2e-6
        y_r = ops.linear_h16(x, w, b, residual=res)                                    # y + r
        assert rel_err(y_r.cpu().numpy(), (ref + res.double()).cpu().numpy()) < 2e-6
        y_p, a_p = ops.linear_h16(x, w, b, want_act=True, residual=res)                # pre-activation untouched
        assert torch.equal(y_p, y) and torch.equal(a_p, a_r)
        dy = torch.randn(rows, nout, device=dev)
        dx = ops.linear_h16(dy, w, None, transposed=True)
        assert rel_err(dx.cpu().numpy(), (dy.double() @ wd).cpu().numpy()) < 2e-6
        with torch.no_grad():
            w.mul_(0.5)                                  # a parameter update must be seen (version-keyed cache)
        y2 = ops.linear_h16(x, w, b)
        assert rel_err(y2.cpu().numpy(), (x.double() @ w.detach().double().t() + b.double()).cpu().numpy()) < 2e-6
    assert ops.tc_timeouts() == 0 and not ops.h16_overflow()


@pytest.mark.parametrize("rows,nout,k,groups", [(39000, 128, 128, 1), (5000, 128, 384, 1), (4097, 64, 128, 1),
                                                (1031, 128, 64, 1), (2304, 256, 256, 5), (2304, 256, 128, 5),
                                                (20000, 100, 72, 1)])
def test_weight_gradient_on_the_tensor_cores_matches_fp64(rows, nout, k, groups):
    """dig3d_wgrad_tc (3xTF32 wgmma, transposed operand tiles built on the fly, csrc/train_tc.cu) vs fp64 and vs the
    FFMA kernel: dW = dY^T X and db = colsum dY, ragged row counts and widths, wide dynamic range of dY, grouped."""
    from dig_b200 import ops
    dev = torch.device("cuda:0")
    torch.manual_seed(rows + nout + k)
    lead = (groups,) if groups > 1 else ()
    x = torch.randn(lead + (rows, k), device=dev)
    dy = torch.randn(lead + (rows, nout), device=dev) * torch.logspace(-9, 0, nout, device=dev)   # gradient-like range
    shape = lead + (nout, k)
    assert ops._lib.load().dig3d_wgrad_tc_supported(rows, nout, k) == 1
    dw, db = ops.wgrad(dy, x, shape, True)
    ops.wgrad_set_mode(False)
    try:
        dw_s, db_s = ops.wgrad(dy, x, shape, True)
    finally:
        ops.wgrad_set_mode(True)
    ref = dy.double().transpose(-1, -2) @ x.double()
    ref_b = dy.double().sum(-2)
    torch.cuda.synchronize()
    assert ops.tc_timeouts() == 0
    # column-wise comparison: every output row n has its own scale (1e-9 .. 1)
    scale = ref.abs().amax(-1, keepdim=True)
    err = ((dw.double() - ref).abs() / scale).max().item()
    err_s = ((dw_s.double() - ref).abs() / scale).max().item()
    assert err < 5e-6, (err, err_s)
    col_scale = dy.double().abs().sum(-2)             # a column sum may cancel: compare against the sum of magnitudes
    assert ((db.double() - ref_b).abs() / col_scale).max().item() < 1e-6
    assert rel_err(db.cpu().numpy(), db_s.cpu().numpy()) < 1e-5
