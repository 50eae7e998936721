"""ComENet forces and training on forces (csrc/comenet.cu dig3d_comenet_features_bwd / _tangent, csrc/train_ops.cu
dig3d_graphnorm_tangent / _bwd, ComENet(energy_and_force=True)).

ComENet's own fp32-vs-fp64 energy gap is 0.26 to 0.41 (the 0/0 noise of phi / tau, DESIGN.md section 3), so, as for
its energies (tests/test_gpu_parity.py::test_comenet_energy_parity), the comparator of the model and of the geometry
derivatives is torch.autograd over the restatement on the same GPU: the forward features are bit for bit the
restatement's there, and its autograd takes ATen's derivatives at the same angles.  The restatement is
tests/comenet_force_ref.py: oracle/restated.py's op sequence with the aliased cross products (a x a, whose ATen value is
an FMA residue) held constant, which is the exact derivative the kernels take.  Plain autograd over oracle/restated.py
adds terms of size |g| / residue that cancel only to their own last bits: O(1) noise in the forces that changes with
the order of the (atomic) sums, so no bound can hold against it."""
import math

import numpy as np
import pytest
import torch

import comenet_force_ref as cfr
from helpers import GOLDEN, case_inputs, formula_state_dict, rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FTOL = 1e-5                # forces, relative to the largest force component
GTOL = 2e-4                # force-training parameter gradients, relative to each tensor's largest entry


def _batch(z, pos, batch):
    from dig_b200.data import Batch
    return Batch(z=z, pos=pos, batch=batch)


# ----------------------------------------------------------------------------- the geometry kernels
def _graph(name):
    """(pos, batch, cutoff) of the graphs the derivative kernels are checked on."""
    gen = torch.Generator().manual_seed(5)
    if name == "oc20":
        _, _, pos, batch = case_inputs("comenet_oc20")
        return pos, batch, 6.0
    if name == "no_out_edge":      # tests/test_gpu_parity.py::test_comenet_reference_atoms_when_a_node_has_no_out_edge
        mol0 = torch.tensor([[0.03, 1.5, 0.07], [0.0, 0.0, 0.0], [1.0, 0.02, -0.05], [0.04, -0.03, 2.2],
                             [2.0, 2.0, 0.3]])
        pos = torch.cat([mol0, 20.0 + torch.rand(70, 3, generator=gen) * 3.0])
        return pos, torch.cat([torch.zeros(5, dtype=torch.long), torch.ones(70, dtype=torch.long)]), 6.0
    if name == "single_in_edge":   # atom 3 sees only atom 1 (e0i == e1i for its one in-edge)
        pos = torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.1, 0.0], [0.2, 1.1, 0.3], [4.5, 0.2, 0.1]])
        return pos, torch.zeros(4, dtype=torch.long), 4.0
    if name == "two_atoms":
        return torch.tensor([[0.0, 0.0, 0.0], [1.1, 0.2, -0.1]]), torch.zeros(2, dtype=torch.long), 5.0
    if name == "isolated_atom":    # a 4-atom molecule and a one-atom molecule (no edge)
        pos = torch.tensor([[0.0, 0.0, 0.0], [1.2, 0.1, 0.0], [0.3, 1.0, 0.4], [-0.8, -0.5, 0.6], [9.0, 9.0, 9.0]])
        return pos, torch.tensor([0, 0, 0, 0, 1]), 5.0
    if name == "planar":           # every atom at z = 0: signed-zero phi / tau planes (SURVEY.md 5.9b)
        ang = torch.arange(6, dtype=torch.float64) * (np.pi / 3)
        ring = torch.stack([1.4 * ang.cos(), 1.4 * ang.sin(), torch.zeros(6, dtype=torch.float64)], 1)
        h = torch.stack([2.5 * ang[:3].cos(), 2.5 * ang[:3].sin(), torch.zeros(3, dtype=torch.float64)], 1)
        return torch.cat([ring, h]).float(), torch.zeros(9, dtype=torch.long), 5.0
    raise KeyError(name)


GRAPHS = ["oc20", "no_out_edge", "single_in_edge", "two_atoms", "isolated_atom", "planar"]


def _setup(name):
    from dig_b200 import ops
    pos, batch, cutoff = _graph(name)
    pos, batch = pos.to(DEV).contiguous(), batch.to(DEV)
    g = ops.build_graph(pos, batch, cutoff, num_graphs=int(batch.max()) + 1)
    f1, f2, ang = ops.comenet_geometry(g, pos, cutoff, want_angles=True)
    gen = torch.Generator().manual_seed(11)
    u1 = torch.randn(g.n_edges, 12, generator=gen).to(DEV)
    u2 = torch.randn(g.n_edges, 6, generator=gen).to(DEV)
    return g, pos, batch, cutoff, f1, f2, ang, u1, u2


def _restated_features(pos, batch, cutoff, ang, planar):
    """(edge_index, (f1, f2)) of the restatement, differentiable in pos.  Its angles equal the kernel's bit for bit,
    except, on an exactly planar molecule, phi / tau of edges whose planes are parallel: their atan2 reads a signed
    zero, and ATen's cross product and the kernel's emulation of it do not always give the zero the same sign, so the
    fold lands on 0 on one side and on pi on the other (SURVEY.md 5.9b; the reference itself is discontinuous there).
    Those values are taken from the kernel (the derivative stays the restatement's), so both differentiate the same
    features."""
    from oracle import restated
    ei = restated.radius_graph(pos, cutoff, batch)
    dist, theta, phi, tau = cfr.comenet_geometry(pos, ei, pos.size(0), cutoff)
    out = []
    for k, t in enumerate((theta, phi, tau)):
        differ = t.detach() != ang[:, k]
        if planar and k > 0:
            pair = torch.stack([t.detach()[differ], ang[differ, k]], 1).sort(1).values
            assert torch.equal(pair, torch.tensor([[0.0, math.pi]], device=DEV).float().expand_as(pair))
            t = t + (ang[:, k] - t).detach()
        else:
            assert not differ.any()
        out.append(t)
    return ei, restated.comenet_features(dist, *out, cutoff)


@pytest.mark.parametrize("name", GRAPHS)
def test_features_bwd_matches_autograd_of_the_restatement(name):
    """dig3d_comenet_features_bwd against torch.autograd (fp32, same GPU) of the restated geometry (aliased cross
    products held constant, tests/comenet_force_ref.py) + restated.comenet_features for random feature gradients,
    element by element within FTOL of the largest component; two runs give the same bits."""
    from dig_b200 import ops
    g, pos, batch, cutoff, f1, f2, ang, u1, u2 = _setup(name)
    p = pos.clone().requires_grad_(True)
    ei, (r1, r2) = _restated_features(p, batch, cutoff, ang, planar=(name == "planar"))
    assert torch.equal(g.edge_index, ei)
    assert torch.equal(f1, r1.detach()) and torch.equal(f2, r2.detach())
    want = torch.autograd.grad((r1 * u1).sum() + (r2 * u2).sum(), p, allow_unused=True)[0]
    if want is None:
        want = torch.zeros_like(pos)
    got = ops.comenet_features_bwd(g, pos, cutoff, u1, u2)
    again = ops.comenet_features_bwd(g, pos, cutoff, u1, u2)
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    assert torch.equal(got, again)
    scale = max(float(want.abs().max()), 1e-30)
    err = (got - want).abs()
    assert float(err.max()) <= FTOL * scale, (name, float(err.max()) / scale, int(err.argmax()) // 3)
    if name == "isolated_atom":
        assert torch.equal(got[4], torch.zeros(3, device=DEV))


@pytest.mark.parametrize("name", GRAPHS)
def test_features_tangent_is_the_transpose_of_bwd(name):
    """<bwd(u), c> = <u, tangent(c)> to fp32 rounding, in fp64 sums."""
    from dig_b200 import ops
    g, pos, batch, cutoff, f1, f2, _, u1, u2 = _setup(name)
    c = torch.randn(pos.size(0), 3, generator=torch.Generator().manual_seed(3)).to(DEV)
    dpos = ops.comenet_features_bwd(g, pos, cutoff, u1, u2).double()
    t1, t2 = ops.comenet_features_tangent(g, pos, cutoff, c)
    lhs = (dpos * c.double()).sum()
    terms = torch.cat([(u1.double() * t1.double()).flatten(), (u2.double() * t2.double()).flatten()])
    rhs = terms.sum()
    scale = float(terms.abs().sum() + (dpos * c.double()).abs().sum()) + 1e-30
    assert abs(float(lhs - rhs)) <= 1e-5 * scale, (name, float(lhs), float(rhs), scale)


def _graphnorm64(h, hd, w, ms, sizes, eps=1e-5):
    """y_dot of GraphNorm in fp64 from the formula: per graph, out = h - ms mean(h), std = sqrt(mean(out^2) + eps)."""
    outs = []
    for hs, hds in zip(torch.split(h, sizes), torch.split(hd, sizes)):
        out = hs - ms * hs.mean(0)
        std = ((out * out).mean(0) + eps).sqrt()
        od = hds - ms * hds.mean(0)
        sd_dot = (out * od).mean(0) / std
        outs.append(w * (od / std - out * sd_dot / std ** 2))
    return torch.cat(outs)


def _graphnorm_value64(h, w, b, ms, sizes, eps=1e-5):
    outs = []
    for hs in torch.split(h, sizes):
        out = hs - ms * hs.mean(0)
        outs.append(w * out / ((out * out).mean(0) + eps).sqrt() + b)
    return torch.cat(outs)


@pytest.mark.parametrize("width,mean_scale", [(256, "scaled"), (128, "scaled"), (256, "ones")])
def test_graphnorm_tangent_and_its_backward_against_fp64(width, mean_scale):
    """dig3d_graphnorm_tangent against torch.func.jvp of GraphNorm in fp64, and dig3d_graphnorm_tangent_bwd against
    fp64 autograd of the tangent formula, on ragged graphs (one with a single node), from the same fp32 inputs.
    mean_scale in [0.5, 0.8] ("scaled"), or 1 (its initial value: a one-node graph's centred value is then exactly 0).
    Conditioning: the tangent is o_dot / std - o std_dot / std^2, two terms of size |h_dot| / std that cancel when a
    channel's values in a graph nearly coincide (std -> sqrt(eps)), and a mean_scale within ~1e-3 of 1 leaves a one-node
    graph's centred value h (1 - mean_scale) with only the leading bits of the fp32 shift; no fixed fp32 bound holds
    there, so the values of each channel are spread around their graph's mean by alternating deviations of 0.5 to 1.5,
    and mean_scale is 1 exactly or at least 0.2 away from it."""
    from dig_b200 import ops
    sizes = [1, 5, 17, 3, 2]
    n = sum(sizes)
    gen = torch.Generator().manual_seed(width)
    r32 = lambda t: t.float().double()                     # the fp32 inputs, exactly, in fp64
    graph = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    rank = torch.cat([torch.arange(s) for s in sizes])
    spread = (1 - 2 * (rank % 2)).double().unsqueeze(1) * (0.5 + torch.rand(n, width, generator=gen, dtype=torch.float64))
    h = r32((torch.randn(len(sizes), width, generator=gen, dtype=torch.float64) * 2 + 0.5)[graph] + spread)
    hd = r32(torch.randn(n, width, generator=gen, dtype=torch.float64))
    w = r32(1 + 0.3 * torch.randn(width, generator=gen, dtype=torch.float64))
    b = r32(0.1 * torch.randn(width, generator=gen, dtype=torch.float64))
    ms = r32(0.5 + 0.3 * torch.rand(width, generator=gen, dtype=torch.float64))
    if mean_scale == "ones":
        ms = torch.ones_like(ms)
    gy = r32(torch.randn(n, width, generator=gen, dtype=torch.float64))
    ptr = torch.tensor([0] + list(np.cumsum(sizes)), dtype=torch.int32, device=DEV)
    f = lambda t: t.float().to(DEV).contiguous()
    _, shift, std = ops.graphnorm(f(h), ptr, f(w), f(b), f(ms))
    yd = ops.graphnorm_tangent(f(h), f(hd), ptr, f(w), f(ms), shift, std)
    _, yd_ref = torch.func.jvp(lambda x: _graphnorm_value64(x, w, b, ms, sizes), (h,), (hd,))
    assert torch.allclose(_graphnorm64(h, hd, w, ms, sizes), yd_ref, rtol=1e-10, atol=1e-12)
    assert rel_err(yd.cpu().numpy(), yd_ref.numpy()) < 1e-5
    dh, dhd, dw, dms = ops.graphnorm_tangent_bwd(f(h), f(hd), f(gy), ptr, f(w), f(ms), shift, std)
    leaves = [t.clone().requires_grad_(True) for t in (h, hd, w, ms)]
    ref = torch.autograd.grad((_graphnorm64(*leaves, sizes) * gy).sum(), leaves)
    for name, got, want in zip(("h", "h_dot", "weight", "mean_scale"), (dh, dhd, dw, dms), ref):
        assert rel_err(got.cpu().numpy(), want.numpy()) < 2e-5, name


# ----------------------------------------------------------------------------- the model
def _fixture(name):
    g = np.load(f"{GOLDEN}/comenet_forces.npz")
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}


def _case(name, energy_and_force=True):
    from dig_b200.threedgraph.method import ComENet
    from oracle.gen_golden_comenet_forces import CASES
    ctor, _, wseed = CASES[name]
    gold = _fixture(name)
    torch.manual_seed(0)
    model = ComENet(energy_and_force=energy_and_force, **ctor)
    sd = formula_state_dict(model.state_dict(), seed=wseed)
    model.load_state_dict(sd)
    model = model.to(DEV)
    z, pos, batch = (torch.from_numpy(gold[k]).to(DEV) for k in ("z", "pos", "batch"))
    return model, {k: v.to(DEV) for k, v in sd.items()}, gold, z, pos, batch, ctor


def _restated(sd, z, pos, batch, ctor):
    from oracle.gen_golden_comenet_forces import restated_kwargs
    return cfr.comenet_forward(sd, z, pos, batch, **restated_kwargs(ctor))


CASE_NAMES = ["aspirin_default", "oc20_capped", "aspirin_generic"]


@pytest.mark.parametrize("name", CASE_NAMES)
def test_forces_match_autograd_over_the_restatement(name):
    """-grad(E, pos) with energy_and_force=True, and with the flag off and pos.requires_grad_() set by the caller, within
    FTOL of the largest force of torch.autograd over the restatement on the same GPU; the energy is bit for bit the
    energy-only training path's."""
    model, sd, gold, z, pos, batch, ctor = _case(name)
    model.eval()
    p2 = pos.clone().requires_grad_(True)
    r = _restated(sd, z, p2, batch, ctor)
    f_ref = -torch.autograd.grad(r.sum(), p2)[0]
    b = _batch(z, pos.clone(), batch)
    e = model(b)
    assert b.pos.requires_grad
    f = -torch.autograd.grad(e.sum(), b.pos)[0]
    assert rel_err(f.cpu().numpy(), f_ref.cpu().numpy()) < FTOL
    assert rel_err(e.detach().cpu().numpy(), r.detach().cpu().numpy()) < 1e-5
    model.energy_and_force = False
    b = _batch(z, pos.clone().requires_grad_(True), batch)
    e2 = model(b)
    f2 = -torch.autograd.grad(e2.sum(), b.pos)[0]
    assert rel_err(f2.cpu().numpy(), f_ref.cpu().numpy()) < FTOL
    e_only = model(_batch(z, pos.clone(), batch))                # grad enabled, pos constant: the training path
    assert torch.equal(e.detach(), e_only.detach()) and torch.equal(e2.detach(), e_only.detach())


@pytest.mark.parametrize("name", CASE_NAMES)
def test_force_training_gradients_match_double_backward(name):
    """d/d(parameters) of L1(E, y) + 100 * L1(F, f), F = -dE/dpos under create_graph=True (model.train()), against
    torch.autograd's double backward over the restatement on the same GPU; every parameter within GTOL of its largest
    entry."""
    model, sd, gold, z, pos, batch, ctor = _case(name)
    model.train()
    y = torch.from_numpy(gold["y"]).to(DEV)
    f_t = torch.from_numpy(gold["force_target"]).to(DEV)

    def total_loss(energy, position):
        force = -torch.autograd.grad(energy, position, grad_outputs=torch.ones_like(energy), create_graph=True,
                                     retain_graph=True)[0]
        return torch.nn.functional.l1_loss(energy, y) + 100.0 * torch.nn.functional.l1_loss(force, f_t), force

    b = _batch(z, pos.clone(), batch)
    loss, force = total_loss(model(b), b.pos)
    assert force.requires_grad, "the force must stay differentiable in the parameters"
    loss.backward()
    sd_ref = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    p2 = pos.clone().requires_grad_(True)
    ref_loss, ref_force = total_loss(_restated(sd_ref, z, p2, batch, ctor), p2)
    ref_loss.backward()
    assert rel_err(force.detach().cpu().numpy(), ref_force.detach().cpu().numpy()) < FTOL
    bad, checked = {}, 0
    for pname, prm in model.named_parameters():
        r = sd_ref[pname].grad
        assert r is not None and prm.grad is not None, pname
        checked += 1
        err = rel_err(prm.grad.cpu().numpy(), r.cpu().numpy())
        if err > GTOL:
            bad[pname] = err
    assert checked == len(list(model.parameters())) and not bad, (checked, bad)


def _molecules(n, seed):
    from dig_b200.data import synthetic_molecules
    return synthetic_molecules(n, "md17-aspirin", seed=seed, variable=True)


def test_run_trains_and_evaluates_on_forces():
    """run().train(..., energy_and_force=True) lowers the loss over 6 epochs; run().val(..., True, ...) gives a finite
    MAE."""
    from dig_b200.data import DataLoader
    from dig_b200.threedgraph.evaluation import ThreeDEvaluator
    from dig_b200.threedgraph.method import ComENet, run
    torch.manual_seed(0)
    model = ComENet(energy_and_force=True, cutoff=5.0, num_layers=2, hidden_channels=128, middle_channels=32).to(DEV)
    mols = _molecules(8, 7)
    loader = DataLoader(mols, 4, shuffle=False)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    r = run()
    losses = [r.train(model, opt, loader, True, 100, torch.nn.L1Loss(), DEV) for _ in range(6)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    mae = r.val(model, DataLoader(mols, 3, shuffle=False), True, 100, ThreeDEvaluator(), DEV)
    assert np.isfinite(float(mae)), mae


def test_pipeline_forces_equal_the_serial_loop():
    """InferencePipeline(forces=True) at depths 1 to 4: energies bit for bit and forces within FTOL of the serial
    forward + grad loop (the rest of the force backward sums rows with float atomics)."""
    from dig_b200.data import collate
    from dig_b200.pipeline import InferencePipeline
    from dig_b200.threedgraph.method import ComENet
    model = ComENet(energy_and_force=True, cutoff=5.0)
    model.load_state_dict(formula_state_dict(model.state_dict(), seed=6))
    model = model.to(DEV).eval()
    host = [collate(_molecules(n, 20 + n), pin_memory=True) for n in (5, 12, 1, 9, 3)]
    want = []
    for hb in host:
        d = hb.to(DEV)
        e = model(d)
        f = -torch.autograd.grad(e, d.pos, torch.ones_like(e), create_graph=True, retain_graph=True)[0]
        want.append((e.detach().cpu(), f.detach().cpu()))
    for depth in (1, 2, 3, 4):
        pipe = InferencePipeline(model, DEV, depth=depth, forces=True)
        got = [(e.clone(), f.clone()) for e, f in pipe.map(host)]
        assert len(got) == len(want)
        for (e, f), (e0, f0) in zip(got, want):
            assert torch.equal(e, e0), depth
            assert rel_err(f.numpy(), f0.numpy()) < FTOL, depth
