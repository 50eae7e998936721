"""Forces and training on forces at triplet-branch widths the fused kernels are not compiled for (SphereNet / DimeNet++
with int_emb_size != 64 or basis_emb_size_* != 8: materialised bases, ordinary linears).

* dig3d_triplet_basis_bwd element by element against an fp64 evaluation of the same closed forms, with a per-element
  bound: |kernel - fp64| <= gamma(c) M + HARMONIC_TOL Mh + c ETA, where M = sum |terms| of the output, Mh the same sum
  without the harmonic factor, and c the longest chain of fp32 roundings:
      per triplet   NR fmas per (l) / (ab) row, then one fma per harmonic (NS, and NY with torsion):  NR + NS + NY + 1
      ddist[kj]     the triplet sums of its n(kj) triplets added in one lane per 32 (n(kj) adds at most), a 5-level
                    butterfly, the product with fl(1 / cutoff) (2 roundings)
  HARMONIC_TOL: the fp32 closed forms (one correctly rounded op per node, CUDA sinf / cosf within 2 ulp) lie within
  7e-6 of their fp64 values for num_spherical = 7 and 5e-7 for 3 over theta in [0, pi], phi in [-pi, pi] (values and
  both derivatives, measured with the same strings on the CPU); 2e-5 leaves room for the device's sin / cos.
* the adjoint identity with dig3d_triplet_basis_tangent, determinism, T = 0, edges that are no triplet's k->j edge.
* model forces against the reference fixture (DimeNet++) and torch.autograd over the restatement on the same GPU
  (SphereNet: the torsion's self-candidate tie-breaks differ between devices), and parameter gradients of force training.
"""
import json
import math
import os
import re

import numpy as np
import pytest
import torch

import triplet_backward_ref as ref
from helpers import GOLDEN, formula_state_dict, rel_err

pytestmark = pytest.mark.gpu
FTOL = 1e-5
HARMONIC_TOL = 2e-5
NR = 6
BASES = [(0, False), (0, True), (1, False), (1, True)]          # (basis_id, torsion)
_CACHE = {}


def _collinear_batch():
    """(pos, batch, cutoff): a straight chain of four atoms (angles exactly 0 and pi) next to a bent triple."""
    pos = torch.tensor([[0, 0, 0], [1.2, 0, 0], [2.4, 0, 0], [3.6, 0, 0],
                        [0, 0, 0], [1.1, 0, 0], [0.3, 1.0, 0.2]], dtype=torch.float32)
    return pos, torch.tensor([0, 0, 0, 0, 1, 1, 1]), 5.0


def _no_triplet_batch():
    """(pos, batch, cutoff): three diatomics: edges, no triplets (T = 0)."""
    pos = torch.tensor([[0, 0, 0], [1.0, 0, 0], [0, 0, 0], [0, 1.5, 0], [0, 0, 0], [0, 0, 0.9]], dtype=torch.float32)
    return pos, torch.tensor([0, 0, 1, 1, 2, 2]), 5.0


def _graph(name):
    from dig_b200 import ops
    from dig_b200.data import synthetic_batch
    if name in _CACHE:
        return _CACHE[name]
    dev = torch.device("cuda:0")
    num_graphs = None
    if name == "qm9":
        b = synthetic_batch(32, "qm9", seed=5, variable=True)
        pos, batch, cutoff = b.pos, b.batch, 5.0
    elif name == "capped":
        pos, batch, cutoff = ref.capped_batch()
    elif name == "ragged":
        pos, batch, cutoff, num_graphs = ref.ragged_batch()
    elif name == "collinear":
        pos, batch, cutoff = _collinear_batch()
    else:
        pos, batch, cutoff = _no_triplet_batch()
    pos, batch = pos.float().contiguous().to(dev), batch.long().to(dev)
    g = ops.build_graph(pos, batch, cutoff, num_graphs=num_graphs)
    ops.triplet_geometry(g, pos, use_torsion=True, want_idx=True)
    _CACHE[name] = (g, cutoff)
    return g, cutoff


def _inputs(name, basis_id, tors, seed):
    """bess / bess_dx of the graph's edges and random upstream gradients of sbf / tbf."""
    from dig_b200 import ops
    g, cutoff = _graph(name)
    ns = 7 if basis_id == 0 else 3
    freq = (torch.arange(1, NR + 1, dtype=torch.float32) * math.pi).cuda()
    _, bess = ops.edge_basis(g.dist, cutoff, 5, freq, basis_id, not tors, NR, ns * NR)
    _, bess_dx = ops.edge_basis_bwd(g.dist, cutoff, 5, None, basis_id, not tors, None, ns * NR, want_ddist=False,
                                    want_bess_dx=True)
    # atoms of the dense box closer than the closed forms can be evaluated in fp32 at: keep the inputs finite
    bess = torch.nan_to_num(bess, nan=0.0, posinf=0.0, neginf=0.0).clamp_(-100.0, 100.0)
    bess_dx = torch.nan_to_num(bess_dx, nan=0.0, posinf=0.0, neginf=0.0).clamp_(-1e3, 1e3)
    gen = torch.Generator().manual_seed(seed)
    t = g.n_triplets
    d_sbf = torch.randn(t, ns * NR, generator=gen).cuda()
    d_tbf = torch.randn(t, ns * ns * NR, generator=gen).cuda() if tors else None
    return g, cutoff, ns, bess, bess_dx, d_sbf, d_tbf


def _harmonics(ns, angle, torsion):
    """fp64 closed forms of the generated headers: yl0, yl0', ylm, dylm/dtheta, dylm/dphi, each [T, K]."""
    from dig_b200.basis import basis_sources
    src = basis_sources("dimenet", ns, NR)
    th = angle.double()
    ph = torsion.double() if torsion is not None else torch.zeros_like(th)
    env = {"sin": torch.sin, "cos": torch.cos, "sqrt": torch.sqrt, "pi": math.pi, "theta": th, "phi": ph}

    def table(key):
        cols = [eval(s, env) for s in src[key]]
        return torch.stack([c if torch.is_tensor(c) else torch.full_like(th, float(c)) for c in cols], 1)
    return {k: table(k) for k in ("yl0", "yl0_dtheta", "ylm", "ylm_dtheta", "ylm_dphi")}


def _reference(g, cutoff, ns, bess, bess_dx, angle, torsion, d_sbf, d_tbf):
    """fp64 (ddist, dangle, dtorsion), their magnitudes M (every factor by its absolute value) and Mh (the harmonic
    factor dropped)."""
    Y = _harmonics(ns, angle, torsion)
    kj = g.idx_kj.long()
    B = bess.double()[kj].view(-1, ns, NR)
    Bd = bess_dx.double()[kj].view(-1, ns, NR)
    ds = d_sbf.double().view(-1, ns, NR)
    out = {}
    for mode in ("v", "m", "h"):
        f = (lambda x: x) if mode == "v" else torch.abs
        y = {k: (torch.ones_like(v) if mode == "h" else f(v)) for k, v in Y.items()}
        s_b, s_bd = (f(ds) * f(B)).sum(2), (f(ds) * f(Bd)).sum(2)           # [T, ns]
        dang = (y["yl0_dtheta"] * s_b).sum(1)
        dx = (y["yl0"] * s_bd).sum(1)
        dtor = None
        if d_tbf is not None:
            dt = d_tbf.double().view(-1, ns, ns, NR)                          # [T, a, b, r]
            h = (f(dt) * f(B)[:, None]).sum(3).reshape(-1, ns * ns)          # [T, ab]
            hd = (f(dt) * f(Bd)[:, None]).sum(3).reshape(-1, ns * ns)
            dang = dang + (y["ylm_dtheta"] * h).sum(1)
            dtor = (y["ylm_dphi"] * h).sum(1)
            dx = dx + (y["ylm"] * hd).sum(1)
        inv = 1.0 / cutoff
        ddist = torch.zeros(g.n_edges, dtype=torch.float64, device=bess.device).index_add_(0, kj, dx) * inv
        out[mode] = (ddist, dang, dtor)
    return out


def _run(g, cutoff, basis_id, bess, bess_dx, d_sbf, d_tbf, tors):
    from dig_b200 import ops
    return ops.triplet_basis_bwd(g, bess, bess_dx, g.angle, g.torsion if tors else None, basis_id, d_sbf, d_tbf,
                                 cutoff, tors)


@pytest.mark.parametrize("graph", ["qm9", "capped", "ragged", "collinear", "none"])
@pytest.mark.parametrize("basis_id,tors", BASES)
def test_triplet_basis_bwd_matches_fp64(graph, basis_id, tors):
    g, cutoff, ns, bess, bess_dx, d_sbf, d_tbf = _inputs(graph, basis_id, tors, seed=3)
    got = _run(g, cutoff, basis_id, bess, bess_dx, d_sbf, d_tbf, tors)
    again = _run(g, cutoff, basis_id, bess, bess_dx, d_sbf, d_tbf, tors)
    torch.cuda.synchronize()
    for a, b in zip(got, again):
        assert (a is None and b is None) or torch.equal(a, b), "two runs on the same input differ"
    if graph == "none":
        assert g.n_triplets == 0 and g.n_edges > 0
    if graph == "collinear":
        a = g.angle.double()
        assert bool((a == 0).any()) and bool((a - math.pi).abs().lt(1e-6).any())
    r = _reference(g, cutoff, ns, bess, bess_dx, g.angle, g.torsion if tors else None, d_sbf, d_tbf)
    counts = torch.bincount(g.idx_kj.long(), minlength=g.n_edges)
    ny = ns * ns if tors else 0
    c_t = NR + ns + ny + 1
    c_e = c_t + counts.double() + 5 + 2
    names = ("ddist", "dangle", "dtorsion")
    for i, name in enumerate(names):
        if got[i] is None:
            assert not tors and name == "dtorsion"
            continue
        c = c_e if name == "ddist" else float(c_t)
        lim = ref.gamma(c) * r["m"][i] + HARMONIC_TOL * r["h"][i] + c * ref.ETA
        ref.check(got[i], r["v"][i], lim, f"{graph} basis {basis_id} torsion {tors}: {name}")
    # an edge that is no triplet's k->j edge gets exactly zero
    assert bool((got[0][counts == 0] == 0).all())


@pytest.mark.parametrize("basis_id,tors", BASES)
def test_triplet_basis_bwd_is_the_adjoint_of_the_tangent(basis_id, tors):
    """<d_sbf, sbf_dot> + <d_tbf, tbf_dot> == <ddist, dist_dot> + <dangle, angle_dot> + <dtorsion, torsion_dot>, with the
    tangents from dig3d_edge_basis_tangent / dig3d_triplet_basis_tangent along random geometry tangents."""
    from dig_b200 import ops
    g, cutoff, ns, bess, bess_dx, d_sbf, d_tbf = _inputs("qm9", basis_id, tors, seed=4)
    gen = torch.Generator().manual_seed(9)
    d_dot = torch.randn(g.n_edges, generator=gen).cuda()
    a_dot = torch.randn(g.n_triplets, generator=gen).cuda()
    t_dot = torch.randn(g.n_triplets, generator=gen).cuda() if tors else None
    _, bess_d = ops.edge_basis_tangent(g.dist, d_dot, cutoff, 5, None, basis_id, not tors, NR, ns * NR,
                                       want_rbf0=False, want_bess=True)
    sbf_d, tbf_d = ops.triplet_basis_tangent(bess, bess_d, g.angle, a_dot, g.torsion if tors else None, t_dot, g.idx_kj,
                                             basis_id, ns, NR, want_tbf=tors)
    ddist, dangle, dtors = _run(g, cutoff, basis_id, bess, bess_dx, d_sbf, d_tbf, tors)
    dot = lambda a, b: float((a.double() * b.double()).sum())
    lhs = dot(d_sbf, sbf_d) + (dot(d_tbf, tbf_d) if tors else 0.0)
    rhs = dot(ddist, d_dot) + dot(dangle, a_dot) + (dot(dtors, t_dot) if tors else 0.0)
    r = _reference(g, cutoff, ns, bess, bess_dx, g.angle, g.torsion if tors else None, d_sbf, d_tbf)["m"]
    mag = dot(r[0], d_dot.abs()) + dot(r[1], a_dot.abs()) + (dot(r[2], t_dot.abs()) if tors else 0.0)
    assert abs(lhs - rhs) <= 1e-5 * mag, (lhs, rhs, mag)


# ---------------------------------------------------------------------------------------------------- the models
def _case(name):
    from dig_b200.threedgraph import method
    from oracle.gen_golden_generic_forces import CASES
    model_name, ctor, wseed = CASES[name]
    g = np.load(os.path.join(GOLDEN, "generic_forces.npz"))
    gold = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}
    with open(os.path.join(GOLDEN, "generic_forces_shapes.json")) as fh:
        shapes = json.load(fh)[name]
    sd = formula_state_dict({k: torch.empty(s) for k, s in shapes.items()}, seed=wseed)
    dev = torch.device("cuda:0")
    model = getattr(method, model_name)(energy_and_force=True, **ctor)
    assert model._triplet_generic
    model.load_state_dict(sd)
    model = model.to(dev)
    z, pos, batch = (torch.from_numpy(gold[k]).to(dev) for k in ("z", "pos", "batch"))
    return model, {k: v.to(dev) for k, v in sd.items()}, gold, z, pos, batch, model_name, ctor


class _B:
    pass


def _batch(z, pos, batch):
    b = _B()
    b.z, b.pos, b.batch = z, pos, batch
    b.num_graphs = int(batch.max().item()) + 1
    return b


def _restated(sd, z, pos, batch, model_name, ctor):
    from oracle import restated
    from oracle.gen_golden_generic_forces import restated_kwargs
    return restated.dimenet_family_forward(sd, z, pos, batch, **restated_kwargs(model_name, ctor))


def test_dimenetpp_generic_forces_match_reference_fixture():
    model, sd, gold, z, pos, batch, model_name, ctor = _case("dimenetpp_wide")
    b = _batch(z, pos.clone(), batch)
    out = model(b)
    force = -torch.autograd.grad(out, b.pos, grad_outputs=torch.ones_like(out))[0]
    assert rel_err(out.detach().cpu().numpy(), gold["energy_f32"]) < 1e-5
    assert rel_err(force.cpu().numpy(), gold["force_f64"]) < FTOL
    assert rel_err(force.cpu().numpy(), gold["force_f32"]) < FTOL


@pytest.mark.parametrize("name", ["spherenet_narrow", "spherenet_ns3"])
def test_spherenet_generic_forces_match_restated_autograd(name):
    model, sd, gold, z, pos, batch, model_name, ctor = _case(name)
    b = _batch(z, pos.clone(), batch)
    out = model(b)
    force = -torch.autograd.grad(out, b.pos, grad_outputs=torch.ones_like(out))[0]
    pos2 = pos.clone().requires_grad_(True)
    r = _restated(sd, z, pos2, batch, model_name, ctor)
    f_ref = -torch.autograd.grad(r.sum(), pos2)[0]
    assert rel_err(out.detach().cpu().numpy(), gold["energy_f32"]) < 1e-5
    assert rel_err(out.detach().cpu().numpy(), r.detach().cpu().numpy()) < 1e-5
    assert rel_err(force.cpu().numpy(), f_ref.cpu().numpy()) < FTOL


@pytest.mark.parametrize("name", ["dimenetpp_wide", "spherenet_narrow", "spherenet_ns3"])
def test_generic_force_training_gradients_match_oracle(name):
    """d/d(parameters) of L1(E, y) + 100 * L1(F, f), F = -dE/dpos under create_graph=True, against torch.autograd's
    double backward over the restatement on the same GPU; every parameter within 2e-4 of its largest entry."""
    model, sd, gold, z, pos, batch, model_name, ctor = _case(name)
    n_mol = int(batch.max()) + 1
    gen = torch.Generator().manual_seed(21)
    y = torch.randn(n_mol, 1, generator=gen).cuda()
    f_t = torch.randn(pos.size(0), 3, generator=gen).cuda()

    def total_loss(energy, position):
        force = -torch.autograd.grad(energy, position, grad_outputs=torch.ones_like(energy), create_graph=True,
                                     retain_graph=True)[0]
        return torch.nn.functional.l1_loss(energy, y) + 100.0 * torch.nn.functional.l1_loss(force, f_t), force

    b = _batch(z, pos.clone(), batch)
    loss, force = total_loss(model(b), b.pos)
    assert force.requires_grad, "the force must stay differentiable in the parameters"
    loss.backward()
    sd_ref = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    pos2 = pos.clone().requires_grad_(True)
    ref_loss, ref_force = total_loss(_restated(sd_ref, z, pos2, batch, model_name, ctor), pos2)
    ref_loss.backward()
    assert rel_err(force.detach().cpu().numpy(), ref_force.detach().cpu().numpy()) < FTOL
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
    assert checked > 30 and not bad, (checked, bad)


def _energy_path_as_before(model, z, pos, g):
    """The generic triplet branch of the energy-only training forward, op for op as it ran before forces existed at
    these widths: ops.triplet_basis on the constant geometry, then the same linears, row gather and segment sum."""
    from dig_b200 import autograd as ag
    from dig_b200 import ops
    m = model
    ns, nr, tors = m.num_spherical, m.num_radial, m._torsion
    ops.triplet_geometry(g, pos, use_torsion=tors, want_idx=False)
    rbf0, bess = ag.edge_basis(m.emb.dist_emb.freq, g.dist, m.cutoff, m.envelope_exponent, m._basis_id, not tors, nr,
                               ns * nr)
    ops.triplet_geometry(g, pos, use_torsion=tors, want_idx=True)
    sbf, tbf = ops.triplet_basis(bess, g.angle, g.torsion, g.idx_kj, m._basis_id, ns, nr, tors)
    lin = ag.lin
    ie = m.init_e
    x = ag.gather_rows(ie.emb.weight, z)
    r0 = ag.lin_swish(ie.lin_rbf_0, rbf0)
    e1 = ag.lin_swish(ie.lin, torch.cat([ag.gather_rows(x, g.dst, g.row_ptr), ag.gather_rows(x, g.src), r0], dim=-1))
    e2_list = [ag.mul(lin(ie.lin_rbf_1, rbf0), e1)]
    for ue in m.update_es:
        x_ji = ag.lin_swish(ue.lin_ji, e1)
        x_kj = ag.mul(ag.lin_swish(ue.lin_kj, e1), lin(ue.lin_rbf2, lin(ue.lin_rbf1, rbf0)))
        x_kj = ag.lin_swish(ue.lin_down, x_kj)
        prod = ag.mul(ag.gather_rows(x_kj, g.idx_kj), lin(ue.lin_sbf2, lin(ue.lin_sbf1, sbf)))
        if tors:
            prod = ag.mul(prod, lin(ue.lin_t2, lin(ue.lin_t1, tbf)))
        x_kj = ag.lin_swish(ue.lin_up, ag.segment_sum(prod, g.trip_ptr, g.idx_ji))
        h = ag.add(x_ji, x_kj)
        for layer in ue.layers_before_skip:
            h = ag.add(h, ag.lin_swish(layer.lin2, ag.lin_swish(layer.lin1, h)))
        h = ag.add(ag.lin_swish(ue.lin, h), e1)
        for layer in ue.layers_after_skip:
            h = ag.add(h, ag.lin_swish(layer.lin2, ag.lin_swish(layer.lin1, h)))
        e1 = h
        e2_list.append(ag.mul(lin(ue.lin_rbf, rbf0), e1))
    v = m._update_v_train([m.init_v] + list(m.update_vs), e2_list, g)
    u = ag.segment_sum(v[0], g.graph_ptr, g.batch)
    for l in range(1, v.size(0)):
        u = ag.add(u, ag.segment_sum(v[l], g.graph_ptr, g.batch))
    return u


@pytest.mark.parametrize("name", ["dimenetpp_wide", "spherenet_narrow", "spherenet_ns3"])
def test_energy_only_path_is_unchanged(name):
    """pos without requires_grad: the energies equal, bit for bit, those of the op sequence the generic branch ran before
    it carried forces, and so do the parameter gradients up to the order of the weight-gradient kernels' atomic
    row-split sums (dig3d_wgrad), which varies from run to run on either path."""
    from dig_b200 import ops
    model, sd, gold, z, pos, batch, model_name, ctor = _case(name)
    model.energy_and_force = False
    model.train()
    target = torch.linspace(-1, 1, int(batch.max()) + 1, device=pos.device).view(-1, 1)
    out = model(_batch(z, pos.clone(), batch))
    torch.nn.functional.l1_loss(out, target).backward()
    got = {k: p.grad.clone() for k, p in model.named_parameters()}
    model.zero_grad()
    g = ops.build_graph(pos, batch, model.cutoff, num_graphs=int(batch.max()) + 1, z=z,
                        z_rows=model.init_e.emb.num_embeddings)
    want = _energy_path_as_before(model, z, pos, g)
    torch.nn.functional.l1_loss(want, target).backward()
    assert torch.equal(out.detach(), want.detach())
    for k, p in model.named_parameters():
        assert rel_err(got[k].cpu().numpy(), p.grad.cpu().numpy()) < 1e-5, k


def test_run_trains_generic_spherenet_on_forces(tmp_path, capsys):
    """run().run(..., energy_and_force=True) for one epoch at a generic SphereNet width: finite energy / force MAEs
    printed and the checkpoint written."""
    from dig_b200.data import synthetic_molecules
    from dig_b200.threedgraph.evaluation import ThreeDEvaluator
    from dig_b200.threedgraph.method import SphereNet, run
    dev = torch.device("cuda:0")
    mols = synthetic_molecules(10, "md17-aspirin", seed=4)
    torch.manual_seed(0)
    model = SphereNet(energy_and_force=True, int_emb_size=32, basis_emb_size_angle=4, basis_emb_size_torsion=6,
                      num_layers=2, hidden_channels=64, out_emb_channels=64, cutoff=5.0)
    run().run(dev, mols[:6], mols[6:8], mols[8:], model, loss_func=torch.nn.L1Loss(), evaluation=ThreeDEvaluator(),
              epochs=1, batch_size=3, vt_batch_size=2, lr=5e-4, lr_decay_factor=0.5, lr_decay_step_size=1,
              energy_and_force=True, p=100, save_dir=str(tmp_path / "ckpt"), log_dir='')
    out = capsys.readouterr().out
    lines = [l for l in out.splitlines() if "'Energy MAE'" in l]
    assert lines, out
    for l in lines:
        for key in ("Energy MAE", "Force MAE"):
            m = re.search(rf"'{key}': (?:tensor\()?([-+\w.]+)", l)
            assert m and np.isfinite(float(m.group(1))), l
    assert os.path.isfile(tmp_path / "ckpt" / "valid_checkpoint.pt")
