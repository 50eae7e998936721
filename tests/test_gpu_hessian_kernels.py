"""The reverse mode of the tangent kernels in their value inputs (the Hessian path of DimeNet++ / SphereNet), element by
element against torch.autograd's fp64 double backward over the restated closed forms (oracle/restated.py), and the
geometry's reverse through the model's _GeometryJVP against fp64 double backward of the restated xyz_to_dat.

With G = d(loss)/d(tangent), each kernel output is d/d(input) of sum G * tangent(dist, dist_dot, angle, ...).  The
comparator evaluates tangent = d/d(eps) basis(dist + eps dist_dot, angle + eps angle_dot, ...) in fp64 and
differentiates sum G * tangent once more.  Every output is held to TOL of its largest component.  The fp32 closed forms
of the order-7 harmonics carry ~1e-5 of cancellation error (tests/test_gpu_generic_triplet_forces.py), and their second
derivatives more: with DimeNet++'s envelope folded into the Bessel values (env'' ~ 2 / x^3 times the values) d_dist
measured 1.03e-4 (QM9-shaped batch) and 1.25e-4 (ragged batch) of its largest component on an H100, the other outputs
and the SphereNet bases below 1e-4.  The basis kernels are not run on the 3 A random cluster of triplet_backward_ref:
its pairs a few hundredths of an Angstrom apart put the fp32 second derivatives (terms up to x^-4) out of range of any
useful bound; the geometry reverse is run on it."""
import math

import pytest
import torch

import triplet_backward_ref as ref

pytestmark = pytest.mark.gpu
NR = 6
TOL = 3e-4
CASES = [(0, False), (0, True), (1, False), (1, True)]          # (basis_id, torsion)


def _close(a, b, what, tol=TOL):
    a, b = a.double().cpu(), b.double().cpu()
    scale = float(b.abs().max()) if b.numel() else 0.0
    err = float((a - b).abs().max()) if b.numel() else 0.0
    assert err <= tol * max(scale, 1e-30), f"{what}: max |got - fp64| = {err / max(scale, 1e-30):.3e} of {scale:.3e}"


def _graph(name):
    from dig_b200 import ops
    from dig_b200.data import synthetic_batch
    dev = torch.device("cuda:0")
    num_graphs = None
    if name == "qm9":
        b = synthetic_batch(16, "qm9", seed=7, variable=True)
        pos, batch, cutoff = b.pos, b.batch, 5.0
    elif name == "capped":
        pos, batch, cutoff = ref.capped_batch()
    else:
        pos, batch, cutoff, num_graphs = ref.ragged_batch()
    pos, batch = pos.float().contiguous().to(dev), batch.long().to(dev)
    g = ops.build_graph(pos, batch, cutoff, num_graphs=num_graphs)
    ops.triplet_geometry(g, pos, use_torsion=True, want_idx=True)
    return g, pos, cutoff


def _restated_basis(basis_id, torsion):
    from oracle import restated
    ns = 7 if basis_id == 0 else 3
    tag = "dimenetpp_7_6" if (basis_id == 0 and not torsion) else f"spherenet_{ns}_{NR}"
    return restated.basis(tag, ns, NR), ns


@pytest.mark.parametrize("name", ["qm9", "ragged"])
@pytest.mark.parametrize("basis_id,torsion", CASES)
def test_triplet_basis_tangent_bwd_matches_fp64_double_backward(name, basis_id, torsion):
    from dig_b200 import autograd_jvp as jv
    from dig_b200 import ops
    g, pos, cutoff = _graph(name)
    bs, ns = _restated_basis(basis_id, torsion)
    gen = torch.Generator().manual_seed(3 + basis_id)
    E, T = g.n_edges, g.n_triplets
    dist, angle, tors = g.dist.view(-1), g.angle.view(-1), g.torsion.view(-1)
    d_dot, a_dot, t_dot = (torch.randn(n, generator=gen).cuda() for n in (E, T, T))
    g_sbf = torch.randn(T, ns * NR, generator=gen).cuda()
    g_tbf = torch.randn(T, ns * ns * NR, generator=gen).cuda() if torsion else None
    freq = (torch.arange(1, NR + 1, dtype=torch.float32) * math.pi).cuda()
    exp = 5
    _, bess = ops.edge_basis(dist, cutoff, exp, freq, basis_id, not torsion, NR, ns * NR)
    inputs = [x.clone().requires_grad_(True) for x in (dist, d_dot, angle, a_dot)]
    if torsion:
        inputs += [x.clone().requires_grad_(True) for x in (tors, t_dot)]
    else:
        inputs += [None, None]
    sbf_d, tbf_d = jv.triplet_basis_tangent(*inputs, bess, g, (cutoff, exp, basis_id, not torsion, ns, NR))
    loss = (sbf_d * g_sbf).sum() + ((tbf_d * g_tbf).sum() if torsion else 0)
    got = torch.autograd.grad(loss, [x for x in inputs if x is not None], retain_graph=True)

    x64 = [None if x is None else x.detach().double().requires_grad_(True) for x in inputs]
    eps = torch.zeros((), dtype=torch.float64, device=dist.device, requires_grad=True)
    kj = g.idx_kj.long()
    d = x64[0] + eps * x64[1]
    a = x64[2] + eps * x64[3]
    if torsion:
        s = (bs.angle_emb(d, a, kj, cutoff) * g_sbf.double()).sum()
        s = s + (bs.torsion_emb(d, a, x64[4] + eps * x64[5], kj, cutoff) * g_tbf.double()).sum()
    else:
        s = (bs.angle_emb(d, a, kj, cutoff, exp) * g_sbf.double()).sum()
    tangent = torch.autograd.grad(s, eps, create_graph=True)[0]
    want = torch.autograd.grad(tangent, [x for x in x64 if x is not None])
    for what, a_, b_ in zip(("dist", "dist_dot", "angle", "angle_dot", "torsion", "torsion_dot"), got, want):
        _close(a_, b_, what)
    # the same bits on a second run (no float atomics)
    again = torch.autograd.grad((jv.triplet_basis_tangent(*inputs, bess, g, (cutoff, exp, basis_id, not torsion,
                                                                             ns, NR))[0] * g_sbf).sum(), inputs[0])[0]
    first = torch.autograd.grad((sbf_d * g_sbf).sum(), inputs[0], retain_graph=True)[0]
    assert torch.equal(again, first)


@pytest.mark.parametrize("basis_id,torsion", CASES)
def test_edge_basis_tangent_bwd_matches_fp64_double_backward(basis_id, torsion):
    from dig_b200 import autograd_jvp as jv
    from oracle import restated
    g, pos, cutoff = _graph("qm9")
    gen = torch.Generator().manual_seed(11)
    dist = g.dist.view(-1).clone().requires_grad_(True)
    d_dot = torch.randn(dist.numel(), generator=gen).cuda().requires_grad_(True)
    freq = (torch.arange(1, NR + 1, dtype=torch.float32) * math.pi * 1.1).cuda().requires_grad_(True)
    G = torch.randn(dist.numel(), NR, generator=gen).cuda()
    ns = 7 if basis_id == 0 else 3
    r_dot = jv.edge_basis_tangent(freq, dist, d_dot, cutoff, 5, basis_id, not torsion, NR, ns * NR)
    got = torch.autograd.grad((r_dot * G).sum(), [dist, d_dot, freq])
    x = [t.detach().double().requires_grad_(True) for t in (dist, d_dot, freq)]
    eps = torch.zeros((), dtype=torch.float64, device=dist.device, requires_grad=True)
    s = (restated.dist_emb(x[0] + eps * x[1], x[2], cutoff, 5) * G.double()).sum()
    tangent = torch.autograd.grad(s, eps, create_graph=True)[0]
    want = torch.autograd.grad(tangent, x)
    for what, a_, b_ in zip(("dist", "dist_dot", "freq"), got, want):
        _close(a_, b_, what)


@pytest.mark.parametrize("name", ["qm9", "capped", "ragged"])
@pytest.mark.parametrize("torsion", [False, True])
def test_geometry_jvp_reverse_matches_fp64_double_backward(name, torsion):
    """d/dpos of sum G . J(pos) c for the model graph's dist / angle / torsion (torsion through g.tors_arg) against the
    restated xyz_to_dat in fp64 at the same torsion candidates (tests/xyz_to_dat_grad_ref.py)."""
    import xyz_to_dat_grad_ref as xref
    from dig_b200 import autograd_jvp as jv
    from dig_b200 import ops
    g, pos, cutoff = _graph(name)
    if torsion:
        ops.triplet_geometry_any_degree_arg(g, pos, 0)
    gen = torch.Generator().manual_seed(5)
    c = torch.randn(pos.shape, generator=gen).cuda()
    E, T = g.n_edges, g.n_triplets
    Gd, Ga, Gt = (torch.randn(n, generator=gen).cuda() for n in (E, T, T))
    p = pos.clone().requires_grad_(True)
    d_dot, a_dot, t_dot = jv.geometry_jvp(p, c, g, torsion)
    loss = (d_dot * Gd).sum() + (a_dot * Ga).sum() + ((t_dot * Gt).sum() if torsion else 0)
    got = torch.autograd.grad(loss, p)[0]

    p64 = pos.detach().double().requires_grad_(True)
    eps = torch.zeros((), dtype=torch.float64, device=pos.device, requires_grad=True)
    ei, n = g.edge_index.long(), pos.size(0)
    geo = xref.geometry_at(p64 + eps * c.double(), ei, n, xref.candidate_atoms(ei, n, g.tors_arg) if torsion else None)
    assert float((geo[1].detach() - g.angle.double()).abs().max()) < 1e-5          # the same triplets, in order
    s = (geo[0] * Gd.double()).sum() + (geo[1] * Ga.double()).sum()
    if torsion:
        s = s + (geo[2] * Gt.double()).sum()
    tangent = torch.autograd.grad(s, eps, create_graph=True)[0]
    want = torch.autograd.grad(tangent, p64)[0]
    _close(got, want, "pos")
