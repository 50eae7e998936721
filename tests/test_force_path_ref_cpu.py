"""CPU checks of the fp64 references and bounds of the first-order force path (tests/triplet_backward_ref.py) that
tests/test_gpu_force_path_fp64.py holds the kernels to: the closed-form tolerance BESSEL_DX_TOL and its X_MIN measured
node by node in fp32, the magnitude transform of a closed form, the moved triplet-basis reverse-mode reference against
autograd of an explicit per-triplet forward, and the envelope magnitudes against dig_b200.basis."""
import math

import pytest
import torch

import triplet_backward_ref as ref


@pytest.mark.parametrize("basis_id", [0, 1])
def test_bessel_closed_forms_in_fp32_stay_within_a_quarter_of_the_tolerance(basis_id):
    """Every "bessel" / "bessel_dx" string evaluated node by node in fp32 (one rounding per node, as the generated code)
    against fp64, over a dense x grid from X_MIN to 1: worst |fp32 - fp64| / magnitude <= BESSEL_DX_TOL / 4.  Below
    1e-6 the fp32 powers leave their range; basis (7, 6) holds from x = 2.3e-6, so its X_MIN is 1e-5, and (3, 6) holds
    over the whole grid, so its X_MIN is 1e-6."""
    from dig_b200.basis import basis_sources
    ns = 7 if basis_id == 0 else 3
    src = basis_sources("dimenet", ns, 6)
    x32 = torch.logspace(-6, 0, 24001, dtype=torch.float64)[:-1].float()
    x64 = x32.double()
    worst = torch.zeros_like(x64)
    for key in ("bessel", "bessel_dx"):
        for s in src[key]:
            got = ref.eval_source(s, x32).double()
            r = (got - ref.eval_source(s, x64)).abs() / ref.source_magnitude(s, x64)
            worst = torch.maximum(worst, torch.where(torch.isfinite(r), r, torch.full_like(r, math.inf)))
    x_min = ref.X_MIN[basis_id]
    held = float(worst[x64 >= x_min].max())
    print(f"basis {basis_id}: worst |fp32 - fp64| / magnitude over [{x_min:g}, 1) = {held / ref.U:.2f} u")
    assert held <= ref.BESSEL_DX_TOL / 4
    bad = (worst > ref.BESSEL_DX_TOL / 4).nonzero()
    if bad.numel():                                  # the measurement holds from the grid point above the last failure
        print(f"basis {basis_id}: holds from x = {float(x64[int(bad.max()) + 1]):.3g}")


def test_magnitude_transform_by_hand():
    x = torch.tensor([0.3, 0.7], dtype=torch.float64)
    cases = [
        ("-2*sin(3.0*x)/x**2 + 0.5", lambda x: 2 * (3 * x).sin().abs() / x ** 2 + 0.5,
         lambda x: 2 * (3 * x) * (3 * x).cos().abs() / x ** 2 + 0.5),
        ("1.5*cos(x)/x - sin(x)/x**2", lambda x: 1.5 * x.cos().abs() / x + x.sin().abs() / x ** 2,
         lambda x: 1.5 * x * x.sin().abs() / x + x * x.cos().abs() / x ** 2),
        ("-0.25*x**3", lambda x: 0.25 * x ** 3, lambda x: 0.25 * x ** 3),
    ]
    for s, mag, arg in cases:
        assert torch.allclose(ref.eval_source(ref.magnitude_source(s), x), mag(x), rtol=1e-15, atol=0), s
        assert torch.allclose(ref.eval_source(ref.magnitude_source(s, arg=True), x), arg(x), rtol=1e-15, atol=0), s
        assert bool((ref.source_magnitude(s, x) >= ref.eval_source(s, x).abs()).all()), s


class _G:
    pass


def _host_graph(seed):
    """A small random triplet list: edges, idx_kj, angles, torsions."""
    gen = torch.Generator().manual_seed(seed)
    g = _G()
    g.n_edges, t = 9, 23
    g.idx_kj = torch.randint(0, 7, (t,), generator=gen)                # edges 7, 8: no triplet reads them
    angle = torch.rand(t, generator=gen, dtype=torch.float64) * math.pi
    torsion = (torch.rand(t, generator=gen, dtype=torch.float64) * 2 - 1) * math.pi
    return g, angle, torsion, gen


@pytest.mark.parametrize("ns", [3, 7])
def test_basis_bwd_reference_against_autograd_of_the_forward(ns):
    """basis_bwd_reference (moved from the generic-width test) against torch.autograd of an explicit per-triplet fp64
    forward sbf[t] = bess(dist_kj / cutoff)[l, r] yl0_l(angle), tbf[t] = bess[b, r] ylm_{ab}(angle, torsion)."""
    from dig_b200.basis import basis_sources
    nr, cutoff = 6, 5.0
    g, angle, torsion, gen = _host_graph(ns)
    src = basis_sources("dimenet", ns, nr)
    dist = (torch.rand(g.n_edges, generator=gen, dtype=torch.float64) * 4 + 0.8)
    d_sbf = torch.randn(angle.numel(), ns * nr, generator=gen, dtype=torch.float64)
    d_tbf = torch.randn(angle.numel(), ns * ns * nr, generator=gen, dtype=torch.float64)

    def bessel(d):
        x = d / cutoff
        return torch.stack([ref.eval_source(s, x) for s in src["bessel"]], 1)

    d_ = dist.clone().requires_grad_(True)
    a_ = angle.clone().requires_grad_(True)
    p_ = torsion.clone().requires_grad_(True)
    Y = ref.harmonics(ns, a_, p_, nr)
    B = bessel(d_)[g.idx_kj].view(-1, ns, nr)
    sbf = (B * Y["yl0"][:, :, None]).reshape(-1, ns * nr)
    tbf = (B[:, None, :, :] * Y["ylm"].view(-1, ns, ns)[:, :, :, None]).reshape(-1, ns * ns * nr)
    gd, ga, gp = torch.autograd.grad([sbf, tbf], [d_, a_, p_], [d_sbf, d_tbf])
    x = dist.clone().requires_grad_(True)
    bess_dx = torch.autograd.functional.jacobian(lambda x: bessel(x * cutoff).sum(0), x / cutoff).permute(1, 0)
    r = ref.basis_bwd_reference(g, cutoff, ns, bessel(dist), bess_dx.contiguous(), angle, torsion, d_sbf, d_tbf)
    for got, want, name in zip(r["v"], (gd, ga, gp), ("ddist", "dangle", "dtorsion")):
        assert torch.allclose(got, want, rtol=1e-10, atol=1e-12 * float(want.abs().max())), name
    for i in range(3):
        assert bool((r["m"][i] >= r["v"][i].abs() * (1 - 1e-12)).all())
    assert bool((r["v"][0][7:] == 0).all())


@pytest.mark.parametrize("exponent", [5, 2, 4])
def test_envelope_magnitudes_against_the_basis_coefficients(exponent):
    """env' of envelope_terms is the derivative of dig_b200.basis's envelope; env_abs / envd_abs take each term by its
    absolute value, so they bound |env| / |env'| everywhere and do not vanish where env(1) = env'(1) = 0 cancel."""
    from dig_b200.basis import envelope_coefficients
    p, a, b, c = envelope_coefficients(exponent)
    x = torch.linspace(0.05, 1.0, 200, dtype=torch.float64).requires_grad_(True)
    env_b = 1.0 / x + a * x ** (p - 1) + b * x ** p + c * x ** (p + 1)
    (denv,) = torch.autograd.grad(env_b.sum(), x)
    env, envd, env_abs, envd_abs = ref.envelope_terms(x.detach(), exponent)
    assert torch.allclose(env, env_b.detach(), rtol=1e-13) and torch.allclose(envd, denv, rtol=1e-12, atol=1e-12)
    xd = x.detach()
    want_abs = 1 / xd + abs(a) * xd ** (p - 1) + abs(b) * xd ** p + abs(c) * xd ** (p + 1)
    want_dabs = 1 / xd ** 2 + abs(a) * (p - 1) * xd ** (p - 2) + abs(b) * p * xd ** (p - 1) + abs(c) * (p + 1) * xd ** p
    assert torch.allclose(env_abs, want_abs, rtol=1e-15) and torch.allclose(envd_abs, want_dabs, rtol=1e-15)
    assert bool((env_abs >= env.abs()).all() and (envd_abs >= envd.abs()).all())
    one = torch.tensor([1.0], dtype=torch.float64)
    e1, d1, ea1, da1 = ref.envelope_terms(one, exponent)
    assert abs(float(e1)) < 1e-12 * float(ea1) and abs(float(d1)) < 1e-12 * float(da1)
