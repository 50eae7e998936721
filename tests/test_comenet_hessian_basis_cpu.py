"""The second-derivative basis sources of ComENet's Hessian path (gemnet flavour, num_spherical=2, num_radial=3)
against central differences of the first-derivative sources, in fp64 (CPU)."""
import math

from dig_b200 import basis

ENV = {"sin": math.sin, "cos": math.cos, "sqrt": math.sqrt, "pi": math.pi}
H = 1e-6


def _ev(s, **kw):
    return float(eval(s, dict(ENV, **kw)))


def test_gemnet_2_3_second_derivatives_match_finite_differences():
    first = basis.basis_sources("gemnet", 2, 3)
    second = basis.basis_sources_second_order("gemnet", 2, 3)
    assert len(second["bessel_dxx"]) == 6 and len(second["yl0_dtheta2"]) == 2
    assert len(second["ylm_dtheta2"]) == len(second["ylm_dtheta_dphi"]) == len(second["ylm_dphi2"]) == 4
    for x in (0.21, 0.37, 0.81):
        for d1, d2 in zip(first["bessel_dx"], second["bessel_dxx"]):
            fd = (_ev(d1, x=x + H) - _ev(d1, x=x - H)) / (2 * H)
            assert abs(_ev(d2, x=x) - fd) <= 2e-5 * max(1.0, abs(fd))
    for th in (0.5, 1.3, 2.2):
        for d1, d2 in zip(first["yl0_dtheta"], second["yl0_dtheta2"]):
            fd = (_ev(d1, theta=th + H) - _ev(d1, theta=th - H)) / (2 * H)
            assert abs(_ev(d2, theta=th) - fd) <= 1e-6 * max(1.0, abs(fd))
        for ph in (0.3, 2.0, 4.1):
            for dt, dp, dtt, dtp, dpp in zip(first["ylm_dtheta"], first["ylm_dphi"], second["ylm_dtheta2"],
                                             second["ylm_dtheta_dphi"], second["ylm_dphi2"]):
                fd_tt = (_ev(dt, theta=th + H, phi=ph) - _ev(dt, theta=th - H, phi=ph)) / (2 * H)
                fd_tp = (_ev(dt, theta=th, phi=ph + H) - _ev(dt, theta=th, phi=ph - H)) / (2 * H)
                fd_pt = (_ev(dp, theta=th + H, phi=ph) - _ev(dp, theta=th - H, phi=ph)) / (2 * H)
                fd_pp = (_ev(dp, theta=th, phi=ph + H) - _ev(dp, theta=th, phi=ph - H)) / (2 * H)
                assert abs(_ev(dtt, theta=th, phi=ph) - fd_tt) <= 1e-6 * max(1.0, abs(fd_tt))
                assert abs(_ev(dtp, theta=th, phi=ph) - fd_tp) <= 1e-6 * max(1.0, abs(fd_tp))
                assert abs(_ev(dtp, theta=th, phi=ph) - fd_pt) <= 1e-6 * max(1.0, abs(fd_pt))
                assert abs(_ev(dpp, theta=th, phi=ph) - fd_pp) <= 1e-6 * max(1.0, abs(fd_pp))
