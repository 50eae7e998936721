"""The second-derivative basis sources of the Hessian path and their generated headers (CPU)."""
import math
import os

from dig_b200 import basis, codegen


def test_second_order_headers_are_up_to_date():
    csrc = os.path.join(os.path.dirname(basis.__file__), "csrc", "generated")
    for tag in codegen.SECOND_ORDER:
        flavor, ns, nr = codegen.CONFIGS[tag]
        want = codegen.emit_header_second_order(tag, flavor, ns, nr, basis.basis_sources_second_order(flavor, ns, nr))
        with open(os.path.join(csrc, f"basis_{tag}_d2.cuh")) as fh:
            assert fh.read() == want, f"stale generated header for {tag}: run python -m dig_b200.codegen --force"


def test_torsion_harmonic_second_derivatives_match_finite_differences():
    """ylm_dtheta2 / ylm_dtheta_dphi / ylm_dphi2 against central differences of the first-derivative sources (fp64)."""
    first = basis.basis_sources("dimenet", 3, 6)
    second = basis.basis_sources_second_order("dimenet", 3, 6)
    env = {"sin": math.sin, "cos": math.cos, "sqrt": math.sqrt, "pi": math.pi}

    def ev(s, **kw):
        return float(eval(s, dict(env, **kw)))

    h = 1e-6
    for th in (0.5, 2.2):
        for ph in (0.3, 4.1):
            for dt, dp, dtt, dtp, dpp in zip(first["ylm_dtheta"], first["ylm_dphi"], second["ylm_dtheta2"],
                                             second["ylm_dtheta_dphi"], second["ylm_dphi2"]):
                fd_tt = (ev(dt, theta=th + h, phi=ph) - ev(dt, theta=th - h, phi=ph)) / (2 * h)
                fd_tp = (ev(dt, theta=th, phi=ph + h) - ev(dt, theta=th, phi=ph - h)) / (2 * h)
                fd_pp = (ev(dp, theta=th, phi=ph + h) - ev(dp, theta=th, phi=ph - h)) / (2 * h)
                assert abs(ev(dtt, theta=th, phi=ph) - fd_tt) <= 1e-6 * max(1.0, abs(fd_tt))
                assert abs(ev(dtp, theta=th, phi=ph) - fd_tp) <= 1e-6 * max(1.0, abs(fd_tp))
                assert abs(ev(dpp, theta=th, phi=ph) - fd_pp) <= 1e-6 * max(1.0, abs(fd_pp))
    assert len(second["ylm_dtheta2"]) == 9
