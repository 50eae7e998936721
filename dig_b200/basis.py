"""Closed-form radial / angular basis tables for the 3D-graph models.

Product-side restatement of the construction the reference performs at model build time:

  * SphereNet / DimeNet++ ("dimenet" flavour): reference
    dig/threedgraph/method/spherenet/features.py:14-148 (identical code in dimenetpp/features.py)
  * ComENet ("gemnet" flavour): reference dig/threedgraph/method/comenet/features.py:16-254

For every (flavour, num_spherical, num_radial) it yields the *expression source strings*
(exactly what sympy.lambdify would hand to Python, e.g.
``(-1.4488*x*cos(4.4934*x) + 0.3224*sin(4.4934*x))/x**2``) for

  bessel[l*nr + n](x)        normalised spherical Bessel j_l(z_ln x)
  yl0[l](theta)              real spherical harmonics, m = 0
  ylm[f](theta, phi)         all real harmonics in the reference's flat order

dig_b200/codegen.py turns those strings into sm_90a device code that evaluates every Python
arithmetic node as ONE correctly-rounded fp32 operation, i.e. with the rounding behaviour of the
reference's op-by-op ATen evaluation (SURVEY.md §5.9c): the high-order closed forms cancel
catastrophically in fp32, so parity requires the same expression tree, not a "better" formula.

The fp32-rounded Bessel zeros and the normalisers are produced with the same numpy/scipy calls as
the reference (Appendix B of SURVEY.md: "regenerate, do not hard-code").
tests/test_basis.py pins the strings against tests/golden/basis_formulas.json, which was written
by the real reference in the build container.
"""
import functools
import math

import numpy as np


def _sym():
    import sympy
    return sympy


# ----------------------------------------------------------------------------- radial part
def _jn_dimenet(r, order):
    from scipy import special
    return np.sqrt(np.pi / (2 * r)) * special.jv(order + 0.5, r)      # features.py:14-15


def _jn_gemnet(r, order):
    from scipy import special
    return special.spherical_jn(order, r)                              # comenet/features.py:16-20


def bessel_zeros(jn, num_orders, num_zeros):
    """First `num_zeros` positive roots of j_l for l < num_orders, stored as float32
    (reference Jn_zeros, features.py:18-30: roots of order l bracket those of order l+1)."""
    from scipy.optimize import brentq
    table = np.zeros((num_orders, num_zeros), dtype="float32")
    table[0] = np.arange(1, num_zeros + 1) * np.pi
    brackets = np.arange(1, num_zeros + num_orders) * np.pi
    found = np.zeros(num_zeros + num_orders - 1, dtype="float32")
    for order in range(1, num_orders):
        for s in range(num_zeros + num_orders - 1 - order):
            found[s] = brentq(jn, brackets[s], brackets[s + 1], (order,))
        brackets = found
        table[order][:num_zeros] = found[:num_zeros]
    return table


def rayleigh_forms(num_orders):
    """Unnormalised j_l(x) via Rayleigh's formula j_l = (-x)^l (1/x d/dx)^l sin(x)/x, each
    simplified by sympy (reference spherical_bessel_formulas, features.py:33-42)."""
    sym = _sym()
    x = sym.symbols("x")
    forms = [sym.sin(x) / x]
    running = sym.sin(x) / x
    for order in range(1, num_orders):
        stepped = sym.diff(running, x) / x
        forms.append(sym.simplify(stepped * (-x) ** order))
        running = sym.simplify(stepped)
    return forms


def bessel_expressions(jn, num_orders, num_zeros):
    """Normalised, rescaled j_l(z_ln x) / sqrt(0.5 j_{l+1}(z_ln)^2) (reference bessel_basis,
    features.py:45-66)."""
    sym = _sym()
    x = sym.symbols("x")
    zeros = bessel_zeros(jn, num_orders, num_zeros)
    forms = rayleigh_forms(num_orders)
    out = []
    for order in range(num_orders):
        norm = []
        for n in range(num_zeros):
            norm += [0.5 * jn(zeros[order, n], order + 1) ** 2]
        norm = 1 / np.array(norm) ** 0.5
        out.append([sym.simplify(norm[n] * forms[order].subs(x, zeros[order, n] * x))
                    for n in range(num_zeros)])
    return out


# ----------------------------------------------------------------------------- angular part
def _prefactor_dimenet(l, m):
    return ((2 * l + 1) * math.factorial(l - abs(m)) /
            (4 * np.pi * math.factorial(l + abs(m)))) ** 0.5          # features.py:69-71


def _prefactor_gemnet(l, m):
    return ((2 * l + 1) / (4 * np.pi) * math.factorial(l - abs(m))
            / math.factorial(l + abs(m))) ** 0.5                        # comenet/features.py:100-104


def _legendre_dimenet(L, zero_m_only):
    """Associated Legendre P_l^m(z), m >= 0 (reference features.py:74-96)."""
    sym = _sym()
    z = sym.symbols("z")
    P = [[0] * (l + 1) for l in range(L)]
    P[0][0] = 1
    if L > 0:
        P[1][0] = z
        for l in range(2, L):
            P[l][0] = sym.simplify(((2 * l - 1) * z * P[l - 1][0] - (l - 1) * P[l - 2][0]) / l)
        if not zero_m_only:
            for m in range(1, L):
                P[m][m] = sym.simplify((1 - 2 * m) * P[m - 1][m - 1])
                if m + 1 < L:
                    P[m + 1][m] = sym.simplify((2 * m + 1) * z * P[m][m])
                for l in range(m + 2, L):
                    P[l][m] = sym.simplify(((2 * l - 1) * z * P[l - 1][m]
                                            - (m + l - 1) * P[l - 2][m]) / (l - m))
    return P


def harmonics_dimenet(L, zero_m_only):
    """Real spherical harmonics in (theta, phi) as the SphereNet/DimeNet++ reference builds
    them (features.py:99-148).  Returns Y[l] = list of 2l+1 entries indexed m = 0..l, then
    negative m from the end (python index -m)."""
    sym = _sym()
    theta, phi = sym.symbols("theta"), sym.symbols("phi")
    xs, ys = sym.symbols("x"), sym.symbols("y")
    if not zero_m_only:
        S, C = [xs * 0], [1 + 0 * xs]
        for m in range(1, L):
            S += [xs * S[m - 1] + ys * C[m - 1]]
            C += [xs * C[m - 1] - ys * S[m - 1]]
    P = _legendre_dimenet(L, zero_m_only)
    zsym = sym.symbols("z")
    for l in range(len(P)):
        for m in range(len(P[l])):
            if type(P[l][m]) != int:
                P[l][m] = P[l][m].subs(zsym, sym.cos(theta))
    if not zero_m_only:
        for m in range(len(S)):
            S[m] = S[m].subs(xs, sym.sin(theta) * sym.cos(phi)).subs(ys, sym.sin(theta) * sym.sin(phi))
        for m in range(len(C)):
            C[m] = C[m].subs(xs, sym.sin(theta) * sym.cos(phi)).subs(ys, sym.sin(theta) * sym.sin(phi))
    Y = [["0"] * (2 * l + 1) for l in range(L)]
    for l in range(L):
        Y[l][0] = sym.simplify(_prefactor_dimenet(l, 0) * P[l][0])
    if not zero_m_only:
        for l in range(1, L):
            for m in range(1, l + 1):
                Y[l][m] = sym.simplify(2 ** 0.5 * _prefactor_dimenet(l, m) * C[m] * P[l][m])
        for l in range(1, L):
            for m in range(1, l + 1):
                Y[l][-m] = sym.simplify(2 ** 0.5 * _prefactor_dimenet(l, -m) * S[m] * P[l][m])
    return Y


def _legendre_gemnet(L, zero_m_only):
    """Reference comenet/features.py:107-165 (pos_m_only=True path)."""
    sym = _sym()
    z = sym.symbols("z")
    P = [[0] * (2 * l + 1) for l in range(L)]
    P[0][0] = 1
    if L > 0:
        if zero_m_only:
            P[1][0] = z
            for l in range(2, L):
                P[l][0] = sym.simplify(((2 * l - 1) * z * P[l - 1][0] - (l - 1) * P[l - 2][0]) / l)
            return P
        for l in range(1, L):
            P[l][l] = sym.simplify((1 - 2 * l) * (1 - z ** 2) ** 0.5 * P[l - 1][l - 1])
        for m in range(0, L - 1):
            P[m + 1][m] = sym.simplify((2 * m + 1) * z * P[m][m])
        for l in range(2, L):
            for m in range(l - 1):
                P[l][m] = sym.simplify(((2 * l - 1) * z * P[l - 1][m]
                                        - (l + m - 1) * P[l - 2][m]) / (l - m))
    return P


def harmonics_gemnet(L, zero_m_only):
    """Reference comenet/features.py:168-254 with spherical_coordinates=True."""
    sym = _sym()
    theta, phi = sym.symbols("theta"), sym.symbols("phi")
    z = sym.symbols("z")
    P = _legendre_gemnet(L, zero_m_only)
    Y = [[0] for _ in range(L)] if zero_m_only else [[0] * (2 * l + 1) for l in range(L)]
    for l in range(L):
        for m in range(len(P[l])):
            if not isinstance(P[l][m], int):
                P[l][m] = P[l][m].subs(z, sym.cos(theta))
    for l in range(L):
        Y[l][0] = sym.simplify(_prefactor_gemnet(l, 0) * P[l][0])
    if not zero_m_only:
        for l in range(1, L):
            for m in range(1, l + 1):
                Y[l][m] = sym.simplify(2 ** 0.5 * (-1) ** m * _prefactor_gemnet(l, m)
                                       * P[l][m] * sym.cos(m * phi))
            for m in range(1, l + 1):
                Y[l][-m] = sym.simplify(2 ** 0.5 * (-1) ** m * _prefactor_gemnet(l, -m)
                                        * P[l][m] * sym.sin(m * phi))
    return Y


# ----------------------------------------------------------------------------- public tables
def _src(expr, args):
    """The expression string sympy.lambdify would emit for `expr` (LambdaPrinter, full
    precision floats) -- the reference lambdifies with a {'sin','cos'[, 'sqrt']} module dict,
    for which sympy uses its plain LambdaPrinter."""
    sym = _sym()
    import inspect
    f = sym.lambdify(args, expr, {"sin": math.sin, "cos": math.cos, "sqrt": math.sqrt})
    return inspect.getsource(f).split("return", 1)[1].strip()


@functools.lru_cache(maxsize=None)
def basis_sources(flavor, num_spherical, num_radial):
    """dict(bessel=[ns*nr strings in x], yl0=[ns strings in theta], ylm=[strings in theta, phi]).

    flavor 'dimenet': SphereNet / DimeNet++ (ylm flat order per l: m = 0, +1..+l, -l..-1 --
    reference features.py:244-251 iterates python indices 0..2l of a list laid out
    [m=0, 1..l, -l..-1]).  flavor 'gemnet': ComENet (same index walk over its own table)."""
    sym = _sym()
    x, theta, phi = sym.symbols("x"), sym.symbols("theta"), sym.symbols("phi")
    if flavor == "dimenet":
        bess = bessel_expressions(_jn_dimenet, num_spherical, num_radial)
        y0 = harmonics_dimenet(num_spherical, zero_m_only=True)
        yall = harmonics_dimenet(num_spherical, zero_m_only=False)
    elif flavor == "gemnet":
        bess = bessel_expressions(_jn_gemnet, num_spherical, num_radial)
        y0 = harmonics_gemnet(num_spherical, zero_m_only=True)
        yall = harmonics_gemnet(num_spherical, zero_m_only=False)
    else:
        raise ValueError(flavor)
    out = {"bessel": [], "yl0": [], "ylm": [], "bessel_dx": [], "yl0_dtheta": [], "ylm_dtheta": [], "ylm_dphi": []}
    for l in range(num_spherical):
        for n in range(num_radial):
            out["bessel"].append(_src(bess[l][n], [x]))
            # d/dx of the same closed form (force path: dE/dpos needs d(basis)/d(dist)); not a reference string --
            # the reference differentiates the lambdified graph with autograd
            out["bessel_dx"].append(_src(sym.diff(bess[l][n], x), [x]))
    for l in range(num_spherical):
        if l == 0:
            out["yl0"].append(repr(float(sym.lambdify([theta], y0[0][0])(0))))
        else:
            out["yl0"].append(_src(y0[l][0], [theta]))
        out["yl0_dtheta"].append("0.0" if l == 0 else _src(sym.diff(y0[l][0], theta), [theta]))
    for l in range(num_spherical):
        if l == 0:
            out["ylm"].append(repr(float(sym.lambdify([theta, phi], yall[0][0])(0, 0))))
            out["ylm_dtheta"].append("0.0")
            out["ylm_dphi"].append("0.0")
        else:
            for k in range(2 * l + 1):
                out["ylm"].append(_src(yall[l][k], [theta, phi]))
                # force path (not reference strings): partial derivatives of the same closed forms
                dth, dph = sym.diff(yall[l][k], theta), sym.diff(yall[l][k], phi)
                out["ylm_dtheta"].append("0.0" if dth == 0 else _src(dth, [theta, phi]))
                out["ylm_dphi"].append("0.0" if dph == 0 else _src(dph, [theta, phi]))
    return out


@functools.lru_cache(maxsize=None)
def basis_sources_second_order(flavor, num_spherical, num_radial):
    """Second derivatives of the closed forms of `basis_sources`: bessel_dxx [ns*nr] in x, yl0_dtheta2 [ns] in theta,
    and ylm_dtheta2 / ylm_dtheta_dphi / ylm_dphi2 [ns*ns] in (theta, phi).  The Hessian path of DimeNet++ / SphereNet
    reads them (csrc/generated/basis_<tag>_d2.cuh, the reverse mode of the tangent kernels in csrc/basis.cu)."""
    sym = _sym()
    x, theta, phi = sym.symbols("x"), sym.symbols("theta"), sym.symbols("phi")
    if flavor == "dimenet":
        bess = bessel_expressions(_jn_dimenet, num_spherical, num_radial)
        y0 = harmonics_dimenet(num_spherical, zero_m_only=True)
        yall = harmonics_dimenet(num_spherical, zero_m_only=False)
    elif flavor == "gemnet":
        bess = bessel_expressions(_jn_gemnet, num_spherical, num_radial)
        y0 = harmonics_gemnet(num_spherical, zero_m_only=True)
        yall = harmonics_gemnet(num_spherical, zero_m_only=False)
    else:
        raise ValueError(flavor)
    out = {"bessel_dxx": [], "yl0_dtheta2": [], "ylm_dtheta2": [], "ylm_dtheta_dphi": [], "ylm_dphi2": []}
    for l in range(num_spherical):
        for n in range(num_radial):
            out["bessel_dxx"].append(_src(sym.diff(bess[l][n], x, 2), [x]))
        out["yl0_dtheta2"].append("0.0" if l == 0 else _src(sym.diff(y0[l][0], theta, 2), [theta]))
    for l in range(num_spherical):
        for k in range(2 * l + 1 if l else 1):
            for key, args in (("ylm_dtheta2", (theta, theta)), ("ylm_dtheta_dphi", (theta, phi)),
                              ("ylm_dphi2", (phi, phi))):
                d = 0 if l == 0 else sym.diff(yall[l][k], *args)
                out[key].append("0.0" if d == 0 else _src(d, [theta, phi]))
    return out


def envelope_coefficients(exponent):
    """Smooth cutoff env(x) = 1/x + a x^(p-1) + b x^p + c x^(p+1), p = exponent + 1
    (reference Envelope, features.py:151-164)."""
    p = exponent + 1
    return p, -(p + 1) * (p + 2) / 2, p * (p + 2), -p * (p + 1) / 2


def harmonics_recurrence(theta, phi, num_spherical, dtype=np.float64):
    """numpy twin of csrc/harmonics.cuh `ylm_recurrence`: the L*L real harmonics in the reference's flat order (per l:
    m = 0, +1..+l, -l..-1) from the recurrences the reference's symbolic construction starts from (features.py:74-148),
    evaluated numerically instead of through the simplified closed forms.  The fused projection kernel uses this form;
    tests/test_basis.py pins it against the closed forms."""
    L = num_spherical
    theta = np.asarray(theta, dtype=dtype)
    phi = np.asarray(phi, dtype=dtype)
    f = dtype

    def norm(l, m):
        v = math.sqrt((2 * l + 1) * math.factorial(l - m) / (4 * math.pi * math.factorial(l + m)))
        return f(v * (math.sqrt(2.0) if m else 1.0))

    st, ct, sp, cp = np.sin(theta), np.cos(theta), np.sin(phi), np.cos(phi)
    x, y, z = st * cp, st * sp, ct
    out = np.zeros(theta.shape + (L * L,), dtype=dtype)
    p2, p1 = np.ones_like(z), z
    out[..., 0] = norm(0, 0)
    if L > 1:
        out[..., 1] = norm(1, 0) * z
    for l in range(2, L):
        p = (f((2.0 * l - 1.0) / l) * z) * p1 - f((l - 1.0) / l) * p2
        out[..., l * l] = norm(l, 0) * p
        p2, p1 = p1, p
    s, c, pmm = np.zeros_like(z), np.ones_like(z), np.ones_like(z)
    for m in range(1, L):
        s, c = x * s + y * c, x * c - y * s
        pmm = f(1 - 2 * m) * pmm
        p2, p1 = np.zeros_like(z), pmm
        for l in range(m, L):
            if l == m:
                p = pmm
            elif l == m + 1:
                p = (f(2 * m + 1) * z) * pmm
            else:
                p = (f((2.0 * l - 1.0) / (l - m)) * z) * p1 - f((l + m - 1) / (l - m)) * p2
            n_p = norm(l, m) * p
            out[..., l * l + m] = n_p * c
            out[..., l * l + 2 * l + 1 - m] = n_p * s
            p2, p1 = p1, p
    return out
