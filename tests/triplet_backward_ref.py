"""fp64 references and per-element bounds for the three triplet-stage backward kernels of the training path.

    sphere_triplet_gather_bwd   (csrc/train_sphere.cu)   d x_down, d sbf_p, d t_p, dW_sbf2, dW_t2
    triplet_basis_project_bwd   (csrc/basis.cu)          dW_sbf1 [32, ns nr], dW_t1 [32, ns^2 nr]
    rbf_freq_grad               (csrc/basis.cu)          d freq

Every forward below is plain differentiable torch; the exact gradients are torch.autograd.grad of it in fp64 on the
kernel's own fp32 inputs cast up.  Every output of these gradients is a sum of products of inputs, so the same autograd
with every input and every upstream gradient replaced by its absolute value gives M = sum |terms| per output element.
A kernel output passes when, for EVERY element,

    |got - exact| <= gamma(c) * M + c * ETA,      gamma(c) = c u / (1 - c u),  u = 2^-24,  ETA = 2^-150 (underflow)

with c the number of fp32 roundings on the longest path from a product to the stored value.  A sum of n addends taken
in ANY order (atomics) is counted as n roundings, each relative to a partial sum of |terms| <= M.

sphere_triplet_gather (forward, spherenet_tc.cu tg_accumulate; "warp" / "edge" organisations are the same arithmetic):
    g = lin_sbf2(sbf_p), h = lin_t2(t_p): 8 fmas each from zero; x g, (x g) h: 2 products; one add per triplet of the edge.
    m[e]        c = 8 + 8 T + 2 + nt(e)            T = 1 with torsion, 0 without (h == 1 exactly), nt(e) triplets of e
sphere_triplet_gather_bwd (one warp per edge e = (j -> i), lanes = channels c and c + 32):
    d x_down[kj] one atomicAdd of dm g h (g, h as above, 2 products) per triplet that reads row kj:
                c = 8 + 8 T + 2 + n(kj)            n(kj) = number of triplets with idx_kj == kj
    d sbf_p[t]  v = fma(a0, w0, a1 w1) with a = (dm x) h: h 8 T, two products, a1 w1, the fma; then the 16-value
                warp reduction adds 32 lanes in 5 levels:      c = 8 T + 2 + 2 + 5
    d t_p[t]    the same with g in place of h:                c = 8 + 2 + 2 + 5
    dW_sbf2     a (8 T + 2 roundings) times sbf_p[t], one fma per triplet into a REGISTER of the warp that owns the
                edge (edge e belongs to warp e mod n_warps, n_warps = 8 min(ceil(E / 8), 296)); then 8 warps are added by
                shared atomics and the CTAs by global atomics.  Longest path, not the triplet total:
                c = 8 T + 2 + max over warps of (triplets of its edges) + 8 + grid
    dW_t2       the same with g: c = 8 + 2 + ...
triplet_basis_project_bwd (one warp per (k -> j) edge, lane = (layer, row)):
    G[l] = sum over the triplets that use kj of d_p[t] Y_l(t): one fma each; G[l] * bess[kj]: one product; shared
    atomicAdd per edge of the CTA; global atomicAdd per CTA.  The reference multiplies d_p with the MATERIALISED basis
    sbf[t] = fl(bess[kj] Y_l(t)) of ops.triplet_basis, which carries one more rounding of the same product:
                c = max n(kj) + 2 + edges per CTA + grid,  edges per CTA = 8 ceil(E / (8 grid)), grid = min(ceil(E / 8), 2 SMs)
    Harmonics: this kernel calls the generated closed forms (BS::yl0 / BS::ylm, one correctly rounded fp32 op per node,
    never contracted) -- the same functions, on the same fp32 angles, as ops.triplet_basis, so the Y it multiplies are
    bit-identical to the ones inside sbf / tbf and the harmonic term of THIS bound is zero.  The recurrence harmonics
    (csrc/harmonics.cuh, the default of the FORWARD projection) differ from the closed forms: tests/test_basis.py
    measured the fp32 recurrences within 3e-6 of the fp64 closed forms and the fp32 closed forms are as far from them,
    so the forward projection is held to gamma(c) M + HARMONIC_TOL sum_c |bess[kj, c]| |w[q, c]| (`project_forward_bound`).
rbf_freq_grad (grid-stride over the edges, 8 partial sums per thread, warp shuffle, one atomicAdd per warp and n):
    d freq[n] = sum_e drbf0[e, n] env(x) cos(freq_n x) x,  x = fl(dist fl(1 / cutoff)).
    env is itself a cancelling sum (1/x + a x^(p-1) + b x^p + c x^(p+1) -> 0 at the cutoff), so its magnitude is
    env_abs = 1/x + |a| x^(p-1) + |b| x^p + |c| x^(p+1) and cos is replaced by |cos|:  M1 = sum |drbf0| env_abs |cos| x.
    x differs from dist / cutoff by 2 u; x d(env)/dx is at most (p + 1) env_abs.  The argument freq x carries 3 u
    (x, and the product), which moves cos by 3 u (freq x) |sin| whatever |cos| is: M2 = sum |drbf0| env_abs (freq x) |sin| x.
    C_ENV = 2 (p + 1) + 1 (rcp) + P (x^(p-1): powf, 4 ulp = 8 u; 1 for x x, 2 for x x x, 0 for x) + 2 (x^p, x^(p+1))
            + 3 (coefficients) + 3 (additions)
    per term: C_ENV + 2 (x as a factor) + 1 (env x) + 4 (cosf, 2 ulp) + 1 (times cos) ; accumulation: one fma per
    grid-stride iteration, 5 shuffle levels, one atomic per warp that holds an edge:
                c1 = C_ENV + 8 + iterations + 5 + warps,   c2 = 3

The first-order force path of the fused widths (tests/test_gpu_force_path_fp64.py):
edge_basis_bwd ddist (one thread per edge, csrc/basis.cu):
    ddist[e] = fl(1/cutoff) sum_n drbf0[e, n] (env'(x) sin(f_n x) + env(x) f_n cos(f_n x)),  x = fl(dist fl(1 / cutoff)).
    The reference is evaluated at the kernel's own fp32 x (`edge_bwd_reference`), so x carries no error of its own.
    env and env' are cancelling sums (env(1) = env'(1) = 0): their magnitudes take every coefficient and power by
    absolute value, env_abs as above and envd_abs = 1/x^2 + |a| (p-1) x^(p-2) + |b| p x^(p-1) + |c| (p+1) x^p.
        M1 = sum_n |drbf0| (envd_abs |sin| + env_abs f |cos|) / cutoff
        M2 = sum_n |drbf0| (envd_abs |cos| + env_abs f |sin|) (f x) / cutoff      the argument f x, counted as 3 u
    Every arithmetic node is counted as one rounding even where nvcc contracts it into an fma (that only removes
    roundings).  env: rcp 1, x^(p-1) 8 (powf, or fewer), two more powers 2, coefficients 1, three adds 3 -> 15.
    env': powf(x, p-2) 8, two powers 2, coefficient times constant and times power 2, x x and the division 2 (the
    shorter branch), three adds 3 -> 15.  Per order: the product with sinf / cosf (4 u each, 2 ulp) 1 + 4, f env 1,
    the add 1, the fma into acc 1 per order; the product with fl(1 / cutoff) 2:
                c1 = 15 + 1 + 4 + 1 + 1 + NR + 2,   c2 = 3
edge_basis_bwd bess_dx (BS::bessel / BS::bessel_dx, the generated closed forms, one fp32 rounding per node):
    the reference is the fp64 evaluation of basis_sources(...)["bessel_dx"] at the kernel's x; folded with the envelope
    (DimeNet++) bess_dx = fma(env', bessel, env bessel_dx).  A closed form is a sum of products with at most one sin /
    cos each; its magnitude (`source_magnitude`) is the same string evaluated in fp64 with every constant and
    subtraction made positive and sin / cos by |sin| / |cos|, plus the first-order sensitivity of each term to a relative
    error in its sin / cos argument (sin(a) -> |a| |cos a|, cos(a) -> |a| |sin a|) -- an fp32 argument z x carries the
    rounding of z and of the product, and near a zero of sin(z x) that is the whole error.  BESSEL_DX_TOL is not derived
    node by node: tests/test_force_path_ref_cpu.py evaluates every string node by node in fp32 on the CPU and asserts
    the worst |fp32 - fp64| / magnitude over x in [X_MIN, 1) is at most BESSEL_DX_TOL / 4; the factor 4 leaves room for
    the device's 2-ulp sinf / cosf and its reciprocal-times-constant divisions.  With the envelope the bound adds
    gamma(15 + 2) (envd_abs |bessel| + env_abs |bessel_dx|) for the envelope's own roundings and the fma.
triplet_basis_project_bwd_geom (one warp per (k -> j) edge, lane = candidate i of the molecule, csrc/basis.cu):
    per edge and lane q = (layer, row): R[q] = sum_r bess[kj, (l, r)] w[q, (l, r)], NR fmas (and R' with bess_dx); per
    triplet h_l = sum_q d[t, q] R[q], 32 fmas (dot32); then one fma per harmonic into d angle / d x / d torsion: NS
    (yl0, yl0'), plus NY (ylm, d ylm / d theta, d ylm / d phi) with torsion:
                c_t = NR + 32 + NS + NY
    ddist[kj]: a lane adds the d x of every triplet it owns (one candidate i per 32-atom chunk of the molecule:
    ceil(atoms / 32) adds at most), a 5-level butterfly, the product with fl(1 / cutoff) (2):
                c_e = c_t + ceil(atoms / 32) + 5 + 2
    The harmonics are the generated closed forms, held to CLOSED_FORM_TOL on every Y (the Mh term, as for
    triplet_basis_bwd).  The reference is `basis_bwd_reference` with d_sbf = sum_l d_s[l] W_s[l] (fp64), and its
    magnitudes with |d_s| |W_s| in place of d_sbf.
"""
import ast
import math

import torch

U = 2.0 ** -24
ETA = 2.0 ** -150
HARMONIC_TOL = 8e-6
# fp32 closed-form harmonics (one correctly rounded op per node, CUDA sinf / cosf within 2 ulp) lie within 7e-6 of their
# fp64 values for num_spherical = 7 and 5e-7 for 3 over theta in [0, pi], phi in [-pi, pi] (values and both derivatives,
# measured with the same strings on the CPU); 2e-5 leaves room for the device's sin / cos.
CLOSED_FORM_TOL = 2e-5
BESSEL_DX_TOL = 16 * U
# smallest x at which the fp32 closed forms of both bases were measured within BESSEL_DX_TOL / 4 of fp64 (relative to
# `source_magnitude`, see test_force_path_ref_cpu.py); below it, 1 / x^k of the high orders leaves the fp32 range
X_MIN = {0: 1e-5, 1: 1e-6}
C_ENV_BWD = 15                   # roundings of env and of env' in edge_basis_bwd (module docstring)
GATHER_BWD_MAX_GRID = 296        # csrc/train_sphere.cu
FREQ_MAX_GRID = 592              # csrc/basis.cu


def gamma(c):
    cu = c * U
    return cu / (1.0 - cu)


# ---------------------------------------------------------------------------------------------------- forwards (fp64)
def gather_forward(x_down, sbf_p, t_p, w_sbf2, w_t2, idx_kj, idx_ji, n_edges):
    """m[e] = sum over the triplets of e of x_down[kj] * lin_sbf2(sbf_p) (* lin_t2(t_p))   (spherenet.py:163-171)."""
    y = x_down[idx_kj] * (sbf_p @ w_sbf2.T)
    if t_p is not None:
        y = y * (t_p @ w_t2.T)
    return torch.zeros(n_edges, x_down.size(1), dtype=y.dtype, device=y.device).index_add(0, idx_ji, y)


def project_forward(sbf, tbf, w_s_rows, w_t_rows):
    """lin_sbf1 / lin_t1 of all layers at once on the materialised bases: (sbf @ w_s^T, tbf @ w_t^T | None)."""
    return sbf @ w_s_rows.T, (tbf @ w_t_rows.T if tbf is not None else None)


def envelope_coefficients(exponent):
    p = exponent + 1
    return p, -(p + 1) * (p + 2) / 2.0, float(p * (p + 2)), -p * (p + 1) / 2.0


def freq_forward(dist, freq, cutoff, exponent):
    """rbf0 = envelope(d / c) * sin(freq * d / c)   (spherenet/features.py:159-182)."""
    p, a, b, c = envelope_coefficients(exponent)
    x = dist.unsqueeze(-1) / cutoff
    env = 1.0 / x + a * x ** (p - 1) + b * x ** p + c * x ** (p + 1)
    return env * torch.sin(freq * x)


def _grads(forward, inputs, upstream):
    """torch.autograd.grad of sum(forward(*inputs) * upstream) w.r.t. every tensor of `inputs` (None passes through)."""
    leaves = [None if t is None else t.detach().double().requires_grad_(True) for t in inputs]
    outs = forward(*leaves)
    outs = outs if isinstance(outs, tuple) else (outs,)
    pairs = [(o, u.detach().double()) for o, u in zip(outs, upstream) if o is not None and u is not None]
    live = [t for t in leaves if t is not None]
    got = iter(torch.autograd.grad([o for o, _ in pairs], live, [u for _, u in pairs], allow_unused=True))
    grads = [None if t is None else next(got) for t in leaves]
    return [o.detach() for o in outs if o is not None], grads


def _abs(ts):
    return [None if t is None else t.detach().abs() for t in ts]


# ---------------------------------------------------------------------------------------------------- references
def gather_reference(x_down, sbf_p, t_p, w_sbf2, w_t2, idx_kj, idx_ji, n_edges, dm):
    """{name: (exact, magnitude)} for m, dx, d_sbf_p, d_t_p, dw_sbf2, dw_t2 (the torsion entries None without t_p)."""
    idx_kj, idx_ji = idx_kj.long(), idx_ji.long()
    fwd = lambda x, s, t, ws, wt: gather_forward(x, s, t, ws, wt, idx_kj, idx_ji, n_edges)
    ins = [x_down, sbf_p, t_p, w_sbf2, w_t2]
    (m,), g = _grads(fwd, ins, [dm])
    (mm,), gm = _grads(fwd, _abs(ins), _abs([dm]))
    names = ["dx", "d_sbf_p", "d_t_p", "dw_sbf2", "dw_t2"]
    out = {"m": (m, mm)}
    out.update({n: (None if v is None else (v, a)) for n, v, a in zip(names, g, gm)})
    return out


def gather_counts(idx_kj, idx_ji, n_edges, torsion):
    """Rounding counts c of the gather outputs (see the module docstring); per row where the count is per row."""
    t = 1 if torsion else 0
    nt = torch.bincount(idx_ji.long(), minlength=n_edges)
    nkj = torch.bincount(idx_kj.long(), minlength=n_edges)
    grid = min(-(-n_edges // 8), GATHER_BWD_MAX_GRID)
    n_warps = 8 * max(grid, 1)
    per_warp = torch.zeros(n_warps, dtype=nt.dtype, device=nt.device)
    per_warp.index_add_(0, torch.arange(n_edges, device=nt.device) % n_warps, nt)
    longest = int(per_warp.max()) if n_edges else 0
    return {"m": (10 + 8 * t + nt).double()[:, None], "dx": (10 + 8 * t + nkj).double()[:, None],
            "d_sbf_p": 8 * t + 9.0, "d_t_p": 17.0,
            "dw_sbf2": 8 * t + 2.0 + longest + 8 + grid, "dw_t2": 10.0 + longest + 8 + grid}


def project_reference(sbf, tbf, d_s, d_t):
    """d_s / d_t: lists (<= 4) of [T, 8] upstream gradients or None -> {"dw_sbf1": (exact [32, NB], magnitude),
    "dw_t1": ... | None}.  A missing layer (None, or past the end of the list) contributes zero rows."""
    def wide(lst, ref):
        z = torch.zeros(ref.size(0), 8, dtype=torch.float64, device=ref.device)
        lst = list(lst) + [None] * (4 - len(lst))
        return torch.cat([z if d is None else d.detach().double() for d in lst], 1)
    sbf = sbf.detach().double()
    tbf = None if tbf is None or d_t is None else tbf.detach().double()
    ups = [wide(d_s, sbf), None if tbf is None else wide(d_t, tbf)]
    zeros = lambda b: None if b is None else torch.zeros(32, b.size(1), dtype=torch.float64, device=b.device)
    fwd = lambda ws, wt: project_forward(sbf, tbf, ws, wt)
    _, g = _grads(fwd, [zeros(sbf), zeros(tbf)], ups)
    sbf, tbf = sbf.abs(), (None if tbf is None else tbf.abs())
    _, gm = _grads(fwd, [zeros(sbf), zeros(tbf)], _abs(ups))
    return {"dw_sbf1": (g[0], gm[0]), "dw_t1": None if tbf is None else (g[1], gm[1])}


def project_count(idx_kj, n_edges, n_sm):
    """Rounding count c of both outputs of triplet_basis_project_bwd."""
    grid = max(min(-(-n_edges // 8), 2 * n_sm), 1)
    per_cta = 8 * -(-n_edges // (8 * grid))
    uses = int(torch.bincount(idx_kj.long(), minlength=1).max()) if idx_kj.numel() else 0
    return float(uses + 2 + per_cta + grid)


def project_forward_bound(basis, bess_kj, w_rows, per_edge_terms):
    """(exact, bound) of the forward projection basis @ w^T for a kernel that evaluates the harmonics by recurrence:
    the fma chains (`per_edge_terms` + the harmonic sum: basis.size(1) roundings at most) plus HARMONIC_TOL on every Y."""
    basis, w = basis.detach().double(), w_rows.detach().double()
    c = basis.size(1) + per_edge_terms + 2.0
    m = basis.abs() @ w.abs().T
    rep = basis.size(1) // bess_kj.size(1)           # tbf repeats the edge's Bessel row once per a of (a, b)
    radial = bess_kj.detach().double().abs().repeat(1, rep) @ w.abs().T
    return basis @ w.T, gamma(c) * m + HARMONIC_TOL * radial + c * ETA


def freq_reference(dist, freq, cutoff, exponent, drbf0):
    """(exact d freq [nr], M1, M2) -- see the module docstring."""
    dist64, freq64, d64 = dist.detach().double(), freq.detach().double(), drbf0.detach().double()
    _, (g,) = _grads(lambda f: freq_forward(dist64, f, cutoff, exponent), [freq64], [d64])
    p, a, b, c = envelope_coefficients(exponent)
    x = dist64.unsqueeze(-1) / cutoff
    env_abs = 1.0 / x + abs(a) * x ** (p - 1) + abs(b) * x ** p + abs(c) * x ** (p + 1)
    arg = freq64 * x
    m1 = (d64.abs() * env_abs * arg.cos().abs() * x).sum(0)
    m2 = (d64.abs() * env_abs * arg.sin().abs() * arg.abs() * x).sum(0)
    return g, m1, m2


def freq_counts(n_edges, exponent):
    p = exponent + 1
    power = {1: 0, 2: 1, 3: 2}.get(p - 1, 8)
    c_env = 2 * (p + 1) + 1 + power + 2 + 3 + 3
    grid = max(min(-(-n_edges // 256), FREQ_MAX_GRID), 1)
    iters = -(-n_edges // (grid * 256))
    warps = min(-(-n_edges // 32), grid * 8)
    return float(c_env + 8 + iters + 5 + warps), 3.0


# ---------------------------------------------------------------------------------------------------- force path (fp64)
def envelope_terms(x, exponent):
    """(env, env', env_abs, envd_abs) at x (fp64) -- see the module docstring."""
    p, a, b, c = envelope_coefficients(exponent)
    env = 1.0 / x + a * x ** (p - 1) + b * x ** p + c * x ** (p + 1)
    envd = -1.0 / x ** 2 + a * (p - 1) * x ** (p - 2) + b * p * x ** (p - 1) + c * (p + 1) * x ** p
    env_abs = 1.0 / x + abs(a) * x ** (p - 1) + abs(b) * x ** p + abs(c) * x ** (p + 1)
    envd_abs = 1.0 / x ** 2 + abs(a) * (p - 1) * x ** (p - 2) + abs(b) * p * x ** (p - 1) + abs(c) * (p + 1) * x ** p
    return env, envd, env_abs, envd_abs


def kernel_x(dist, cutoff):
    """x = fl(dist fl(1 / cutoff)) as the edge kernels form it, returned in fp64."""
    inv = torch.tensor(1.0 / cutoff, dtype=torch.float32)
    return (dist.detach().float() * inv.to(dist.device)).double()


def edge_bwd_reference(x, freq, cutoff, exponent, drbf0):
    """(exact ddist [E], M1, M2) of edge_basis_bwd at the kernel's x (fp64) -- see the module docstring."""
    env, envd, env_abs, envd_abs = envelope_terms(x.unsqueeze(-1), exponent)
    f, d = freq.detach().double(), drbf0.detach().double()
    arg = f * x.unsqueeze(-1)
    exact = (d * (envd * arg.sin() + env * f * arg.cos())).sum(1) / cutoff
    m1 = (d.abs() * (envd_abs * arg.sin().abs() + env_abs * f.abs() * arg.cos().abs())).sum(1) / cutoff
    m2 = (d.abs() * (envd_abs * arg.cos().abs() + env_abs * f.abs() * arg.sin().abs()) * arg.abs()).sum(1) / cutoff
    return exact, m1, m2


def edge_bwd_count(nr):
    return float(C_ENV_BWD + 1 + 4 + 1 + 1 + nr + 2), 3.0


class _Magnitude(ast.NodeTransformer):
    """Every constant positive, every subtraction an addition, sin / cos -> |sin| / |cos| (`arg`: -> the sensitivity to
    a relative error in the argument, |a| |cos a| / |a| |sin a|)."""

    def __init__(self, arg):
        self.arg = arg

    def visit_BinOp(self, node):
        self.generic_visit(node)
        if isinstance(node.op, ast.Sub):
            node.op = ast.Add()
        return node

    def visit_UnaryOp(self, node):
        self.generic_visit(node)
        return node.operand if isinstance(node.op, (ast.USub, ast.UAdd)) else node

    def visit_Constant(self, node):
        return ast.Constant(abs(node.value))

    def visit_Call(self, node):
        self.generic_visit(node)
        if node.func.id not in ("sin", "cos"):
            return node
        call = lambda fn, args: ast.Call(ast.Name(fn, ast.Load()), args, [])
        if not self.arg:
            return call("abs", [node])
        other = call("cos" if node.func.id == "sin" else "sin", node.args)
        return ast.BinOp(call("abs", node.args), ast.Mult(), call("abs", [other]))


def magnitude_source(src, arg=False):
    """The closed form `src` with every term made non-negative (see _Magnitude), as a string."""
    return ast.unparse(_Magnitude(arg).visit(ast.parse(src, mode="eval")))


def eval_source(src, x):
    """A basis_sources string evaluated on the tensor x: one rounding per node in x's dtype."""
    env = {"sin": torch.sin, "cos": torch.cos, "sqrt": torch.sqrt, "abs": torch.abs, "pi": math.pi, "x": x}
    v = eval(src, env)
    return v if torch.is_tensor(v) else torch.full_like(x, float(v))


def source_magnitude(src, x):
    """fp64 magnitude of the closed form `src` at x: the abs-transform plus the argument sensitivity."""
    return eval_source(magnitude_source(src), x) + eval_source(magnitude_source(src, arg=True), x)


def bessel_tables(ns, nr, x):
    """{key: (fp64 values [E, ns nr], magnitudes)} of the closed forms "bessel" and "bessel_dx" at x (fp64)."""
    from dig_b200.basis import basis_sources
    src = basis_sources("dimenet", ns, nr)
    return {k: (torch.stack([eval_source(s, x) for s in src[k]], 1),
                torch.stack([source_magnitude(s, x) for s in src[k]], 1)) for k in ("bessel", "bessel_dx")}


def bess_dx_reference(x, ns, nr, exponent, env_on_bessel):
    """(exact bess_dx [E, ns nr], bound) of edge_basis_bwd's second output at the kernel's x (fp64)."""
    t = bessel_tables(ns, nr, x)
    (b, mb), (bd, mbd) = t["bessel"], t["bessel_dx"]
    if not env_on_bessel:
        return bd, BESSEL_DX_TOL * mbd
    env, envd, env_abs, envd_abs = (v.unsqueeze(-1) for v in envelope_terms(x, exponent))
    exact = envd * b + env * bd
    return exact, (BESSEL_DX_TOL * (envd_abs * mb + env_abs * mbd)
                   + gamma(C_ENV_BWD + 2) * (envd_abs * b.abs() + env_abs * bd.abs()) + (C_ENV_BWD + 2) * ETA)


def harmonics(ns, angle, torsion, nr=6):
    """fp64 closed forms of the generated headers: yl0, yl0', ylm, dylm/dtheta, dylm/dphi, each [T, K]."""
    from dig_b200.basis import basis_sources
    src = basis_sources("dimenet", ns, nr)
    th = angle.double()
    ph = torsion.double() if torsion is not None else torch.zeros_like(th)
    env = {"sin": torch.sin, "cos": torch.cos, "sqrt": torch.sqrt, "pi": math.pi, "theta": th, "phi": ph}

    def table(key):
        cols = [eval(s, env) for s in src[key]]
        return torch.stack([c if torch.is_tensor(c) else torch.full_like(th, float(c)) for c in cols], 1)
    return {k: table(k) for k in ("yl0", "yl0_dtheta", "ylm", "ylm_dtheta", "ylm_dphi")}


def basis_bwd_reference(g, cutoff, ns, bess, bess_dx, angle, torsion, d_sbf, d_tbf):
    """fp64 (ddist, dangle, dtorsion) of the triplet bases' reverse mode (g needs idx_kj and n_edges), under "v", their
    magnitudes M (every factor by its absolute value) under "m" and Mh (the harmonic factor dropped) under "h"."""
    nr = bess.size(1) // ns
    Y = harmonics(ns, angle, torsion, nr)
    kj = g.idx_kj.long()
    B = bess.double()[kj].view(-1, ns, nr)
    Bd = bess_dx.double()[kj].view(-1, ns, nr)
    ds = d_sbf.double().view(-1, ns, nr)
    out = {}
    for mode in ("v", "m", "h"):
        f = (lambda x: x) if mode == "v" else torch.abs
        y = {k: (torch.ones_like(v) if mode == "h" else f(v)) for k, v in Y.items()}
        s_b, s_bd = (f(ds) * f(B)).sum(2), (f(ds) * f(Bd)).sum(2)           # [T, ns]
        dang = (y["yl0_dtheta"] * s_b).sum(1)
        dx = (y["yl0"] * s_bd).sum(1)
        dtor = None
        if d_tbf is not None:
            dt = d_tbf.double().view(-1, ns, ns, nr)                          # [T, a, b, r]
            h = (f(dt) * f(B)[:, None]).sum(3).reshape(-1, ns * ns)          # [T, ab]
            hd = (f(dt) * f(Bd)[:, None]).sum(3).reshape(-1, ns * ns)
            dang = dang + (y["ylm_dtheta"] * h).sum(1)
            dtor = (y["ylm_dphi"] * h).sum(1)
            dx = dx + (y["ylm"] * hd).sum(1)
        inv = 1.0 / cutoff
        ddist = torch.zeros(g.n_edges, dtype=torch.float64, device=bess.device).index_add_(0, kj, dx) * inv
        out[mode] = (ddist, dang, dtor)
    return out


# ---------------------------------------------------------------------------------------------------- the check
def bound(mag, c):
    return gamma(c) * mag + c * ETA


def check(got, exact, limit, what):
    """Assert finiteness, then |got - exact| <= limit on every element.  Returns the largest |got - exact| / limit."""
    got = got.detach().double()
    assert got.shape == exact.shape, (what, tuple(got.shape), tuple(exact.shape))
    assert torch.isfinite(got).all(), (f"{what}: {int((~torch.isfinite(got)).sum())} non-finite elements -- the output "
                                       "buffer is allocated uninitialised, so a row the kernel never wrote shows up here")
    limit = torch.broadcast_to(torch.as_tensor(limit, dtype=torch.float64, device=got.device), got.shape)
    err = (got - exact).abs()
    bad = err > limit
    if bad.any():
        i = int(torch.nonzero(bad.flatten())[0])
        where = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), got.shape)) if got.dim() else ()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound; first at {where}: "
                             f"kernel {float(got.flatten()[i])!r} fp64 {float(exact.flatten()[i])!r} "
                             f"|err| {float(err.flatten()[i]):.3e} bound {float(limit.flatten()[i]):.3e}")
    return float((err / limit.clamp_min(1e-300)).max()) if err.numel() else 0.0


# ---------------------------------------------------------------------------------------------------- graphs (host side)
def capped_batch():
    """(pos, batch, cutoff): 90 atoms uniform in a 3 A box as one molecule (every atom has > 33 candidates within 6 A,
    so the neighbour cap binds: in-degree 33 where the atom itself is not among its first 33 hits, asymmetric in / out
    lists) followed by a 40-atom molecule of QM9-like spacing; both have more than 32 atoms."""
    from dig_b200.data import synthetic_molecules
    dense = torch.rand(90, 3, generator=torch.Generator().manual_seed(1)) * 3.0
    mol = synthetic_molecules(1, "qm9", seed=7, natoms=40)[0]
    pos = torch.cat([dense, mol.pos + 100.0]).float()
    batch = torch.cat([torch.zeros(90), torch.ones(40)]).long()
    return pos, batch, 6.0


def ragged_batch():
    """(pos, batch, cutoff, num_graphs): two atoms 30 A apart (no edge), a single atom, a diatomic (edges, no triplets),
    an empty graph slot, a bonded quadruple."""
    pos = torch.tensor([[0, 0, 0], [30, 0, 0], [5, 5, 5], [0, 0, 0], [1.1, 0, 0],
                        [0, 0, 0], [1, 0.1, 0], [0.2, 1.2, 0], [0.9, 1.0, 0.8]], dtype=torch.float32)
    batch = torch.tensor([0, 0, 1, 2, 2, 4, 4, 4, 4])
    return pos, batch, 5.0, 5


def tiny_batch():
    """(pos, batch, cutoff): one bonded triple -- 6 edges, 6 triplets: fewer edges than the 8 warps of the only CTA."""
    pos = torch.tensor([[0, 0, 0], [1, 0, 0], [0, 1.2, 0]], dtype=torch.float32)
    return pos, torch.zeros(3, dtype=torch.long), 5.0


def collinear_batch():
    """(pos, batch, cutoff): a straight chain of four atoms (angles exactly 0 and pi) next to a bent triple."""
    pos = torch.tensor([[0, 0, 0], [1.2, 0, 0], [2.4, 0, 0], [3.6, 0, 0],
                        [0, 0, 0], [1.1, 0, 0], [0.3, 1.0, 0.2]], dtype=torch.float32)
    return pos, torch.tensor([0, 0, 0, 0, 1, 1, 1]), 5.0
