"""fp64 restatement with a running error bound, for checking the dense chains element by element.

A `Bounded` value carries three fp64 tensors of the same shape:
    v  the exact result of the op sequence on the kernel's own fp32 inputs,
    m  the magnitude chain: the same sequence with every input, weight and bias replaced by its absolute value and
       swish(t) by 1.1 |t| (1.1 bounds |swish'|, so it is a Lipschitz constant of swish),
    e  a bound on |kernel - v|: each op adds its own rounding error, TOL * A + FLOOR with the constants below, where A
       is the magnitude of what the kernel actually multiplies (|v| + e of the op's inputs through |W|: for one layer
       on exact inputs A = M, the magnitude chain of that layer), and carries the error of its inputs forward through
       |W| and swish's Lipschitz constant.
For one layer e = TOL * M + FLOOR.  Through a chain, e stays below q * TOL * M after q layers (every later layer
multiplies an earlier error by at most what it multiplies the magnitude by), but is much smaller: M grows ~10x per
layer (sum|w| of a 128-wide Glorot row) while the values do not, so the bound of a deep output is built from the
rounding of the values actually computed, not from M.  A kernel passes when |y - v| <= e for EVERY element, so a
row far below the batch maximum is held to its own bound.

Rounding model of one 3xFP16 layer (csrc/spherenet_h16.cu: activations x pre-scaled by H_SA = 8, weights w by
H_SW = 64; each split into hi = fp16(s) and lo = fp16(s - hi); D = lo_x w_hi + hi_x lo_w + hi_x w_hi):
  * hi carries 11 bits, so |s - hi| <= 2^-11 |s|, and lo rounds that residual to 11 bits: |s - hi - lo| <= 2^-22 |s|
    while lo is normal.  lo goes subnormal below 2^-14: fp16's subnormal spacing 2^-24 leaves an ABSOLUTE error of
    at most 2^-25, i.e. 2^-25 / 8 = 2^-28 on an activation and 2^-25 / 64 = 2^-31 on a weight (FLOOR).
  * the dropped product lo_x lo_w is at most 2^-11 |x| * 2^-11 |w| = 2^-22 |x w|.
    Together: 3 * 2^-22 of sum|w||x| (second-order terms are below 2^-43).
  * the products of fp16 pairs are exact in fp32.  Each wgmma instruction (m64nNk16) adds its k16 products to the
    fp32 accumulator and truncates once: at most 1 ulp = 2^-23 of the chunk's sum|w||x|.  A K = 64 chunk is
    4 k-steps x 3 products = 12 instructions.
  * the K = 64 chunks are summed in fp32 with round-to-nearest (K/64 - 1 additions of 2^-24) and the bias is added
    by one fma (2^-24): K/64 * 2^-24.
  TOL_H16(K) = 3 * 2^-22 + 12 * 2^-23 + K/64 * 2^-24          (K = 128: 38 * 2^-24 = 2.3e-6)
  FLOOR_H16  = 2^-28 * sum|w| + 2^-31 * sum|x|
  K = 256 / 384 (`linear_h16_kernel` with two / three operand panels): the epilogue rebuilds the operand tile between
  panels, but a panel only changes WHICH columns of x the next K = 64 chunks read.  Every chunk still starts from a
  zeroed accumulator (scale-d = 0), so its 12 truncations are bounded by 2^-23 of that chunk's own sum|w||x| (<= the
  row's), and the epilogue adds the chunk sums into the same fp32 registers with __fadd_rn in chunk order across panel
  boundaries (h_drain<FIRST = false> for panels p > 0): K/64 - 1 additions, each below 2^-24 of a partial sum of
  |terms|, then the bias fma.  The split terms are per element and do not see panels at all.  So the same TOL_H16(K)
  holds with K/64 = 4 / 6 chunk terms; the residual of the fused epilogue is one more fp32 addition (`add`).
Aggregations and GraphNorm (ComENet):
  * filter_sum (dig3d_comenet_filter_sum): per edge and channel w = sum_q f_q W_q by Q fmas from zero (Q roundings of
    2^-24 of sum_q |f_q||W_q|), then acc = fma(w, x_j, acc) once per in-edge: c roundings of sum_e |w||x_j| for a node
    with c in-edges.  An error of W (the fold) and of x is carried through |f| and |w|, |x|.
  * the filter fold W_eff^T = W1^T W2^T (ComENet._filter_t: one exact-fp32 `ops.linear`, K = middle) is a K-term
    dot product: (K + 1) * 2^-24 of (|W1|^T |W2|^T), NOT of |W_eff| -- the middle sum can cancel (`fold`).
  * graphnorm (graphnorm_fwd_kernel, comenet_graphnorm_stats_kernel + comenet_norm_final_kernel): see `graphnorm`.
The 3xTF32 chain (csrc/spherenet_tc.cu) splits the same way (TF32 also carries 11 bits, fp32 range: no floor) but
accumulates K = 32 chunks of 4 k8-steps x 3 products: TOL_TF32(K) = 3 * 2^-22 + 12 * 2^-23 + K/32 * 2^-24.
The exact-fp32 FFMA kernels (the twins, the small rbf / sbf linears): a K-term dot product plus the bias is
K + 1 roundings of 2^-24 of sum|w||x| (gamma_{K+1}); a sum of n terms is n - 1 roundings; a product one.
swish: libdevice expf + IEEE division, or the MUFU ex2 / rcp approximations (2^-22 and 2^-23 relative) of the fast
form, plus the rounding of the scaled argument: below 2^-20 of |t| either way (TOL_ACT).
Underflow: the kernels keep fp32 subnormals (no flush to zero), so a rounding below 2^-126 is off by at most half the
subnormal spacing, 2^-150, ABSOLUTE (ETA): every op adds one ETA per rounding it counts.  It only matters where the
values themselves are ~1e-40, e.g. the edge features of edges at the cutoff, whose envelope goes to zero.
SchNet (csrc/schnet.cu, the training kernels of csrc/train_ops.cu / train_geom.cu).  Libdevice expf, log1pf, cosf and
sinf are within 2 ulp (4u of the result, u = 2^-24); the products, sums and quotients round once each:
  * ssp(t) = (t > 20 ? t : log1pf(expf(t))) - ln2_f (`ssp`): Lipschitz 1, so an input error passes unchanged.  expf's
    4u enter log1p as 4u * e^t / (1 + e^t) = 4u sigmoid(t), log1pf adds 4u of softplus(t), the subtraction u of the
    result.  The t > 20 branch is exact (the identity); an input error that straddles 20 may take the other branch,
    which differs by log1p(e^-20) < 2.1e-9.  Below t = -87 e^t is subnormal or 0: absolute, and far below u * ln2.
  * gauss = expf(c_f * (d - mu)^2) (`gauss`): the argument a = c_f ((d - mu)^2) takes three roundings, t = d - mu
    counted twice by the square (4u relative, c_f = fp32(coeff) being what the kernel receives), which exp turns into
    a relative error 4u |a| (magnified by |a|, up to ~1e3 for a Gaussian far from the edge), plus expf's own 4u;
    subnormal results 4 ETA absolute (2 ulp).
  * C = 0.5 (cosf((d pi_f) inv_f) + 1) (`cutoff_fn`): pi_f and inv_f = fp32(1/cutoff) are kernel inputs.  The
    argument x takes two roundings (2u |x|, moved by |sin x|), cosf 4u |cos x|, the + 1 one u.  Near C = 0 (x -> pi)
    cos x = -1 + O(C) and its 4u is an ABSOLUTE term next to C: the bound there is ~2u, not relative to C.
  * the cfconv aggregation (schnet_cfconv_kernel's tile_segment_accumulate): per 64-edge tile a running fp32 sum over
    each target's edges; a target whose edges cross a tile boundary gets two partial sums, added onto the zeroed row
    by atomics (the first is exact).  With at most 64 edges per target (33 under the neighbour cap) that is c - 1
    roundings for c in-edges, inside `index_add`'s c.
  * act' and act'' (`act_d1`, `act_d2`): s = sigmoid_f(x) = 1 / (1 + expf(-x)) is within 6u of s (4u expf, the add,
    the division); sm = sigmoid_f(-x) = 1 - s likewise, with no cancellation.  swish' = s (1 + x (1 - s)) evaluates
    1.0f - s, whose error is 6u s (absolute): <= 12u s (1 + |x| (1 - s)) + 7u |x| s^2.  swish'' = s sm (2 + x (1 - 2s))
    (1 - 2 s is exact after s): <= 17u s sm (2 + |x| |1 - 2s|) + 12u |x| s^2 sm.  ssp' = s: 6u s; ssp'' = s sm: 13u s
    sm, and 0 for x > 20 (the forward is the identity there, as in torch's softplus with threshold 20).  For |x| > 87
    s or sm is subnormal or 0: 2^-126 ABSOLUTE on each (SIG_FLOOR), times the factors it multiplies.  The kernel's
    dx = dy * d and out = (g * dy) * d2 add one and two roundings.
"""
import torch

U = 2.0 ** -24                       # fp32 round-to-nearest
ETA = 2.0 ** -150                    # fp32 gradual underflow: absolute error of one rounding below 2^-126
TOL_SPLIT = 3 * 2.0 ** -22
TOL_WGMMA_CHUNK = 12 * 2.0 ** -23
FLOOR_A, FLOOR_W = 2.0 ** -28, 2.0 ** -31
TOL_ACT = 2.0 ** -20
SWISH_LIP = 1.1


def tol_h16(k):
    return TOL_SPLIT + TOL_WGMMA_CHUNK + (k // 64 if k >= 64 else 1) * U


def tol_tf32(k):
    return TOL_SPLIT + TOL_WGMMA_CHUNK + max(k // 32, 1) * U


def tol_fp32(k):
    return (k + 1) * U


class Bounded:
    """(value, magnitude, error bound), fp64.  `split_max` records the largest operand each split layer multiplies."""
    __slots__ = ("v", "m", "e")
    split_max = []

    def __init__(self, v, m, e):
        self.v, self.m, self.e = v, m, e

    @classmethod
    def exact(cls, x):
        """A kernel input: taken as exact (only the kernel's own arithmetic is under test)."""
        x = x.detach().double()
        return cls(x, x.abs(), torch.zeros_like(x))

    def __getitem__(self, idx):
        return Bounded(self.v[idx], self.m[idx], self.e[idx])

    def check(self, y, what=""):
        """Assert |y - v| <= e element by element; returns the largest ratio |y - v| / e."""
        y = y.detach().double()
        assert y.shape == self.v.shape, (what, tuple(y.shape), tuple(self.v.shape))
        assert torch.isfinite(y).all(), f"{what}: non-finite output"
        err = (y - self.v).abs()
        bad = err > self.e
        if bad.any():
            i = int(torch.nonzero(bad.flatten())[0])
            raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound; first at flat "
                                 f"index {i}: kernel {float(y.flatten()[i])!r} fp64 {float(self.v.flatten()[i])!r} "
                                 f"|err| {float(err.flatten()[i]):.3e} bound {float(self.e.flatten()[i]):.3e} "
                                 f"magnitude {float(self.m.flatten()[i]):.3e}")
        return float((err / self.e.clamp_min(1e-300)).max()) if err.numel() else 0.0


def linear(x, w, b=None, engine="h16"):
    """x @ w^T + b on `engine`: 'h16' (3xFP16), 'tf32' (3xTF32) or 'fp32' (FFMA)."""
    w = w.detach().double()
    aw = w.abs()
    k = w.size(1)
    xm = x.v.abs() + x.e                             # magnitude of what the kernel actually multiplies
    v = x.v @ w.T
    m = x.m @ aw.T
    mu = xm @ aw.T
    if b is not None:
        b = b.detach().double()
        v, m, mu = v + b, m + b.abs(), mu + b.abs()
    e = x.e @ aw.T
    if engine != "fp32":
        Bounded.split_max.append(float(x.v.abs().max()) if x.v.numel() else 0.0)
    e = e + (k + 1) * ETA
    if engine == "h16":
        e = e + tol_h16(k) * mu + FLOOR_A * aw.sum(1) + FLOOR_W * xm.sum(-1, keepdim=True)
    elif engine == "tf32":
        e = e + tol_tf32(k) * mu
    else:
        e = e + tol_fp32(k) * mu
    return Bounded(v, m, e)


def swish(x):
    t = x.v.abs() + x.e
    return Bounded(x.v * torch.sigmoid(x.v), SWISH_LIP * x.m, SWISH_LIP * x.e + TOL_ACT * t + 4 * ETA)


def add(x, y):
    return Bounded(x.v + y.v, x.m + y.m, x.e + y.e + U * ((x.v + y.v).abs() + x.e + y.e) + ETA)


def mul(x, y):
    xa, ya = x.v.abs() + x.e, y.v.abs() + y.e
    return Bounded(x.v * y.v, x.m * y.m, x.e * ya + x.v.abs() * y.e + U * xa * ya + ETA)


def cat(parts):
    return Bounded(*(torch.cat([getattr(p, f) for p in parts], -1) for f in ("v", "m", "e")))


def index_add(x, idx, n):
    """Sum of the rows of x into n rows by idx, in any order: a row with c terms takes c - 1 roundings (+ one more:
    the kernels may split a segment and add the parts onto a zeroed row)."""
    idx = idx.long()
    cnt = torch.bincount(idx, minlength=n).double()[:, None]
    z = lambda t: torch.zeros(n, t.size(1), dtype=t.dtype, device=t.device).index_add_(0, idx, t)
    v, m, e = z(x.v), z(x.m), z(x.e)
    return Bounded(v, m, e + cnt * (U * (z(x.v.abs()) + e) + ETA))


def fold(w1, w2):
    """W_eff^T = W1^T W2^T [Q, hidden] of a TwoLayerLinear(bias=False) filter (W1 [middle, Q], W2 [hidden, middle]) as
    one exact-fp32 linear with K = middle: m and the rounding term are relative to |W1|^T |W2|^T."""
    return linear(Bounded.exact(w1.detach().T), w2, None, "fp32")


def filter_sum(feat, weff_t, x, src, row_ptr, n):
    """agg[i] = sum over the in-edges e = (j -> i) (CSR rows of row_ptr) of (feat[e] @ weff_t) * x[src[e]].
    feat: the exact [E, Q] features; weff_t, x: Bounded."""
    feat = feat.detach().double()
    q = feat.size(1)
    cnt = (row_ptr[1:] - row_ptr[:-1]).long()
    dst = torch.repeat_interleave(torch.arange(n, device=feat.device), cnt)
    af = feat.abs()
    wv, wm = feat @ weff_t.v, af @ weff_t.m
    we = af @ weff_t.e + q * (U * (af @ (weff_t.v.abs() + weff_t.e)) + ETA)      # Q fmas from zero
    src = src.long()
    xv, xm, xe = x.v[src], x.m[src], x.e[src]
    wa, xa = wv.abs() + we, xv.abs() + xe
    z = lambda t: torch.zeros(n, t.size(1), dtype=t.dtype, device=t.device).index_add_(0, dst, t)
    c = cnt.double()[:, None]
    return Bounded(z(wv * xv), z(wm * xm), z(we * xa + wv.abs() * xe) + c * (U * z(wa * xa) + ETA))   # one fma per in-edge


def graphnorm(h, graph_ptr, weight, bias, mean_scale, eps):
    """GraphNorm in the order of graphnorm_fwd_kernel (and of the fused stats / norm kernels), per graph and channel with
    cnt = max(nodes, 1) (an empty graph slot gives shift 0, sd = sqrt(eps)):
        sum = sum_n h          cnt - 1 fp32 additions                       |err| <= e_h summed + (cnt - 1) u A
        sh  = (sum / cnt) * ms  two roundings                               A = sum |h| + e_h
        o   = h - sh            one rounding; carries e_h + e_sh
        sq  = sum_n o * o       cnt products + cnt - 1 additions: cnt u sum (|o| + e_o)^2, plus 2 |o| e_o + e_o^2
        sd  = sqrt(sq / cnt + eps)  three roundings; |sqrt(a) - sqrt(b)| = |a - b| / (sqrt(a) + sqrt(b))
        y   = (w * o) / sd + b  three roundings; an error of o enters as |w| e_o / sd, one of sd as |w| |o| e_sd / sd^2.
    A kernel's sd is never below sqrt(fp32(eps)) (1 - u): sq >= 0 whatever its error, so that is the lower end of sd
    used for the 1/sd factors (at most |w| / 3.2e-3 with eps = 1e-5).  Returns (y, shift, sd) as Bounded."""
    dev = h.v.device
    ptr = graph_ptr.long()
    ng = ptr.numel() - 1
    counts = ptr[1:] - ptr[:-1]
    gid = torch.repeat_interleave(torch.arange(ng, device=dev), counts)
    cnt = counts.clamp_min(1).double()[:, None]
    w, b, ms = (t.detach().double().to(dev) for t in (weight, bias, mean_scale))
    aw, ams = w.abs(), ms.abs()
    eps32 = float(torch.tensor(eps, dtype=torch.float32))
    seg = lambda t: torch.zeros(ng, t.size(1), dtype=t.dtype, device=dev).index_add_(0, gid, t)
    hv, he = h.v, h.e
    S, A = seg(hv), seg(hv.abs() + he)
    mean = S / cnt
    e_mean = seg(he) / cnt + U * A                      # (cnt - 1) additions and the division, each <= u A / cnt .. u A
    sh = mean * ms
    e_sh = ams * e_mean + U * ams * (mean.abs() + e_mean)
    m_sh = ams * seg(h.m) / cnt
    o = hv - sh[gid]
    e_o = he + e_sh[gid] + U * (o.abs() + he + e_sh[gid])
    oa = o.abs() + e_o
    sq = seg(o * o)
    e_sq = seg(2 * o.abs() * e_o + e_o * e_o) + (cnt + 1) * U * seg(oa * oa)
    v = sq / cnt + eps32
    e_v = e_sq / cnt + 2 * U * ((sq + e_sq) / cnt + eps32)
    sd = v.sqrt()
    sd_min = eps32 ** 0.5 * (1 - 2 * U)
    e_sd = e_v / (sd + (v - e_v).clamp_min(0).sqrt()) + U * sd
    e_sd = e_sd + U * e_sd
    sd_lo = (sd - e_sd).clamp_min(sd_min)
    sdg, sdlg, esdg = sd[gid], sd_lo[gid], e_sd[gid]
    y = w * o / sdg + b
    t_a = aw * oa / sdlg
    e_y = aw * e_o / sdlg + aw * o.abs() * esdg / (sdg * sdlg) + 3 * U * t_a + U * (b.abs() + t_a) + 4 * ETA
    m_y = aw * (h.m + m_sh[gid]) / sdg + b.abs()
    return Bounded(y, m_y, e_y), Bounded(sh, m_sh, e_sh), Bounded(sd, sd, e_sd)


LN2_F = 0.693147182464599609375     # fp32(ln 2), the constant the kernels subtract
PI_F = 3.14159274101257324           # fp32(pi)
SIG_FLOOR = 2.0 ** -126              # sigmoid_f(x) or sigmoid_f(-x) subnormal or 0 (|x| > 87): absolute error


def f32(x):
    """The fp32 value the kernel receives for a host double."""
    return float(torch.tensor(x, dtype=torch.float32))


def ssp(x):
    """Shifted softplus with threshold 20 (see the module docstring)."""
    t = x.v
    hi = t + x.e                                     # sigmoid and softplus are increasing: their largest value in reach
    v = torch.nn.functional.softplus(t, threshold=20.0) - LN2_F
    e = (x.e + 4 * U * torch.sigmoid(hi) + 4 * U * torch.nn.functional.softplus(hi) + U * (v.abs() + x.e)
         + 2.1e-9 * ((t - 20.0).abs() <= x.e) + 2 * ETA)
    return Bounded(v, x.m, e)


def gauss(dist, offset, coeff):
    """expf(c_f * (d - mu)^2) for exact fp32 dist [E] and offset [G] -> [E, G]."""
    c = f32(coeff)
    t = dist.detach().double()[:, None] - offset.detach().double()[None, :]
    a = c * t * t
    v = torch.exp(a)
    rel = torch.expm1(4 * U * a.abs() + 2 * abs(c) * ETA) * (1 + 4 * U) + 4 * U
    return Bounded(v, v, v * rel + 4 * ETA)


def cutoff_fn(dist, cutoff):
    """0.5 (cosf((d pi_f) inv_f) + 1) for exact fp32 dist [E], inv_f = fp32(1 / cutoff)."""
    x = dist.detach().double() * PI_F * f32(1.0 / cutoff)
    ex = 2 * U * x.abs() * (1 + 2 * U)
    c = torch.cos(x)
    e_cos = x.sin().abs() * ex + ex * ex / 2 + 4 * U * (c.abs() + ex)
    e_sum = e_cos + U * ((c + 1).abs() + e_cos)
    v = 0.5 * (c + 1)
    return Bounded(v, v, 0.5 * e_sum + ETA)


def act_d1(x, mode):
    """act'(x) (mode 0 swish, 1 ssp, 2 relu) of exact fp32 x, as act_bwd_kernel evaluates it."""
    x = x.detach().double()
    s, sm, ax = torch.sigmoid(x), torch.sigmoid(-x), x.abs()
    if mode == 0:
        v = s * (1 + x * sm)
        e = 12 * U * s * (1 + ax * sm) + 7 * U * ax * s * s + SIG_FLOOR * (1 + 2 * ax)
    elif mode == 1:
        v, e = s, 6 * U * s + SIG_FLOOR
    else:
        v, e = (x > 0).double(), torch.zeros_like(x)
    return Bounded(v, v.abs(), e)


def act_d2(x, mode):
    """act''(x) of exact fp32 x, as act_bwd2_kernel evaluates it (ssp'' = 0 above the threshold 20)."""
    x = x.detach().double()
    s, sm, ax = torch.sigmoid(x), torch.sigmoid(-x), x.abs()
    if mode == 0:
        v = s * sm * (2 + x * (1 - 2 * s))
        e = 17 * U * s * sm * (2 + ax * (1 - 2 * s).abs()) + 12 * U * ax * s * s * sm + SIG_FLOOR * (2 + 2 * ax)
    elif mode == 1:
        keep = (x <= 20).double()
        v, e = keep * s * sm, keep * (13 * U * s * sm + SIG_FLOOR)
    else:
        v, e = torch.zeros_like(x), torch.zeros_like(x)
    return Bounded(v, v.abs(), e)


def split16(x, scale):
    """The kernels' operand split, exactly: s = fp32(x * scale), hi = fp16_rn(s), lo = fp16_rn(fp32(s - hi))."""
    s = x.float() * scale
    hi = s.half()
    lo = (s - hi.float()).half()
    return hi, lo
