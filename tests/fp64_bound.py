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


def split16(x, scale):
    """The kernels' operand split, exactly: s = fp32(x * scale), hi = fp16_rn(s), lo = fp16_rn(fp32(s - hi))."""
    s = x.float() * scale
    hi = s.half()
    lo = (s - hi.float()).half()
    return hi, lo
