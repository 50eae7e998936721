"""CPU self-check of the element-wise bound used by tests/test_gpu_dense_fp64.py (tests/fp64_bound.py).

The 3xFP16 product is emulated exactly as the kernels split their operands (fp16 round-to-nearest of x * 8 and of
the residual, the same for w * 64), with the three products summed in fp64.  The bound must accept it in every
activation / weight regime the GPU tests use, and must reject (a) the same product with the A_lo * W_hi correction
of one k16 step dropped and (b) an error confined to a row 100x below the batch maximum, which the old max-normalised
metric (`helpers.rel_err < 1e-5`) lets through.  So the GPU test is sharp enough to see a missing correction.
The same holds for the ComENet ops of tests/test_gpu_comenet_fp64.py: the split product at K = 256 / 384 (chunk sums
carried across operand panels; rejects a dropped chunk), the folded edge-filter sum (rejects a dropped q term) and
GraphNorm (cnt = 1, an empty slot, constant / large-offset channels, mean_scale 0 / 0.5 / 1; rejects a one-pass
variance, a dropped eps and an ignored mean_scale), each emulated in fp32 in its kernel's operation order."""
import pytest
import torch

from fp64_bound import (LN2_F, PI_F, U, Bounded, act_d1, act_d2, cutoff_fn, filter_sum, fold, gauss, graphnorm, linear,
                        mul, split16, ssp)
from helpers import rel_err

ROWS, K, N = 512, 128, 128
ACT_SCALES = [1e-4, 1e-2, 1.0, 4000.0, 8100.0]
WEIGHT_SCALES = [2.0 ** -8, 2.0 ** -4, 1.0, 4.0]


def _operands(act, ws, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(ROWS, K, generator=g, dtype=torch.float64) * act / 3).clamp(-act, act).float()
    a = (6.0 / (K + N)) ** 0.5                                    # formula (uniform Glorot) weights, then scaled
    w = ((torch.rand(N, K, generator=g, dtype=torch.float64) * 2 - 1) * a * ws).float()
    b = (0.1 * act * (torch.rand(N, generator=g, dtype=torch.float64) * 2 - 1)).float()
    return x, w, b


def _emulate(x, w, b, drop_lo_hi_step=None):
    """fp32 result of the kernels' three-product form (sum in fp64, then the fp32 epilogue rounding)."""
    xh, xl = (t.double() for t in split16(x, 8.0))
    wh, wl = (t.double() for t in split16(w, 64.0))
    lo_hi = xl @ wh.T
    if drop_lo_hi_step is not None:                              # one k16 step of the A_lo * W_hi correction missing
        s = slice(16 * drop_lo_hi_step, 16 * drop_lo_hi_step + 16)
        lo_hi = lo_hi - xl[:, s] @ wh[:, s].T
    return ((lo_hi + xh @ wl.T + xh @ wh.T) / 512.0 + b.double()).float()


@pytest.mark.parametrize("ws", WEIGHT_SCALES)
@pytest.mark.parametrize("act", ACT_SCALES)
def test_bound_accepts_the_emulated_split_product(act, ws):
    x, w, b = _operands(act, ws)
    ref = linear(Bounded.exact(x), w, b, "h16")
    y = _emulate(x, w, b)
    assert torch.isfinite(y).all()
    ratio = ref.check(y, f"act={act} ws={ws}")
    assert ratio < 0.5, ratio                                      # the model is not at the edge of its bound


def test_split_is_exact_below_the_range_edge_and_overflows_above():
    """8189 * 8 rounds to 65504 (fp16's largest finite value); 8191 * 8 = 65528 rounds to inf."""
    hi, lo = split16(torch.tensor([8189.0, -8189.0, 8191.0]), 8.0)
    assert torch.isfinite(hi[:2]).all() and (hi[:2].float() + lo[:2].float() == torch.tensor([65512.0, -65512.0])).all()
    assert torch.isinf(hi[2])


@pytest.mark.parametrize("ws", WEIGHT_SCALES)
@pytest.mark.parametrize("act", [1.0, 4000.0, 8100.0])
@pytest.mark.parametrize("step", [0, 7])
def test_bound_rejects_a_dropped_correction_step(act, ws, step):
    """Activations above 0.03 keep lo normal: the missing 2^-11-sized correction is far outside the bound."""
    x, w, b = _operands(act, ws, seed=1)
    ref = linear(Bounded.exact(x), w, b, "h16")
    y = _emulate(x, w, b, drop_lo_hi_step=step)
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.check(y)


def test_bound_rejects_a_row_local_error_that_rel_err_accepts():
    x, w, b = _operands(1.0, 1.0, seed=2)
    x[7] *= 0.01                                                   # a row 100x below the others (a near-cutoff edge)
    b[:] = 0.0
    ref = linear(Bounded.exact(x), w, b, "h16")
    y = _emulate(x, w, b)
    ref.check(y)
    y[7] += 20 * ref.e[7].float()                                  # 20x that row's own bound
    assert rel_err(y.numpy(), ref.v.numpy()) < 1e-5
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.check(y)


# ------------------------------------------------------------------------------------------------ K = 256 / 384 panels
def _emulate_chunks(x, w, b, drop_chunk=None):
    """The kernel's order at any K: each K = 64 chunk's three split products rounded to fp32 on their own (the
    accumulator of a chunk starts from zero), the chunk sums added in fp32 in chunk order across the operand panels
    (128 columns each), then the 1 / (H_SA H_SW) scale and the bias in one fma (emulated in fp64, rounded once)."""
    xh, xl = (t.double() for t in split16(x, 8.0))
    wh, wl = (t.double() for t in split16(w, 64.0))
    acc = None
    for c in range(x.size(1) // 64):
        if c == drop_chunk:
            continue
        s = slice(64 * c, 64 * c + 64)
        d = (xl[:, s] @ wh[:, s].T + xh[:, s] @ wl[:, s].T + xh[:, s] @ wh[:, s].T).float()
        acc = d if acc is None else acc + d
    return (acc.double() / 512.0 + b.double()).float()


def _operands_k(k, n, act, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(ROWS, k, generator=g, dtype=torch.float64) * act / 3).clamp(-act, act).float()
    x = x * 10.0 ** (torch.rand(ROWS, 1, generator=g, dtype=torch.float64) * 4 - 4).float()     # rows over 4 decades
    a = (6.0 / (k + n)) ** 0.5
    w = ((torch.rand(n, k, generator=g, dtype=torch.float64) * 2 - 1) * a).float()
    b = (0.1 * (torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1)).float()
    return x, w, b


@pytest.mark.parametrize("act", [1e-4, 1.0, 8100.0])
@pytest.mark.parametrize("k", [256, 384])
def test_bound_holds_across_operand_panels(k, act):
    """tol_h16(K) for two / three panels: the chunk sums carried across panels are K/64 - 1 fp32 additions."""
    x, w, b = _operands_k(k, 192, act, seed=k)
    ratio = linear(Bounded.exact(x), w, b, "h16").check(_emulate_chunks(x, w, b), f"K={k} act={act}")
    assert ratio < 0.5, ratio


@pytest.mark.parametrize("k", [256, 384])
def test_bound_rejects_a_dropped_chunk_of_the_second_panel(k):
    x, w, b = _operands_k(k, 192, 1.0, seed=k + 1)
    ref = linear(Bounded.exact(x), w, b, "h16")
    ref.check(_emulate_chunks(x, w, b))
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.check(_emulate_chunks(x, w, b, drop_chunk=2), f"K={k} chunk 2 (columns 128-191) dropped")


# ------------------------------------------------------------------------------------------------ filter_sum
def _filter_case(seed=3, n=40, q=12, width=32):
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(1, 9, (n,), generator=g)
    row_ptr = torch.zeros(n + 1, dtype=torch.long)
    row_ptr[1:] = torch.cumsum(deg, 0)
    e = int(row_ptr[-1])
    src = torch.randint(0, n, (e,), generator=g)
    feat = torch.rand(e, q, generator=g).float()
    weff_t = (torch.randn(q, width, generator=g) * 0.3).float()
    x = (torch.randn(n, width, generator=g) * 10.0 ** (torch.rand(n, 1, generator=g) * 4 - 3)).float()
    return feat, weff_t, x, src, row_ptr, n


def _filter_emulate(feat, weff_t, x, src, row_ptr, n, drop_q=None):
    """dig3d_comenet_filter_sum's order: w by Q fmas from zero, then one fma per in-edge (fma = exact fp64 product and
    sum, rounded to fp32)."""
    fma = lambda a, b, c: (a.double() * b.double() + c.double()).float()
    out = torch.zeros(n, x.size(1))
    for i in range(n):
        acc = torch.zeros(x.size(1))
        for e in range(int(row_ptr[i]), int(row_ptr[i + 1])):
            w = torch.zeros(x.size(1))
            for q in range(feat.size(1)):
                if q != drop_q:
                    w = fma(weff_t[q], feat[e, q].expand(x.size(1)), w)
            acc = fma(w, x[src[e]], acc)
        out[i] = acc
    return out


def test_filter_sum_bound_accepts_the_kernel_order_and_rejects_a_dropped_q_term():
    feat, weff_t, x, src, row_ptr, n = _filter_case()
    ref = filter_sum(feat, Bounded.exact(weff_t), Bounded.exact(x), src, row_ptr, n)
    assert ref.check(_filter_emulate(feat, weff_t, x, src, row_ptr, n), "filter_sum") < 0.5
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.check(_filter_emulate(feat, weff_t, x, src, row_ptr, n, drop_q=5), "filter_sum without q = 5")


def test_fold_bound_is_relative_to_the_factor_magnitudes():
    """W1^T W2^T in exact fp32 with a cancelling middle sum: the bound is built on |W1|^T |W2|^T."""
    g = torch.Generator().manual_seed(4)
    w1, w2 = torch.randn(64, 12, generator=g).float(), torch.randn(32, 64, generator=g).float()
    w2[:, 32:] = -w2[:, :32] * (w1[:32, :].abs().mean() / w1[32:, :].abs().mean())   # partial cancellation
    ref = fold(w1, w2)
    y = (w1.T.double() @ w2.T.double())                           # fp64, then one fp32 rounding per K-term sum
    assert ref.check(y.float(), "fold") < 0.5
    assert torch.allclose(ref.m, w1.T.double().abs() @ w2.T.double().abs())


# ------------------------------------------------------------------------------------------------ graphnorm
GN_SIZES = [1, 0, 16, 2, 3, 40]                 # cnt = 1, an empty graph slot, small and large graphs
GN_W = 8


def _gn_case(ms_value, seed=5):
    """Channel 0 constant, 1 a large offset (mean 1e3, spread 1e-2), 2 a small spread (1e-2 around 0), the rest randn
    over four decades."""
    g = torch.Generator().manual_seed(seed)
    ptr = torch.zeros(len(GN_SIZES) + 1, dtype=torch.int32)
    ptr[1:] = torch.cumsum(torch.tensor(GN_SIZES), 0)
    n = int(ptr[-1])
    h = torch.randn(n, GN_W, generator=g) * 10.0 ** (torch.rand(1, GN_W, generator=g) * 4 - 2)
    h[:, 0] = 0.37
    h[:, 1] = 1e3 + 1e-2 * torch.randn(n, generator=g)
    h[:, 2] = 1e-2 * torch.randn(n, generator=g)
    w = (1.0 + 0.1 * (torch.rand(GN_W, generator=g) * 2 - 1)).float()
    b = (0.1 * (torch.rand(GN_W, generator=g) * 2 - 1)).float()
    ms = torch.full((GN_W,), ms_value).float()
    return h.float(), ptr, w, b, ms


def _gn_emulate(h, ptr, w, b, ms, eps=1e-5, fault=None):
    """graphnorm_fwd_kernel in fp32, node by node (vectorised over channels).  fault: 'one_pass' (E[h^2] - E[h]^2),
    'no_eps', 'no_mean_scale'."""
    eps = torch.tensor(eps, dtype=torch.float32)
    y = torch.empty_like(h)
    for gi in range(ptr.numel() - 1):
        n0, n1 = int(ptr[gi]), int(ptr[gi + 1])
        cnt = torch.tensor(float(max(n1 - n0, 1)))
        s = torch.zeros(h.size(1))
        for n in range(n0, n1):
            s = s + h[n]
        sh = s / cnt if fault == "no_mean_scale" else (s / cnt) * ms
        sq = torch.zeros(h.size(1))
        if fault == "one_pass":
            for n in range(n0, n1):
                sq = sq + h[n] * h[n]
            var = sq / cnt - sh * sh
        else:
            for n in range(n0, n1):
                o = h[n] - sh
                sq = sq + o * o
            var = sq / cnt
        sd = torch.sqrt(var if fault == "no_eps" else var + eps)
        for n in range(n0, n1):
            y[n] = (w * (h[n] - sh)) / sd + b
    return y


@pytest.mark.parametrize("ms_value", [0.0, 0.5, 1.0])
def test_graphnorm_bound_accepts_the_kernel_order(ms_value):
    h, ptr, w, b, ms = _gn_case(ms_value)
    y_ref, sh_ref, sd_ref = graphnorm(Bounded.exact(h), ptr, w, b, ms, 1e-5)
    assert y_ref.check(_gn_emulate(h, ptr, w, b, ms), f"graphnorm ms={ms_value}") < 0.5
    assert float(sd_ref.v[1].min()) == pytest.approx(1e-5 ** 0.5, rel=1e-6)     # the empty slot: sd = sqrt(eps)
    assert float(sh_ref.v[1].abs().max()) == 0.0


@pytest.mark.parametrize("fault", ["one_pass", "no_eps", "no_mean_scale"])
def test_graphnorm_bound_rejects_a_wrong_kernel(fault):
    """one_pass cancels on the large-offset channel (var 1e-4 under a mean of 1e3); no_eps moves sd by 5 % on the
    1e-2-spread channel and divides by zero on the constant one; no_mean_scale shifts by the mean at mean_scale 0.5."""
    h, ptr, w, b, ms = _gn_case(0.5 if fault == "no_mean_scale" else 1.0)
    y_ref = graphnorm(Bounded.exact(h), ptr, w, b, ms, 1e-5)[0]
    cols = {"one_pass": [1], "no_eps": [2], "no_mean_scale": list(range(GN_W))}[fault]
    y = _gn_emulate(h, ptr, w, b, ms, fault=fault)
    y_ref[:, cols].check(_gn_emulate(h, ptr, w, b, ms)[:, cols])
    with pytest.raises(AssertionError, match="outside the bound|non-finite"):
        y_ref[:, cols].check(y[:, cols], f"graphnorm with {fault}")


# ------------------------------------------------------------------------------------------------ SchNet ops, act', act''
def _ssp32(x):
    """ssp in the kernels' fp32 order: (x > 20 ? x : log1pf(expf(x))) - fp32(ln 2)."""
    return torch.where(x > 20, x, torch.log1p(torch.exp(x))) - torch.tensor(LN2_F)


def _sigmoid32(x):
    return 1.0 / (1.0 + torch.exp(-x))


def _act_x():
    """Dense around 0, dense over [8, 20] and around the ssp threshold, out to the expf under- / overflow at +-88."""
    return torch.cat([torch.linspace(-100, 100, 4001), torch.linspace(-3, 3, 2001), torch.linspace(8, 20, 3001),
                      torch.linspace(19.99, 20.01, 201)]).float()


def test_ssp_bound_accepts_the_kernel_order():
    """Near ssp = -ln 2 (x < -8) the subtraction's half-ulp rounding (2^-25) is the whole error and the bound u |v| is
    0.69 u: the emulation reaches ~0.72 of it there."""
    x = _act_x()
    assert ssp(Bounded.exact(x)).check(_ssp32(x), "ssp") < 0.8


def test_ssp_bound_rejects_the_unshifted_softplus():
    x = _act_x()
    with pytest.raises(AssertionError, match="outside the bound"):
        ssp(Bounded.exact(x)).check(_ssp32(x) + torch.tensor(LN2_F), "softplus without the shift")


def _d_case(n=512, cutoff=10.0, g=50, seed=6):
    """Distances over [0, cutoff] with coincident atoms (d = 0) and pairs at 0.99 - 1.0 x cutoff; Gaussian centres of
    the model (far ones underflow into subnormals and 0)."""
    gen = torch.Generator().manual_seed(seed)
    d = torch.cat([torch.zeros(2), torch.rand(n, generator=gen) * cutoff,
                   cutoff * (0.99 + 0.01 * torch.rand(64, generator=gen)), torch.tensor([cutoff])]).float()
    offset = torch.linspace(0.0, cutoff, g)
    return d, offset, -0.5 / (offset[1] - offset[0]).item() ** 2


def _gauss32(d, offset, coeff):
    t = d[:, None] - offset[None, :]
    return torch.exp(torch.tensor(coeff, dtype=torch.float32) * (t * t))


def _cut32(d, cutoff):
    x = (d * torch.tensor(PI_F, dtype=torch.float32)) * torch.tensor(1.0 / cutoff, dtype=torch.float32)
    return 0.5 * (torch.cos(x) + 1.0)


@pytest.mark.parametrize("g", [2, 50, 64, 70])
def test_gauss_and_cutoff_bounds_accept_the_kernel_order(g):
    d, offset, coeff = _d_case(g=g)
    gs = _gauss32(d, offset, coeff)
    assert (gs[gs > 0] < 2.0 ** -126).any() or g == 2                # subnormal Gaussians are part of the case
    # the argument's rounding, magnified by |a|, is the whole error of a far Gaussian: the emulation (the kernel's own
    # fp32 argument) reaches 0.9 of its worst case there
    assert gauss(d, offset, coeff).check(gs, f"gauss G={g}") < 0.95
    assert cutoff_fn(d, 10.0).check(_cut32(d, 10.0), "cutoff") < 0.8


def test_gauss_bound_rejects_an_unrounded_coefficient_and_the_cutoff_bound_a_relative_model():
    d, offset, coeff = _d_case()
    ref = gauss(d, offset, coeff)
    t = d.double()[:, None] - offset.double()[None, :]
    with pytest.raises(AssertionError, match="outside the bound"):  # (coeff + 1e-4 relative): far Gaussians move
        ref.check(torch.exp(coeff * (1 + 1e-4) * t * t).float(), "coeff off by 1e-4")
    c = cutoff_fn(d, 10.0)
    near = d > 9.9
    assert (c.e[near] > 16 * U * c.v[near]).any()                    # the absolute term near C = 0
    with pytest.raises(AssertionError, match="outside the bound"):
        c.check(_cut32(d, 10.0 * (1 + 1e-6)), "cutoff 1e-6 off")


def _filter(d, offset, coeff, w0, b0, w2, b2, fault=None):
    """update_e's filter in fp32: W = (ssp(gauss @ w0^T + b0) @ w2^T + b2) * C, with a seeded fault."""
    h = _ssp32(_gauss32(d, offset, coeff) @ w0.T + b0)
    f = h @ w2.T + (0.0 if fault == "no_b2" else b2)
    c = _cut32(d, 10.0)
    w = f * c[:, None]
    return w * c[:, None] if fault == "cutoff_twice" else w


@pytest.mark.parametrize("fault", [None, "no_b2", "cutoff_twice"])
def test_filter_bound_accepts_the_kernel_order_and_rejects_a_seeded_fault(fault):
    d, offset, coeff = _d_case(g=50)
    gen = torch.Generator().manual_seed(7)
    a0, a2 = (6.0 / (50 + 64)) ** 0.5, (6.0 / 128) ** 0.5
    w0 = ((torch.rand(64, 50, generator=gen) * 2 - 1) * a0 * 300).float()   # pre-activations beyond +-88
    w2 = ((torch.rand(64, 64, generator=gen) * 2 - 1) * a2).float()
    b0, b2 = (0.1 * (torch.rand(2, 64, generator=gen) * 2 - 1)).float()
    pre = linear(gauss(d, offset, coeff), w0, b0, "fp32")
    assert (pre.v > 20).any() and (pre.v < -88).any()
    ref = mul(linear(ssp(pre), w2, b2, "fp32"), cutoff_fn(d, 10.0)[:, None])
    y = _filter(d, offset, coeff, w0, b0, w2, b2, fault)
    if fault is None:
        assert ref.check(y, "filter") < 0.5
    else:
        with pytest.raises(AssertionError, match="outside the bound"):
            ref.check(y, f"filter with {fault}")


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_act_derivative_bounds_accept_the_kernel_order(mode):
    x = _act_x()
    s, sm = _sigmoid32(x), _sigmoid32(-x)
    d1 = [s * (1.0 + x * (1.0 - s)), s, (x > 0).float()][mode]
    d2 = [s * sm * (2.0 + x * (1.0 - 2.0 * s)), torch.where(x > 20, 0.0, s * sm), torch.zeros_like(x)][mode]
    assert act_d1(x, mode).check(d1, f"act' mode {mode}") < 0.5
    assert act_d2(x, mode).check(d2, f"act'' mode {mode}") < 0.5


@pytest.mark.parametrize("mode", [0, 1])
def test_act_second_derivative_bound_rejects_the_cancelling_one_minus_s(mode):
    """1.0f - s loses every digit of 1 - s as s -> 1: the parent kernel's form at x in [10, 17]."""
    x = torch.linspace(10, 17, 701).float()
    s = _sigmoid32(x)
    y = s * (1.0 - s) * (2.0 + x * (1.0 - 2.0 * s)) if mode == 0 else s * (1.0 - s)
    with pytest.raises(AssertionError, match="outside the bound"):
        act_d2(x, mode).check(y, f"act'' mode {mode} with 1 - s")
