"""CPU self-check of the element-wise bound used by tests/test_gpu_dense_fp64.py (tests/fp64_bound.py).

The 3xFP16 product is emulated exactly as the kernels split their operands (fp16 round-to-nearest of x * 8 and of
the residual, the same for w * 64), with the three products summed in fp64.  The bound must accept it in every
activation / weight regime the GPU tests use, and must reject (a) the same product with the A_lo * W_hi correction
of one k16 step dropped and (b) an error confined to a row 100x below the batch maximum, which the old max-normalised
metric (`helpers.rel_err < 1e-5`) lets through.  So the GPU test is sharp enough to see a missing correction."""
import pytest
import torch

from fp64_bound import Bounded, linear, split16
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
