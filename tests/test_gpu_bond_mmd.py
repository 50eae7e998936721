"""GPU tests of the bond-length MMD (csrc/mmd.cu through dig_b200.ggraph3D.utils.compute_mmd / ops.mmd_terms): the
reference's values on every fixture case, the fp64 restatement (oracle/restated_mmd.py) run on CUDA at sizes past 2^32
pairs, determinism, symmetry and the reference's nan / error cases."""
import math

import pytest
import torch

from test_bond_mmd_cpu import fixture_cases

pytestmark = pytest.mark.gpu
F64 = torch.float64


def _restated_terms(s, t, **kw):
    from oracle import restated_mmd
    b, xx, yy, xy = restated_mmd.compute_mmd_terms(s.to("cuda", F64), t.to("cuda", F64), **kw)
    return [float(b), float(xx), float(yy), float(xy)]


def _lengths(n, mean, std, seed):
    g = torch.Generator().manual_seed(seed)
    return mean + std * torch.randn(n, generator=g, dtype=F64)


def test_fixture_cases_match_the_reference():
    from dig_b200.ggraph3D.utils import compute_mmd
    from oracle import restated_mmd
    for meta, s, t, ref in fixture_cases():
        src, tgt, kw = torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda(), meta["kwargs"]
        if meta["outcome"] == "raises":
            with pytest.raises(ZeroDivisionError):
                compute_mmd(src, tgt, **kw)
            continue
        got = compute_mmd(src, tgt, **kw)
        if math.isnan(ref):
            assert math.isnan(got), meta["name"]
        elif src.dtype == torch.float32 and tgt.dtype == torch.float32:
            # the reference computes this case in fp32, the port in fp64: the fp64 restatement of the same values is the
            # 1e-10 yardstick, the reference's fp32 value agrees to fp32 rounding
            want = restated_mmd.compute_mmd(src.double().cpu(), tgt.double().cpu(), **kw)
            assert abs(got - want) <= 1e-10, (meta["name"], got, want)
            assert abs(got - ref) <= 1e-5, (meta["name"], got, ref)
        else:
            assert abs(got - ref) <= 1e-10, (meta["name"], got, ref)


@pytest.mark.parametrize("n_source", [1, 9000])
def test_terms_match_the_fp64_restatement_past_2_32_pairs(n_source):
    from dig_b200 import ops
    n_target = 100_000                                  # 1e10 target pairs: every pair index past 2^32 is visited
    src = _lengths(n_source, 1.095, 0.02, seed=1).float()
    tgt = _lengths(n_target, 1.09, 0.012, seed=2)
    got = ops.mmd_terms(src.cuda(), tgt.cuda()).tolist()
    want = _restated_terms(src, tgt)
    for name, g, w in zip(("bandwidth", "XX", "YY", "XY"), got, want):
        assert abs(g - w) <= 1e-12 * abs(w), (name, g, w)
    mmd_got, mmd_want = got[1] + got[2] - 2 * got[3], want[1] + want[2] - 2 * want[3]
    assert abs(mmd_got - mmd_want) <= 1e-10, (mmd_got, mmd_want)


@pytest.mark.parametrize("kw", [dict(kernel_num=7), dict(kernel_num=2), dict(kernel_mul=1.5, kernel_num=5),
                                dict(fix_sigma=2e-4)])
def test_other_kernel_settings_match_the_fp64_restatement(kw):
    from dig_b200 import ops
    src, tgt = _lengths(3000, 1.1, 0.03, seed=3), _lengths(5000, 1.09, 0.02, seed=4)
    got = ops.mmd_terms(src.cuda(), tgt.cuda(), **kw).tolist()
    want = _restated_terms(src, tgt, **kw)
    for name, g, w in zip(("bandwidth", "XX", "YY", "XY"), got, want):
        assert abs(g - w) <= 1e-12 * abs(w), (kw, name, g, w)


def test_deterministic_and_permutation_invariant():
    from dig_b200.ggraph3D.utils import compute_mmd
    src, tgt = _lengths(5000, 1.1, 0.03, seed=5).cuda(), _lengths(20000, 1.09, 0.02, seed=6).cuda()
    a, b = compute_mmd(src, tgt), compute_mmd(src, tgt)
    assert a == b                                       # bit-identical: fixed-order reduction, no atomics
    g = torch.Generator().manual_seed(0)
    ps, pt = torch.randperm(src.numel(), generator=g).cuda(), torch.randperm(tgt.numel(), generator=g).cuda()
    assert abs(compute_mmd(src[ps], tgt[pt]) - a) <= 1e-12


def test_symmetry_and_self_distance():
    from dig_b200.ggraph3D.utils import compute_mmd
    a, b = _lengths(3000, 1.1, 0.03, seed=7).cuda(), _lengths(7000, 1.09, 0.02, seed=8).cuda()
    assert abs(compute_mmd(a, b) - compute_mmd(b, a)) <= 1e-12
    assert abs(compute_mmd(a, a)) <= 1e-12


def test_nan_and_error_cases_as_the_reference():
    from dig_b200.ggraph3D.utils import compute_mmd
    x = _lengths(50, 1.1, 0.03, seed=9).cuda()
    assert math.isnan(compute_mmd(x[:0], x))                               # XX = 0 / 0
    assert math.isnan(compute_mmd(torch.full((40,), 1.09, dtype=F64), torch.full((60,), 1.09, dtype=F64)))
    assert math.isnan(compute_mmd(torch.full((1,), 1.09, dtype=F64), torch.full((1,), 1.09, dtype=F64)))
    with pytest.raises(ZeroDivisionError):
        compute_mmd(x, x[:0])


def test_cpu_and_cuda_inputs_agree():
    from dig_b200.ggraph3D.utils import compute_mmd
    src, tgt = _lengths(900, 1.1, 0.03, seed=10).float(), _lengths(4000, 1.09, 0.02, seed=11)
    ref = compute_mmd(src.cuda(), tgt.cuda())
    assert compute_mmd(src, tgt) == ref
    assert compute_mmd(src.cuda(), tgt) == ref
