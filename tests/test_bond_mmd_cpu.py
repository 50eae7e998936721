"""CPU tests of the bond-length MMD: the travelling restatement (oracle/restated_mmd.py) reproduces the reference's
compute_mmd bit for bit on every fixture case, collect_bond_dists reproduces the reference's output exactly, and
compute_mmd has no CPU fallback."""
import json
import math
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN


def _fixture():
    return np.load(os.path.join(GOLDEN, "bond_mmd.npz"))


def fixture_cases():
    f = _fixture()
    for k, meta in enumerate(json.loads(str(f["cases"]))):
        yield meta, f[f"case{k}_source"], f[f"case{k}_target"], float(f[f"case{k}_ref"])


@pytest.fixture
def fixture_threads():
    from oracle import FIXTURE_THREADS
    old = torch.get_num_threads()
    torch.set_num_threads(FIXTURE_THREADS)
    yield
    torch.set_num_threads(old)


def test_fixture_covers_the_cases():
    names = [m["name"] for m, *_ in fixture_cases()]
    for want in ("sizes_1_2", "sizes_127_128", "sizes_128_129", "sizes_1000_4097", "sizes_4097_128", "fix_sigma",
                 "mul3_num4", "num1", "f32_f32", "f32_f64", "f64_f64", "outlier", "qm9_ch", "qm9_cc", "empty_source",
                 "empty_target", "constant"):
        assert want in names
    assert os.path.getsize(os.path.join(GOLDEN, "bond_mmd.npz")) < 1 << 20


def test_restated_compute_mmd_equals_reference_fixture(fixture_threads):
    from oracle import restated_mmd
    for meta, s, t, ref in fixture_cases():
        src, tgt = torch.from_numpy(s), torch.from_numpy(t)
        if meta["outcome"] == "raises":
            with pytest.raises(ZeroDivisionError):
                restated_mmd.compute_mmd(src, tgt, **meta["kwargs"])
            continue
        got = restated_mmd.compute_mmd(src, tgt, **meta["kwargs"])
        if math.isnan(ref):
            assert math.isnan(got), meta["name"]
        else:
            assert got == ref, (meta["name"], got, ref)


def _bond_inputs(f):
    mols = {int(n): {"_atomic_numbers": f[f"mols{n}_z"], "_positions": f[f"mols{n}_pos"]} for n in f["mol_sizes"]}
    valid = [bool(v) for v in f["valid"]]
    cons = [f[f"con{i}"] for i in range(len(valid))]
    return mols, valid, cons


def test_collect_bond_dists_equals_reference_fixture():
    from dig_b200.ggraph3D.utils import collect_bond_dists
    f = _fixture()
    mols, valid, cons = _bond_inputs(f)
    assert not all(valid) and any(valid)
    out = collect_bond_dists(mols, valid, cons)
    assert [tuple(int(x) for x in k) for k in out] == [tuple(k) for k in f["bond_keys"].tolist()]   # keys and order
    assert [len(v) for v in out.values()] == f["bond_counts"].tolist()
    lengths = [x for v in out.values() for x in v]
    assert all(type(x) is np.float32 for x in lengths)
    assert np.array_equal(np.array(lengths, dtype=np.float32).view(np.int32), f["bond_lengths"].view(np.int32))
    assert {int(o) for k in out for o in k[2:]} <= {1, 2, 3}


def test_compute_mmd_has_no_cpu_fallback(monkeypatch):
    from dig_b200.ggraph3D.utils import compute_mmd
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    a = torch.tensor([1.0, 1.1, 1.2], dtype=torch.float64)
    with pytest.raises(RuntimeError, match="CUDA"):
        compute_mmd(a, a + 0.05)


def test_compute_mmd_input_checks():
    from dig_b200.ggraph3D.utils import compute_mmd
    a = torch.tensor([1.0, 1.1, 1.2], dtype=torch.float64)
    with pytest.raises(ZeroDivisionError):                   # as the reference: the target term divides by n_t^2
        compute_mmd(a, a[:0])
    with pytest.raises(TypeError):
        compute_mmd(a.view(3, 1), a)
    with pytest.raises(TypeError):
        compute_mmd(a.long(), a)


def test_public_api_mirrors_the_reference_names():
    import dig_b200.ggraph3D.utils as utils
    assert utils.__all__ == ["collect_bond_dists", "compute_mmd"]
    assert not hasattr(utils, "xyz2mol") and not hasattr(utils, "compute_prop")
