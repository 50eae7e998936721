"""CPU tests of xyz2mol (csrc/xyz2mol.cu / xyz2mol.cuh, dig_b200.ggraph3D.evaluation): the travelling restatement
(oracle/restated_validity.py) reproduces the reference fixture tests/golden/xyz2mol.npz bit for bit and the fixture
covers every branch; the input checks of ops.xyz2mol; no CPU fallback; and a host build of xyz2mol.cuh (the code the
kernel runs) against networkx's matching on random graphs and against the restatement on every fixture molecule."""
import ctypes
import json
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from helpers import ROOT

GOLD = os.path.join(ROOT, "tests", "golden", "xyz2mol.npz")


def fixture():
    return np.load(GOLD)


def fixture_molecules(f=None):
    """-> [(z int64 [n], positions fp64 [n, 3], bo int64 [n, n], valid)] in fixture order."""
    f = fixture() if f is None else f
    z, pos, bo = f["z"], f["pos"], f["bo"]                # each NpzFile access decompresses the array again
    out, a, b = [], 0, 0
    for n, ok in zip(f["n_atoms"].tolist(), f["valid"].tolist()):
        out.append((z[a:a + n], pos[a:a + n], bo[b:b + n * n].reshape(n, n).astype(np.int64), ok))
        a, b = a + n, b + n * n
    return out


def test_restatement_matches_the_fixture():
    from oracle import restated_validity as rv
    for k, (z, pos, bo, ok) in enumerate(fixture_molecules()):
        got, valid = rv.xyz2mol(z, pos)
        assert valid == ok and np.array_equal(got, bo), k


def test_fixture_covers_every_branch():
    from oracle.gen_golden_validity import MIN_COUNTS
    f = fixture()
    counts = json.loads(str(f["counts"]))
    for k, v in MIN_COUNTS.items():
        assert counts[k] >= v, (k, counts[k], v)
    names = json.loads(str(f["source_names"]))
    assert set(names) == {"gsphere", "grown", "idealised", "planted"}
    per_source = np.bincount(f["source"], minlength=len(names))
    assert per_source.min() > 0
    n = f["n_atoms"]
    assert n.min() == 1 and n.max() == 64 and 2 in set(n.tolist())
    assert bool(f["float32"].any())                       # G-SphereNet output keeps its float32 positions
    assert str(f["networkx_version"])


def test_input_checks():
    from dig_b200 import ops
    z, pos = torch.ones(3, 5, dtype=torch.int64), torch.zeros(3, 5, 3)
    with pytest.raises(ValueError, match="1 to 64"):
        ops.xyz2mol(torch.ones(2, 65, dtype=torch.int64), torch.zeros(2, 65, 3))
    with pytest.raises(ValueError, match="1 to 64"):
        ops.xyz2mol(torch.ones(2, 0, dtype=torch.int64), torch.zeros(2, 0, 3))
    with pytest.raises(TypeError, match="integer dtype"):
        ops.xyz2mol(z.double(), pos)
    with pytest.raises(TypeError, match="integer dtype"):
        ops.xyz2mol(z.bool(), pos)
    with pytest.raises(TypeError, match="float32 / float64"):
        ops.xyz2mol(z, pos.half())
    with pytest.raises(TypeError, match="torch.Tensor"):
        ops.xyz2mol(z.numpy(), pos)
    for bad_z, bad_pos in ((z[0], pos), (z, pos[..., :2]), (z, pos[:2]), (z, pos.view(3, 15))):
        with pytest.raises(ValueError, match="expected z"):
            ops.xyz2mol(bad_z, bad_pos)


def test_no_cpu_fallback():
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    from dig_b200 import ops
    from dig_b200.ggraph3D.evaluation import RandGenEvaluator, xyz2mol_batch
    z, pos = torch.tensor([[6, 8]]), torch.tensor([[[0.0, 0, 0], [1.2, 0, 0]]])
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.xyz2mol(z, pos)
    mols = {2: {"_atomic_numbers": z.numpy(), "_positions": pos.numpy()}}
    with pytest.raises(RuntimeError, match="CUDA"):
        xyz2mol_batch(mols)
    with pytest.raises(RuntimeError, match="CUDA"):
        RandGenEvaluator.eval_validity(mols)


def test_empty_mol_dicts_raise_zero_division_like_the_reference():
    from dig_b200.ggraph3D.evaluation import RandGenEvaluator, xyz2mol_batch
    assert xyz2mol_batch({}) == ([], [])
    with pytest.raises(ZeroDivisionError):
        RandGenEvaluator.eval_validity({})


def test_public_names():
    import dig_b200.ggraph3D.evaluation as ev
    import dig_b200.ggraph3D.utils as utils
    assert ev.__all__ == ["RandGenEvaluator", "xyz2mol_batch"]
    assert not hasattr(ev, "PropOptEvaluator")
    assert not hasattr(utils, "xyz2mol")


# ---------------------------------------------------------------------------------------------------- host build
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    cxx = shutil.which(os.environ.get("CXX", "g++")) or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler for the test build of xyz2mol.cuh")
    out = str(tmp_path_factory.mktemp("x2m") / "x2m_host.so")
    res = subprocess.run([cxx, "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", out,
                          os.path.join(ROOT, "tests", "xyz2mol_host.cpp")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lib = ctypes.CDLL(out)
    lib.x2m_host_match.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    lib.x2m_host_xyz2mol.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p,
                                     ctypes.c_void_p]
    lib.x2m_host_xyz2mol.restype = None
    return lib


def host_xyz2mol(lib, z, pos):
    """z [G, n] int64, pos [G, n, 3] fp64 -> (bo int8 [G, n, n], valid int8 [G])."""
    z = np.ascontiguousarray(z, np.int64)
    pos = np.ascontiguousarray(pos, np.float64)
    g, n = z.shape
    bo = np.zeros((g, n, n), np.int8)
    valid = np.zeros(g, np.int8)
    lib.x2m_host_xyz2mol(z.ctypes.data, pos.ctypes.data, g, n, bo.ctypes.data, valid.ctypes.data)
    return bo, valid


def _networkx_matching(n, edges):
    import networkx as nx
    g = nx.Graph()
    g.add_edges_from(sorted(edges))                       # the order get_bonds builds the list in
    return {tuple(sorted(e)) for e in nx.max_weight_matching(g)}


def test_host_build_matching_equals_networkx_on_random_graphs(host_lib):
    """The blossom port picks networkx's matching, not just a maximum one, on dense and sparse random graphs."""
    pytest.importorskip("networkx")
    rng = np.random.default_rng(5)
    for it in range(6000):
        n = int(rng.integers(2, 17)) if it % 10 else int(rng.integers(17, 65))
        p = rng.uniform(0.05, 0.6) if it % 2 else rng.uniform(1.0 / n, 3.5 / n)
        edges = [(i, j) for i in range(n) for j in range(i + 1, n) if rng.random() < p]
        if not edges:
            continue
        adj = np.zeros(n, np.uint64)
        for i, j in edges:
            adj[i] |= np.uint64(1) << np.uint64(j)
            adj[j] |= np.uint64(1) << np.uint64(i)
        mate = np.full(n, -1, np.int8)
        assert host_lib.x2m_host_match(n, adj.ctypes.data, mate.ctypes.data) == 0
        got = {tuple(sorted((i, int(mate[i])))) for i in range(n) if mate[i] >= 0}
        assert got == _networkx_matching(n, edges), (n, edges)


def test_host_build_equals_the_fixture(host_lib):
    mols = fixture_molecules()
    for n in sorted({len(z) for z, _, _, _ in mols}):
        idx = [k for k, m in enumerate(mols) if len(m[0]) == n]
        bo, valid = host_xyz2mol(host_lib, np.stack([mols[k][0] for k in idx]), np.stack([mols[k][1] for k in idx]))
        for r, k in enumerate(idx):
            assert valid[r] == mols[k][3] and np.array_equal(bo[r], mols[k][2]), k


def test_host_build_equals_the_restatement_on_seeded_molecules(host_lib):
    pytest.importorskip("networkx")
    from oracle import gen_golden_validity as gv
    from oracle import restated_validity as rv
    mols = [(z, p) for _, z, p in gv.molecules(seed=3, scale=1, with_gsphere=False)]
    for n in sorted({len(z) for z, _ in mols}):
        group = [m for m in mols if len(m[0]) == n]
        bo, valid = host_xyz2mol(host_lib, np.stack([z for z, _ in group]), np.stack([p for _, p in group]))
        for r, (z, p) in enumerate(group):
            want, ok = rv.xyz2mol(z, p)
            assert valid[r] == ok and np.array_equal(bo[r], want), (z.tolist(), p.tolist())
