"""CPU tests of dig_b200.ggraph3D.dataset: the SDF reader on handwritten records, the dataset's files, indexing and
errors, collate_fn against the reference's on the fixture (tests/golden/qm93dgen.npz, oracle/gen_golden_qm93dgen.py),
and the host restatement of get() (oracle/restated_qm93dgen.py) against the fixture bit for bit."""
import os
import sys

import numpy as np
import pytest
import torch

from helpers import GOLDEN

FIELDS = ("atom_type", "position", "batch", "focus", "c1_focus", "c2_c1_focus", "new_atom_type", "new_dist",
          "new_angle", "new_torsion", "cannot_focus")
SHAPES = {"position": (-1, 3), "focus": (-1, 1), "c1_focus": (-1, 2), "c2_c1_focus": (-1, 3), "new_dist": (-1, 1),
          "new_angle": (-1, 1), "new_torsion": (-1, 1)}


def fixture():
    return dict(np.load(os.path.join(GOLDEN, "qm93dgen.npz")))


def fixture_molecules(fx):
    """[(atom_type, position, con_mat)] of the fixture's inputs."""
    n = fx["n_atoms"]
    a = np.concatenate([[0], np.cumsum(n)])
    c = np.concatenate([[0], np.cumsum(n * n)])
    return [(fx["in_atom_type"][a[i]:a[i + 1]], fx["in_position"][a[i]:a[i + 1]],
             fx["in_con_mat"][c[i]:c[i + 1]].reshape(n[i], n[i])) for i in range(len(n))]


def fixture_dicts(fx):
    """The reference's get() dict of every fixture molecule."""
    offs = {k: np.concatenate([[0], np.cumsum(fx["lens_" + k])]) for k in FIELDS}
    return [{k: torch.from_numpy(fx[k][offs[k][i]:offs[k][i + 1]]).reshape(SHAPES.get(k, (-1,))) for k in FIELDS}
            for i in range(len(fx["n_atoms"]))]


def same(a, b):
    """Equal dtype, shape and values (NaN where the other has NaN)."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.is_floating_point():
        return torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(torch.nan_to_num(a), torch.nan_to_num(b))
    return torch.equal(a, b)


def test_sdf_reader_on_handwritten_records():
    from dig_b200.ggraph3D.dataset.ggraph3D_dataset import read_sdf
    mols = read_sdf(os.path.join(GOLDEN, "qm93dgen_records.sdf"))
    assert len(mols) == 4
    t, p, c = mols[0]                                   # CH4, carbon first: kept as written
    assert t.tolist() == [1, 0, 0, 0, 0] and t.dtype == np.int64
    assert p.dtype == np.float32 and p[0].tolist() == np.float32([-0.0127, 1.0858, 0.0080]).tolist()
    assert c.dtype == np.int64 and c[0].tolist() == [0, 1, 1, 1, 1] and c[1:, 1:].sum() == 0
    t, p, c = mols[1]                                   # water: no carbon, so no swap
    assert t.tolist() == [3, 0, 0] and c.tolist() == [[0, 1, 1], [1, 0, 0], [1, 0, 0]]
    t, p, c = mols[2]                                   # N#C-CH3 written N first: N and the first carbon swap
    assert t.tolist() == [1, 2, 1, 0, 0, 0]
    assert p[0].tolist() == np.float32([1.15, 0, 0]).tolist() and p[1].tolist() == np.float32([2.3, 0, 0]).tolist()
    assert c.tolist() == [[0, 3, 1, 0, 0, 0], [3, 0, 0, 0, 0, 0], [1, 0, 0, 1, 1, 1],
                          [0, 0, 1, 0, 0, 0], [0, 0, 1, 0, 0, 0], [0, 0, 1, 0, 0, 0]]
    t, p, c = mols[3]                                   # O=CH2 written O first, bond listed C -> O
    assert t.tolist() == [1, 3, 0, 0]
    assert c.tolist() == [[0, 2, 1, 1], [2, 0, 0, 0], [1, 0, 0, 0], [1, 0, 0, 0]]
    assert p[2].tolist() == np.float32([0.0, 0.943, -0.587]).tolist()


def test_sdf_reader_rejects_what_the_reference_cannot_map(tmp_path):
    from dig_b200.ggraph3D.dataset.ggraph3D_dataset import read_sdf
    with open(os.path.join(GOLDEN, "qm93dgen_records.sdf")) as fh:
        text = fh.read()
    bad = tmp_path / "s.sdf"
    bad.write_text(text.replace(" O   0", " S   0", 1))
    with pytest.raises(ValueError, match="element 'S'"):
        read_sdf(str(bad))
    bad.write_text(text.replace("  1  2  1  0", "  1  2  4  0", 1))
    with pytest.raises(ValueError, match="bond type 4"):
        read_sdf(str(bad))


def _root(tmp_path, sdf=True):
    raw = tmp_path / "raw"
    raw.mkdir()
    if sdf:
        (raw / "gdb9.sdf").write_text(open(os.path.join(GOLDEN, "qm93dgen_records.sdf")).read())
    return str(tmp_path)


def test_dataset_files_indexing_and_split(tmp_path):
    from dig_b200.ggraph3D.dataset import QM93DGEN
    from dig_b200.ggraph3D.dataset.ggraph3D_dataset import read_sdf
    root = _root(tmp_path)
    ds = QM93DGEN(root=root)
    saved = torch.load(os.path.join(root, "processed", "data.pt"))          # the reference's format: three lists
    assert isinstance(saved, tuple) and len(saved) == 3 and all(isinstance(x, list) for x in saved)
    for (t, p, c), a, b, d in zip(read_sdf(ds.raw_paths[0]), *saved):
        assert torch.equal(a, torch.tensor(t)) and torch.equal(b, torch.tensor(p)) and torch.equal(d, torch.tensor(c))
    # a second instance loads data.pt instead of reading the SDF again
    (tmp_path / "raw" / "gdb9.sdf").write_text("")
    ds = QM93DGEN(root=root)
    assert len(ds) == 4 and ds.len() == 4
    sub = ds[[3, 1]]
    assert isinstance(sub, QM93DGEN) and len(sub) == 2 and list(sub.indices()) == [3, 1]
    assert list(ds[1:3].indices()) == [1, 2] and list(ds[torch.tensor([0, 2])].indices()) == [0, 2]
    assert list(ds[np.array([False, True, False, True])].indices()) == [1, 3]
    assert list(sub[[1]].indices()) == [1]
    assert sub._cache is ds._cache                       # subsets share the trajectory cache
    np.savez(tmp_path / "raw" / "split.npz", train_idx=np.array([2, 0, 3]), val_idx=np.array([1]))
    np.savez(tmp_path / "raw" / "gap.npz", train_idx=np.array([1]), val_idx=np.array([0]))
    assert ds.get_idx_split("rand_gen") == {"train": [2, 0, 3], "valid": [1]}
    assert ds.get_idx_split("gap_opt") == {"train": [1], "valid": [0]}
    with pytest.raises(AssertionError):
        ds.get_idx_split("homo")
    assert QM93DGEN(root=root, subset_idxs=[2]).indices() == [2]


def test_missing_raw_file_raises_and_downloads_nothing(tmp_path):
    from dig_b200.ggraph3D.dataset import QM93DGEN
    root = _root(tmp_path, sdf=False)
    with pytest.raises(FileNotFoundError, match="does not download"):
        QM93DGEN(root=root)
    assert sorted(os.listdir(os.path.join(root, "raw"))) == []


def test_collate_fn_matches_the_reference():
    from dig_b200.ggraph3D.dataset import collate_fn
    from oracle.gen_golden_qm93dgen import COLLATE_BATCHES
    fx = fixture()
    dicts = fixture_dicts(fx)
    for b, idx in enumerate(COLLATE_BATCHES):
        got = collate_fn([dicts[i] for i in idx])
        assert set(got) == set(FIELDS)
        for k in FIELDS:
            want = torch.from_numpy(fx[f"collate{b}_{k}"])
            assert same(got[k], want), (b, k)


def test_restatement_matches_the_reference_bit_for_bit():
    from oracle import restated_qm93dgen as rq
    fx = fixture()
    for i, ((t, p, c), want) in enumerate(zip(fixture_molecules(fx), fixture_dicts(fx))):
        got = rq.get(t, p, c, atan2="libm")
        for k in FIELDS:
            assert same(got[k], want[k]), (i, k)
    for t, p, c in __import__("oracle.gen_golden_qm93dgen", fromlist=["RAISING"]).RAISING:
        with pytest.raises(ValueError):
            rq.get(t, p, c)


def test_fixture_covers_the_planted_cases():
    fx = fixture()
    tags = set(fx["tag"].tolist())
    assert {"grown", "lattice", "collinear", "coplanar", "coincident", "first_not_carbon", "coincident_focus_c1"} <= tags
    assert fx["n_atoms"].min() == 2 and fx["n_atoms"].max() == 29
    assert np.isnan(fx["new_torsion"]).sum() == 1 and not np.isnan(fx["new_angle"]).any()


def test_trajectories_are_not_computed_inside_loader_workers(tmp_path, monkeypatch):
    """A DataLoader worker that finds no computed trajectories raises instead of starting CUDA in a forked process."""
    from dig_b200.ggraph3D.dataset import QM93DGEN
    ds = QM93DGEN(root=_root(tmp_path))
    monkeypatch.setattr(torch.utils.data, "get_worker_info", lambda: object())
    with pytest.raises(RuntimeError, match="dataset.trajectories\\(\\) in the main process"):
        ds[0]


@pytest.mark.reference
def test_reference_example_imports_resolve_with_dig_aliased():
    """examples/ggraph3D/G_SphereNet/run_rand_gen.py's imports, with `dig` served by dig_b200 (INTEGRATION.md)."""
    import ast
    import importlib
    from oracle.ref_loader import REFERENCE_ROOT
    import dig_b200
    path = os.path.join(REFERENCE_ROOT, "examples", "ggraph3D", "G_SphereNet", "run_rand_gen.py")
    with open(path) as fh:
        tree = ast.parse(fh.read())
    saved = {k: v for k, v in sys.modules.items() if k == "dig" or k.startswith("dig.")}
    try:
        for k in saved:
            del sys.modules[k]
        sys.modules["dig"] = dig_b200
        for sub in ("ggraph3D", "ggraph3D.dataset", "ggraph3D.method", "ggraph3D.evaluation"):
            sys.modules["dig." + sub] = importlib.import_module("dig_b200." + sub)
        seen = 0
        for node in ast.walk(tree):
            if isinstance(node, ast.ImportFrom) and node.module and node.module.startswith("dig."):
                mod = importlib.import_module(node.module)
                for alias in node.names:
                    assert hasattr(mod, alias.name), (node.module, alias.name)
                    seen += 1
        assert seen == 4                    # QM93DGEN, collate_fn, G_SphereNet, RandGenEvaluator
    finally:
        for k in [k for k in sys.modules if k == "dig" or k.startswith("dig.")]:
            del sys.modules[k]
        sys.modules.update(saved)
