"""Writes tests/golden/qm93dgen.npz from the UNMODIFIED reference dig/ggraph3D/dataset/ggraph3D_dataset.py
(QM93DGEN.get, collate_fn), loaded by file path with rdkit stubbed (get and collate_fn never call it), torch_geometric
from oracle/shim.py and nx.from_numpy_matrix aliased to nx.from_numpy_array (networkx 3 removed it).  get runs on an
instance built without __init__ that holds synthetic QM9-shaped molecules (`molecules(seed)`):
  * grown molecules of 2 to 29 atoms with QM9's element frequencies, bonds of order 1-3 between close atoms;
  * integer-lattice coordinates (exact distance ties for the spanning tree and for c1 / c2);
  * collinear and coplanar molecules, a molecule with two coincident atoms, first atoms other than carbon, and one
    whose focus and c1 coincide at a torsion step (NaN torsion).
One atom and three coincident atoms are recorded as raising.  Every dict is also checked against
oracle/restated_qm93dgen.py (atan2="libm") bit for bit.  collate_fn is run on three lists of the dicts.

    python -m oracle.gen_golden_qm93dgen          (needs the reference checkout, see oracle/ref_loader.py)
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

from oracle import restated_qm93dgen as rq
from oracle.ref_loader import REFERENCE_ROOT

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
FIELDS = ("atom_type", "position", "batch", "focus", "c1_focus", "c2_c1_focus", "new_atom_type", "new_dist",
          "new_angle", "new_torsion", "cannot_focus")
QM9_P = np.array([0.510, 0.351, 0.056, 0.078, 0.005])       # H, C, N, O, F as type ids 0-4
COLLATE_BATCHES = ([0, 1, 2], list(range(10, 40)), [7])


def load_reference_dataset():
    """-> the reference's ggraph3D_dataset module over the stand-ins."""
    from oracle import shim
    import networkx as nx
    shim.install()
    data = sys.modules["torch_geometric.data"]
    if not hasattr(data, "extract_tar"):
        def extract_tar(*a, **k):
            raise RuntimeError("no network")
        data.extract_tar = extract_tar
    if not hasattr(nx, "from_numpy_matrix"):
        nx.from_numpy_matrix = nx.from_numpy_array
    chem = types.ModuleType("rdkit.Chem")
    rdchem = types.ModuleType("rdkit.Chem.rdchem")
    rdchem.BondType = types.SimpleNamespace(SINGLE="SINGLE", DOUBLE="DOUBLE", TRIPLE="TRIPLE")
    chem.rdchem = rdchem
    rdkit = types.ModuleType("rdkit")
    rdkit.Chem = chem
    sys.modules.update({"rdkit": rdkit, "rdkit.Chem": chem, "rdkit.Chem.rdchem": rdchem})
    path = os.path.join(REFERENCE_ROOT, "dig", "ggraph3D", "dataset", "ggraph3D_dataset.py")
    if not os.path.isfile(path):
        raise RuntimeError(f"reference file not found: {path}")
    spec = importlib.util.spec_from_file_location("ref_ggraph3D_dataset", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _bonds(pos, rng, cutoff=1.65):
    n = len(pos)
    d = np.linalg.norm(pos[:, None].astype(np.float64) - pos[None].astype(np.float64), axis=-1)
    con = np.zeros((n, n), dtype=np.int64)
    for i in range(n):
        for j in range(i + 1, n):
            if 0 < d[i, j] < cutoff:
                con[i, j] = con[j, i] = rng.choice([1, 1, 1, 2, 3])
    return con


def grown(rng, n):
    pos = np.zeros((n, 3))
    for k in range(1, n):
        v = rng.standard_normal(3)
        pos[k] = pos[rng.integers(k)] + v / np.linalg.norm(v) * rng.uniform(0.95, 1.6)
    return pos.astype(np.float32)


def molecules(seed=0, n_random=360):
    """[(atom_type int64 [n], position float32 [n, 3], con_mat int64 [n, n], tag)], seeded."""
    rng = np.random.default_rng(seed)
    out = []

    def add(pos, tag, types_=None):
        pos = np.asarray(pos, dtype=np.float32)
        n = len(pos)
        t = rng.choice(5, size=n, p=QM9_P) if types_ is None else np.asarray(types_)
        out.append((t.astype(np.int64), pos, _bonds(pos, rng), tag))

    for k in range(n_random):
        n = 2 + k % 28
        add(grown(rng, n), "grown")
    for n in (4, 7, 12, 20, 29):
        for _ in range(6):
            cells = rng.choice(27, size=n, replace=False) if n <= 27 else rng.choice(64, size=n, replace=False)
            side = 3 if n <= 27 else 4
            add(np.stack([cells // side ** 2, (cells // side) % side, cells % side], 1) * 1.0, "lattice")
    for n in (3, 5, 9):
        add(np.outer(np.arange(n) * 1.25 + rng.uniform(0, 0.1, n), [1.0, 0.0, 0.0]), "collinear")
        add(np.outer(rng.permutation(n) * 1.5, [0.6, 0.8, 0.0]), "collinear")
    for n in (4, 8, 15):
        p = grown(rng, n)
        p[:, 2] = 0
        add(p, "coplanar")
    p = grown(rng, 6)
    p[4] = p[1]
    add(p, "coincident")
    for first in (0, 2, 3, 4):
        add(grown(rng, 8), "first_not_carbon", types_=[first] + list(rng.choice(5, size=7, p=QM9_P)))
    # atom 2 sits on atom 0 (no tree edge between them): the order is 0, 1, 2, 3, and at step 2 the focus of atom 3 is
    # atom 0 and its c1 is atom 2, so the torsion's |focus - c1| is 0 and the torsion is 0 / 0 = NaN
    add([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 0.0], [0.0, 1.2, 0.0]], "coincident_focus_c1")
    return out


RAISING = ((np.zeros(1, np.int64), np.zeros((1, 3), np.float32), np.zeros((1, 1), np.int64)),
           (np.ones(3, np.int64), np.full((3, 3), 0.5, np.float32), np.zeros((3, 3), np.int64)))


def pack(dicts, prefix=""):
    """Concatenate the dicts' fields; lens_<field> holds each dict's row count."""
    out = {}
    for k in FIELDS:
        out[prefix + k] = np.concatenate([d[k].numpy() for d in dicts])
        out[prefix + "lens_" + k] = np.array([len(d[k]) for d in dicts], dtype=np.int64)
    return out


def main():
    ref = load_reference_dataset()
    mols = molecules()
    ds = ref.QM93DGEN.__new__(ref.QM93DGEN)
    ds.atom_type_list = [torch.tensor(t) for t, _, _, _ in mols]
    ds.position_list = [torch.tensor(p) for _, p, _, _ in mols]
    ds.con_mat_list = [torch.tensor(c) for _, _, c, _ in mols]
    dicts = [ds.get(i) for i in range(len(mols))]
    for i, (d, (t, p, c, _)) in enumerate(zip(dicts, mols)):
        r = rq.get(t, p, c, atan2="libm")
        assert set(d) == set(FIELDS) == set(r), i
        for k in FIELDS:
            assert d[k].dtype == r[k].dtype and d[k].shape == r[k].shape, (i, k, d[k].dtype, r[k].dtype)
            assert torch.equal(torch.nan_to_num(d[k]), torch.nan_to_num(r[k])), (i, k)
            assert torch.equal(torch.isnan(d[k]) if d[k].is_floating_point() else d[k] * 0,
                               torch.isnan(r[k]) if r[k].is_floating_point() else r[k] * 0), (i, k)
    for t, p, c in RAISING:
        dr = ref.QM93DGEN.__new__(ref.QM93DGEN)
        dr.atom_type_list, dr.position_list, dr.con_mat_list = [torch.tensor(t)], [torch.tensor(p)], [torch.tensor(c)]
        try:
            dr.get(0)
        except ValueError:
            pass
        else:
            raise AssertionError("expected the reference's get to raise")
    arrays = {"n_atoms": np.array([len(t) for t, _, _, _ in mols], dtype=np.int64),
              "in_atom_type": np.concatenate([t for t, _, _, _ in mols]),
              "in_position": np.concatenate([p for _, p, _, _ in mols]),
              "in_con_mat": np.concatenate([c.reshape(-1) for _, _, c, _ in mols]),
              "tag": np.array([tag for _, _, _, tag in mols])}
    arrays.update(pack(dicts))
    for b, idx in enumerate(COLLATE_BATCHES):
        batch = ref.collate_fn([dicts[i] for i in idx])
        for k in FIELDS:
            arrays[f"collate{b}_{k}"] = batch[k].numpy()
    os.makedirs(GOLDEN, exist_ok=True)
    path = os.path.join(GOLDEN, "qm93dgen.npz")
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {len(mols)} molecules, {len(arrays['atom_type'])} trajectory rows, "
          f"{int(np.isnan(arrays['new_torsion']).sum())} NaN torsions")
    assert np.isnan(arrays["new_torsion"]).any()


if __name__ == "__main__":
    main()
