"""Writes tests/golden/xyz2mol.npz from the UNMODIFIED reference dig/ggraph3D/utils/eval_validity_utils.py (xyz2mol)
and dig/ggraph3D/evaluation/metric.py (RandGenEvaluator), loaded by file path over a small RDKit stand-in: on this path
RDKit only holds the atomic numbers and a conformer, the logic is numpy, scipy and networkx.

Molecule sources (all seeded; `molecules(seed, scale)` re-creates them for the GPU tests):
  * idealised molecules built from ring / chain templates (benzene, pyridine, pyrimidine, pyrrole, furan, imidazole,
    cyclopentadiene, fulvene, a fused 5-7 ring system, propyne, acetonitrile, CO2, formic and acetic acid, formamide,
    small saturated molecules, bare carbon rings of 3 to 9 atoms), randomly rotated, bare and with 0.02 / 0.05 / 0.1 A Gaussian noise;
  * grown geometries: each atom 0.95-1.8 A (or 0.8-1.0 times the bond threshold) from a random earlier one, elements
    with QM9's frequencies;
  * G-SphereNet output of the fixture weights (oracle/restated_gsphere.py, seeded draws), float32 positions;
  * planted cases: n = 1 and 2, F, elements 0 and 16, an atom j with five candidate partners (the greedy cap binds),
    pairs 1e-6 A and one ulp either side of every threshold, and n = 64.
Every molecule is checked against oracle/restated_validity.py bit for bit, and the branch counts are asserted.
RandGenEvaluator.eval_validity / eval_bond_mmd are run on one mol_dicts against a subsample of the shipped QM9
bond-length table.

    python -m oracle.gen_golden_validity          (needs the reference checkout, see oracle/ref_loader.py)
"""
import contextlib
import importlib.util
import io
import json
import os
import sys
import types

import numpy as np
import torch

from oracle import FIXTURE_THREADS
from oracle import restated_validity as rv
from oracle.ref_loader import REFERENCE_ROOT

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
QM9_ELEMENTS = (np.array([1, 6, 7, 8, 9]), np.array([0.510, 0.351, 0.056, 0.078, 0.005]))
BOND_TYPES = [(1, 8, 1), (1, 7, 1), (6, 7, 1), (6, 8, 1), (6, 6, 1), (1, 6, 1)]
MIN_COUNTS = dict(disconnected=50, over_valence=30, unknown_element=10, no_ua=50, bo_ok=200, bo_not_ok=50,
                  two_rounds=20, odd_cycle=50, multiple_maximum=300)


# ---------------------------------------------------------------------------------------------------- RDKit stand-in
def install_rdkit_standin():
    """rdkit.Chem with what get_proto_mol / xyz2AC_vdW call: MolFromSmarts("[#z]"), RWMol, Atom, Conformer."""
    class Atom:
        def __init__(self, z):
            self._z = int(z)

        def GetAtomicNum(self):
            return self._z

    class Mol:
        def __init__(self, atoms=()):
            self._atoms = list(atoms)
            self._conformers = []

        def GetNumAtoms(self):
            return len(self._atoms)

        def GetAtomWithIdx(self, i):
            return self._atoms[i]

        def AddConformer(self, conf):
            self._conformers.append(conf)

    class RWMol(Mol):
        def __init__(self, mol):
            super().__init__(mol._atoms)

        def AddAtom(self, atom):
            self._atoms.append(atom)

        def GetMol(self):
            return Mol(self._atoms)

    class Conformer:
        def __init__(self, n):
            self._pos = [None] * n

        def SetAtomPosition(self, i, p):
            self._pos[i] = p

    def mol_from_smarts(s):
        assert s.startswith("[#") and s.endswith("]"), s
        return Mol([Atom(int(s[2:-1]))])

    chem = types.ModuleType("rdkit.Chem")
    chem.Atom, chem.RWMol, chem.Conformer, chem.MolFromSmarts = Atom, RWMol, Conformer, mol_from_smarts
    rdkit = types.ModuleType("rdkit")
    rdkit.Chem = chem
    sys.modules["rdkit"], sys.modules["rdkit.Chem"] = rdkit, chem


def _load(name, *parts):
    path = os.path.join(REFERENCE_ROOT, *parts)
    if not os.path.isfile(path):
        raise RuntimeError(f"reference file not found: {path}")
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_reference_validity():
    """-> (eval_validity_utils module, metric module) of the reference, over the stand-in; metric.py's
    `from dig.ggraph3D.utils import ...` is served by a stand-in package holding the reference's own functions
    (compute_prop, PySCF, is a stub that raises)."""
    from oracle.gen_golden_mmd import load_reference_bond_mmd
    install_rdkit_standin()
    vu = _load("ref_eval_validity_utils", "dig", "ggraph3D", "utils", "eval_validity_utils.py")
    mmd = load_reference_bond_mmd()
    utils = types.ModuleType("dig.ggraph3D.utils")
    utils.xyz2mol, utils.collect_bond_dists, utils.compute_mmd = vu.xyz2mol, mmd.collect_bond_dists, mmd.compute_mmd

    def compute_prop(*a, **k):
        raise NotImplementedError("compute_prop needs PySCF")
    utils.compute_prop = compute_prop
    saved = {k: sys.modules.get(k) for k in ("dig", "dig.ggraph3D", "dig.ggraph3D.utils")}
    sys.modules["dig"] = types.ModuleType("dig")
    sys.modules["dig.ggraph3D"] = types.ModuleType("dig.ggraph3D")
    sys.modules["dig.ggraph3D.utils"] = utils
    try:
        metric = _load("ref_ggraph3d_metric", "dig", "ggraph3D", "evaluation", "metric.py")
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return vu, metric


# ---------------------------------------------------------------------------------------------------- molecule sources
def _rotation(rng):
    q, r = np.linalg.qr(rng.standard_normal((3, 3)))
    return q * np.sign(np.diag(r))


def _ring(k, length):
    r = length / (2 * np.sin(np.pi / k))
    a = 2 * np.pi * np.arange(k) / k
    return np.stack([r * np.cos(a), r * np.sin(a), np.zeros(k)], axis=1)


def _radial_h(p, center, length=1.08):
    u = p - center
    return p + length * u / np.linalg.norm(u)


def _ch2(p, center, length=1.09):
    u = (p - center) / np.linalg.norm(p - center)
    up = np.array([0.0, 0.0, 1.0])
    return [p + length * (0.55 * u + 0.835 * up), p + length * (0.55 * u - 0.835 * up)]


def _ring_molecule(elements, length, h_on, ch2_at=()):
    pos = _ring(len(elements), length)
    z, out = list(elements), list(pos)
    for i in range(len(elements)):
        if i in ch2_at:
            for h in _ch2(pos[i], np.zeros(3)):
                z.append(1)
                out.append(h)
        elif i in h_on:
            z.append(1)
            out.append(_radial_h(pos[i], np.zeros(3), 1.01 if elements[i] == 7 else 1.08))
    return z, np.array(out)


def _chain(elements, lengths, end_h=(), methyl=()):
    """Linear heavy-atom chain along x; end_h: indices with one H continuing the line; methyl: indices with three H."""
    x = np.concatenate([[0.0], np.cumsum(lengths)])
    z, pos = list(elements), [np.array([xi, 0.0, 0.0]) for xi in x]
    for i in end_h:
        z.append(1)
        pos.append(pos[i] + np.array([1.06 if i else -1.06, 0.0, 0.0]))
    for i in methyl:
        s = 1.0 if i else -1.0
        for phi in (0.0, 2.0944, 4.18879):
            z.append(1)
            pos.append(pos[i] + 1.09 * np.array([s * 0.334, 0.943 * np.cos(phi), 0.943 * np.sin(phi)]))
    return z, np.array(pos)


def _planar(atoms):
    """atoms: [(z, x, y)] -> (z list, positions in the plane z = 0)."""
    return [a[0] for a in atoms], np.array([[a[1], a[2], 0.0] for a in atoms])


def _fused_5_7():
    seven = _ring(7, 1.40)
    a, b = seven[0], seven[1]
    mid, edge = (a + b) / 2, b - a
    out = mid / np.linalg.norm(mid)                       # the 5-ring lies outside the 7-ring, across edge a-b
    r5 = 1.40 / (2 * np.sin(np.pi / 5))
    c5 = mid + out * r5 * np.cos(np.pi / 5)
    ang0 = np.arctan2(*(a - c5)[[1, 0]])
    sgn = 1 if np.cross(a - c5, b - c5)[2] > 0 else -1
    five = [c5 + r5 * np.array([np.cos(ang0 + sgn * 2 * np.pi * k / 5), np.sin(ang0 + sgn * 2 * np.pi * k / 5), 0.0])
            for k in range(5)]
    heavy = list(seven) + five[2:]
    z, pos = [6] * len(heavy), list(heavy)
    for i in range(2, 7):
        z.append(1)
        pos.append(_radial_h(seven[i], np.zeros(3)))
    for p in five[2:]:
        z.append(1)
        pos.append(_radial_h(p, c5))
    return z, np.array(pos)


def idealised_templates():
    t = {}
    t["benzene"] = _ring_molecule([6] * 6, 1.39, range(6))
    t["pyridine"] = _ring_molecule([7, 6, 6, 6, 6, 6], 1.38, range(1, 6))
    t["pyrimidine"] = _ring_molecule([7, 6, 7, 6, 6, 6], 1.37, (1, 3, 4, 5))
    t["pyrrole"] = _ring_molecule([7, 6, 6, 6, 6], 1.38, range(5))
    t["furan"] = _ring_molecule([8, 6, 6, 6, 6], 1.38, range(1, 5))
    t["imidazole"] = _ring_molecule([7, 6, 7, 6, 6], 1.36, (0, 1, 3, 4))
    t["cyclopentadiene"] = _ring_molecule([6] * 5, 1.44, (1, 2, 3, 4), ch2_at=(0,))
    z, pos = _ring_molecule([6] * 5, 1.44, (1, 2, 3, 4))
    c = pos[0] * (1 + 1.35 / np.linalg.norm(pos[0]))
    t["fulvene"] = (z + [6, 1, 1], np.vstack([pos, c, c + [0.55, 0.93, 0.0], c + [0.55, -0.93, 0.0]]))
    t["fused_5_7"] = _fused_5_7()
    t["propyne"] = _chain([6, 6, 6], [1.20, 1.46], end_h=(0,), methyl=(2,))
    t["acetonitrile"] = _chain([7, 6, 6], [1.16, 1.46], methyl=(2,))
    t["co2"] = _chain([8, 6, 8], [1.16, 1.16])
    t["hcn"] = _chain([1, 6, 7], [1.07, 1.16])
    t["formic_acid"] = _planar([(6, 0, 0), (8, 1.20, 0.05), (8, -0.67, 1.13), (1, -0.55, -0.93), (1, -0.1, 1.85)])
    t["acetic_acid"] = _planar([(6, 0, 0), (8, 1.21, 0.0), (8, -0.66, 1.15), (1, -0.05, 1.85), (6, -0.75, -1.30),
                                (1, -1.83, -1.10), (1, -0.50, -1.90), (1, -0.40, -1.75)])
    t["formamide"] = _planar([(6, 0, 0), (8, 1.22, 0.0), (7, -0.68, 1.17), (1, -0.55, -0.94), (1, -1.68, 1.20),
                              (1, -0.17, 2.04)])
    t["ethene"] = _planar([(6, 0, 0), (6, 1.33, 0), (1, -0.56, 0.93), (1, -0.56, -0.93), (1, 1.89, 0.93),
                           (1, 1.89, -0.93)])
    t["ethane"] = _chain([6, 6], [1.53], methyl=(0, 1))
    t["methanol"] = _chain([6, 8], [1.43], methyl=(0,))
    t["methylamine"] = _chain([6, 7], [1.47], methyl=(0,))
    t["fluoromethane"] = _chain([9, 6], [1.35], methyl=(1,))
    t["water"] = _planar([(8, 0, 0), (1, 0.96, 0), (1, -0.24, 0.93)])
    t["formaldehyde"] = _planar([(6, 0, 0), (8, 1.21, 0), (1, -0.55, 0.94), (1, -0.55, -0.94)])
    t["azide_like"] = _chain([7, 7, 7], [1.13, 1.13])
    t["nitroso"] = _planar([(7, 0, 0), (8, 1.21, 0), (1, -0.35, 0.96)])
    t["methane"] = ([6, 1, 1, 1, 1], np.array([[0, 0, 0], [0.63, 0.63, 0.63], [-0.63, -0.63, 0.63], [-0.63, 0.63, -0.63],
                                              [0.63, -0.63, -0.63]]))
    t["ammonia"] = ([7, 1, 1, 1], np.array([[0, 0, 0], [0.94, 0, -0.38], [-0.47, 0.81, -0.38], [-0.47, -0.81, -0.38]]))
    for k in (3, 5, 7, 9):                                # bare carbon rings: odd cycles in the unsaturated graph
        t[f"c{k}_ring"] = ([6] * k, _ring(k, 1.40))
    return t


def idealised(rng, replicas):
    out = []
    for name, (z, pos) in idealised_templates().items():
        for noise in (0.0, 0.02, 0.05, 0.1):
            for _ in range(replicas):
                p = (pos - pos.mean(axis=0)) @ _rotation(rng).T + rng.standard_normal(3)
                out.append((np.array(z, np.int64), p + noise * rng.standard_normal(p.shape)))
    return out


def grown(rng, count, n_range=(2, 30), bonded=False):
    """Each atom 0.95-1.8 A from a random earlier one; bonded: 0.8-1.0 times the pair's threshold where it has one."""
    out = []
    for _ in range(count):
        n = int(rng.integers(*n_range))
        z = rng.choice(QM9_ELEMENTS[0], size=n, p=QM9_ELEMENTS[1] / QM9_ELEMENTS[1].sum())
        pos = np.zeros((n, 3))
        for k in range(1, n):
            u = rng.standard_normal(3)
            parent = rng.integers(k)
            thr = rv.THRESHOLD.get((min(z[k], z[parent]), max(z[k], z[parent])))
            r = rng.uniform(0.8, 1.0) * thr if bonded and thr else rng.uniform(0.95, 1.8)
            pos[k] = pos[parent] + r * u / np.linalg.norm(u)
        out.append((z.astype(np.int64), pos))
    return out


def gsphere(seed, num_gen, max_atoms=35):
    """G-SphereNet molecules of the fixture weights through the restated generator: [(z, float32 positions)]."""
    from oracle import restated_gsphere as rg
    with open(os.path.join(GOLDEN, "gsphere_state_shapes.json")) as fh:
        sd = rg.gsphere_state_dict({k: torch.empty(v) for k, v in json.load(fh).items()})
    with torch.no_grad():
        mols = rg.generate(sd, rg.SeededDraws(seed), np.array([1, 6, 7, 8, 9]), num_gen=num_gen,
                           temperature=(0.5, 0.3, 0.4, 1.0), min_atoms=2, max_atoms=max_atoms)
    return [(z.astype(np.int64), p) for n in mols for z, p in zip(mols[n]["_atomic_numbers"], mols[n]["_positions"])]


def planted(rng):
    out = []

    def add(z, pos):
        out.append((np.array(z, np.int64), np.array(pos, np.float64).reshape(-1, 3)))
    for z in (1, 6, 7, 8, 9, 0, 16, 35, 2, 3, 5, 14, 15, 17, 53, -1, 118):
        add([z], [0, 0, 0])
    for pair, d in ((6, 8), 1.2), ((1, 1), 0.74), ((9, 9), 1.42), ((6, 16), 1.8), ((0, 6), 1.0), ((1, 9), 0.92), \
            ((6, 8), 2.0), ((7, 7), 1.1):
        add(pair, [[0, 0, 0], [d, 0, 0]])
    add([6, 9, 9, 9, 9], [[0, 0, 0], [1.35, 0, 0], [-0.45, 1.27, 0], [-0.45, -0.64, 1.1], [-0.45, -0.64, -1.1]])
    add([6, 16, 1, 1], [[0, 0, 0], [1.8, 0, 0], [-0.5, 0.9, 0], [-0.5, -0.9, 0]])
    add([0, 6, 1], [[0, 0, 0], [1.0, 0, 0], [2.0, 0, 0]])
    # five candidate partners of one j: only the first four bond (then the molecule is disconnected)
    ring5 = [[np.cos(a), np.sin(a), 0.3] for a in 2 * np.pi * np.arange(5) / 5]
    add([6, 1, 1, 1, 1, 1], [[0, 0, 0]] + ring5)
    add([6, 6, 6, 6, 6, 6], [[0, 0, 0]] + [[1.5 * c for c in p] for p in ring5])
    # an i with five earlier partners: i is not capped, the molecule is over-valent
    add([1, 1, 1, 1, 1, 6], ring5 + [[0, 0, 0]])
    add([1, 1, 1, 1, 1, 7], ring5 + [[0, 0, 0]])
    # every threshold: 1e-6 and one ulp either side, and the value itself, along the x axis and rotated
    for (a, b), thr in rv.THRESHOLD.items():
        for d in (thr - 1e-6, thr + 1e-6, thr, np.nextafter(thr, 0), np.nextafter(thr, 2)):
            add([a, b], [[0, 0, 0], [d, 0, 0]])
            add([b, a], [[0.25, -0.5, 0.125], [0.25 + d, -0.5, 0.125]])
            u = rng.standard_normal(3)
            p0 = rng.standard_normal(3)
            add([a, b], [p0, p0 + d * u / np.linalg.norm(u)])
            add([a, 6, b], [p0 + [0, 0, 0], p0 + [0, 0, 1.1], p0 + [d, 0, 0]])
    # n = 64: an even and an odd carbon ring, a hydrogenated chain and grown geometries
    add([6] * 64, _ring(64, 1.40))
    add([6] * 63 + [1], np.vstack([_ring(63, 1.40), [[0, 0, 0.0]]]))
    chain = [[1.25 * k, 0.35 * (k % 2), 0] for k in range(32)]
    add([6] * 32 + [1] * 32, chain + [[1.25 * k, 0.35 * (k % 2) + (1.08 if k % 2 else -1.08), 0] for k in range(32)])
    for z, p in grown(rng, 3, (64, 65), bonded=True):
        add(z, p)
    return out


def molecules(seed=0, scale=1, with_gsphere=True):
    """The fixture's molecule sources: [(source name, z int64 [n], positions [n, 3])] (float32 positions for
    G-SphereNet output, float64 otherwise)."""
    rng = np.random.default_rng(seed)
    out = [("idealised", z, p) for z, p in idealised(rng, 8 * scale)]
    out += [("grown", z, p) for z, p in grown(rng, 250 * scale)]
    out += [("grown", z, p) for z, p in grown(rng, 1600 * scale, bonded=True)]
    if with_gsphere:
        out += [("gsphere", z, p) for z, p in gsphere(seed, 40 * scale)]
    out += [("planted", z, p) for z, p in planted(rng)]
    return out


def group(mols):
    """[(z, pos)] -> mol_dicts {n: {'_atomic_numbers', '_positions'}} in order of first appearance of each size."""
    d = {}
    for z, p in mols:
        d.setdefault(len(z), ([], []))
        d[len(z)][0].append(z)
        d[len(z)][1].append(p)
    return {n: {"_atomic_numbers": np.stack(zs), "_positions": np.stack(ps)} for n, (zs, ps) in d.items()}


def main():
    import networkx
    torch.set_num_threads(FIXTURE_THREADS)
    vu, metric = load_reference_validity()
    mols = molecules(0)
    counts = dict.fromkeys(MIN_COUNTS, 0)
    sources = sorted({s for s, _, _ in mols})
    out = {"source": np.array([sources.index(s) for s, _, _ in mols], np.int8),
           "source_names": np.array(json.dumps(sources)),
           "n_atoms": np.array([len(z) for _, z, _ in mols], np.int64)}
    zs, ps, bos, valid, f32 = [], [], [], [], []
    for _, z, p in mols:
        bo, ok = vu.xyz2mol(z, p)
        info = {}
        bo_r, ok_r = rv.xyz2mol(z, p, info)
        assert ok == ok_r and bo.dtype == np.int64 and np.array_equal(bo, bo_r), (z, p)
        counts["disconnected"] += info["outcome"] == "disconnected"
        counts["over_valence"] += info["outcome"] == "over_valence"
        counts["unknown_element"] += info["outcome"] == "unknown_element"
        counts["no_ua"] += info["outcome"] == "no_ua"
        if info["outcome"] == "matched":
            counts["bo_ok"] += info["bo_ok"]
            counts["bo_not_ok"] += not info["bo_ok"]
            counts["two_rounds"] += info["rounds"] >= 2
            counts["odd_cycle"] += info["odd_cycle"]
            counts["multiple_maximum"] += info["multiple_maximum"]
        zs.append(z)
        ps.append(np.asarray(p, np.float64))
        f32.append(p.dtype == np.float32)
        bos.append(bo.astype(np.int8).ravel())
        valid.append(ok)
    print(f"{len(mols)} molecules, {sum(valid)} valid; branch counts {counts}")
    for k, v in MIN_COUNTS.items():
        assert counts[k] >= v, (k, counts[k], v)
    out.update(z=np.concatenate(zs), pos=np.concatenate(ps), float32=np.array(f32), bo=np.concatenate(bos),
               valid=np.array(valid, np.int8), counts=np.array(json.dumps(counts)),
               networkx_version=np.array(networkx.__version__))
    # RandGenEvaluator on one mol_dicts (G-SphereNet output and grown geometries, float32, keys in arbitrary order)
    rng = np.random.default_rng(11)
    ev = [(z, p) for s, z, p in mols if s == "gsphere"]
    ev += [(z, p.astype(np.float32)) for z, p in grown(rng, 300, (3, 30), bonded=True)]
    mol_dicts = group(ev)
    keys = list(mol_dicts)
    rng.shuffle(keys)
    mol_dicts = {k: mol_dicts[k] for k in keys}
    from oracle.gen_golden_mmd import reference_target_bond_lengths
    table = reference_target_bond_lengths()
    target = {}
    for bt in BOND_TYPES:
        real = np.asarray(table[bt], np.float64)
        target[bt] = [np.float64(x) for x in real[rng.choice(real.size, 1500, replace=False)]]
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        validity = metric.RandGenEvaluator.eval_validity(mol_dicts)
        mmd = metric.RandGenEvaluator.eval_bond_mmd({"mol_dicts": mol_dicts, "target_bond_dists": target})
    print(buf.getvalue(), end="")
    out["eval_keys"] = np.array(keys, np.int64)
    for n in keys:
        out[f"eval{n}_z"] = mol_dicts[n]["_atomic_numbers"]
        out[f"eval{n}_pos"] = mol_dicts[n]["_positions"]
    for bt in BOND_TYPES:
        out["target_{}_{}_{}".format(*bt)] = np.array(target[bt], np.float64)
    out["eval_valid_ratio"] = np.float64(validity["valid_ratio"])
    out["eval_stdout"] = np.array(buf.getvalue())
    out["eval_mmd_keys"] = np.array([list(k) for k in mmd], np.int64)
    out["eval_mmd"] = np.array([float(v) for v in mmd.values()], np.float64)
    path = os.path.join(GOLDEN, "xyz2mol.npz")
    np.savez_compressed(path, **out)
    print(f"{path}: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
