"""Writes tests/golden/bond_mmd.npz from the UNMODIFIED reference dig/ggraph3D/utils/eval_bond_mmd_utils.py
(load_reference_bond_mmd below), run on the CPU with oracle.FIXTURE_THREADS intra-op threads:

  * compute_mmd on seeded cases: sizes 1 .. 4097 (tile edges 127 / 128 / 129 and 4097 = 4 x 1024 + 1), fix_sigma,
    kernel_mul = 3 / kernel_num = 4, kernel_num = 1, float32 + float32 / float32 + float64 / float64 + float64 inputs, a
    source with one far outlier, subsamples of the shipped QM9 C-H and C-C lengths (target_bond_lengths.dict), an empty
    source and constant input (nan) and an empty target (the reference raises ZeroDivisionError);
  * collect_bond_dists on a seeded mol_dicts (float32 positions, 5 / 8 / 12 atoms) with bond orders 0-3 and invalid
    molecules.

Case k is stored as case{k}_source / case{k}_target (their own dtypes) and case{k}_ref (the reference's float, nan when
it raised); `cases` is a JSON list of the keyword arguments and the outcome ("value" / "raises").

    python -m oracle.gen_golden_mmd          (needs the reference checkout, see oracle/ref_loader.py)
"""
import json
import os

import numpy as np
import torch

from oracle import FIXTURE_THREADS
from oracle.ref_loader import REFERENCE_ROOT

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
MOL_SIZES = {5: 3, 8: 4, 12: 2}                 # atoms -> molecules
ATOM_TYPES = np.array([1, 6, 7, 8])


def load_reference_bond_mmd():
    """The reference's dig/ggraph3D/utils/eval_bond_mmd_utils.py (compute_mmd, collect_bond_dists), loaded by file path:
    the package dig.ggraph3D.utils imports RDKit (xyz2mol) and PySCF (compute_prop), which the oracle does not need."""
    import importlib.util
    path = os.path.join(REFERENCE_ROOT, "dig", "ggraph3D", "utils", "eval_bond_mmd_utils.py")
    if not os.path.isfile(path):
        raise RuntimeError(f"reference file not found: {path}")
    spec = importlib.util.spec_from_file_location("ref_eval_bond_mmd_utils", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference_target_bond_lengths():
    """The shipped QM9 bond-length table examples/ggraph3D/G_SphereNet/target_bond_lengths.dict
    ({(z1, z2, order): [length, ...]})."""
    import pickle
    path = os.path.join(REFERENCE_ROOT, "examples", "ggraph3D", "G_SphereNet", "target_bond_lengths.dict")
    with open(path, "rb") as fh:
        return pickle.load(fh)


def _lengths(rng, n, dtype, mean=1.09, std=0.05):
    return (mean + std * rng.standard_normal(n)).astype(dtype)


def mmd_cases():
    """-> list of (name, source ndarray, target ndarray, kwargs)."""
    rng = np.random.default_rng(20240611)
    f32, f64 = np.float32, np.float64
    cases = []
    for ns, nt in ((1, 2), (2, 1), (2, 127), (127, 128), (128, 129), (129, 1000), (1000, 4097), (4097, 128)):
        cases.append((f"sizes_{ns}_{nt}", _lengths(rng, ns, f64), _lengths(rng, nt, f64, 1.1, 0.07), {}))
    cases.append(("fix_sigma", _lengths(rng, 300, f64), _lengths(rng, 500, f64, 1.12), dict(fix_sigma=0.003)))
    cases.append(("mul3_num4", _lengths(rng, 300, f64), _lengths(rng, 700, f64, 1.1, 0.08),
                  dict(kernel_mul=3.0, kernel_num=4)))
    cases.append(("num1", _lengths(rng, 200, f64), _lengths(rng, 300, f64, 1.08), dict(kernel_num=1)))
    cases.append(("f32_f32", _lengths(rng, 500, f32), _lengths(rng, 700, f32, 1.1), {}))
    cases.append(("f32_f64", _lengths(rng, 500, f32), _lengths(rng, 700, f64, 1.1), {}))
    cases.append(("f64_f64", _lengths(rng, 500, f64), _lengths(rng, 700, f64, 1.1), {}))
    src = _lengths(rng, 400, f64)
    src[123] = 40.0
    cases.append(("outlier", src, _lengths(rng, 600, f64), {}))
    target = reference_target_bond_lengths()
    for name, key, n_t, n_s in (("qm9_ch", (1, 6, 1), 3000, 400), ("qm9_cc", (6, 6, 1), 2000, 300)):
        real = np.asarray(target[key], dtype=f64)
        pick = rng.choice(real.size, n_t + n_s, replace=False)
        gen = (real[pick[n_t:]] + 0.02 * rng.standard_normal(n_s)).astype(f32)   # generated lengths come as float32
        cases.append((name, gen, real[pick[:n_t]], {}))
    cases.append(("empty_source", np.zeros(0, f64), _lengths(rng, 50, f64), {}))
    cases.append(("empty_target", _lengths(rng, 50, f64), np.zeros(0, f64), {}))
    cases.append(("constant", np.full(40, 1.09, f64), np.full(60, 1.09, f64), {}))
    return cases


def bond_inputs():
    """Seeded mol_dicts / valid_list / con_mat_list in the layout RandGenEvaluator.eval_bond_mmd builds them."""
    rng = np.random.default_rng(7)
    mols, valid, cons = {}, [], []
    for n_atoms, g in MOL_SIZES.items():
        z = rng.choice(ATOM_TYPES, size=(g, n_atoms))
        pos = (1.4 * rng.standard_normal((g, n_atoms, 3))).astype(np.float32)
        mols[n_atoms] = {"_atomic_numbers": z, "_positions": pos}
        for _ in range(g):
            upper = np.triu(rng.choice(4, size=(n_atoms, n_atoms), p=[0.55, 0.25, 0.15, 0.05]), 1)
            cons.append((upper + upper.T).astype(np.int64))
            valid.append(bool(rng.random() > 0.3))
    valid[0], valid[4] = False, False
    return mols, valid, cons


def main():
    torch.set_num_threads(FIXTURE_THREADS)
    ref = load_reference_bond_mmd()
    out, meta = {}, []
    for k, (name, s, t, kw) in enumerate(mmd_cases()):
        out[f"case{k}_source"], out[f"case{k}_target"] = s, t
        try:
            val, outcome = ref.compute_mmd(torch.from_numpy(s), torch.from_numpy(t), **kw), "value"
        except ZeroDivisionError:
            val, outcome = float("nan"), "raises"
        out[f"case{k}_ref"] = np.float64(val)
        meta.append(dict(name=name, kwargs=kw, outcome=outcome))
        print(f"{name:14s} ns={s.size:5d} nt={t.size:5d} {kw} -> {outcome} {val!r}")
    out["cases"] = np.array(json.dumps(meta))
    mols, valid, cons = bond_inputs()
    for n_atoms in mols:
        out[f"mols{n_atoms}_z"] = mols[n_atoms]["_atomic_numbers"]
        out[f"mols{n_atoms}_pos"] = mols[n_atoms]["_positions"]
    out["mol_sizes"] = np.array(list(mols), dtype=np.int64)
    out["valid"] = np.array(valid)
    for i, c in enumerate(cons):
        out[f"con{i}"] = c
    dists = ref.collect_bond_dists(mols, valid, cons)
    out["bond_keys"] = np.array([[int(x) for x in key] for key in dists], dtype=np.int64)
    out["bond_counts"] = np.array([len(v) for v in dists.values()], dtype=np.int64)
    lengths = [x for v in dists.values() for x in v]
    assert all(type(x) is np.float32 for x in lengths)
    out["bond_lengths"] = np.array(lengths, dtype=np.float32)
    path = os.path.join(GOLDEN, "bond_mmd.npz")
    np.savez_compressed(path, **out)
    print(f"{path}: {os.path.getsize(path)} bytes, {len(meta)} compute_mmd cases, {len(dists)} bond types")


if __name__ == "__main__":
    main()
