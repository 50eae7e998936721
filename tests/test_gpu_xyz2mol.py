"""GPU tests of xyz2mol (csrc/xyz2mol.cu through ops.xyz2mol / dig_b200.ggraph3D.evaluation): every fixture molecule's
bond-order matrix and flag exactly as the reference computed them (tests/golden/xyz2mol.npz), freshly seeded molecules
and live G-SphereNet output exactly as the restatement (oracle/restated_validity.py) computes them, large and mixed
batches, repeatability, and RandGenEvaluator against the reference's results on the fixture's mol_dicts."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from test_xyz2mol_cpu import fixture, fixture_molecules

pytestmark = pytest.mark.gpu


def _by_size(mols):
    """[(z, pos, ...)] -> {n: [index, ...]} in order of first appearance."""
    groups = {}
    for k, m in enumerate(mols):
        groups.setdefault(len(m[0]), []).append(k)
    return groups


def _gpu(mols):
    """(bo [n, n] int64, valid) of each molecule, one ops.xyz2mol call per atom count."""
    from dig_b200 import ops
    out = [None] * len(mols)
    for n, idx in _by_size(mols).items():
        z = torch.from_numpy(np.stack([mols[k][0] for k in idx]))
        pos = torch.from_numpy(np.stack([mols[k][1] for k in idx]))
        bo, valid = ops.xyz2mol(z, pos)
        bo, valid = bo.cpu().numpy().astype(np.int64), valid.cpu().numpy()
        for r, k in enumerate(idx):
            out[k] = (bo[r], int(valid[r]))
    return out


def _check_against_restatement(mols):
    pytest.importorskip("networkx", reason="the restatement needs networkx")
    from oracle import restated_validity as rv
    for k, ((z, pos), (bo, ok)) in enumerate(zip(mols, _gpu(mols))):
        want, want_ok = rv.xyz2mol(z, pos)
        assert ok == want_ok and np.array_equal(bo, want), (k, z.tolist(), np.asarray(pos).tolist())


def test_every_fixture_molecule_matches_the_reference():
    mols = fixture_molecules()
    for k, ((_, _, bo, ok), (got, got_ok)) in enumerate(zip(mols, _gpu([(z, p) for z, p, _, _ in mols]))):
        assert got_ok == ok and np.array_equal(got, bo), k


def test_float32_positions_are_widened_exactly():
    from dig_b200 import ops
    mols = [(z, p) for (z, p, _, _), f32 in zip(fixture_molecules(), fixture()["float32"]) if f32]
    n, idx = next(iter(_by_size(mols).items()))
    z = torch.from_numpy(np.stack([mols[k][0] for k in idx]))
    pos64 = torch.from_numpy(np.stack([mols[k][1] for k in idx]))
    pos32 = pos64.float()
    assert torch.equal(pos32.double(), pos64)                # the fixture stored them widened
    a, b = ops.xyz2mol(z, pos32), ops.xyz2mol(z, pos64)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_fifty_thousand_seeded_molecules_match_the_restatement():
    from oracle import gen_golden_validity as gv
    mols = [(z, p) for _, z, p in gv.molecules(seed=1, scale=10, with_gsphere=False)]
    mols += [(z, p) for z, p in gv.grown(np.random.default_rng(2), 50_000 - len(mols), bonded=True)]
    assert len(mols) == 50_000
    _check_against_restatement(mols)


def _generated(n_mols, seed=0, num_max_node=35):
    """G_SphereNet.generate with the fixture weights (tests/golden/gsphere_state_shapes.json)."""
    from dig_b200.ggraph3D.method import G_SphereNet
    from oracle import restated_gsphere as rg
    with open(os.path.join(os.path.dirname(__file__), "golden", "gsphere_state_shapes.json")) as fh:
        sd = rg.gsphere_state_dict({k: torch.empty(v) for k, v in json.load(fh).items()})
    with tempfile.TemporaryDirectory() as tmp:
        ckpt = os.path.join(tmp, "ckpt.pth")
        torch.save(sd, ckpt)
        torch.manual_seed(seed)
        return G_SphereNet().generate(dict(rg.CONFIG), ckpt, n_mols=n_mols, chunk_size=1000, num_min_node=2,
                                      num_max_node=num_max_node, temperature=[0.5, 0.3, 0.4, 1.0], focus_th=0.5)


def test_generated_molecules_match_the_restatement():
    mol_dicts = _generated(1000)
    mols = [(z, p) for n in mol_dicts for z, p in zip(mol_dicts[n]["_atomic_numbers"], mol_dicts[n]["_positions"])]
    assert len(mols) == 1000 and mols[0][1].dtype == np.float32
    _check_against_restatement(mols)


def test_batch_follows_key_and_row_order_with_mixed_sizes():
    from dig_b200.ggraph3D.evaluation import xyz2mol_batch
    from oracle import gen_golden_validity as gv
    from oracle import restated_validity as rv
    rng = np.random.default_rng(4)
    mol_dicts = gv.group(gv.grown(rng, 600, (1, 40), bonded=True))
    keys = list(mol_dicts)
    rng.shuffle(keys)
    mol_dicts = {k: {"_atomic_numbers": torch.from_numpy(mol_dicts[k]["_atomic_numbers"]),
                     "_positions": torch.from_numpy(mol_dicts[k]["_positions"]).float().cuda()} for k in keys}
    mol_dicts[45] = {"_atomic_numbers": np.zeros((0, 45), np.int64), "_positions": np.zeros((0, 45, 3))}
    con, valid = xyz2mol_batch(mol_dicts)
    k = 0
    for n in mol_dicts:
        for z, p in zip(mol_dicts[n]["_atomic_numbers"], mol_dicts[n]["_positions"]):
            want, ok = rv.xyz2mol(np.asarray(z), p.cpu().numpy())
            assert con[k].dtype == np.int64 and con[k].shape == (n, n)
            assert valid[k] is bool(ok) and np.array_equal(con[k], want), k
            k += 1
    assert k == len(con) == len(valid) == 600


def test_two_hundred_thousand_molecules_in_one_call_and_repeatable():
    """One launch over 200,000 molecules of 40 atoms (3.2e8 bond-order entries, int64 offsets), twice, bit-identical."""
    from dig_b200 import ops
    from oracle import gen_golden_validity as gv
    from oracle import restated_validity as rv
    rng = np.random.default_rng(6)
    seed_mols = gv.grown(rng, 2000, (40, 41), bonded=True)
    z = torch.from_numpy(np.stack([m[0] for m in seed_mols])).repeat(100, 1)
    pos = torch.from_numpy(np.stack([m[1] for m in seed_mols])).repeat(100, 1, 1)
    shift = torch.randn(200_000, 1, 3, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    pos = pos + shift                                        # a translation of each copy: rounding differs per copy
    bo, valid = ops.xyz2mol(z.cuda(), pos.cuda())
    bo2, valid2 = ops.xyz2mol(z.cuda(), pos.cuda())
    assert torch.equal(bo, bo2) and torch.equal(valid, valid2)
    pick = np.concatenate([np.arange(50), np.arange(200_000 - 50, 200_000), rng.choice(200_000, 1500, replace=False)])
    bo_h, valid_h = bo.cpu().numpy(), valid.cpu().numpy()
    for k in pick.tolist():
        want, ok = rv.xyz2mol(z[k].numpy(), pos[k].numpy())
        assert valid_h[k] == ok and np.array_equal(bo_h[k].astype(np.int64), want), k


def _fixture_eval_inputs():
    f = fixture()
    mol_dicts = {int(n): {"_atomic_numbers": f[f"eval{n}_z"], "_positions": f[f"eval{n}_pos"]}
                 for n in f["eval_keys"].tolist()}
    from oracle.gen_golden_validity import BOND_TYPES
    target = {bt: list(f["target_{}_{}_{}".format(*bt)]) for bt in BOND_TYPES}
    return f, mol_dicts, target


def test_eval_validity_matches_the_reference(capsys):
    from dig_b200.ggraph3D.evaluation import RandGenEvaluator
    f, mol_dicts, _ = _fixture_eval_inputs()
    got = RandGenEvaluator.eval_validity(mol_dicts)
    assert got == {"valid_ratio": float(f["eval_valid_ratio"])}
    assert capsys.readouterr().out == str(f["eval_stdout"]).splitlines(keepends=True)[0]


def test_eval_bond_mmd_matches_the_reference(capsys):
    from dig_b200.ggraph3D.evaluation import RandGenEvaluator
    f, mol_dicts, target = _fixture_eval_inputs()
    got = RandGenEvaluator.eval_bond_mmd({"mol_dicts": mol_dicts, "target_bond_dists": target})
    assert [list(k) for k in got] == f["eval_mmd_keys"].tolist()
    # float32 generated lengths against the float64 table: the reference computes in fp64, so does the port
    for (k, v), want in zip(got.items(), f["eval_mmd"].tolist()):
        assert abs(v - want) <= 1e-10, (k, v, want)
    lines = capsys.readouterr().out.splitlines()
    want_lines = str(f["eval_stdout"]).splitlines()[1:]
    assert len(lines) == len(want_lines)
    for a, b in zip(lines, want_lines):
        assert a.rsplit(" ", 1)[0] == b.rsplit(" ", 1)[0]
        assert abs(float(a.rsplit(" ", 1)[1]) - float(b.rsplit(" ", 1)[1])) <= 1e-10
