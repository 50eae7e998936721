"""GPU tests of QM93DGEN's trajectories (csrc/gen_traj.cu): every fixture molecule against the reference's get(), a
5000-molecule ragged batch across chunk boundaries against the host restatement, repeatability, DataLoader batches
against the reference's collate_fn, and the call sequence of the reference's run_rand_gen.py.

atan2 is the one op that is not bit-reproducible: CPU torch calls the C library's atan2f, which is not correctly rounded,
and the kernel gives the correctly rounded value.  new_angle / new_torsion are therefore held bit for bit to the
restatement with atan2="rn" and to within one fp32 ulp of pi of the reference."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from test_qm93dgen_cpu import FIELDS, fixture, fixture_dicts, fixture_molecules, same

pytestmark = pytest.mark.gpu
ATAN2_FIELDS = ("new_angle", "new_torsion")
ATAN2_BOUND = np.pi * 2.0 ** -23 * 1.0001          # one fp32 ulp at |atan2| <= pi, plus the fp64 shift by 2 pi


def _gpu_dicts(mols, chunk=4096):
    from dig_b200.ggraph3D.dataset.ggraph3D_dataset import compute_trajectories
    ds = _Holder(mols)
    ds._cache["traj"] = compute_trajectories(ds.atom_type_list, ds.position_list, ds.con_mat_list, chunk=chunk)
    return [ds.get(i) for i in range(len(mols))], ds._cache["traj"]


class _Holder:
    """A QM93DGEN without files: only the three molecule lists and the cache."""

    def __init__(self, mols):
        from dig_b200.ggraph3D.dataset import QM93DGEN
        self.atom_type_list = [torch.tensor(t) for t, _, _ in mols]
        self.position_list = [torch.tensor(p) for _, p, _ in mols]
        self.con_mat_list = [torch.tensor(c) for _, _, c in mols]
        self._cache = {}
        self.get = QM93DGEN.get.__get__(self)
        self.trajectories = QM93DGEN.trajectories.__get__(self)


def _check_reference(got, want, where):
    for k in FIELDS:
        if k in ATAN2_FIELDS:
            assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, (where, k)
            nan = torch.isnan(want[k])
            assert torch.equal(torch.isnan(got[k]), nan), (where, k)
            d = (got[k] - want[k])[~nan]
            assert d.numel() == 0 or float(d.abs().max()) <= ATAN2_BOUND, (where, k)
        else:
            assert same(got[k], want[k]), (where, k)


def test_every_fixture_molecule_matches_the_reference():
    from oracle import restated_qm93dgen as rq
    fx = fixture()
    mols = fixture_molecules(fx)
    got, _ = _gpu_dicts(mols)
    differ = 0
    for i, (g, w, (t, p, c)) in enumerate(zip(got, fixture_dicts(fx), mols)):
        _check_reference(g, w, i)
        r = rq.get(t, p, c, atan2="rn")
        for k in ATAN2_FIELDS:
            assert same(g[k], r[k]), (i, k)
            differ += int((g[k] != w[k]).sum())
    n = sum(len(g[k]) for g in got for k in ATAN2_FIELDS)
    assert differ < 0.3 * n, (differ, n)                # the C library's atan2f is off by one ulp on a minority


def _ragged(n_mols, seed):
    from oracle.gen_golden_qm93dgen import grown, _bonds
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_mols):
        n = int(rng.integers(2, 30))
        if k % 10 == 0:                                   # lattice molecules: exact distance ties
            cells = rng.choice(64, size=n, replace=False)
            pos = (np.stack([cells // 16, (cells // 4) % 4, cells % 4], 1) * 1.1).astype(np.float32)
        else:
            pos = grown(rng, n)
        out.append((rng.integers(0, 5, n).astype(np.int64), pos, _bonds(pos, rng)))
    return out


def test_five_thousand_ragged_molecules_across_chunks_match_the_restatement():
    from oracle import restated_qm93dgen as rq
    mols = _ragged(5000, seed=3)
    got, _ = _gpu_dicts(mols, chunk=1024)                # 4 full chunks and a partial one
    for i in list(range(0, 5000, 3)) + [1023, 1024, 1025, 2047, 2048, 4095, 4096, 4999]:
        t, p, c = mols[i]
        want = rq.get(t, p, c, atan2="rn")
        for k in FIELDS:
            assert same(got[i][k], want[k]), (i, k)


def test_two_runs_are_bit_identical_and_chunking_does_not_matter():
    mols = _ragged(3000, seed=5)
    _, (a, pa) = _gpu_dicts(mols, chunk=3000)
    _, (b, pb) = _gpu_dicts(mols, chunk=3000)
    _, (c, pc) = _gpu_dicts(mols, chunk=777)
    assert torch.equal(pa, pb) and torch.equal(pa, pc)
    for k in a:
        for other in (b, c):
            assert torch.equal(a[k].view(torch.uint8) if a[k].is_floating_point() else a[k],
                               other[k].view(torch.uint8) if other[k].is_floating_point() else other[k]), k


def test_one_atom_and_coincident_atoms_raise():
    from dig_b200.ggraph3D.dataset.ggraph3D_dataset import compute_trajectories
    from oracle.gen_golden_qm93dgen import RAISING
    good = fixture_molecules(fixture())[:3]
    for t, p, c in RAISING:
        mols = good + [(t, p, c)]
        with pytest.raises(ValueError, match="molecule 3"):
            compute_trajectories(*([torch.tensor(x[j]) for x in mols] for j in range(3)))
    big = [(np.zeros(33, np.int64), np.arange(99, dtype=np.float32).reshape(33, 3), np.zeros((33, 33), np.int64))]
    with pytest.raises(ValueError, match="up to 32"):
        compute_trajectories(*([torch.tensor(x[j]) for x in big] for j in range(3)))


def _dataset_root(tmp, mols):
    os.makedirs(os.path.join(tmp, "raw"))
    os.makedirs(os.path.join(tmp, "processed"))
    open(os.path.join(tmp, "raw", "gdb9.sdf"), "w").close()
    torch.save(([torch.tensor(t) for t, _, _ in mols], [torch.tensor(p) for _, p, _ in mols],
                [torch.tensor(c) for _, _, c in mols]), os.path.join(tmp, "processed", "data.pt"))
    return tmp


def test_dataloader_batches_match_the_reference_collate():
    from dig_b200.ggraph3D.dataset import QM93DGEN, collate_fn
    from oracle.gen_golden_qm93dgen import COLLATE_BATCHES
    fx = fixture()
    mols = fixture_molecules(fx)
    ref = fixture_dicts(fx)
    with tempfile.TemporaryDirectory() as tmp:
        ds = QM93DGEN(root=_dataset_root(tmp, mols))
        subset = [int(i) for i in np.random.default_rng(0).permutation(len(mols))[:300]]
        loader = torch.utils.data.DataLoader(ds[subset], batch_size=64, collate_fn=collate_fn)
        n = 0
        for b, batch in enumerate(loader):
            _check_reference(batch, collate_fn([ref[i] for i in subset[64 * b:64 * (b + 1)]]), b)
            n += 1
        assert n == 5
        last = ds.get(len(mols) - 1)
        assert all(torch.equal(torch.nan_to_num(v), torch.nan_to_num(ds.get(-1)[k])) for k, v in last.items())
        for bad in (len(mols), -len(mols) - 1):
            with pytest.raises(IndexError):
                ds.get(bad)
        for b, idx in enumerate(COLLATE_BATCHES):    # the reference's own collate_fn output
            (batch,) = list(torch.utils.data.DataLoader(ds[idx], batch_size=64, collate_fn=collate_fn))
            _check_reference(batch, {k: torch.from_numpy(fx[f"collate{b}_{k}"]) for k in FIELDS}, b)


def test_run_rand_gen_call_sequence():
    """The steps of the reference's examples/ggraph3D/G_SphereNet/run_rand_gen.py: the dataset with its split and
    loader, then generation from a checkpoint and the RandGenEvaluator."""
    from dig_b200.ggraph3D.dataset import QM93DGEN, collate_fn
    from dig_b200.ggraph3D.evaluation import RandGenEvaluator
    from dig_b200.ggraph3D.method import G_SphereNet
    from oracle import restated_gsphere as rg
    from helpers import GOLDEN
    mols = fixture_molecules(fixture())
    with tempfile.TemporaryDirectory() as tmp:
        root = _dataset_root(tmp, mols)
        np.savez(os.path.join(root, "raw", "split.npz"), train_idx=np.arange(0, 400), val_idx=np.arange(400, 405))
        dataset = QM93DGEN(root=root)
        idxs = dataset.get_idx_split("rand_gen")
        train_set = dataset[idxs["train"]]
        loader = torch.utils.data.DataLoader(train_set, batch_size=32, shuffle=True, collate_fn=collate_fn)
        batch = next(iter(loader))
        assert batch["focus"].shape[1] == 1 and int(batch["batch"].max()) + 1 == len(batch["new_atom_type"])
        with open(os.path.join(GOLDEN, "gsphere_state_shapes.json")) as fh:
            sd = rg.gsphere_state_dict({k: torch.empty(v) for k, v in json.load(fh).items()})
        ckpt = os.path.join(tmp, "rand_gen.pth")
        torch.save(sd, ckpt)
        torch.manual_seed(0)
        with torch.no_grad():
            mol_dicts = G_SphereNet().generate(model_conf_dict=dict(rg.CONFIG), checkpoint_path=ckpt, n_mols=200,
                                               chunk_size=200, num_min_node=2, num_max_node=35,
                                               temperature=[0.5, 0.3, 0.4, 1.0], focus_th=0.5)
    assert sum(len(v["_atomic_numbers"]) for v in mol_dicts.values()) > 0
    results = RandGenEvaluator().eval_validity(mol_dicts)
    assert 0.0 <= results["valid_ratio"] <= 100.0
    target = {bt: np.random.default_rng(1).normal(1.2, 0.1, 500) for bt in
              [(1, 8, 1), (1, 7, 1), (6, 7, 1), (6, 8, 1), (6, 6, 1), (1, 6, 1)]}
    mmd = RandGenEvaluator().eval_bond_mmd({"mol_dicts": mol_dicts, "target_bond_dists": target})
    assert all(np.isfinite(v) for v in mmd.values())
