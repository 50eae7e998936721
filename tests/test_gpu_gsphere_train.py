"""GPU tests of SphGen.forward, G-SphereNet's training likelihood (model/sphgen.py, model/spherenet.py forward_train,
csrc/gsphere_train.cu): the reference fixture (outputs, dtypes, loss, every gradient against its sketch, the None-gradient set), a 64-molecule
QM9-sized batch against the fp64 restatement on the GPU, the feature network against its inference forward,
repeatability, a batch without torsion steps, and a short Adam loop.  Generation stays pinned by
tests/test_gpu_gsphere.py and tests/test_gpu_gsphere_kernels.py."""
import os

import numpy as np
import pytest
import torch

from helpers import ROOT, rel_err
from test_gsphere_train_cpu import (GTOL, check_fixture_grad, fixture, fixture_batch, residue_only, residue_scale,
                                    train_sd)

pytestmark = pytest.mark.gpu
# Gradients of the 64-molecule batch (~1,200 step graphs, ~12,000 atoms) against fp64: the weight gradients are fp32
# sums over ~10^5 edge rows, whose rounding alone reaches ~1e-4 of the largest entry.
BATCH_GTOL = 5e-4


def _model(sd=None):
    from dig_b200.ggraph3D.method.G_SphereNet.model import SphGen
    from oracle import restated_gsphere as rg
    m = SphGen(**rg.CONFIG)
    m.load_state_dict(train_sd() if sd is None else sd)
    return m


def _loss(out, cannot_focus):
    from oracle import restated_gsphere_train as rt
    return rt.loss(out, cannot_focus)


def _synthetic_batch(n_mols, seed, min_atoms=9, max_atoms=29):
    """collate_fn over QM93DGEN trajectories of seeded QM9-sized molecules (bonded random walks with no two atoms
    closer than 0.9 A, H/C/N/O/F)."""
    from dig_b200.ggraph3D.dataset import collate_fn
    from test_gpu_qm93dgen import _gpu_dicts
    rng = np.random.default_rng(seed)
    mols = []
    for _ in range(n_mols):
        n = int(rng.integers(min_atoms, max_atoms + 1))
        pos = np.zeros((n, 3))
        for k in range(1, n):
            while True:             # no pair closer than 0.9 A (see oracle.restated_gsphere_train.select_molecules)
                v = rng.standard_normal(3)
                pos[k] = pos[rng.integers(k)] + v / np.linalg.norm(v) * rng.uniform(1.0, 1.6)
                if np.linalg.norm(pos[:k] - pos[k], axis=1).min() >= 0.9:
                    break
        pos = pos.astype(np.float32)
        d = np.linalg.norm(pos[:, None].astype(np.float64) - pos[None], axis=-1)
        con = ((d > 0) & (d < 1.65)).astype(np.int64)
        types = rng.choice(5, size=n, p=[0.5, 0.35, 0.06, 0.08, 0.01]).astype(np.int64)
        types[0] = 1
        mols.append((types, pos, con))
    dicts, _ = _gpu_dicts(mols)
    return collate_fn(dicts)


def _to(batch, dev="cuda"):
    return {k: v.to(dev) for k, v in batch.items()}


def test_fixture_parity():
    fx = fixture()
    m = _model()
    data = fixture_batch(fx, "cuda")
    out = m(data, deq_noise=torch.from_numpy(fx["noise"]).cuda())
    from oracle import restated_gsphere_train as rt
    for k, v in rt.flat_outputs(out).items():
        ref = fx["out_" + k]
        assert v.dtype == torch.from_numpy(ref).dtype and tuple(v.shape) == ref.shape, k
        assert rel_err(v.detach().cpu().numpy(), ref) <= GTOL, k
    loss = _loss(out, data["cannot_focus"])
    assert loss.dtype == torch.float64
    assert abs(loss.item() - float(fx["loss"])) <= GTOL * abs(float(fx["loss"]))
    loss.backward()
    none = sorted(k for k, p in m.named_parameters() if p.grad is None)
    assert none == sorted(str(s) for s in fx["none_grads"])
    for k, p in m.named_parameters():
        if p.grad is not None:
            check_fixture_grad(fx, k, p.grad)


def test_qm9_sized_batch_against_fp64():
    from oracle import restated_gsphere_train as rt
    batch = _to(_synthetic_batch(64, seed=5))
    assert int(batch["batch"].max()) + 1 == batch["new_atom_type"].numel()
    m = _model()
    noise = torch.rand(batch["new_atom_type"].numel(), 5, generator=torch.Generator().manual_seed(1)).cuda()
    out = m(batch, deq_noise=noise)
    loss = _loss(out, batch["cannot_focus"])
    loss.backward()
    sd_leaves = rt.leaf_state_dict({k: v.double().cuda() for k, v in train_sd().items()})
    data64 = dict(batch, position=batch["position"].double())
    out64 = rt.sphgen_forward(sd_leaves, data64, noise.double())
    for k, v in rt.flat_outputs(out).items():
        ref = rt.flat_outputs(out64)[k]
        assert rel_err(v.detach().double().cpu().numpy(), ref.detach().cpu().numpy()) <= GTOL, k
    loss64 = _loss(out64, batch["cannot_focus"])
    assert abs(loss.item() - loss64.item()) <= GTOL * abs(loss64.item())
    loss64.backward()
    ref_grads = {k: v.grad.cpu().numpy() for k, v in sd_leaves.items() if v.grad is not None}
    for k, p in m.named_parameters():
        ref = sd_leaves[k].grad
        assert (p.grad is None) == (ref is None), k
        if ref is None:
            continue
        got = p.grad.double().cpu().numpy()
        if residue_only(k):
            gmax = lambda n: float(np.abs(ref_grads[n]).max())                  # noqa: E731
            assert np.abs(got - ref_grads[k]).max() <= GTOL * residue_scale(gmax, k), k
        else:
            assert rel_err(got, ref_grads[k]) <= BATCH_GTOL, (k, rel_err(got, ref_grads[k]))


def test_feature_network_training_output_equals_inference():
    batch = _to(_synthetic_batch(64, seed=6))
    m = _model()
    n_steps = batch["new_atom_type"].numel()
    train = m.feat_net.forward_train(batch["atom_type"], batch["position"], batch["batch"], num_graphs=n_steps)
    infer = m.feat_net(batch["atom_type"], batch["position"], batch["batch"], num_graphs=n_steps)
    assert rel_err(train.detach().cpu().numpy(), infer.cpu().numpy()) <= 1e-5


def test_two_runs_with_the_same_noise_are_bit_identical():
    from oracle import restated_gsphere_train as rt
    batch = _to(_synthetic_batch(16, seed=7))
    m = _model()
    noise = torch.rand(batch["new_atom_type"].numel(), 5, device="cuda")
    a, b = rt.flat_outputs(m(batch, deq_noise=noise)), rt.flat_outputs(m(batch, deq_noise=noise))
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_default_noise_is_drawn_on_the_device():
    batch = _to(_synthetic_batch(4, seed=8))
    m = _model()
    torch.manual_seed(3)
    a = m(batch)[0][0]
    torch.manual_seed(3)
    b = m(batch)[0][0]
    assert torch.equal(a, b)
    with pytest.raises(ValueError, match="deq_noise"):
        m(batch, deq_noise=torch.rand(1, 5, device="cuda"))


def test_batch_without_torsion_steps():
    from oracle import restated_gsphere_train as rt
    npz = np.load(os.path.join(ROOT, "tests", "golden", "qm93dgen.npz"))
    small = [k for k, n in enumerate(npz["n_atoms"]) if n <= 3][:4]
    batch = _to(rt.batch_from_fixture(npz, small))
    assert batch["c2_c1_focus"].shape[0] == 0
    m = _model()
    out = m(batch)
    tors = out[4]
    assert tuple(tors[0].shape) == (0, 1) and tuple(tors[1].shape) == (0, 1)
    assert tors[0].dtype == torch.float64 and tors[1].dtype == torch.float32
    loss = _loss(out, batch["cannot_focus"])
    assert torch.isnan(loss)                       # torch.mean of an empty tensor, as in the reference


def test_adam_steps_lower_the_loss():
    batch = _to(_synthetic_batch(16, seed=9))
    m = _model()
    noise = torch.rand(batch["new_atom_type"].numel(), 5, generator=torch.Generator().manual_seed(2)).cuda()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    losses = []
    for _ in range(8):
        opt.zero_grad()
        loss = _loss(m(batch, deq_noise=noise), batch["cannot_focus"])
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(np.isfinite(losses))
    assert losses[-1] < losses[0], losses

