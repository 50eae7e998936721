"""CPU tests of G-SphereNet's training likelihood: the travelling restatement (oracle/restated_gsphere_train.py) reproduces
the reference fixture tests/golden/gsphere_train.npz (outputs, loss, every parameter gradient through its sketch -- the
largest |g|, sampled values and random projections -- and the set of parameters without one), and a CPU-resident model's forward still refuses before it reads the batch."""
import os

import numpy as np
import pytest
import torch

from helpers import ROOT, rel_err
from test_gsphere_cpu import _fixture_sd

GOLD = os.path.join(ROOT, "tests", "golden")
GTOL = 1e-4


def fixture():
    return np.load(os.path.join(GOLD, "gsphere_train.npz"))


def fixture_batch(fx, device="cpu"):
    from oracle import restated_gsphere_train as rt
    return {k: torch.from_numpy(fx["in_" + k]).to(device) for k in rt.KEYS}


def train_sd():
    from oracle import restated_gsphere_train as rt
    return rt.train_state_dict(_fixture_sd())


def residue_only(name, num_layers=4):
    """Parameters whose gradient is mathematically zero, so that both sides only hold fp32 rounding residue:
    update_es[l].lin_rbf for l < L - 1 (a flagged edge's value is overwritten by the next layer, an unflagged edge
    never takes layer l's; exactly 0 here) and the attention key biases (a bias shifts every score of a query by the
    same q . b, which the softmax cancels)."""
    return (any(name == f"feat_net.update_es.{l}.lin_rbf.weight" for l in range(num_layers - 1))
            or name.endswith("_att.k_proj.bias"))


def residue_scale(gmax, name, num_layers=4):
    """Absolute scale a residue-only gradient is judged on: the largest gradient of its live counterpart (the last
    layer's lin_rbf, the same attention's query bias).  gmax: name -> largest |gradient|."""
    if name.endswith("_att.k_proj.bias"):
        return gmax(name.replace("k_proj", "q_proj"))
    return gmax(f"feat_net.update_es.{num_layers - 1}.lin_rbf.weight")


def check_fixture_grad(fx, name, grad):
    """grad against the fixture's sketch of the reference gradient: within GTOL of the reference's largest |g| (rel_err),
    or, for a residue-only gradient, within GTOL of its live counterpart's."""
    from oracle import restated_gsphere_train as rt
    names = [str(k) for k in fx["grad_names"]]
    gmax = lambda k: float(fx["grad_max"][names.index(k)])                  # noqa: E731
    scale = residue_scale(gmax, name) if residue_only(name) else gmax(name)
    return rt.check_grad_sketch(name, grad, rt.sketch_from(fx, name, grad.numel()), GTOL * scale)


def test_fixture_shape():
    fx = fixture()
    assert fx["in_new_atom_type"].shape[0] == fx["out_node_latent"].shape[0]
    assert set(np.unique(np.bincount(fx["in_batch"]))) >= {1, 2}          # 1- and 2-atom step graphs occur
    assert fx["out_torsion_latent"].shape[0] > 0 and np.isfinite(fx["out_torsion_latent"]).all()
    assert fx["out_dist_latent"].dtype == np.float64 and fx["out_node_latent"].dtype == np.float32


def test_restatement_reproduces_the_reference():
    from oracle import restated_gsphere_train as rt
    fx = fixture()
    sd = rt.leaf_state_dict(train_sd())
    data = fixture_batch(fx)
    out = rt.sphgen_forward(sd, data, torch.from_numpy(fx["noise"]))
    for k, v in rt.flat_outputs(out).items():
        ref = fx["out_" + k]
        assert v.dtype == torch.from_numpy(ref).dtype and tuple(v.shape) == ref.shape, k
        assert rel_err(v.detach().numpy(), ref) <= 1e-5, k
    loss = rt.loss(out, data["cannot_focus"])
    assert abs(loss.item() - float(fx["loss"])) <= 1e-6 * abs(float(fx["loss"]))
    loss.backward()
    none = sorted(k for k, v in sd.items() if v.grad is None)
    want_none = sorted(str(s) for s in fx["none_grads"])
    assert none == want_none
    for k, v in sd.items():
        if v.grad is not None:
            check_fixture_grad(fx, k, v.grad)
    # the sketch rejects a gradient that is 1% off, and one with a single wrong element among its sampled positions
    k = "torsion_flow_layers.0.linear1.weight"
    with pytest.raises(AssertionError):
        check_fixture_grad(fx, k, sd[k].grad * 1.01)
    bad = sd[k].grad.clone().view(-1)
    bad[int(rt.sketch_from(fx, k, bad.numel())["idx"][7])] += 1e-3 * float(bad.abs().max())
    with pytest.raises(AssertionError):
        check_fixture_grad(fx, k, bad)


def test_cpu_model_forward_refuses_before_reading_the_batch():
    from dig_b200.ggraph3D.method.G_SphereNet.model import SphGen
    from oracle import restated_gsphere as rg
    m = SphGen(**dict(rg.CONFIG, use_gpu=False))
    with pytest.raises(NotImplementedError, match="DESIGN.md"):
        m(None)
