"""CPU tests of G-SphereNet at model sizes other than config_dict.json's (oracle/restated_gsphere_sizes.SIZES): SphGen's
parameter tree is the reference's at each size (a reference checkpoint loads with strict=True), the restatement
reproduces the reference fixture tests/golden/gsphere_sizes.npz, and the only sizes refused are those the reference
cannot run or whose basis is not generated."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import ROOT, rel_err
from test_gsphere_cpu import TYPES, fixture_threads  # noqa: F401  (pytest fixture)

GOLD = os.path.join(ROOT, "tests", "golden")
SIZE_NAMES = ["narrow", "wide_heads"]


def sizes_fixture():
    return np.load(os.path.join(GOLD, "gsphere_sizes.npz"))


def size_shapes(name):
    with open(os.path.join(GOLD, "gsphere_sizes_shapes.json")) as fh:
        return json.load(fh)[name]


def size_sd(name):
    """The fixture's generation weights at size `name`."""
    from oracle import restated_gsphere as rg
    return rg.gsphere_state_dict({k: torch.empty(v) for k, v in size_shapes(name).items()})


def size_train_sd(name):
    from oracle import restated_gsphere_train as rt
    return rt.train_state_dict(size_sd(name))


def section(fx, prefix):
    """The fixture arrays under `prefix` ("<size>/gen/" or "<size>/train/") with the prefix stripped."""
    return {k[len(prefix):]: fx[k] for k in fx.files if k.startswith(prefix)}


def size_draws(gen, device="cpu"):
    from oracle import restated_gsphere as rg
    n_focus = len([k for k in gen if k.startswith("draw_focus_")])
    n_norm = len([k for k in gen if k.startswith("draw_normal_kind_")])
    focus = [torch.from_numpy(gen[f"draw_focus_{k}"]) for k in range(n_focus)]
    normals = [(int(gen[f"draw_normal_kind_{k}"]), torch.from_numpy(gen[f"draw_normal_{k}"])) for k in range(n_norm)]
    return rg.RecordedDraws(focus, normals, device=device)


def out_sizes(gen):
    return sorted(int(k[3:k.index("_")]) for k in gen if k.startswith("out") and k.endswith("_positions"))


@pytest.mark.parametrize("name", SIZE_NAMES)
def test_state_dict_matches_the_reference(name):
    from dig_b200.ggraph3D.method.G_SphereNet.model import SphGen
    from oracle.restated_gsphere_sizes import SIZES
    model = SphGen(**dict(SIZES[name], use_gpu=False))
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == size_shapes(name)
    model.load_state_dict(size_sd(name), strict=True)
    assert model.node_att.d_k == SIZES[name]["hidden_channels"] // SIZES[name]["n_att_heads"]


@pytest.mark.parametrize("name", SIZE_NAMES)
def test_restated_generation_equals_reference(name, fixture_threads):  # noqa: F811
    from oracle import restated_gsphere as rg
    from oracle.restated_gsphere_sizes import SIZES, sized
    fx = sizes_fixture()
    gen = section(fx, f"{name}/gen/")
    run = json.loads(str(fx["run"]))
    trace = []
    with sized(SIZES[name]), torch.no_grad():
        out = rg.generate(size_sd(name), size_draws(gen), TYPES, **run, trace=trace)
    assert len(trace) == int(gen["n_steps"])
    for s in trace:
        i = s["i"]
        assert torch.equal(s["focus_score"], torch.from_numpy(gen[f"step{i}_focus_score"])), i
        for key in ("focus_id", "node_type", "dist", "angle", "torsion", "new_pos"):
            if s.get(key) is not None:
                assert torch.equal(s[key], torch.from_numpy(gen[f"step{i}_{key}"])), (i, key)
    assert sorted(out) == out_sizes(gen)
    for n in out:
        for key in out[n]:
            assert np.array_equal(out[n][key], gen[f"out{n}{key}"]), (n, key)


@pytest.mark.parametrize("name", SIZE_NAMES)
def test_restated_forward_equals_reference(name):
    from oracle import restated_gsphere_train as rt
    from oracle.restated_gsphere_sizes import SIZES, sized
    from test_gsphere_train_cpu import fixture as train_fixture, fixture_batch
    tr = section(sizes_fixture(), f"{name}/train/")
    data = fixture_batch(train_fixture())                # the same 8 molecules as tests/golden/gsphere_train.npz
    assert np.array_equal(tr["picks"], train_fixture()["picks"])
    sd = rt.leaf_state_dict(size_train_sd(name))
    with sized(SIZES[name]):
        out = rt.sphgen_forward(sd, data, torch.from_numpy(tr["noise"]))
    for k, v in rt.flat_outputs(out).items():
        ref = tr["out_" + k]
        assert v.dtype == torch.from_numpy(ref).dtype and tuple(v.shape) == ref.shape, k
        assert rel_err(v.detach().numpy(), ref) <= 1e-5, k
    loss = rt.loss(out, data["cannot_focus"])
    assert abs(loss.item() - float(tr["loss"])) <= 1e-6 * abs(float(tr["loss"]))


def test_refused_sizes():
    from dig_b200.ggraph3D.method.G_SphereNet.model import SphGen
    from oracle import restated_gsphere as rg
    with pytest.raises(ValueError, match="n_att_heads"):
        SphGen(**dict(rg.CONFIG, hidden_channels=100, n_att_heads=3, use_gpu=False))
    with pytest.raises(NotImplementedError, match="basis"):
        SphGen(**dict(rg.CONFIG, num_spherical=5, use_gpu=False))
    # any head width and triplet-branch width otherwise builds
    for kw in (dict(hidden_channels=120, n_att_heads=5), dict(hidden_channels=128, n_att_heads=16),
               dict(hidden_channels=128, n_att_heads=1), dict(int_emb_size=48, basis_emb_size=8),
               dict(int_emb_size=64, basis_emb_size=6)):
        m = SphGen(**dict(rg.CONFIG, use_gpu=False, **kw))
        assert m.feat_net._triplet_generic == (kw.get("int_emb_size", 64) != 64 or kw.get("basis_emb_size", 8) != 8)
