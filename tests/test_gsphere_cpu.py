"""CPU tests of G-SphereNet generation: the travelling restatement (oracle/restated_gsphere.py) reproduces the reference
fixtures bit for bit, and SphGen's parameter tree is the reference's (a reference checkpoint loads unchanged)."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import ROOT

GOLD = os.path.join(ROOT, "tests", "golden")
TYPES = np.array([1, 6, 7, 8, 9])


def _shapes():
    with open(os.path.join(GOLD, "gsphere_state_shapes.json")) as fh:
        return json.load(fh)


def _fixture_sd():
    from oracle import restated_gsphere as rg
    return rg.gsphere_state_dict({k: torch.empty(v) for k, v in _shapes().items()})


@pytest.fixture
def fixture_threads():
    from oracle import FIXTURE_THREADS
    old = torch.get_num_threads()
    torch.set_num_threads(FIXTURE_THREADS)
    yield
    torch.set_num_threads(old)


def recorded_draws(gen, device="cpu"):
    from oracle import restated_gsphere as rg
    n_focus = len([k for k in gen.files if k.startswith("draw_focus_")])
    n_norm = len([k for k in gen.files if k.startswith("draw_normal_kind_")])
    focus = [torch.from_numpy(gen[f"draw_focus_{k}"]) for k in range(n_focus)]
    normals = [(int(gen[f"draw_normal_kind_{k}"]), torch.from_numpy(gen[f"draw_normal_{k}"])) for k in range(n_norm)]
    return rg.RecordedDraws(focus, normals, device=device)


def test_state_dict_matches_the_reference():
    from dig_b200.ggraph3D.method.G_SphereNet.model import SphGen
    from oracle import restated_gsphere as rg
    model = SphGen(**dict(rg.CONFIG, use_gpu=False))
    ours = {k: list(v.shape) for k, v in model.state_dict().items()}
    assert ours == _shapes()
    model.load_state_dict(_fixture_sd())                       # strict: a reference checkpoint loads unchanged


def test_training_entry_points_raise():
    from dig_b200.ggraph3D.method import G_SphereNet
    from dig_b200.ggraph3D.method.G_SphereNet.model import SphGen
    from oracle import restated_gsphere as rg
    model = SphGen(**dict(rg.CONFIG, use_gpu=False))
    with pytest.raises(NotImplementedError, match="DESIGN.md"):
        model({})
    with pytest.raises(NotImplementedError, match="DESIGN.md"):
        G_SphereNet().train(None, 1e-4, 0.0, 1, dict(rg.CONFIG), None, 1, "/nonexistent")


def test_restated_feat_net_equals_reference_fixture(fixture_threads):
    from oracle import restated_gsphere as rg
    f = np.load(os.path.join(GOLD, "gsphere_feat.npz"))
    sd = _fixture_sd()
    z, pos, batch = (torch.from_numpy(f[k]) for k in ("z", "pos", "batch"))
    with torch.no_grad():
        out = rg.feat_net_forward(sd, z, pos, batch)
        out_d = rg.feat_net_forward(sd, z, pos, batch, dist_only=True)
    assert torch.equal(out, torch.from_numpy(f["forward"]))
    assert torch.equal(out_d, torch.from_numpy(f["dist_only"]))
    # the isolated atom (index 11) gets its node-type embedding (forward) / zero (dist_only)
    assert torch.equal(out[11], sd["feat_net.init_e.emb.weight"][z[11]])
    assert not out_d[11].any()


def test_restated_generation_equals_reference_trace(fixture_threads):
    from oracle import restated_gsphere as rg
    gen = np.load(os.path.join(GOLD, "gsphere_generate.npz"))
    run = json.loads(str(gen["run"]))
    trace = []
    with torch.no_grad():
        out = rg.generate(_fixture_sd(), recorded_draws(gen), TYPES, **run, trace=trace)
    assert len(trace) == int(gen["n_steps"])
    for s in trace:
        i = s["i"]
        assert torch.equal(s["focus_score"], torch.from_numpy(gen[f"step{i}_focus_score"])), i
        assert torch.equal(s["continue"], torch.from_numpy(gen[f"step{i}_continue"])), i
        for key in ("focus_id", "node_latent", "node_type", "dist", "angle", "torsion", "c1", "c2", "new_pos"):
            if s.get(key) is not None:
                assert torch.equal(s[key], torch.from_numpy(gen[f"step{i}_{key}"])), (i, key)
    sizes = sorted(int(k[3:k.index("_")]) for k in gen.files if k.startswith("out") and k.endswith("_positions"))
    assert sorted(out) == sizes
    for n in sizes:
        for key in ("_atomic_numbers", "_positions", "_focus"):
            assert np.array_equal(out[n][key], gen[f"out{n}{key}"]), (n, key)
