"""G-SphereNet generation on the sm_90a kernels against the reference fixtures (tests/golden/gsphere_*.npz) and the
travelling restatement run on the same GPU."""
import json
import os

import numpy as np
import pytest
import torch

from test_gsphere_cpu import GOLD, TYPES, _fixture_sd, recorded_draws

pytestmark = pytest.mark.gpu

DEV = "cuda"
TOL = 1e-4


def _model(sd=None):
    from dig_b200.ggraph3D.method.G_SphereNet.model import SphGen
    from oracle import restated_gsphere as rg
    model = SphGen(**rg.CONFIG)
    model.load_state_dict(sd if sd is not None else _fixture_sd())
    return model.to(DEV).eval()


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _gen_fixture():
    return np.load(os.path.join(GOLD, "gsphere_generate.npz"))


def test_feat_net_matches_fixture_and_restatement():
    from oracle import restated_gsphere as rg
    f = np.load(os.path.join(GOLD, "gsphere_feat.npz"))
    model = _model()
    sd = {k: v.to(DEV) for k, v in _fixture_sd().items()}
    z, pos, batch = (torch.from_numpy(f[k]).to(DEV) for k in ("z", "pos", "batch"))
    out = model.feat_net(z, pos, batch)
    out_d = model.feat_net.dist_only_forward(z, pos, batch)
    ref, ref_d = torch.from_numpy(f["forward"]).to(DEV), torch.from_numpy(f["dist_only"]).to(DEV)
    assert _rel(out, ref) < 1e-5 and _rel(out_d, ref_d) < 1e-5, (_rel(out, ref), _rel(out_d, ref_d))
    with torch.no_grad():
        gpu_ref = rg.feat_net_forward(sd, z, pos, batch)
        gpu_ref_d = rg.feat_net_forward(sd, z, pos, batch, dist_only=True)
    assert _rel(out, gpu_ref) < 1e-5 and _rel(out_d, gpu_ref_d) < 1e-5
    assert torch.equal(out[11], sd["feat_net.init_e.emb.weight"][z[11]]) and not out_d[11].any()


def _margins(trace, focus_th):
    """Distances of every traced decision from a tie: focus threshold, node-type argmax, c1 / c2 nearest atoms."""
    m = {"threshold": float("inf"), "type": float("inf"), "neighbour": float("inf")}
    for s in trace:
        m["threshold"] = min(m["threshold"], float((s["focus_score"] - focus_th).abs().min()))
        if "node_latent" not in s:
            continue
        top = torch.topk(s["node_latent"], 2, dim=1).values
        m["type"] = min(m["type"], float((top[:, 0] - top[:, 1]).min()))
        z, pos, _, _ = s["state"]
        g = torch.arange(z.size(0))
        for near, ref in (("c1", s["focus_id"]), ("c2", s["c1"])):
            if s.get(near) is None or pos.size(1) < (3 if near == "c1" else 4):
                continue
            d = ((pos - pos[g, ref][:, None]) ** 2).sum(-1)
            d[g, ref] = float("inf")
            if near == "c2":
                d[g, s["focus_id"]] = float("inf")
            two = torch.topk(d, 2, dim=1, largest=False).values
            m["neighbour"] = min(m["neighbour"], float((two[:, 1] - two[:, 0]).min()))
    return m


def _reference_trace():
    """The reference run, replayed on the CPU by the restatement (bit-identical to the fixture, see the CPU tests)."""
    from oracle import restated_gsphere as rg
    gen = _gen_fixture()
    run = json.loads(str(gen["run"]))
    trace = []
    with torch.no_grad():
        rg.generate(_fixture_sd(), recorded_draws(gen), TYPES, **run, trace=trace)
    return gen, run, trace


def test_fixture_decisions_are_not_near_ties():
    _, run, trace = _reference_trace()
    m = _margins(trace, run["focus_th"])
    assert min(m.values()) > 10 * TOL, m


def test_teacher_forced_single_steps():
    """Each step from the reference's state and recorded draws: same focus, node type, dist / angle / torsion, position."""
    from oracle import restated_gsphere as rg
    gen, run, trace = _reference_trace()
    model = _model()
    plan = model._plan()
    checked = 0
    for s in trace:
        if "state" not in s:
            continue
        i, n = s["i"], s["i"] + 1
        z, pos, focuses, can = (t.to(DEV) for t in s["state"])
        g = z.size(0)
        zb = torch.zeros(g, n + 1, dtype=torch.int64, device=DEV)
        pb = torch.zeros(g, n + 1, 3, device=DEV)
        fb = torch.zeros(g, n + 1, dtype=torch.int64, device=DEV)
        zb[:, :n], pb[:, :n], fb[:, :i] = z, pos, focuses
        feat = model._node_features(i, z.contiguous(), pos.contiguous(), g)
        draws = rg.RecordedDraws([s["focus_id"]], s["draws"], device=DEV)
        step = {"can_focus": can}
        with torch.no_grad():
            model._place(i, plan, feat, zb, pb, fb, draws, run["temperature"], trace=step)
        assert torch.equal(step["focus_id"].cpu(), s["focus_id"])
        assert torch.equal(step["node_type"].cpu(), torch.from_numpy(gen[f"step{i}_node_type"])), i
        for key in ("dist", "angle", "torsion", "new_pos"):
            if s.get(key) is not None:
                err = float((step[key].cpu() - torch.from_numpy(gen[f"step{i}_{key}"])).abs().max())
                assert err < TOL, (i, key, err)
        assert torch.equal(zb[:, n].cpu(), s["node_type"]) and torch.equal(fb[:, i].cpu(), s["focus_id"])
        checked += 1
    assert checked >= 3


def test_whole_generate_run_with_recorded_draws():
    gen, run, trace = _reference_trace()
    model = _model()
    gtrace = []
    out = model.generate(TYPES, run["num_gen"], run["temperature"], run["min_atoms"], run["max_atoms"],
                         run["focus_th"], draws=recorded_draws(gen, device=DEV), trace=gtrace)
    sizes = sorted(int(k[3:k.index("_")]) for k in gen.files if k.startswith("out") and k.endswith("_positions"))
    assert sorted(out) == sizes
    for n in sizes:
        assert np.array_equal(out[n]["_atomic_numbers"], gen[f"out{n}_atomic_numbers"]), n
        assert np.array_equal(out[n]["_focus"], gen[f"out{n}_focus"]), n
        assert np.abs(out[n]["_positions"] - gen[f"out{n}_positions"]).max() < TOL, n
    assert len(gtrace) == len(trace)
    for a, b in zip(gtrace, trace):            # scores: well inside the 1e-3 decision margins asserted above
        assert float((a["focus_score"].cpu().view(b["focus_score"].shape) - b["focus_score"]).abs().max()) < 1e-3


def _finish_at_step_one_state_dict(hidden=128):
    """Weights under which every molecule completes with two atoms: the focus classifier accepts the node-type
    embedding of a carbon and rejects a zero feature vector (what an atom without neighbours gets from
    dist_only_forward), the distance flow places the second atom ~60 A away, the type flow favours the last type."""
    sd = _fixture_sd()
    sd["focus_mlp.layers.0.weight"] = torch.eye(hidden)
    sd["focus_mlp.layers.0.bias"] = torch.zeros(hidden)
    sd["focus_mlp.layers.2.weight"] = torch.full((1, hidden), -0.2)
    sd["focus_mlp.layers.2.bias"] = torch.full((1,), 3.0)
    for l in range(6):
        sd[f"dist_flow_layers.{l}.linear2.weight"] = torch.zeros(2, hidden)
        sd[f"dist_flow_layers.{l}.linear2.bias"] = torch.tensor([0.0, -10.0])
        sd[f"node_flow_layers.{l}.linear2.weight"] = torch.zeros(10, hidden)
        sd[f"node_flow_layers.{l}.linear2.bias"] = torch.tensor([0.0] * 5 + [0.0, -1.0, -2.0, -3.0, -4.0])
    return sd


def test_chunks_that_finish_at_step_one_and_uneven_chunking(tmp_path):
    """n_mols=5 in chunks of 2 (2 + 2 + 1), num_min_node=2, every molecule complete after its second atom: the
    method-level API returns the reference's dict; positions / types match the restatement on the same draws."""
    from dig_b200.ggraph3D.method import G_SphereNet
    from oracle import restated_gsphere as rg
    sd = _finish_at_step_one_state_dict()
    path = tmp_path / "ckpt.pth"
    torch.save(sd, path)
    conf = dict(rg.CONFIG)
    temps = [0.5, 0.3, 0.4, 1.0]
    out = G_SphereNet().generate(conf, str(path), n_mols=5, chunk_size=2, num_min_node=2, num_max_node=8,
                                 temperature=temps, focus_th=0.5, draws=rg.SeededDraws(3, device=DEV))
    assert sorted(out) == [2]
    assert out[2]["_atomic_numbers"].shape == (5, 2) and out[2]["_positions"].shape == (5, 2, 3)
    assert out[2]["_focus"].shape == (5, 1) and not out[2]["_focus"].any()
    draws = rg.SeededDraws(3, device=DEV)
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    ref = [rg.generate(sd_dev, draws, TYPES, num_gen=k, temperature=temps, min_atoms=2, max_atoms=8, device=DEV)
           for k in (2, 2, 1)]
    ref_types = np.concatenate([r[2]["_atomic_numbers"] for r in ref])
    ref_pos = np.concatenate([r[2]["_positions"] for r in ref])
    assert np.array_equal(out[2]["_atomic_numbers"], ref_types)
    assert np.abs(out[2]["_positions"] - ref_pos).max() < TOL
    assert (out[2]["_positions"][:, 1, 0] > 50).all()


def test_nan_and_inf_focus_scores_drop_a_molecule():
    """sphgen.py:116-142 on crafted focus logits: a NaN score drops a molecule that still has a candidate, a molecule
    whose scores are all NaN counts as complete (and is emitted), order is kept."""
    from dig_b200 import ops
    nan, inf = float("nan"), float("inf")
    logit = torch.tensor([[-3.0, 2.0, -1.0],      # candidates -> continues
                          [-3.0, nan, 2.0],       # candidate + NaN -> dropped
                          [2.0, 3.0, 4.0],        # no candidate -> complete
                          [nan, nan, nan],        # no candidate (NaN compares false) -> complete
                          [-inf, 1.0, 1.0],       # score 0 -> candidate -> continues
                          [-2.0, -2.0, -2.0]],    # z == 0 rows only -> complete
                         device=DEV)
    z = torch.tensor([[1, 1, 1], [1, 1, 1], [1, 1, 1], [1, 1, 1], [1, 0, 2], [0, 0, 0]], device=DEV)
    for emit in (0, 1):
        score, can, cont_src, emit_src, counts = ops.gsphere_focus_select(logit.view(-1), z, 6, 3, 0.5, emit)
        n_cont, n_emit = counts.tolist()
        ref_score = torch.sigmoid(logit)
        ref_can = (ref_score < 0.5) & (z > 0)
        complete = ref_can.sum(-1) == 0
        cont = ~complete & ~torch.isnan(ref_score).any(-1) & ~torch.isinf(ref_score).any(-1)
        assert torch.allclose(score, ref_score, equal_nan=True, rtol=1e-6)
        assert cont_src[:n_cont].tolist() == torch.nonzero(cont)[:, 0].tolist() == [0, 4]
        assert torch.equal(can[:n_cont], ref_can[cont].float())
        assert emit_src[:n_emit].tolist() == (torch.nonzero(complete)[:, 0].tolist() if emit else [])
