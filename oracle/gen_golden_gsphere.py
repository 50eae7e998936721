"""Writes tests/golden/gsphere_feat.npz, tests/golden/gsphere_generate.npz and tests/golden/gsphere_state_shapes.json
from the UNMODIFIED reference G-SphereNet (dig/ggraph3D/method/G_SphereNet/model/*.py) run on the CPU over
oracle/shim.py (+ torch_geometric.utils.softmax, oracle/restated_gsphere.py):

  * feat_net forward / dist_only_forward on a fixed batch (one atom placed out of every other atom's reach);
  * one SphGen.generate run (config_dict.json model, formula weights) with its two random calls -- torch.multinomial
    and Normal.sample -- recorded, plus per step: focus scores (focus_mlp output), the flow outputs (node latent, dist,
    angle, torsion), the output dict; new positions come from the restatement replaying the recorded draws, which is
    checked here to reproduce every recorded value bit for bit.

    python -m oracle.gen_golden_gsphere          (needs the reference checkout, see oracle/ref_loader.py)
"""
import importlib
import importlib.util
import json
import math
import os
import sys

import numpy as np
import torch

from oracle import restated_gsphere as rg
from oracle.ref_loader import REFERENCE_ROOT

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
TYPES = np.array([1, 6, 7, 8, 9])
RUN = dict(num_gen=12, temperature=[0.5, 0.1, 0.2, 1.0], min_atoms=2, max_atoms=7, focus_th=0.5)
SEED = 8


def load_reference_sphgen():
    rg.install_shim()
    if not hasattr(np, "math"):
        np.math = math
    d = os.path.join(REFERENCE_ROOT, "dig", "ggraph3D", "method", "G_SphereNet", "model")
    spec = importlib.util.spec_from_file_location("gsn_ref_model", os.path.join(d, "__init__.py"),
                                                  submodule_search_locations=[d])
    pkg = importlib.util.module_from_spec(spec)
    sys.modules["gsn_ref_model"] = pkg
    spec.loader.exec_module(pkg)
    return importlib.import_module("gsn_ref_model.sphgen")


def feat_batch():
    """Three molecules (5, 7, 4 atoms) with node types 0..4; the last atom of the second one is 20 A away from the rest."""
    g = torch.Generator().manual_seed(17)
    sizes = [5, 7, 4]
    pos = torch.cat([torch.randn(s, 3, generator=g) * 1.3 + 10.0 * k for k, s in enumerate(sizes)])
    pos[11] += torch.tensor([20.0, 0.0, 0.0])
    z = torch.randint(0, 5, (sum(sizes),), generator=g)
    batch = torch.cat([torch.full((s,), k, dtype=torch.long) for k, s in enumerate(sizes)])
    return z, pos, batch


def main():
    from oracle import FIXTURE_THREADS
    torch.set_num_threads(FIXTURE_THREADS)
    sphgen = load_reference_sphgen()
    cfg = dict(rg.CONFIG, use_gpu=False)
    torch.manual_seed(0)
    with torch.no_grad():          # features.py:181 fills a Parameter through arange(out=...), refused under autograd
        model = sphgen.SphGen(**cfg)
    shapes = {k: list(v.shape) for k, v in model.state_dict().items()}
    sd = rg.gsphere_state_dict(model.state_dict())
    model.load_state_dict(sd)
    model.eval()

    feat = {}
    z, pos, batch = feat_batch()
    with torch.no_grad():
        feat["z"], feat["pos"], feat["batch"] = z.numpy(), pos.numpy(), batch.numpy()
        feat["forward"] = model.feat_net(z, pos, batch).numpy()
        feat["dist_only"] = model.feat_net.dist_only_forward(z, pos, batch).numpy()

    # ---- one generate run with the random calls recorded
    rec = {"focus": [], "normal": [], "score": [], "flow": []}
    real_multinomial, real_sample = torch.multinomial, torch.distributions.normal.Normal.sample
    real_flow = sphgen.flow_reverse
    kinds = {}

    def multinomial(inp, k, *a, **kw):
        out = real_multinomial(inp, k, *a, **kw)
        rec["focus"].append(out.view(-1).clone())
        kinds["next"] = 0
        return out

    def sample(self, shape=torch.Size()):
        out = real_sample(self, shape)
        rec["normal"].append((kinds["next"], out.clone()))
        kinds["next"] += 1
        return out

    def flow(layers, latent, f):
        out = real_flow(layers, latent, f)
        rec["flow"].append(out.clone())
        return out

    hook = model.focus_mlp.register_forward_hook(lambda m, i, o: rec["score"].append(o.detach().clone()))
    torch.multinomial, torch.distributions.normal.Normal.sample = multinomial, sample
    sphgen.flow_reverse = flow
    try:
        torch.manual_seed(SEED)
        out = model.generate(TYPES, RUN["num_gen"], RUN["temperature"], RUN["min_atoms"], RUN["max_atoms"],
                             RUN["focus_th"])
    finally:
        torch.multinomial, torch.distributions.normal.Normal.sample = real_multinomial, real_sample
        sphgen.flow_reverse = real_flow
        hook.remove()

    # ---- the restatement replays the draws and must reproduce every recorded value bit for bit
    sd = model.state_dict()
    trace = []
    draws = rg.RecordedDraws(rec["focus"], rec["normal"])
    out_r = rg.generate(sd, draws, TYPES, **RUN, trace=trace)
    flows = iter(rec["flow"])
    for s, score in zip(trace, rec["score"]):
        assert torch.equal(s["focus_score"].view(-1), score), s["i"]
        if "node_latent" in s:
            for key in ("node_latent", "dist", "angle", "torsion"):
                if s[key] is not None:
                    assert torch.equal(s[key], next(flows)), (s["i"], key)
    assert sorted(out) == sorted(out_r)
    for n in out:
        for key in out[n]:
            assert np.array_equal(out[n][key], out_r[n][key]), (n, key)
    print("restatement == reference (scores, flows, output) over", len(trace), "steps; margins",
          rg.margin_report(trace, RUN["focus_th"]), "; molecules per size", {n: len(v["_atomic_numbers"])
                                                                              for n, v in out.items()})

    gen = {"run": np.array(json.dumps(RUN)), "seed": np.array(SEED), "n_steps": np.array(len(trace))}
    for k, f in enumerate(rec["focus"]):
        gen[f"draw_focus_{k}"] = f.numpy()
    for k, (kind, v) in enumerate(rec["normal"]):
        gen[f"draw_normal_{k}"] = v.numpy()
        gen[f"draw_normal_kind_{k}"] = np.array(kind)
    for s in trace:
        i = s["i"]
        gen[f"step{i}_focus_score"] = s["focus_score"].numpy()
        gen[f"step{i}_continue"] = s["continue"].numpy()
        for key in ("focus_id", "node_latent", "node_type", "dist", "angle", "torsion", "c1", "c2", "new_pos"):
            if s.get(key) is not None:
                gen[f"step{i}_{key}"] = s[key].numpy()
    for n, d in out.items():
        for key, v in d.items():
            gen[f"out{n}{key}"] = v
    np.savez_compressed(os.path.join(GOLDEN, "gsphere_feat.npz"), **feat)
    np.savez_compressed(os.path.join(GOLDEN, "gsphere_generate.npz"), **gen)
    with open(os.path.join(GOLDEN, "gsphere_state_shapes.json"), "w") as fh:
        json.dump(shapes, fh, indent=0)
    print("wrote", len(feat), "+", len(gen), "arrays")


if __name__ == "__main__":
    main()
