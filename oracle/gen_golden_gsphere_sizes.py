"""Writes tests/golden/gsphere_sizes.npz and tests/golden/gsphere_sizes_shapes.json from the UNMODIFIED reference SphGen
(dig/ggraph3D/method/G_SphereNet/model/*.py) at the non-default sizes of oracle/restated_gsphere_sizes.SIZES, run on the
CPU over oracle/shim.py as oracle/gen_golden_gsphere.py loads it.  Per size (array names prefixed "<size>/"):

  * one generate run (formula weights of oracle.restated_gsphere.gsphere_state_dict) with its random calls recorded,
    and per step the focus scores, decisions, flow outputs and new positions; the restatement replaying the draws must
    reproduce every recorded value bit for bit, every decision must lie at least MARGIN from a tie, and no position may
    move by more than CONDITIONED when the attention outputs are perturbed at fp32 rounding level;
  * one SphGen.forward on the 8 molecules of oracle/gen_golden_gsphere_train.py (training weights,
    oracle.restated_gsphere_train.train_state_dict) with recorded dequantisation noise: the five outputs, the training
    loss, a sketch of every parameter gradient and the names of the parameters without one.

    python -m oracle.gen_golden_gsphere_sizes          (needs the reference checkout, see oracle/ref_loader.py)
"""
import json
import os

import numpy as np
import torch

from oracle import restated_gsphere as rg
from oracle import restated_gsphere_train as rt
from oracle.gen_golden_gsphere import GOLDEN, RUN, TYPES, load_reference_sphgen
from oracle.restated_gsphere_sizes import SIZES, sized

SEEDS = {"narrow": 12, "wide_heads": 12}   # draw seeds whose runs keep every decision MARGIN from a tie and positions
                                           # CONDITIONED
NOISE_SEED = 23
MARGIN = 1e-3
CONDITIONED = 1e-5        # largest position shift under a 2e-7 relative perturbation of every attention output


def position_sensitivity(sd, cfg, focus, normals, out):
    """Largest |position change| of the replayed run when every attention output is perturbed by fp32-rounding-sized
    relative noise: a run whose positions move by ~1e-4 under it cannot pin an fp32 implementation to 1e-4."""
    g = torch.Generator().manual_seed(0)
    orig = rg.mh_att
    with sized(cfg), torch.no_grad():
        att = rg.mh_att
        rg.mh_att = lambda *a, **kw: (lambda o: o * (1 + 2e-7 * torch.randn(o.shape, generator=g)))(att(*a, **kw))
        try:
            out_p = rg.generate(sd, rg.RecordedDraws(focus, normals), TYPES, **RUN)
        finally:
            rg.mh_att = att
    assert rg.mh_att is orig
    return max(float(np.abs(out_p[n]["_positions"] - out[n]["_positions"]).max()) for n in out)


def neighbour_margin(trace):
    """Smallest gap between the nearest and second-nearest candidate of every c1 / c2 choice of a traced run."""
    m = float("inf")
    for s in trace:
        if s.get("c1") is None:
            continue
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
            m = min(m, float((two[:, 1] - two[:, 0]).min()))
    return m


def generation_record(sphgen, model, cfg, seed):
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
        torch.manual_seed(seed)
        with torch.no_grad():
            out = model.generate(TYPES, RUN["num_gen"], RUN["temperature"], RUN["min_atoms"], RUN["max_atoms"],
                                 RUN["focus_th"])
    finally:
        torch.multinomial, torch.distributions.normal.Normal.sample = real_multinomial, real_sample
        sphgen.flow_reverse = real_flow
        hook.remove()

    trace = []
    with sized(cfg), torch.no_grad():
        out_r = rg.generate(model.state_dict(), rg.RecordedDraws(rec["focus"], rec["normal"]), TYPES, **RUN,
                            trace=trace)
    flows = iter(rec["flow"])
    for s, score in zip(trace, rec["score"]):
        assert torch.equal(s["focus_score"].view(-1), score), s["i"]
        if "node_latent" in s:
            for key in ("node_latent", "dist", "angle", "torsion"):
                if s[key] is not None:
                    assert torch.equal(s[key], next(flows)), (s["i"], key)
    assert sorted(out) == sorted(out_r) and len(out) >= 2, sorted(out)
    for n in out:
        for key in out[n]:
            assert np.array_equal(out[n][key], out_r[n][key]), (n, key)
    margins = dict(rg.margin_report(trace, RUN["focus_th"]), neighbour=neighbour_margin(trace))
    assert min(margins.values()) >= MARGIN, margins
    margins["position_sensitivity"] = position_sensitivity(model.state_dict(), cfg, rec["focus"], rec["normal"], out)
    assert margins["position_sensitivity"] <= CONDITIONED, margins
    print("  generate: restatement == reference over", len(trace), "steps; margins", margins, "; molecules per size",
          {n: len(v["_atomic_numbers"]) for n, v in out.items()})

    gen = {"seed": np.array(seed), "n_steps": np.array(len(trace))}
    for k, f in enumerate(rec["focus"]):
        gen[f"draw_focus_{k}"] = f.numpy()
    for k, (kind, v) in enumerate(rec["normal"]):
        gen[f"draw_normal_{k}"] = v.numpy()
        gen[f"draw_normal_kind_{k}"] = np.array(kind)
    for s in trace:
        i = s["i"]
        gen[f"step{i}_focus_score"] = s["focus_score"].numpy()
        for key in ("focus_id", "node_type", "dist", "angle", "torsion", "new_pos"):
            if s.get(key) is not None:
                gen[f"step{i}_{key}"] = s[key].numpy()
    for n, d in out.items():
        for key, v in d.items():
            gen[f"out{n}{key}"] = v
    return gen


def training_record(model, cfg):
    model.load_state_dict(rt.train_state_dict(rg.gsphere_state_dict(model.state_dict())))
    model.train()
    npz = np.load(os.path.join(GOLDEN, "qm93dgen.npz"))
    picks = rt.select_molecules(npz)
    batch = rt.batch_from_fixture(npz, picks)
    noise = torch.rand(batch["new_atom_type"].size(0), cfg["num_node_types"],
                       generator=torch.Generator().manual_seed(NOISE_SEED))
    real_rand = torch.rand

    def rand(size, *a, **kw):                       # sphgen.py:56, the one random call of the forward
        assert tuple(size) == tuple(noise.shape)
        return noise.clone()

    torch.rand = rand
    try:
        out = model(batch)
    finally:
        torch.rand = real_rand
    loss = rt.loss(out, batch["cannot_focus"])
    model.zero_grad(set_to_none=True)
    loss.backward()
    rec = {"picks": np.array(picks), "noise": noise.numpy(), "loss": np.array(loss.item())}
    for k, v in rt.flat_outputs(out).items():
        rec["out_" + k] = v.detach().numpy()
    none, sketches = [], {}
    for name, p in model.named_parameters():
        if p.grad is None:
            none.append(name)
        else:
            sketches[name] = rt.grad_sketch(name, p.grad)
    rec.update(rt.pack_sketches(sketches))
    rec["none_grads"] = np.array(none)

    with sized(cfg):
        out_r = rt.sphgen_forward(rt.leaf_state_dict(model.state_dict()), batch, noise)
    for k, v in rt.flat_outputs(out_r).items():
        ref = torch.from_numpy(rec["out_" + k])
        assert v.dtype == ref.dtype and v.shape == ref.shape, k
        assert torch.allclose(v.detach(), ref, rtol=1e-5, atol=1e-6), k
    print("  forward: loss", loss.item(), "| steps", batch["new_atom_type"].size(0), "| None gradients:", len(none))
    return rec


def main():
    from oracle import FIXTURE_THREADS
    torch.set_num_threads(FIXTURE_THREADS)
    sphgen = load_reference_sphgen()
    arrays, shapes = {}, {}
    for name, cfg in SIZES.items():
        print(name, {k: cfg[k] for k in ("hidden_channels", "n_att_heads", "int_emb_size", "basis_emb_size",
                                         "out_emb_channels", "num_spherical")})
        torch.manual_seed(0)
        with torch.no_grad():      # features.py:181 fills a Parameter through arange(out=...), refused under autograd
            model = sphgen.SphGen(**dict(cfg, use_gpu=False))
        shapes[name] = {k: list(v.shape) for k, v in model.state_dict().items()}
        model.load_state_dict(rg.gsphere_state_dict(model.state_dict()))
        model.eval()
        rec = {"gen/" + k: v for k, v in generation_record(sphgen, model, cfg, SEEDS[name]).items()}
        rec.update({"train/" + k: v for k, v in training_record(model, cfg).items()})
        arrays.update({f"{name}/{k}": v for k, v in rec.items()})
    arrays["run"] = np.array(json.dumps(RUN))
    np.savez_compressed(os.path.join(GOLDEN, "gsphere_sizes.npz"), **arrays)
    with open(os.path.join(GOLDEN, "gsphere_sizes_shapes.json"), "w") as fh:
        json.dump(shapes, fh, indent=0)
    print("wrote", len(arrays), "arrays")


if __name__ == "__main__":
    main()
