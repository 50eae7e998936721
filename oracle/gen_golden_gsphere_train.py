"""Writes tests/golden/gsphere_train.npz from the UNMODIFIED reference SphGen.forward (dig/ggraph3D/method/G_SphereNet/
model/sphgen.py:44-79), loaded over oracle/shim.py as oracle/gen_golden_gsphere.py loads it, run on the CPU:

  * inputs: collate_fn over 8 molecules of tests/golden/qm93dgen.npz (a 2-atom and a 3-atom one among them, so that
    step graphs of 1 and 2 atoms occur; none with a NaN torsion), recorded dequantisation noise;
  * weights: formula weights (oracle.restated_gsphere_train.train_state_dict), under which every flow and every
    attention weight is non-trivial;
  * records: the five outputs, the reference training loss (gspherenet.py:62-71), a sketch of every parameter gradient
    after loss.backward() (rt.grad_sketch: largest |g|, 256 sampled values, 8 random +-1 projections) and the names of
    the parameters whose gradient is None.

    python -m oracle.gen_golden_gsphere_train          (needs the reference checkout, see oracle/ref_loader.py)
"""
import os

import numpy as np
import torch

from oracle import restated_gsphere as rg
from oracle import restated_gsphere_train as rt
from oracle.gen_golden_gsphere import GOLDEN, load_reference_sphgen

NOISE_SEED = 23


def main():
    from oracle import FIXTURE_THREADS
    torch.set_num_threads(FIXTURE_THREADS)
    sphgen = load_reference_sphgen()
    cfg = dict(rg.CONFIG, use_gpu=False)
    torch.manual_seed(0)
    with torch.no_grad():
        model = sphgen.SphGen(**cfg)
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
    for k in rt.KEYS:
        rec["in_" + k] = batch[k].numpy()
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

    # the restatement must reproduce the reference on the same inputs
    sd = rt.leaf_state_dict(model.state_dict())
    out_r = rt.sphgen_forward(sd, batch, noise)
    for k, v in rt.flat_outputs(out_r).items():
        ref = torch.from_numpy(rec["out_" + k])
        assert v.dtype == ref.dtype and v.shape == ref.shape, k
        assert torch.allclose(v.detach(), ref, rtol=1e-5, atol=1e-6), k
    loss_r = rt.loss(out_r, batch["cannot_focus"])
    loss_r.backward()
    assert abs(loss_r.item() - loss.item()) <= 1e-6 * abs(loss.item()), (loss_r.item(), loss.item())
    print("loss", loss.item(), "| molecules", picks, "| steps", batch["new_atom_type"].size(0), "| atoms",
          batch["atom_type"].size(0), "| None gradients:", len(none))
    np.savez_compressed(os.path.join(GOLDEN, "gsphere_train.npz"), **rec)
    print("wrote", len(rec), "arrays")


if __name__ == "__main__":
    main()
