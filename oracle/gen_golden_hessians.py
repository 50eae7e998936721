"""Writes tests/golden/hessians.npz and tests/golden/hessians_shapes.json from the UNMODIFIED reference SchNet, DimeNetPP
and SphereNet (dig/threedgraph/method, run on the CPU over oracle/shim.py): torch.autograd.functional.hessian of the
summed energy in the positions, in fp64, for two small molecules per case (the batch's Hessian; its off-diagonal
molecule blocks are zero).  Cases: default triplet widths and one non-default SphereNet width (the generic branch),
weights from formula_state_dict.  Per case (array names prefixed "<case>/"): z, pos, batch, energy, hessian [3N, 3N]
and buffer/<key> for the state_dict buffers formula_state_dict copies from the reference (SchNet's Gaussian centres).

Before writing anything it checks that the restated models (oracle/restated.py) give the same fp64 Hessian, which the
GPU Hessian tests use as their comparator.

    python -m oracle.gen_golden_hessians          (needs the reference checkout, see oracle/ref_loader.py)
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.ref_loader import load_reference  # noqa: E402
from oracle.weights import formula_state_dict  # noqa: E402
from dig_b200.data import Batch, synthetic_batch  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
warnings.filterwarnings("ignore")

# name: (model, ctor kwargs, weight seed)
CASES = {
    "schnet": ("SchNet", dict(cutoff=5.0, num_layers=2, hidden_channels=32, num_filters=32, num_gaussians=20), 41),
    "dimenetpp": ("DimeNetPP", dict(cutoff=5.0, num_layers=2), 42),
    "spherenet": ("SphereNet", dict(cutoff=5.0, num_layers=2), 43),
    "spherenet_narrow": ("SphereNet", dict(cutoff=5.0, num_layers=2, int_emb_size=32, basis_emb_size_angle=4,
                                           basis_emb_size_torsion=6), 44),
}
DATA = dict(nmol=2, shape="qm9", seed=23, natoms=9)
AGREE_TOL = 1e-6          # restated vs reference fp64 Hessian, relative to the largest entry (op order differs:
#                           the closed forms cancel, measured up to 1.7e-8)


def restated_forward(model_name, ctor, sd, z, pos, batch):
    from oracle import restated
    if model_name == "SchNet":
        return restated.schnet_forward(sd, z, pos, batch, cutoff=ctor["cutoff"], num_layers=ctor["num_layers"],
                                       num_gaussians=ctor["num_gaussians"])
    return restated.dimenet_family_forward(sd, z, pos, batch, torsion=(model_name == "SphereNet"),
                                           cutoff=ctor["cutoff"], num_layers=ctor["num_layers"])


def run_case(method, name):
    model_name, ctor, wseed = CASES[name]
    torch.manual_seed(0)
    model = getattr(method, model_name)(**ctor)
    sd = formula_state_dict(model.state_dict(), seed=wseed)
    model.load_state_dict(sd)
    model.eval()
    model.to(torch.float64)
    b = synthetic_batch(**DATA)
    pos64 = b.pos.double()

    def energy(p):
        return model(Batch(z=b.z, pos=p, batch=b.batch)).sum()
    n = pos64.size(0)
    hess = torch.autograd.functional.hessian(energy, pos64).reshape(3 * n, 3 * n)
    e = model(Batch(z=b.z, pos=pos64.clone(), batch=b.batch))
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    ref = torch.autograd.functional.hessian(
        lambda p: restated_forward(model_name, ctor, sd64, b.z, p, b.batch).sum(), pos64).reshape(3 * n, 3 * n)
    err = float((ref - hess).abs().max() / hess.abs().max())
    assert err < AGREE_TOL, (name, err)
    print(name, "atoms", n, "max |H|", f"{float(hess.abs().max()):.3e}", "restated rel-err", f"{err:.2e}")
    out = {"z": b.z.numpy(), "pos": b.pos.numpy(), "batch": b.batch.numpy(), "energy": e.detach().numpy(),
           "hessian": hess.numpy()}
    # buffers formula_state_dict keeps as the reference builds them (SchNet's Gaussian centres)
    out.update({f"buffer/{k}": v.numpy() for k, v in sd.items() if k.split(".")[-1] == "offset"})
    return out, {k: list(v.shape) for k, v in sd.items()}


def main():
    from oracle import FIXTURE_THREADS
    torch.set_num_threads(FIXTURE_THREADS)
    method = load_reference()
    arrays, shapes = {}, {}
    for name in CASES:
        out, shapes[name] = run_case(method, name)
        arrays.update({f"{name}/{k}": v for k, v in out.items()})
    np.savez_compressed(os.path.join(GOLD, "hessians.npz"), **arrays)
    with open(os.path.join(GOLD, "hessians_shapes.json"), "w") as fh:
        json.dump(shapes, fh)


if __name__ == "__main__":
    main()
