"""Writes tests/golden/generic_forces.npz and tests/golden/generic_forces_shapes.json from the UNMODIFIED reference
SphereNet / DimeNetPP (dig/threedgraph/method, run on the CPU over oracle/shim.py) at triplet-branch widths the fused
kernels are not compiled for (the generic branch: materialised bases, ordinary linears).  Per case (array names
prefixed "<case>/"): the inputs, energies and forces -dE/dpos in fp32 and fp64 from formula_state_dict weights.

It also checks, before writing anything, that oracle/restated.dimenet_family_forward reproduces the reference at these
sizes: energies bit for bit (CPU fp32, FIXTURE_THREADS threads) and its autograd forces to fp32 rounding level.

    python -m oracle.gen_golden_generic_forces          (needs the reference checkout, see oracle/ref_loader.py)
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

# name: (model, ctor kwargs, weight seed).  The generic sizes of tests/test_gpu_parity.py::test_generic_channel_sizes.
CASES = {
    "dimenetpp_wide": ("DimeNetPP", dict(int_emb_size=96, basis_emb_size=16, num_layers=2, cutoff=5.0), 31),
    "spherenet_narrow": ("SphereNet", dict(int_emb_size=32, basis_emb_size_angle=4, basis_emb_size_torsion=6,
                                           num_layers=2, cutoff=5.0), 32),
    "spherenet_ns3": ("SphereNet", dict(int_emb_size=48, num_spherical=3, num_layers=2, cutoff=5.0), 33),
}
DATA = dict(nmol=3, shape="md17-aspirin", seed=17)
FORCE_TOL = 1e-5          # restated vs reference forces, relative to the largest component (fp32 level)


def restated_kwargs(model_name, ctor):
    """The keyword arguments of restated.dimenet_family_forward for a case (widths come from the state_dict)."""
    kw = {k: v for k, v in ctor.items() if k in ("cutoff", "num_layers", "num_spherical")}
    return dict(torsion=(model_name == "SphereNet"), **kw)


def _np(t):
    return t.detach().cpu().numpy()


def run_case(method, name):
    from oracle import restated
    model_name, ctor, wseed = CASES[name]
    torch.manual_seed(0)
    model = getattr(method, model_name)(**ctor)
    sd = formula_state_dict(model.state_dict(), seed=wseed)
    model.load_state_dict(sd)
    model.eval()
    b = synthetic_batch(**DATA)
    out = {"z": _np(b.z), "pos": _np(b.pos), "batch": _np(b.batch)}
    for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        m = model.to(dtype)
        pos = b.pos.to(dtype).clone().requires_grad_(True)
        e = m(Batch(z=b.z, pos=pos, batch=b.batch))
        f = -torch.autograd.grad(e.sum(), pos)[0]
        out[f"energy_{tag}"], out[f"force_{tag}"] = _np(e), _np(f)
    model.to(torch.float32)
    # the restatement at the same sizes: energies bit for bit, forces at fp32 level
    pos = b.pos.clone().requires_grad_(True)
    u = restated.dimenet_family_forward(sd, b.z, pos, b.batch, **restated_kwargs(model_name, ctor))
    f = -torch.autograd.grad(u.sum(), pos)[0]
    assert np.array_equal(_np(u), out["energy_f32"]), (name, _np(u), out["energy_f32"])
    ferr = float(np.abs(_np(f) - out["force_f32"]).max() / np.abs(out["force_f64"]).max())
    assert ferr < FORCE_TOL, (name, ferr)
    print(name, "energy", out["energy_f32"].ravel(), "restated force rel-err", f"{ferr:.2e}",
          "f32 vs f64 force", f"{np.abs(out['force_f32'] - out['force_f64']).max() / np.abs(out['force_f64']).max():.2e}")
    shapes = {k: list(v.shape) for k, v in model.state_dict().items()}
    return out, shapes


def main():
    from oracle import FIXTURE_THREADS
    torch.set_num_threads(FIXTURE_THREADS)
    method = load_reference()
    arrays, shapes = {}, {}
    for name in CASES:
        out, shapes[name] = run_case(method, name)
        arrays.update({f"{name}/{k}": v for k, v in out.items()})
    np.savez_compressed(os.path.join(GOLD, "generic_forces.npz"), **arrays)
    with open(os.path.join(GOLD, "generic_forces_shapes.json"), "w") as fh:
        json.dump(shapes, fh)


if __name__ == "__main__":
    main()
