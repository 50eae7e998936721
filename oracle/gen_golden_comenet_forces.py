"""Writes tests/golden/comenet_forces.npz and tests/golden/comenet_forces_shapes.json from the UNMODIFIED reference
ComENet (dig/threedgraph/method/comenet, run on the CPU over oracle/shim.py).  Per case (array names prefixed
"<case>/"): the inputs, energies and forces -dE/dpos in fp32 and fp64 from formula_state_dict weights, seeded energy /
force targets, and the fp32 parameter gradients of the force-training loss of run.py:110-123,
L1(E, y) + P * L1(F, f) with F = -grad(E, pos, create_graph=True): in full ("grad/<name>") for tensors of at most
FULL_GRAD_NUMEL entries, as N_PROJ seeded random projections ("grad_proj/<name>", fp64, see `projection`) for the
weight matrices, which would make the fixture tens of megabytes.

It also checks, before writing anything, that oracle/restated.comenet_forward reproduces the reference: energies bit
for bit, forces and parameter gradients at fp32 rounding level (CPU fp32).  Everything runs on ONE thread: the
reference's position gradient adds pairs of opposite ~1e7-sized terms (the derivative of the FMA residue a x a of an
aliased cross product, SURVEY.md 5.9b and csrc/comenet.cu), so its last bits -- O(1) in the forces -- depend on the
order of the multi-threaded CPU sums and change from run to run with several threads.

    python -m oracle.gen_golden_comenet_forces          (needs the reference checkout, see oracle/ref_loader.py)
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

# name: (ctor kwargs, data, weight seed).  data: synthetic_batch kwargs, or the name of an existing golden case whose
# inputs are reused ("comenet_oc20": two OC20-shaped structures where the 32-neighbour cap binds).
CASES = {
    "aspirin_default": (dict(cutoff=5.0, num_layers=2), dict(nmol=3, shape="md17-aspirin", seed=17), 41),
    "oc20_capped": (dict(cutoff=6.0), "comenet_oc20", 4),
    "aspirin_generic": (dict(cutoff=5.0, num_layers=2, hidden_channels=128, middle_channels=32, num_output_layers=2),
                        dict(nmol=3, shape="md17-aspirin", seed=18), 43),
}
P_FORCE = 100.0           # run.py's default force weight p
TARGET_SEED = 5
FORCE_TOL = 1e-5          # restated vs reference forces, relative to the largest component (fp32 level)
GRAD_TOL = 1e-4           # restated vs reference parameter gradients, relative to each tensor's largest entry
FIXTURE_THREADS = 1       # see the module docstring
FULL_GRAD_NUMEL = 4096
N_PROJ = 4


def projection(numel, index):
    """[numel, N_PROJ] fp64 standard-normal matrix of the index-th parameter's gradient projections."""
    return torch.randn(numel, N_PROJ, generator=torch.Generator().manual_seed(1000 + index), dtype=torch.float64)


def gradient_record(names, grads):
    out = {}
    for idx, (k, gr) in enumerate(zip(names, grads)):
        if gr.numel() <= FULL_GRAD_NUMEL:
            out[f"grad/{k}"] = _np(gr)
        else:
            out[f"grad_proj/{k}"] = _np(gr.detach().double().reshape(-1) @ projection(gr.numel(), idx))
    return out


def restated_kwargs(ctor):
    """The keyword arguments of restated.comenet_forward for a case."""
    return {k: v for k, v in ctor.items() if k in ("cutoff", "num_layers", "num_output_layers")}


def inputs(data):
    if isinstance(data, str):
        g = np.load(os.path.join(GOLD, data + ".npz"))
        return torch.from_numpy(g["z"]), torch.from_numpy(g["pos"]), torch.from_numpy(g["batch"])
    b = synthetic_batch(**data)
    return b.z, b.pos, b.batch


def targets(n_graphs, n_atoms):
    gen = torch.Generator().manual_seed(TARGET_SEED)
    return torch.randn(n_graphs, 1, generator=gen), torch.randn(n_atoms, 3, generator=gen)


def force_loss(e, f, y, ft):
    l1 = torch.nn.L1Loss()
    return l1(e, y) + P_FORCE * l1(f, ft)


def _np(t):
    return t.detach().cpu().numpy()


def run_case(method, name):
    from oracle import restated
    ctor, data, wseed = CASES[name]
    torch.manual_seed(0)
    model = method.ComENet(**ctor)
    sd = formula_state_dict(model.state_dict(), seed=wseed)
    model.load_state_dict(sd)
    model.eval()
    z, pos0, batch = inputs(data)
    n_graphs = int(batch.max()) + 1
    y, ft = targets(n_graphs, pos0.size(0))
    out = {"z": _np(z), "pos": _np(pos0), "batch": _np(batch), "y": _np(y), "force_target": _np(ft)}
    for dtype, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
        m = model.to(dtype)
        pos = pos0.to(dtype).clone().requires_grad_(True)
        e = m(Batch(z=z, pos=pos, batch=batch))
        f = -torch.autograd.grad(e.sum(), pos, create_graph=(tag == "f32"))[0]
        out[f"energy_{tag}"], out[f"force_{tag}"] = _np(e), _np(f)
    names = [k for k, _ in model.named_parameters()]
    grads = torch.autograd.grad(force_loss(e, f, y, ft), [p for _, p in model.named_parameters()])
    out.update(gradient_record(names, grads))
    # the restatement: energies bit for bit, forces and parameter gradients at fp32 level
    sd_r = {k: v.clone().requires_grad_(k in names) for k, v in sd.items()}
    pos = pos0.clone().requires_grad_(True)
    u = restated.comenet_forward(sd_r, z, pos, batch, **restated_kwargs(ctor))
    fr = -torch.autograd.grad(u.sum(), pos, create_graph=True)[0]
    assert np.array_equal(_np(u), out["energy_f32"]), (name, _np(u), out["energy_f32"])
    ferr = float(np.abs(_np(fr) - out["force_f32"]).max() / np.abs(out["force_f32"]).max())
    assert ferr < FORCE_TOL, (name, ferr)
    grads_r = torch.autograd.grad(force_loss(u, fr, y, ft), [sd_r[k] for k in names])
    gerr = max(float(np.abs(_np(a) - _np(b)).max() / max(float(b.abs().max()), 1e-30)) for a, b in zip(grads_r, grads))
    assert gerr < GRAD_TOL, (name, gerr)
    print(name, "E", out["energy_f32"].ravel(), f"restated force rel-err {ferr:.2e}, grad rel-err {gerr:.2e}",
          f"f32 vs f64 force {np.abs(out['force_f32'] - out['force_f64']).max() / np.abs(out['force_f64']).max():.2e}")
    model.to(torch.float32)
    shapes = {k: list(v.shape) for k, v in model.state_dict().items()}
    return out, shapes


def main():
    torch.set_num_threads(FIXTURE_THREADS)
    method = load_reference()
    arrays, shapes = {}, {}
    for name in CASES:
        out, shapes[name] = run_case(method, name)
        arrays.update({f"{name}/{k}": v for k, v in out.items()})
    np.savez_compressed(os.path.join(GOLD, "comenet_forces.npz"), **arrays)
    with open(os.path.join(GOLD, "comenet_forces_shapes.json"), "w") as fh:
        json.dump(shapes, fh)


if __name__ == "__main__":
    main()
