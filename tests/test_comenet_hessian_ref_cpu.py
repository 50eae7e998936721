"""CPU test of the comparator of ComENet's Hessian tests (tests/comenet_hessian_ref.py), in fp64.

The reference itself gives no usable Hessian (DESIGN.md §6): on every graph an aliased cross product (plane1 =
(-pos_ji) x pos_ji on each node's nearest in-edge) is exactly zero in fp64, and the double backward of its norm and of
phi = atan2(0, 0) is NaN, which reaches every entry through the network.  Nor can its forces be differenced: the signed
zeros of the aliased products pick the branch of atan2 (0 or pi after the fold), which a step of any size can flip.  So
the comparator is held to the reference's fp64 forces (tests/golden/comenet_forces.npz) and to a finite, symmetric
double backward.  The GPU tests compare the kernels and models with its fp64 variant at the kernels' fp32 inputs
(comenet_hessian_ref.geometry_at_kernel_inputs)."""
import json
import os

import numpy as np
import pytest
import torch

import comenet_hessian_ref
from helpers import GOLDEN, formula_state_dict

CASES = {"aspirin_default": dict(cutoff=5.0, num_layers=2),
         "aspirin_generic": dict(cutoff=5.0, num_layers=2, num_output_layers=2)}


def _case(name):
    g = np.load(os.path.join(GOLDEN, "comenet_forces.npz"))
    with open(os.path.join(GOLDEN, "comenet_forces_shapes.json")) as fh:
        shapes = json.load(fh)[name]
    g = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}
    return g, shapes


@pytest.mark.parametrize("name", list(CASES))
def test_comparator_is_twice_differentiable_and_gives_the_reference_forces(name):
    g, shapes = _case(name)
    wseed = {"aspirin_default": 41, "aspirin_generic": 43}[name]
    sd = formula_state_dict({k: torch.empty(s) for k, s in shapes.items()}, seed=wseed)
    sd = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    z, batch = torch.from_numpy(g["z"]), torch.from_numpy(g["batch"])
    keep = batch == 0                                   # the first molecule: 21 atoms, 63 columns
    z, batch = z[keep], batch[keep]
    pos0 = torch.from_numpy(g["pos"]).double()[keep]
    kw = CASES[name]

    p = pos0.clone().requires_grad_(True)
    f = -torch.autograd.grad(comenet_hessian_ref.comenet_forward(sd, z, p, batch, **kw).sum(), p)[0]
    want_f = torch.from_numpy(g["force_f64"])[keep]
    assert float((f - want_f).abs().max() / want_f.abs().max()) < 1e-6
    n = pos0.size(0)
    hess = torch.autograd.functional.hessian(
        lambda p: comenet_hessian_ref.comenet_forward(sd, z, p, batch, **kw).sum(), pos0).reshape(3 * n, 3 * n)
    assert bool(torch.isfinite(hess).all())
    scale = float(hess.abs().max())
    assert float((hess - hess.T).abs().max()) <= 1e-12 * scale
