"""CPU test of the Hessian fixture (tests/golden/hessians.npz, written by the unmodified reference through
oracle/gen_golden_hessians.py): the restated models, which the GPU Hessian tests use as their comparator, give the
reference's fp64 Hessian in the positions (torch.autograd double backward), SchNet, DimeNet++ and SphereNet at the
default and a non-default triplet width."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, formula_state_dict
from oracle import FIXTURE_THREADS
from oracle.gen_golden_hessians import CASES, restated_forward


@pytest.fixture(autouse=True)
def _fixture_thread_count():
    saved = torch.get_num_threads()
    torch.set_num_threads(FIXTURE_THREADS)
    yield
    torch.set_num_threads(saved)


@pytest.mark.parametrize("name", list(CASES))
def test_restated_double_backward_matches_reference_hessian(name):
    model_name, ctor, wseed = CASES[name]
    g = np.load(os.path.join(GOLDEN, "hessians.npz"))
    with open(os.path.join(GOLDEN, "hessians_shapes.json")) as fh:
        shapes = json.load(fh)[name]
    g = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}
    sd = formula_state_dict({k: torch.from_numpy(g["buffer/" + k]) if "buffer/" + k in g else torch.empty(s)
                             for k, s in shapes.items()}, seed=wseed)
    sd = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    z, batch = torch.from_numpy(g["z"]), torch.from_numpy(g["batch"])
    pos = torch.from_numpy(g["pos"]).double()
    n = pos.size(0)
    hess = torch.autograd.functional.hessian(lambda p: restated_forward(model_name, ctor, sd, z, p, batch).sum(), pos)
    want = g["hessian"]
    assert np.abs(hess.reshape(3 * n, 3 * n).numpy() - want).max() <= 1e-6 * np.abs(want).max()
    # molecules do not interact: the off-diagonal blocks are zero
    b = np.repeat(g["batch"], 3)
    assert np.abs(want[b[:, None] != b[None, :]]).max() == 0.0
