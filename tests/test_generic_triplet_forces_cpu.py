"""CPU tests of the generic-triplet-branch force fixture (tests/golden/generic_forces.npz, written by the unmodified
reference through oracle/gen_golden_generic_forces.py): the restatement the GPU tests compare against reproduces the
reference at these widths, and the drop-in classes hold the reference's parameters."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, formula_state_dict
from oracle import FIXTURE_THREADS, restated
from oracle.gen_golden_generic_forces import CASES, restated_kwargs


@pytest.fixture(autouse=True)
def _fixture_thread_count():
    saved = torch.get_num_threads()
    torch.set_num_threads(FIXTURE_THREADS)
    yield
    torch.set_num_threads(saved)


def _fixture(name):
    g = np.load(os.path.join(GOLDEN, "generic_forces.npz"))
    with open(os.path.join(GOLDEN, "generic_forces_shapes.json")) as fh:
        shapes = json.load(fh)[name]
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}, shapes


@pytest.mark.parametrize("name", list(CASES))
def test_restated_matches_reference_energies_and_forces(name):
    model_name, ctor, wseed = CASES[name]
    g, shapes = _fixture(name)
    sd = formula_state_dict({k: torch.empty(s) for k, s in shapes.items()}, seed=wseed)
    pos = torch.from_numpy(g["pos"]).clone().requires_grad_(True)
    u = restated.dimenet_family_forward(sd, torch.from_numpy(g["z"]), pos, torch.from_numpy(g["batch"]),
                                        **restated_kwargs(model_name, ctor))
    assert np.array_equal(u.detach().numpy(), g["energy_f32"])
    f = -torch.autograd.grad(u.sum(), pos)[0].numpy()
    assert np.abs(f - g["force_f32"]).max() < 1e-5 * np.abs(g["force_f64"]).max()


@pytest.mark.parametrize("name", list(CASES))
def test_state_dict_shapes_match_reference(name):
    from dig_b200.threedgraph import method
    model_name, ctor, _ = CASES[name]
    _, shapes = _fixture(name)
    model = getattr(method, model_name)(energy_and_force=True, **ctor)
    assert model._triplet_generic
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == shapes
