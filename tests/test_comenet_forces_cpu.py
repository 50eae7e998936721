"""CPU tests of the ComENet force fixture (tests/golden/comenet_forces.npz, written by the unmodified reference through
oracle/gen_golden_comenet_forces.py): the restatement the GPU tests build their comparator on reproduces the
reference's forces and force-training gradients, the comparator (tests/comenet_force_ref.py) computes the same values
and well-conditioned forces, ComENet(energy_and_force=True) holds the reference's parameters, and the new C entry points
have ctypes signatures."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, ROOT, formula_state_dict
from oracle import restated
from oracle.gen_golden_comenet_forces import (CASES, FIXTURE_THREADS, force_loss, projection, restated_kwargs)


@pytest.fixture(autouse=True)
def _fixture_thread_count():
    saved = torch.get_num_threads()
    torch.set_num_threads(FIXTURE_THREADS)        # one thread: the reference's force sums are order-sensitive
    yield
    torch.set_num_threads(saved)


def _fixture(name):
    g = np.load(os.path.join(GOLDEN, "comenet_forces.npz"))
    with open(os.path.join(GOLDEN, "comenet_forces_shapes.json")) as fh:
        shapes = json.load(fh)[name]
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}, shapes


@pytest.mark.parametrize("name", list(CASES))
def test_restated_forces_and_force_training_gradients_match_reference(name):
    ctor, _, wseed = CASES[name]
    g, shapes = _fixture(name)
    sd = formula_state_dict({k: torch.empty(s) for k, s in shapes.items()}, seed=wseed)
    names = list(shapes)                        # every state-dict entry of ComENet is a parameter
    sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    pos = torch.from_numpy(g["pos"]).clone().requires_grad_(True)
    u = restated.comenet_forward(sd, torch.from_numpy(g["z"]), pos, torch.from_numpy(g["batch"]),
                                 **restated_kwargs(ctor))
    assert np.array_equal(u.detach().numpy(), g["energy_f32"])
    f = -torch.autograd.grad(u.sum(), pos, create_graph=True)[0]
    assert np.abs(f.detach().numpy() - g["force_f32"]).max() < 1e-5 * np.abs(g["force_f32"]).max()
    grads = torch.autograd.grad(force_loss(u, f, torch.from_numpy(g["y"]), torch.from_numpy(g["force_target"])),
                                [sd[k] for k in names])
    checked = 0
    for idx, (k, gr) in enumerate(zip(names, grads)):
        if f"grad/{k}" in g:
            want = g[f"grad/{k}"]
            assert np.abs(gr.numpy() - want).max() <= 1e-4 * max(np.abs(want).max(), 1e-30), k
        else:
            r = projection(gr.numel(), idx)
            got = gr.double().reshape(-1) @ r
            bound = gr.double().abs().reshape(-1) @ r.abs()
            assert (np.abs(got.numpy() - g[f"grad_proj/{k}"]) <= 1e-4 * bound.numpy()).all(), k
        checked += 1
    assert checked == len(names) > 40


@pytest.mark.parametrize("name", list(CASES))
def test_comparator_has_the_restated_values_and_order_independent_forces(name):
    """tests/comenet_force_ref.py: the restatement's angles bit for bit; with the aliased cross products held constant
    its forces no longer depend on the order of the CPU's multi-threaded sums (the plain restatement's change by O(1)
    from run to run there, see the module docstring of comenet_force_ref)."""
    import comenet_force_ref as cfr
    ctor, _, wseed = CASES[name]
    g, shapes = _fixture(name)
    sd = formula_state_dict({k: torch.empty(s) for k, s in shapes.items()}, seed=wseed)
    z, pos, batch = (torch.from_numpy(g[k]) for k in ("z", "pos", "batch"))
    ei = restated.radius_graph(pos, ctor["cutoff"], batch)
    for a, b in zip(restated.comenet_geometry(pos, ei, pos.size(0), ctor["cutoff"]),
                    cfr.comenet_geometry(pos, ei, pos.size(0), ctor["cutoff"])):
        assert torch.equal(a, b)
    u = cfr.comenet_forward(sd, z, pos, batch, **restated_kwargs(ctor))
    assert np.array_equal(u.numpy(), g["energy_f32"])
    torch.set_num_threads(8)
    forces = []
    for _ in range(3):
        p = pos.clone().requires_grad_(True)
        u = cfr.comenet_forward(sd, z, p, batch, **restated_kwargs(ctor))
        forces.append(torch.autograd.grad(u.sum(), p)[0])
    for f in forces[1:]:
        assert float((f - forces[0]).abs().max()) < 1e-5 * float(forces[0].abs().max())


@pytest.mark.parametrize("name", list(CASES))
def test_state_dict_shapes_and_parameter_count_match_reference(name):
    from dig_b200.threedgraph.method import ComENet
    ctor, _, _ = CASES[name]
    _, shapes = _fixture(name)
    model = ComENet(energy_and_force=True, **ctor)
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == shapes
    assert sum(p.numel() for p in model.parameters()) == sum(int(np.prod(s)) for s in shapes.values())
    assert model.energy_and_force
    # the reference's positional arguments keep their meaning
    m2 = ComENet(ctor["cutoff"], ctor.get("num_layers", 4), ctor.get("hidden_channels", 256),
                 ctor.get("middle_channels", 64), 1, 3, 2, ctor.get("num_output_layers", 3))
    assert not m2.energy_and_force
    assert {k: list(v.shape) for k, v in m2.state_dict().items()} == shapes


def test_new_entry_points_have_ctypes_signatures():
    import ctypes
    import re
    from dig_b200 import _lib
    with open(os.path.join(ROOT, "include", "dig3d.h")) as fh:
        text = re.sub(r"/\*.*?\*/", " ", fh.read(), flags=re.S)
    decls = dict(re.findall(r"\b(dig3d_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", text, flags=re.S))
    for name in ("dig3d_comenet_features_bwd", "dig3d_comenet_features_tangent", "dig3d_graphnorm_tangent",
                 "dig3d_graphnorm_tangent_bwd"):
        params = [p.strip() for p in " ".join(decls[name].split()).split(",")]
        sig = _lib.SIGNATURES[name]
        assert len(params) == len(sig), name
        for decl, ct in zip(params, sig):
            if "*" in decl:
                assert ct is ctypes.c_void_p, (name, decl)
            elif "double" in decl:
                assert ct is ctypes.c_double, (name, decl)
            elif "int64_t" in decl:
                assert ct is ctypes.c_int64, (name, decl)
            else:
                assert ct is ctypes.c_int32, (name, decl)
