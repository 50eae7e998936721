"""CPU tests of the ComENet-OCP force fixture (tests/golden/comenet_ocp_forces.npz, written by the unmodified reference
through oracle/gen_golden_ocp_forces.py): the restatement the GPU tests build their comparator on reproduces the
reference's energies, forces, cell gradients and force-training gradients; the comparator
(tests/comenet_ocp_force_ref.py) computes the restatement's angles and energies bit for bit; the model class holds the
reference's parameters; the new C entry points have ctypes signatures."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, ROOT
from oracle import restated
from oracle.gen_golden_comenet_forces import FIXTURE_THREADS, force_loss, projection
from oracle.gen_golden_ocp_forces import CASES, CTOR, batch_from, make_batch, restated_kwargs, state_dict


@pytest.fixture(autouse=True)
def _fixture_thread_count():
    saved = torch.get_num_threads()
    torch.set_num_threads(FIXTURE_THREADS)        # one thread: the reference's force sums are order-sensitive
    yield
    torch.set_num_threads(saved)


def _fixture(name):
    g = np.load(os.path.join(GOLDEN, "comenet_ocp_forces.npz"))
    with open(os.path.join(GOLDEN, "comenet_ocp_forces_shapes.json")) as fh:
        shapes = json.load(fh)[name]
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}, shapes


def _sd(name, shapes):
    return state_dict({k: torch.empty(s) for k, s in shapes.items()}, CASES[name][1])


@pytest.mark.parametrize("name", list(CASES))
def test_fixture_inputs_are_the_case_batches(name):
    """The stored inputs are make_batch's, and the small cell holds self-image edges and a zero-length edge."""
    g, _ = _fixture(name)
    b = make_batch(name)
    for k in ("atomic_numbers", "pos", "cell", "edge_index", "cell_offsets", "neighbors", "batch"):
        assert np.array_equal(getattr(b, k).numpy(), g[k]), k
    if name == "small_cell":
        ei, off = g["edge_index"], g["cell_offsets"]
        self_edge = ei[0] == ei[1]
        assert (self_edge & (np.abs(off).sum(1) > 0)).sum() > 10
        assert (self_edge & (np.abs(off).sum(1) == 0)).sum() == 1


@pytest.mark.parametrize("name", list(CASES))
def test_restated_forces_cell_gradients_and_training_gradients_match_reference(name):
    g, shapes = _fixture(name)
    sd = {k: v.clone().requires_grad_(True) for k, v in _sd(name, shapes).items()}
    names = list(shapes)                        # every state-dict entry is a parameter
    b = batch_from(g)
    b.pos, b.cell = b.pos.clone().requires_grad_(True), b.cell.clone().requires_grad_(True)
    u = restated.comenet_ocp_forward(sd, b, **restated_kwargs())
    assert np.array_equal(u.detach().numpy(), g["energy"])
    dpos, dcell = torch.autograd.grad(u.sum(), [b.pos, b.cell])
    assert np.abs(-dpos.numpy() - g["force"]).max() < 1e-5 * np.abs(g["force"]).max()
    assert np.abs(dcell.numpy() - g["dcell"]).max() < 1e-5 * np.abs(g["dcell"]).max()
    b = batch_from(g)
    b.pos = b.pos.clone().requires_grad_(True)
    u = restated.comenet_ocp_forward(sd, b, **restated_kwargs())
    f = -torch.autograd.grad(u.sum(), b.pos, create_graph=True)[0]
    grads = torch.autograd.grad(force_loss(u, f, torch.from_numpy(g["y"]), torch.from_numpy(g["force_target"])),
                                [sd[k] for k in names])
    for idx, (k, gr) in enumerate(zip(names, grads)):
        if f"grad/{k}" in g:
            want = g[f"grad/{k}"]
            assert np.abs(gr.numpy() - want).max() <= 1e-4 * max(np.abs(want).max(), 1e-30), k
        else:
            r = projection(gr.numel(), idx)
            got = gr.double().reshape(-1) @ r
            bound = gr.double().abs().reshape(-1) @ r.abs()
            assert (np.abs(got.numpy() - g[f"grad_proj/{k}"]) <= 1e-4 * bound.numpy()).all(), k
    assert len(names) > 40


@pytest.mark.parametrize("name", list(CASES))
def test_comparator_has_the_restated_angles_and_energies(name):
    """tests/comenet_ocp_force_ref.py: over get_pbc_distances' vectors, the geometry with the products of vectors on one
    line held constant gives the restatement's distances and angles bit for bit, and the comparator's energies are the
    reference's."""
    import comenet_ocp_force_ref as ocfr
    from oracle.ocp_stub import get_pbc_distances
    g, shapes = _fixture(name)
    b = batch_from(g)
    out = get_pbc_distances(b.pos, b.edge_index, b.cell, b.cell_offsets, b.neighbors, return_distance_vec=True)
    n = b.pos.size(0)
    assert out["edge_index"].size(1) == b.edge_index.size(1) - (1 if name == "small_cell" else 0)
    for a, c in zip(restated.comenet_geometry(None, out["edge_index"], n, CTOR["cutoff"], vecs=out["distance_vec"]),
                    ocfr.comenet_geometry(None, out["edge_index"], n, CTOR["cutoff"], vecs=out["distance_vec"])):
        assert torch.equal(a, c)
    u = ocfr.comenet_ocp_forward(_sd(name, shapes), b, **restated_kwargs())
    assert np.array_equal(u.numpy(), g["energy"])


@pytest.mark.parametrize("name", list(CASES))
def test_periodic_line_rule_fires_on_the_tiny_cells(name):
    """The tiny cells hold cross products of two distinct self-image edges of one atom on one line (an atom's images at
    +a and -a), which the kernels and the comparator hold aliased; the slabs and the small cell hold none, so only the
    tiny cells exercise that rule."""
    import comenet_ocp_force_ref as ocfr
    from oracle.ocp_stub import get_pbc_distances
    g, _ = _fixture(name)
    b = batch_from(g)
    out = get_pbc_distances(b.pos, b.edge_index, b.cell, b.cell_offsets, b.neighbors, return_distance_vec=True)
    pairs = ocfr.periodic_line_pairs(out["edge_index"], out["distance_vec"], b.pos.size(0), CTOR["cutoff"])
    if name == "tiny_cell":
        assert pairs >= 10, pairs
    else:
        assert pairs == 0, pairs


@pytest.mark.parametrize("name", list(CASES))
def test_state_dict_shapes_match_reference(name):
    from dig_b200.threedgraph.method.comenet_ocp import ComENet
    _, shapes = _fixture(name)
    model = ComENet(**CTOR)
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == shapes


def test_new_entry_points_have_ctypes_signatures():
    import ctypes
    import re
    from dig_b200 import _lib
    with open(os.path.join(ROOT, "include", "dig3d.h")) as fh:
        text = re.sub(r"/\*.*?\*/", " ", fh.read(), flags=re.S)
    decls = dict(re.findall(r"\b(dig3d_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", text, flags=re.S))
    for name in ("dig3d_comenet_features_bwd_vec", "dig3d_comenet_features_tangent_vec", "dig3d_pbc_cell_bwd"):
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
