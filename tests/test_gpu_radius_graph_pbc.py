"""GPU tests of the periodic radius graph kernels (csrc/graph_pbc.cu) and of ComENet-OCP with otf_graph=True.

The kernels' edge_index, cell_offsets and neighbors are bit-equal to the torch restatement of ocpmodels'
radius_graph_pbc (oracle/ocp_pbc.py, checked on the CPU in tests/test_radius_graph_pbc_cpu.py) run on the same GPU;
the model built with otf_graph=True matches the oracle forward and the fixture of the unmodified reference."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import formula_state_dict, rel_err

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _batch(cells, fracs, dev):
    from dig_b200.data import Batch
    cells = [torch.as_tensor(c, dtype=torch.float32) for c in cells]
    pos = torch.cat([torch.as_tensor(f, dtype=torch.float32).reshape(-1, 3) @ c for f, c in zip(fracs, cells)])
    natoms = torch.tensor([len(f) for f in fracs], dtype=torch.int64)
    return Batch(pos=pos, cell=torch.stack(cells), natoms=natoms).to(dev)


def _tri(a, b, c, s=(0.0, 0.0, 0.0)):
    return [[a, 0.0, 0.0], [s[0] * b, b, 0.0], [s[1] * c, s[2] * c, c]]


def _cases(dev):
    from dig_b200.data import synthetic_pbc_batch
    gen = torch.Generator().manual_seed(3)
    oc20 = synthetic_pbc_batch(64, natoms=73, seed=0).to(dev)
    # batch-maximum image range pads the large cells: rep 3 from the 2.4 A axis, rep 1 on its own for the 12 A cell
    mixed = _batch([_tri(12.0, 11.0, 13.0, (0.2, 0.1, 0.0)), _tri(6.0, 5.0, 2.4, (0.3, 0.0, 0.2)),
                    _tri(9.0, 9.0, 14.0, (0.3, 0.0, 0.0))],
                   [torch.rand(20, 3, generator=gen), torch.rand(4, 3, generator=gen), torch.rand(15, 3, generator=gen)],
                   dev)
    # simple cubic lattice, a = 2.5 A, as a 2 x 2 x 2 supercell: every distance is exact, ties everywhere
    lattice = torch.tensor([[x, y, z] for x in (0, 0.5) for y in (0, 0.5) for z in (0, 0.5)])
    dense = _batch([_tri(5.0, 5.0, 5.0), _tri(5.0, 5.0, 5.0)], [lattice, lattice], dev)
    one = _batch([_tri(3.0, 3.0, 3.0)], [torch.zeros(1, 3)], dev)
    # a lone atom in a 20 A cell (no neighbour within 6 A, not even its own images) and an empty structure, mid-batch
    gap = _batch([_tri(8.0, 8.0, 8.0), _tri(20.0, 20.0, 20.0), _tri(7.0, 7.0, 7.0), _tri(9.0, 8.5, 10.0, (0.1, 0.2, 0.0))],
                 [torch.rand(10, 3, generator=gen), torch.full((1, 3), 0.5), torch.zeros(0, 3),
                  torch.rand(12, 3, generator=gen)], dev)
    small = synthetic_pbc_batch(4, natoms=40, seed=2).to(dev)
    return [("oc20_64x73", oc20, 50), ("mixed_cells", mixed, 50), ("dense_ties_cap20", dense, 20),
            ("dense_ties_cap7", dense, 7), ("one_atom", one, 12), ("one_atom_nocap", one, 0),
            ("zero_edges_mid_batch", gap, 50), ("cap_zero", small, 0), ("cap_negative", small, -1)]


CASE_IDS = ["oc20_64x73", "mixed_cells", "dense_ties_cap20", "dense_ties_cap7", "one_atom", "one_atom_nocap",
            "zero_edges_mid_batch", "cap_zero", "cap_negative"]


@pytest.mark.parametrize("case", CASE_IDS)
def test_kernel_bit_equal_to_restatement(case):
    from dig_b200.threedgraph.utils import radius_graph_pbc
    from oracle import ocp_pbc
    dev = torch.device("cuda:0")
    _, b, cap = next(c for c in _cases(dev) if c[0] == case)
    ei, off, nb = radius_graph_pbc(b, 6.0, cap)
    ei_r, off_r, nb_r = ocp_pbc.radius_graph_pbc(b, 6.0, cap)
    assert ei.dtype == torch.int64 and off.dtype == torch.float32 and nb.dtype == torch.int64
    assert ei.shape == ei_r.shape, (ei.shape, ei_r.shape)
    assert torch.equal(ei, ei_r) and torch.equal(off, off_r) and torch.equal(nb, nb_r)
    assert int(nb.sum()) == ei.size(1)
    if case == "zero_edges_mid_batch":
        assert nb.tolist()[1:3] == [0, 0] and nb[0] > 0 and nb[3] > 0
    if case.startswith("dense_ties"):
        assert torch.all(torch.bincount(ei[1], minlength=b.pos.size(0)) == cap)
    if case == "one_atom_nocap":
        assert ei.size(1) == 32
    if case == "mixed_cells":
        reps = ocp_pbc.image_range(b.cell, 6.0)
        assert reps.max(0).values.tolist() != reps[0].tolist()          # structure 0 is padded by the batch maximum


def test_two_runs_are_bit_identical():
    from dig_b200 import ops
    from dig_b200.data import synthetic_pbc_batch
    b = synthetic_pbc_batch(64, natoms=73, seed=1).to("cuda:0")
    a = ops.radius_graph_pbc(b.pos, b.cell, b.natoms, 6.0, 50)
    c = ops.radius_graph_pbc(b.pos, b.cell, b.natoms, 6.0, 50)
    assert all(torch.equal(x, y) for x, y in zip(a, c))


def test_bad_input_raises_value_error():
    from dig_b200 import ops
    dev = torch.device("cuda:0")
    pos = torch.rand(4, 3, device=dev)
    cell = (5.0 * torch.eye(3, device=dev))[None]
    flat = cell.clone()
    flat[0, 2] = flat[0, 0] + flat[0, 1]                                     # coplanar lattice vectors: zero volume
    with pytest.raises(ValueError, match="volume"):
        ops.radius_graph_pbc(pos, flat, torch.tensor([4], device=dev), 6.0, 50)
    nan = cell.clone()
    nan[0, 1, 1] = float("nan")
    with pytest.raises(ValueError, match="volume"):
        ops.radius_graph_pbc(pos, nan, torch.tensor([4], device=dev), 6.0, 50)
    for natoms in ([3], [5], [-1]):
        with pytest.raises(ValueError, match="natoms"):
            ops.radius_graph_pbc(pos, cell, torch.tensor(natoms, device=dev), 6.0, 50)
    with pytest.raises(ValueError, match="natoms"):
        ops.radius_graph_pbc(pos, cell.repeat(2, 1, 1), torch.tensor([2, 1], device=dev), 6.0, 50)
    # the library is still usable after a rejected call
    ei, _, nb = ops.radius_graph_pbc(pos, cell, torch.tensor([4], device=dev), 6.0, 50)
    assert int(nb.sum()) == ei.size(1) > 0


def _ocp_model(dev, otf_graph):
    from dig_b200.threedgraph.method.comenet_ocp import ComENet
    g = np.load(os.path.join(GOLDEN, "comenet_ocp_otf.npz"))
    with open(os.path.join(GOLDEN, "comenet_ocp_checkpoint_shapes.json")) as fh:
        pin = json.load(fh)
    sd = formula_state_dict({k[len("module."):]: torch.empty(s) for k, s in pin["keys"].items()},
                            seed=int(g["weight_seed"]))
    sd["lin_out.weight"] = sd["lin_out.weight"] + 0.05
    model = ComENet(0, 0, hidden_channels=256, num_blocks=4, cutoff=6.0, num_radial=3, num_spherical=2,
                    otf_graph=otf_graph)
    model.load_state_dict({"module." + k: v for k, v in sd.items()})
    return model.to(dev), sd


def _otf_batch(dev):
    from dig_b200.data import Batch
    g = np.load(os.path.join(GOLDEN, "comenet_ocp_otf.npz"))
    b = Batch(**{k: torch.from_numpy(g[k]) for k in ("atomic_numbers", "pos", "tags", "cell", "natoms", "batch")})
    b.num_graphs = int(g["natoms"].size)
    return b.to(dev), g


def test_comenet_ocp_otf_graph():
    """ComENet(otf_graph=True) on a batch without edges: builds the graph on the GPU and writes it onto the batch;
    energies within 1e-5 and every parameter gradient within 1e-4 of the oracle forward on the restated graph;
    bit-identical to otf_graph=False on the GPU-built graph; within 2e-5 of the unmodified reference's fixture."""
    from oracle import ocp_pbc, restated
    dev = torch.device("cuda:0")
    model, sd = _ocp_model(dev, otf_graph=True)
    b, g = _otf_batch(dev)
    assert not hasattr(b, "edge_index")
    out = model(b)
    for k in ("edge_index", "cell_offsets", "neighbors"):
        assert isinstance(getattr(b, k, None), torch.Tensor) and getattr(b, k).is_cuda, k
    ei_r, off_r, nb_r = ocp_pbc.radius_graph_pbc(b, 6.0, 50)
    assert torch.equal(b.edge_index, ei_r) and torch.equal(b.cell_offsets, off_r) and torch.equal(b.neighbors, nb_r)
    # oracle forward on the restated graph
    b_ref, _ = _otf_batch(dev)
    b_ref.edge_index, b_ref.cell_offsets, b_ref.neighbors = ei_r, off_r, nb_r
    sd_ref = {k: v.to(dev).clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    ref = restated.comenet_ocp_forward(sd_ref, b_ref, cutoff=6.0)
    assert out.shape == ref.shape == (3, 1)
    assert rel_err(out.detach().cpu().numpy(), ref.detach().cpu().numpy()) < 1e-5
    out.sum().backward()
    ref.sum().backward()
    for name, p in model.named_parameters():
        r = sd_ref[name].grad
        assert p.grad is not None and r is not None, name
        assert rel_err(p.grad.cpu().numpy(), r.cpu().numpy()) < 1e-4, name
    # otf_graph=False over the graph the GPU just built: the same forward, bit for bit (the weight-gradient kernels
    # combine row splits with atomics, so gradients agree to rounding only)
    pre, _ = _ocp_model(dev, otf_graph=False)
    out_pre = pre(b)
    assert torch.equal(out.detach(), out_pre.detach())
    out_pre.sum().backward()
    for (name, p), (_, q) in zip(model.named_parameters(), pre.named_parameters()):
        assert rel_err(p.grad.cpu().numpy(), q.grad.cpu().numpy()) < 1e-5, name
    # the unmodified reference (CPU, fp32, graph from the restatement)
    assert rel_err(out.detach().cpu().numpy(), g["energy_f32"]) < 2e-5
