"""GPU edge cases: empty / ragged inputs, isolated atoms, the neighbour cap, error behaviour."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_isolated_atoms_and_single_atom_graphs():
    from dig_b200 import ops
    from oracle import restated
    dev = torch.device("cuda:0")
    # graph 0: two atoms 20 A apart (no edges); graph 1: one atom; graph 2: a bonded triple
    pos = torch.tensor([[0, 0, 0], [20, 0, 0], [5, 5, 5], [0, 0, 0], [1, 0, 0], [0, 1.2, 0]],
                       dtype=torch.float32, device=dev)
    batch = torch.tensor([0, 0, 1, 2, 2, 2], device=dev)
    gr = ops.build_graph(pos, batch, 5.0)
    ops.triplet_geometry(gr, pos, use_torsion=True, want_idx64=True)
    ei = restated.radius_graph(pos, 5.0, batch)
    res = restated.xyz_to_dat(pos, ei, 6, use_torsion=True)
    assert torch.equal(gr.edge_index, ei) and gr.n_edges == 6
    assert torch.equal(gr.idx_kj64, res[-2]) and torch.equal(gr.torsion, res[2])


def test_no_edges_at_all():
    from dig_b200.threedgraph.method import DimeNetPP
    from dig_b200.data import Batch
    dev = torch.device("cuda:0")
    model = DimeNetPP().to(dev)
    b = Batch(z=torch.tensor([1, 6], device=dev), pos=torch.tensor([[0., 0, 0], [50, 0, 0]], device=dev),
              batch=torch.tensor([0, 1], device=dev))
    with torch.no_grad():
        u = model(b)
    assert u.shape == (2, 1) and torch.isfinite(u).all()


def test_neighbour_cap_matches_torch_cluster_semantics():
    from dig_b200 import ops
    from oracle import restated
    dev = torch.device("cuda:0")
    torch.manual_seed(1)
    pos = (torch.rand(90, 3) * 3.0).to(dev)       # dense: > 33 candidates per node
    batch = torch.zeros(90, dtype=torch.long, device=dev)
    gr = ops.build_graph(pos, batch, 6.0)
    ei = restated.radius_graph(pos, 6.0, batch)
    assert torch.equal(gr.edge_index, ei)
    deg = torch.bincount(ei[1], minlength=90)
    assert int(deg.max()) == 33 and int(deg.min()) == 32
    ops.triplet_geometry(gr, pos, use_torsion=True, want_idx64=True)
    res = restated.xyz_to_dat(pos, ei, 90, use_torsion=True)
    assert torch.equal(gr.idx_kj64, res[-2]) and torch.equal(gr.idx_ji64, res[-1])
    assert torch.equal(gr.angle, res[1]) and torch.equal(gr.torsion, res[2])


def test_ragged_batch_with_empty_graph_slot():
    from dig_b200 import ops
    dev = torch.device("cuda:0")
    pos = torch.rand(7, 3, device=dev)
    batch = torch.tensor([0, 0, 0, 2, 2, 2, 2], device=dev)     # graph 1 is empty
    gr = ops.build_graph(pos, batch, 5.0, num_graphs=3)
    assert gr.graph_ptr.tolist() == [0, 3, 3, 7]
    assert gr.n_edges == 3 * 2 + 4 * 3


def test_errors_are_loud():
    from dig_b200 import ops
    from dig_b200._lib import Dig3dError
    dev = torch.device("cuda:0")
    with pytest.raises(ValueError):
        ops.build_graph(torch.rand(4, 2, device=dev), None, 5.0)
    with pytest.raises(TypeError):
        ops.build_graph(torch.rand(4, 3, device=dev, dtype=torch.float64), None, 5.0)
    with pytest.raises(Dig3dError):
        ops.build_graph(torch.rand(4, 3, device=dev), torch.zeros(4, dtype=torch.long, device=dev), 5.0,
                        max_num_neighbors=200)


@pytest.mark.parametrize("cls_name", ["SphereNet", "DimeNetPP", "SchNet"])      # the reference ComENet indexes out of range for atoms without neighbours (comenet.py:305-327)
def test_training_path_with_isolated_atoms_and_no_triplets(cls_name):
    """Training forward+backward (and forces where the model has them) on a batch with a no-edge graph, a single atom, a
    diatomic (edges but no triplets) and a bonded quadruple; then on a batch with no edges at all."""
    from dig_b200.data import Batch
    from dig_b200.threedgraph import method
    from oracle import restated
    from helpers import formula_state_dict, rel_err
    dev = torch.device("cuda:0")
    pos = torch.tensor([[0, 0, 0], [30, 0, 0], [5, 5, 5], [0, 0, 0], [1.1, 0, 0],
                        [0, 0, 0], [1, 0.1, 0], [0.2, 1.2, 0], [0.9, 1.0, 0.8]], dtype=torch.float32, device=dev)
    batch = torch.tensor([0, 0, 1, 2, 2, 3, 3, 3, 3], device=dev)
    z = torch.tensor([1, 6, 7, 8, 1, 6, 1, 1, 8], device=dev)
    kw = dict(cutoff=5.0)
    if cls_name in ("SphereNet", "DimeNetPP", "SchNet"):
        kw["energy_and_force"] = True
    if cls_name == "SchNet":
        kw.update(num_layers=2, hidden_channels=32, num_filters=32)
    model = getattr(method, cls_name)(**kw)
    sd = formula_state_dict(model.state_dict(), seed=21)
    model.load_state_dict(sd)
    model = model.to(dev)
    b = Batch(z=z, pos=pos.clone(), batch=batch)
    out = model(b)
    assert out.shape == (4, 1) and torch.isfinite(out).all()
    target = torch.tensor([[0.1], [-0.2], [0.3], [0.4]], device=dev)
    torch.nn.functional.l1_loss(out, target).backward()
    sd_ref = {k: v.to(dev).clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    pos2 = pos.clone().requires_grad_(True)
    fwd = {"SphereNet": restated.spherenet_forward, "DimeNetPP": restated.dimenetpp_forward,
           "SchNet": lambda s, *a, **k: restated.schnet_forward(s, *a, num_layers=2, **k)}[cls_name]
    ref = fwd(sd_ref, z, pos2, batch, cutoff=5.0, num_graphs=4)
    torch.nn.functional.l1_loss(ref, target).backward()
    assert rel_err(out.detach().cpu().numpy(), ref.detach().cpu().numpy()) < 1e-5
    for name, p in model.named_parameters():
        r = sd_ref[name].grad
        scale = max(float(r.abs().max()), 1e-6)
        assert p.grad is not None and float((p.grad - r).abs().max()) / scale < 2e-4, name
    if "energy_and_force" in kw:
        scale = max(float(pos2.grad.abs().max()), 1e-6)
        assert float((b.pos.grad - pos2.grad).abs().max()) / scale < 1e-4
    # no edges at all: still differentiable, finite
    b2 = Batch(z=z[:3], pos=torch.tensor([[0., 0, 0], [40, 0, 0], [80, 0, 0]], device=dev),
               batch=torch.tensor([0, 0, 1], device=dev))
    model.zero_grad()
    out2 = model(b2)
    out2.sum().backward()
    assert out2.shape == (2, 1) and torch.isfinite(out2).all()


def test_out_of_range_indices_raise_instead_of_reading_out_of_bounds():
    """ADVICE r1: an atomic number outside the embedding table, a batch id >= num_graphs or an unsorted batch vector
    raise ValueError at the forward's one sync point (the reference's nn.Embedding / scatter assert on the device)."""
    from dig_b200 import ops
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph.method import DimeNetPP, SchNet
    dev = torch.device("cuda:0")
    b = synthetic_batch(3, "qm9", seed=1).to(dev)
    model = DimeNetPP().to(dev)
    with torch.no_grad():
        ok = model(b)
        assert torch.isfinite(ok).all()
        bad = synthetic_batch(3, "qm9", seed=1).to(dev)
        bad.z[4] = 95
        with pytest.raises(ValueError, match="atomic numbers"):
            model(bad)
        bad.z[4] = -1
        with pytest.raises(ValueError, match="atomic numbers"):
            SchNet(num_layers=2, hidden_channels=32, num_filters=32).to(dev)(bad)
    with pytest.raises(ValueError, match="batch ids"):
        ops.build_graph(b.pos, b.batch, 5.0, num_graphs=2)
    unsorted = b.batch.clone()
    unsorted[0] = 2
    with pytest.raises(ValueError, match="not sorted"):
        ops.build_graph(b.pos, unsorted, 5.0, num_graphs=3)
    g = ops.build_graph(b.pos, b.batch, 5.0, num_graphs=3)       # the context is still healthy afterwards
    assert g.n_edges > 0


def test_out_edge_lists_of_the_graph_build():
    """out_ptr / out_list / pos_in (CSR by SOURCE, left by the graph build for the triplet kernels) against their
    definition computed from edge_index: capped dense graph (out-degree != in-degree), isolated atom, > 32 atoms per
    molecule -- and the triplet gather / projection are bit-identical with and without the lists."""
    import ctypes
    from dig_b200 import ops
    from dig_b200.data import synthetic_batch, collate, Molecule
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    dense = (torch.rand(70, 3) * 3.0)
    mols = synthetic_batch(6, "qm9", seed=9, variable=True)
    b = collate([Molecule(torch.full((70,), 6), dense), Molecule(torch.tensor([8]), torch.tensor([[90.0, 0, 0]])),
                 Molecule(mols.z, mols.pos + 200.0)]).to(dev)
    b.batch = torch.cat([torch.zeros(70), torch.ones(1), torch.full((mols.z.numel(),), 2.0)]).long().to(dev)
    g = ops.build_graph(b.pos, b.batch, 5.0, num_graphs=3)
    src, dst = g.edge_index[0].cpu().numpy(), g.edge_index[1].cpu().numpy()
    n, e = g.n_nodes, g.n_edges
    out_ptr, out_list, pos_in = g.out_ptr.cpu().numpy(), g.out_list.cpu().numpy(), g.pos_in.cpu().numpy()
    row_ptr = g.row_ptr.cpu().numpy()
    assert np.array_equal(out_ptr, np.concatenate([[0], np.cumsum(np.bincount(src, minlength=n))]))
    assert not np.array_equal(np.diff(out_ptr), np.diff(row_ptr))           # the cap broke the symmetry somewhere
    order = np.lexsort((dst, src))                                           # by source, then target
    assert np.array_equal(out_list, order)
    for ed in range(e):
        j, i = src[ed], dst[ed]
        ins = src[row_ptr[j]:row_ptr[j + 1]]
        hit = np.nonzero(ins == i)[0]
        assert pos_in[ed] == (hit[0] if hit.size else ins.size)
    # consumers: lists vs search
    ops.triplet_geometry(g, b.pos, use_torsion=True, want_idx=False)
    t = g.n_triplets
    x_down = torch.randn(e, 64, device=dev)
    sbf_p, t_p = torch.randn(t, 8, device=dev), torch.randn(t, 8, device=dev)
    w_s, w_t = torch.randn(64, 8, device=dev), torch.randn(64, 8, device=dev)
    bess = torch.randn(e, 42, device=dev)
    w1s, w1t = torch.randn(32, 42, device=dev), torch.randn(32, 294, device=dev)
    lists = (g.out_ptr, g.out_list, g.pos_in)
    outs = []
    for use in (True, False):
        g.out_ptr, g.out_list, g.pos_in = lists if use else (None, None, None)
        m = torch.full((e, 64), float("nan"), device=dev)
        ops.triplet_gather(x_down, ctypes.c_void_p(sbf_p.data_ptr()), ctypes.c_void_p(t_p.data_ptr()), g,
                           w_s.data_ptr(), w_t.data_ptr(), m, ops._stream())
        sp, tp = ops.triplet_basis_project(g, bess, 0, w1s, w1t)
        outs.append((m, sp.clone(), tp.clone()))
    g.out_ptr, g.out_list, g.pos_in = lists
    for a, c in zip(outs[0], outs[1]):
        assert torch.isfinite(a).all() and torch.equal(a, c)


@pytest.mark.parametrize("cls_name", ["SphereNet", "DimeNetPP"])
def test_inference_paths_with_isolated_atoms_and_an_empty_graph_slot(cls_name):
    """The inference forward (cached plan, fused chain, out-edge lists) on a batch with an isolated atom, a two-atom
    molecule without triplets and an empty graph slot: bit-identical to the op-by-op chain and within 1e-5 of the
    oracle."""
    from dig_b200 import ops
    from dig_b200.data import synthetic_molecules, collate, Molecule
    from dig_b200.threedgraph import method
    from helpers import formula_state_dict, rel_err, sphere_forward_op_by_op
    from oracle import restated
    dev = torch.device("cuda:0")
    m0, m1 = synthetic_molecules(2, "qm9", seed=11, variable=True)
    items = [Molecule(m0.z, m0.pos), Molecule(torch.tensor([8]), torch.tensor([[60.0, 0.0, 0.0]])),
             Molecule(torch.tensor([6, 1]), torch.tensor([[0.0, 0.0, 0.0], [1.1, 0.0, 0.0]])), Molecule(m1.z, m1.pos)]
    b = collate(items).to(dev)
    b.batch = torch.where(b.batch >= 3, b.batch + 1, b.batch)            # graph 3 is an empty slot
    b.num_graphs = 5
    model = getattr(method, cls_name)()
    sd = formula_state_dict(model.state_dict(), seed=6)
    model.load_state_dict(sd)
    model = model.to(dev).eval()
    with torch.no_grad():
        lean = model(b)
        general = sphere_forward_op_by_op(model, b)
        ref = restated.dimenet_family_forward({k: v.to(dev) for k, v in sd.items()}, b.z, b.pos, b.batch,
                                              torsion=cls_name == "SphereNet", num_graphs=5)
    assert not ops.h16_overflow()
    assert lean.shape == (5, 1) and torch.isfinite(lean).all()
    assert torch.equal(lean, general)
    assert float(lean[3].abs().max()) == 0.0                              # the empty slot sums nothing
    assert rel_err(lean.cpu().numpy(), ref.cpu().numpy()) < 1e-5
