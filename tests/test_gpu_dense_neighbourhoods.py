"""Radius graphs and triplet geometry at any neighbour count: `radius_graph(max_num_neighbors >= 64)` (the builder
without a neighbour table, csrc/graph_dense.cu), `xyz_to_dat` / G-SphereNet's `xyztodat` at any in-degree (the
heavy-edge geometry kernel, csrc/graph.cu) and ProNet with `max_num_neighbors >= 64`, all against the restated
reference ops run by ATen on the same GPU."""
import pytest
import torch

from helpers import formula_state_dict, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
CAPS = [63, 64, 65, 100, 255, 256, 1000]


def _cluster(n=100, seed=0):
    """n atoms in a 3 A box: at cutoff 6 every atom sees every other one (in-degree n - 1)."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 3, generator=g) * 3.0


def _molecule(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 3, generator=g) * 4.0 + 0.5 * seed


def _ragged():
    """A QM9-sized molecule, the 100-atom cluster, two more molecules: one batch of four graphs."""
    parts = [_molecule(18, 1), _cluster(100, 2), _molecule(9, 3), _molecule(25, 4)]
    batch = torch.repeat_interleave(torch.arange(4), torch.tensor([p.size(0) for p in parts]))
    return torch.cat(parts).to(DEV), batch.to(DEV)


def _corner_cases():
    """An empty graph slot (graph 1), isolated atoms, coincident atoms (d2 = 0), a pair at exactly the cutoff (2.0:
    d2 == r^2 is not a hit) and one just inside it, then a dense 70-atom graph."""
    g0 = torch.tensor([[0, 0, 0], [0, 0, 0], [0, 0, 0], [0.5, 0, 0], [50, 50, 50]], dtype=torch.float32)
    g2 = torch.tensor([[10, 0, 0], [12, 0, 0], [10, 1.9999999, 0], [-40, 0, 0]], dtype=torch.float32)
    g3 = _cluster(70, 5) * 0.6
    pos = torch.cat([g0, g2, g3])
    batch = torch.tensor([0] * 5 + [2] * 4 + [3] * 70)
    return pos.to(DEV), batch.to(DEV), 4


def _inputs():
    pos_c = _cluster().to(DEV)
    yield "cluster", pos_c, torch.zeros(100, dtype=torch.long, device=DEV), 1
    pos_r, batch_r = _ragged()
    yield "ragged", pos_r, batch_r, 4
    yield "corners", *_corner_cases()


def _check_csr(g, ei):
    assert torch.equal(g.src.long(), ei[0]) and torch.equal(g.dst.long(), ei[1])
    deg = torch.bincount(ei[1], minlength=g.n_nodes)
    assert g.row_ptr[0] == 0 and torch.equal(torch.diff(g.row_ptr.long()), deg)


@pytest.mark.parametrize("case", ["cluster", "ragged", "corners"])
def test_radius_graph_matches_torch_cluster_semantics_at_any_cap(case):
    from dig_b200 import ops
    from dig_b200.threedgraph.utils import radius_graph
    from oracle import restated
    name, pos, batch, n_graphs = next(c for c in _inputs() if c[0] == case)
    n = pos.size(0)
    r = 2.0 if case == "corners" else 6.0
    for m in CAPS + [n + 5]:
        want = restated.radius_graph(pos, r, batch, max_num_neighbors=m)
        got = radius_graph(pos, r, batch, max_num_neighbors=m)
        assert torch.equal(got, want), (case, m)
        g = ops.radius_graph_dense(pos, batch, r, num_graphs=n_graphs, max_num_neighbors=m)
        assert torch.equal(g.edge_index, want) and g.n_edges == want.size(1) and g.n_graphs == n_graphs
        _check_csr(g, want)
    if case == "cluster":
        assert int(torch.bincount(want[1]).min()) == 99                # uncapped: everyone sees everyone
    if case == "corners":
        assert g.graph_ptr.tolist() == [0, 5, 5, 9, 79]
        deg = torch.bincount(want[1], minlength=n)
        assert deg[4] == 0 and deg[8] == 0 and deg[0] == 3             # isolated atoms; coincident atoms see each other
        pairs = set(map(tuple, want.t().tolist()))
        assert (6, 5) not in pairs and (7, 5) in pairs                  # exactly at the cutoff: out; just inside: in


def test_dense_builder_equals_the_capped_builder_below_the_old_limit():
    from dig_b200 import ops
    for _, pos, batch, n_graphs in _inputs():
        for m in (0, 1, 8, 32, 63):
            ref = ops.build_graph(pos, batch, 2.5, num_graphs=n_graphs, max_num_neighbors=m)
            g = ops.radius_graph_dense(pos, batch, 2.5, num_graphs=n_graphs, max_num_neighbors=m)
            assert torch.equal(g.edge_index, ref.edge_index) and torch.equal(g.row_ptr, ref.row_ptr)
            assert torch.equal(g.graph_ptr, ref.graph_ptr) and torch.equal(g.src, ref.src) and torch.equal(g.dst, ref.dst)


def _hub_graph(d, seed=0):
    """Node 0 is a hub with in-degree d (sources 1..d).  Its out-edges go to node 1 and node d // 2 (both among its
    in-neighbours: their triplets skip them) and to nodes d + 1, d + 2 (not in-neighbours); node 1 also feeds d + 1,
    so light and heavy edges meet.  Returns (pos, edge_index sorted by (target, source))."""
    g = torch.Generator().manual_seed(seed)
    n = d + 3
    pos = torch.randn(n, 3, generator=g) * 2.0
    src = list(range(1, d + 1)) + [0, 0, 0, 0, 1]
    dst = [0] * d + [1, d // 2, d + 1, d + 2, d + 1]
    ei = torch.tensor([src, dst])
    order = torch.sort(ei[1] * n + ei[0]).indices
    return pos.to(DEV), ei[:, order].contiguous().to(DEV)


def _straddle_graph(seed=0):
    """Hubs with in-degree 63, 64, 65 and 66 in one graph, wired to each other: the edges out of the 65 and 66 hubs are
    heavy, all others light."""
    g = torch.Generator().manual_seed(seed)
    degs = [63, 64, 65, 66]
    hubs = list(range(4))
    n = 4 + 80
    pos = torch.randn(n, 3, generator=g) * 2.0
    pairs = set()
    for h, d in zip(hubs, degs):
        others = [x for x in range(n) if x != h]
        pick = torch.randperm(len(others), generator=g)[:d].tolist()
        pairs.update((others[p], h) for p in pick)
    for a in hubs:
        for b in hubs:
            if a != b:
                pairs.add((a, 4 + b))                                   # hub -> a spoke of another hub
    ei = torch.tensor(sorted(pairs, key=lambda p: (p[1], p[0]))).t().contiguous()
    return pos.to(DEV), ei.to(DEV)


def _geometry_cases():
    from oracle import restated
    pos_c = _cluster().to(DEV)
    yield "cluster_m1000", pos_c, restated.radius_graph(pos_c, 6.0, torch.zeros(100, dtype=torch.long, device=DEV),
                                                        max_num_neighbors=1000)
    pos_r, batch_r = _ragged()
    yield "ragged_m65", pos_r, restated.radius_graph(pos_r, 6.0, batch_r, max_num_neighbors=65)
    for d in (65, 128, 129, 300, 1000):
        yield f"hub{d}", *_hub_graph(d, seed=d)
    yield "straddle", *_straddle_graph()


def _heavy_edges(ei, n):
    deg = torch.bincount(ei[1], minlength=n)
    return int((deg[ei[0]] > 64).sum())


@pytest.mark.parametrize("case", ["cluster_m1000", "ragged_m65", "hub65", "hub128", "hub129", "hub300", "hub1000",
                                  "straddle"])
def test_xyz_to_dat_matches_the_restatement_at_any_in_degree(case):
    from dig_b200.threedgraph.utils import xyz_to_dat
    from oracle import restated
    _, pos, ei = next(c for c in _geometry_cases() if c[0] == case)
    n = pos.size(0)
    assert 0 < _heavy_edges(ei, n)
    for tors in (False, True):
        got = xyz_to_dat(pos, ei, n, use_torsion=tors)
        want = restated.xyz_to_dat(pos, ei, n, use_torsion=tors)
        assert len(got) == len(want)
        for k, (a, b) in enumerate(zip(got, want)):
            assert a.dtype == b.dtype and torch.equal(a, b), (case, tors, k)
        del want


@pytest.mark.parametrize("case", ["cluster_m1000", "ragged_m65", "hub65", "hub300", "hub1000", "straddle"])
def test_gsphere_xyztodat_matches_the_restatement_at_any_in_degree(case):
    from dig_b200.ggraph3D.method.G_SphereNet.model.geometric_computing import xyztodat
    from oracle import restated
    _, pos, ei = next(c for c in _geometry_cases() if c[0] == case)
    n = pos.size(0)
    if case == "ragged_m65":
        _, batch = _ragged()
    else:
        batch = torch.zeros(n, dtype=torch.long, device=DEV)
    got = xyztodat(pos, ei, n, batch)
    want = restated.xyztodat_knn(pos, ei, n, batch)
    for k, (a, b) in enumerate(zip(got, want)):
        assert a.dtype == b.dtype and torch.equal(a, b), (case, k)


def test_unsorted_edge_list_with_a_heavy_hub():
    """An edge list in no particular order: the same (k->j, j->i) pair carries the same values as in the sorted call,
    the way test_xyz_to_dat_api_matches_reference_outputs checks it."""
    from dig_b200.threedgraph.utils import xyz_to_dat
    pos, ei_sorted = _hub_graph(300, seed=7)
    n = pos.size(0)
    g = torch.Generator().manual_seed(3)
    ei_u = ei_sorted[:, torch.randperm(ei_sorted.size(1), generator=g).to(DEV)].contiguous()
    for tors in (False, True):
        got = xyz_to_dat(pos, ei_u, n, use_torsion=tors)
        order = torch.sort(ei_u[1] * n + ei_u[0], stable=True).indices
        srt = xyz_to_dat(pos, ei_u[:, order].contiguous(), n, use_torsion=tors)
        e_n = ei_u.size(1)
        key_s = order[srt[-1]] * e_n + order[srt[-2]]
        key_u = got[-1] * e_n + got[-2]
        ps, pu = torch.argsort(key_s), torch.argsort(key_u)
        assert torch.equal(key_s[ps], key_u[pu]) and torch.equal(srt[1][ps], got[1][pu])
        inv = torch.empty_like(order)
        inv[order] = torch.arange(e_n, device=DEV)
        assert torch.equal(got[0], srt[0][inv])
        if tors:
            assert torch.equal(srt[2][ps], got[2][pu])


def _light_cases():
    """Graphs whose in-degrees are all <= 64, so that the warp-per-edge kernel can run every edge."""
    from oracle import restated
    pos_r, batch_r = _ragged()
    yield pos_r, restated.radius_graph(pos_r, 6.0, batch_r, max_num_neighbors=63), batch_r
    pos_h, ei_h = _hub_graph(64, seed=11)
    yield pos_h, ei_h, torch.zeros(pos_h.size(0), dtype=torch.long, device=DEV)
    pos_c, batch_c, _ = _corner_cases()
    yield pos_c[5:], restated.radius_graph(pos_c[5:], 2.0, batch_c[5:] - 2, max_num_neighbors=63), batch_c[5:] - 2


def test_heavy_edge_kernel_matches_the_warp_kernel_bit_for_bit(monkeypatch):
    from dig_b200.threedgraph.utils import geometric_computing as gc
    from dig_b200.ggraph3D.method.G_SphereNet.model.geometric_computing import xyztodat
    for pos, ei, batch in _light_cases():
        n = pos.size(0)
        assert int(torch.bincount(ei[1], minlength=n).max()) <= 64 and ei.size(1) > 0
        outs = {}
        for forced in (False, True):
            monkeypatch.setattr(gc, "_HEAVY_KERNEL_FOR_ALL_EDGES", forced)
            outs[forced] = [gc.xyz_to_dat(pos, ei, n, use_torsion=False), gc.xyz_to_dat(pos, ei, n, use_torsion=True),
                            xyztodat(pos, ei, n, batch)]
        for a_set, b_set in zip(outs[False], outs[True]):
            for a, b in zip(a_set, b_set):
                assert torch.equal(a, b)


def _dense_proteins():
    """synthetic_proteins with every chain pulled towards its centroid until more than 96 C-alpha atoms lie within
    10 A of one another."""
    from dig_b200.data import synthetic_proteins
    b = synthetic_proteins(3, length=110, seed=4)
    for g in range(3):
        sel = b.batch == g
        c = b.coords_ca[sel].mean(0)
        for key in ("coords_ca", "coords_n", "coords_c"):
            v = getattr(b, key)
            v[sel] = c + (v[sel] - c) * 0.3
    return b.to(DEV)


@pytest.mark.parametrize("m", [64, 96])
@pytest.mark.parametrize("level", ["aminoacid", "backbone", "allatom"])
def test_pronet_beyond_63_neighbours_matches_the_restatement(level, m):
    from dig_b200 import ops
    from dig_b200.threedgraph.method import ProNet
    from oracle import restated
    ctor = {"aminoacid": dict(level="aminoacid"), "backbone": dict(level="backbone", num_blocks=2),
            "allatom": dict(level="allatom", num_blocks=2, out_channels=3, out_layers=3)}[level]
    b = _dense_proteins()
    full = restated.radius_graph(b.coords_ca, 10.0, b.batch, max_num_neighbors=10 ** 6)
    assert int(torch.bincount(full[1]).max()) > 96                       # the cap binds at both values
    want_ei = restated.radius_graph(b.coords_ca, 10.0, b.batch, max_num_neighbors=m)
    g = ops.radius_graph_dense(b.coords_ca, b.batch, 10.0, num_graphs=b.num_graphs, max_num_neighbors=m)
    assert torch.equal(g.edge_index, want_ei)
    model = ProNet(max_num_neighbors=m, **ctor)
    sd = formula_state_dict(model.state_dict(), seed=6)
    model.load_state_dict(sd)
    model = model.to(DEV)
    kw = {k: v for k, v in ctor.items() if k != "out_channels"}
    sd_ref = {k: v.to(DEV).clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    ref = restated.pronet_forward(sd_ref, b, max_num_neighbors=m, **kw)
    out = model(b)
    assert rel_err(out.detach().cpu().numpy(), ref.detach().cpu().numpy()) < 1e-5
    target = torch.linspace(-1, 1, ref.numel(), device=DEV).view_as(ref)
    torch.nn.functional.l1_loss(out, target).backward()
    torch.nn.functional.l1_loss(ref, target).backward()
    bad = {}
    for pname, p in model.named_parameters():
        r = sd_ref[pname].grad
        assert p.grad is not None and r is not None, pname
        err = rel_err(p.grad.cpu().numpy(), r.cpu().numpy()) if float(r.abs().max()) > 0 else float(p.grad.abs().max())
        if err > 1e-4:
            bad[pname] = err
    assert not bad, bad


def test_totals_of_2_pow_31_are_refused_before_they_are_allocated():
    """E >= 2^31: 46 342 coincident atoms see each other (46 342 * 46 341 edges); T >= 2^31: a two-way star whose hub
    has in- and out-degree 46 342 (46 342 * 46 341 triplets from 92 684 edges).  Both raise ValueError from the count
    pass, with peak memory far below what the edges or triplets would take."""
    from dig_b200 import ops
    from dig_b200._lib import Dig3dError
    from dig_b200.threedgraph.utils import radius_graph, xyz_to_dat
    n = 46342
    pos = torch.zeros(n, 3, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match="2\\^31"):
        radius_graph(pos, 1.0, None, max_num_neighbors=10 ** 9)
    assert torch.cuda.max_memory_allocated() - base < 64 << 20
    leaves = torch.arange(1, n + 1, device=DEV)
    hub = torch.zeros_like(leaves)
    ei = torch.cat([torch.stack([leaves, hub]), torch.stack([hub, leaves])], 1)
    ei = ei[:, torch.sort(ei[1] * (n + 1) + ei[0]).indices].contiguous()
    pos_s = torch.randn(n + 1, 3, device=DEV)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match="2\\^31"):
        xyz_to_dat(pos_s, ei, n + 1, use_torsion=True)
    assert torch.cuda.max_memory_allocated() - base < 64 << 20
    # the capped builder keeps its limit
    with pytest.raises(Dig3dError):
        ops.build_graph(torch.rand(4, 3, device=DEV), torch.zeros(4, dtype=torch.long, device=DEV), 5.0,
                        max_num_neighbors=200)


def test_dense_builder_validates_nodes_like_the_capped_builder():
    from dig_b200 import ops
    pos = torch.rand(6, 3, device=DEV)
    with pytest.raises(ValueError, match="batch ids"):
        ops.radius_graph_dense(pos, torch.tensor([0, 0, 1, 1, 2, 7], device=DEV), 5.0, num_graphs=3,
                               max_num_neighbors=100)
    with pytest.raises(ValueError, match="not sorted"):
        ops.radius_graph_dense(pos, torch.tensor([0, 1, 0, 1, 1, 1], device=DEV), 5.0, num_graphs=2,
                               max_num_neighbors=100)
    with pytest.raises(ValueError, match="atomic numbers"):
        ops.radius_graph_dense(pos, None, 5.0, max_num_neighbors=100, z=torch.tensor([0, 1, 2, 3, 4, 30], device=DEV),
                               z_rows=26)
    g = ops.radius_graph_dense(torch.zeros(0, 3, device=DEV), torch.zeros(0, dtype=torch.long, device=DEV), 5.0,
                               max_num_neighbors=100)
    assert g.n_edges == 0 and g.edge_index.shape == (2, 0) and g.row_ptr.tolist() == [0]
