"""`xyz_to_dat` / `radius_graph` with the reference's call signatures, on the sm_90a kernels.

reference: dig/threedgraph/utils/geometric_computing.py:12-80 (xyz_to_dat);
           torch_cluster.radius_graph as called at spherenet.py:304.
The model classes do not go through these wrappers (they keep int32 CSR internally and never
materialise idx_kj / idx_ji); they exist for users of the reference's utility API and for tests.
"""
import torch

from ... import autograd_dd, ops
from ...ops import _p, _stream, call


def radius_graph(x, r, batch=None, loop=False, max_num_neighbors=32, flow='source_to_target', num_workers=1):
    """edge_index [2, E] int64 = (source j, target i), sorted by (i, j); torch_cluster CUDA semantics, any
    max_num_neighbors."""
    if loop or flow != 'source_to_target':
        raise NotImplementedError("radius_graph: only loop=False, flow='source_to_target' (the reference's use)")
    if int(max_num_neighbors) <= 63:
        g = ops.build_graph(x, batch, r, max_num_neighbors=max_num_neighbors)
    else:                                           # beyond the capped builder's neighbour table
        g = ops.radius_graph_dense(x, batch, r, max_num_neighbors=max_num_neighbors)
    return g.edge_index


# Tests only: run every edge on the heavy-edge geometry kernel, which otherwise takes the edges whose source has
# in-degree > 64, to hold it bit for bit against the warp-per-edge kernel on the graphs both can run.
_HEAVY_KERNEL_FOR_ALL_EDGES = False


def _xyz_to_dat_sorted(pos, ei, n, use_torsion, knn_batch=None, want_grad=False):
    """Kernel path for an edge_index sorted by (target, source); returns None when it is not sorted.
    knn_batch: the `batch` vector -- selects G-SphereNet's single-reference torsion (nearest neighbour of j).
    want_grad: with the torsion, record each triplet's winning candidate (g.tors_arg) for the derivative kernels."""
    dev = pos.device
    e = ei.size(1)
    g = ops.Graph3D()
    g.n_nodes, g.n_edges = n, e
    g.src = torch.empty(max(e, 1), dtype=torch.int32, device=dev)[:e]
    g.dst = torch.empty(max(e, 1), dtype=torch.int32, device=dev)[:e]
    g.row_ptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
    g.trip_ptr = torch.empty(e + 1, dtype=torch.int32, device=dev)
    g.dist = torch.empty(max(e, 1), dtype=torch.float32, device=dev)[:e]
    ws = torch.empty(2 * e + 2, dtype=torch.int32, device=dev)
    flags = torch.empty(6, dtype=torch.int32, device=dev)
    call("dig3d_edges_to_csr", _p(pos.detach(), torch.float32, "pos"), _p(ei, torch.int64, "edge_index"), e, n,
         _p(g.src), _p(g.dst), _p(g.row_ptr), _p(ws), _p(g.trip_ptr), _p(g.dist), _p(flags), _stream())
    fl = flags.tolist()
    if fl[0] & 1:
        return None
    t = (fl[4] & 0xFFFFFFFF) | (fl[5] << 32)                           # the int64 triplet total
    ops.check_int32_total(t, "triplets")
    g.n_triplets = t
    n_heavy = e if _HEAVY_KERNEL_FOR_ALL_EDGES else fl[1]
    if knn_batch is None:
        if want_grad and use_torsion:
            return ops.triplet_geometry_any_degree_arg(g, pos, n_heavy)
        return ops.triplet_geometry_any_degree(g, pos, int(bool(use_torsion)), n_heavy)
    n_graphs = int(knn_batch[-1].item()) + 1 if n else 0
    graph_ptr = torch.empty(n_graphs + 1, dtype=torch.int32, device=dev)
    call("dig3d_graph_ptr", _p(knn_batch, torch.int64, "batch"), n, n_graphs, _p(graph_ptr), _stream())
    nn = torch.empty(2, max(n, 1), dtype=torch.int32, device=dev)
    call("dig3d_knn2", _p(pos.detach(), torch.float32, "pos"), _p(knn_batch), _p(graph_ptr), n, n_graphs, _p(nn[0]),
         _p(nn[1]), _stream())
    if n and int(nn.min()) < 0:
        raise ValueError("xyztodat: every graph needs at least three atoms (nearest and second-nearest neighbour)")
    return ops.triplet_geometry_any_degree(g, pos, 2, n_heavy, nn)


def xyz_to_dat(pos, edge_index, num_nodes, use_torsion=False, _knn_batch=None):
    """(dist, angle[, torsion], i, j, idx_kj, idx_ji) exactly as the reference returns them
    (utils/geometric_computing.py:12-80).  (`_knn_batch`: internal, see dig_b200.ggraph3D ... xyztodat.)

    An `edge_index` sorted by (target, source) -- what `radius_graph` returns -- goes straight to the kernels.  Any other
    order is handled like the reference's SparseTensor does: the edges are sorted (stable, by target then source), the
    kernels run on the sorted list, and the results are mapped back: `dist` in the caller's edge order, triplets grouped
    by the caller's edge order with k ascending inside a group, `idx_kj` / `idx_ji` holding the caller's edge ids (the
    re-ordering is index plumbing with torch; all geometry is computed by the kernels).

    Any in-degree: a node of in-degree d and out-degree d' has about d * d' triplets, and the torsion takes the min
    over d candidates per triplet (the sets the reference materialises).  Raises ValueError for 2^31 edges or
    triplets or more (int32 indices), before the triplet buffers are allocated.

    Derivatives: when `pos` requires grad and grad mode is on, `dist`, `angle` and `torsion` are differentiable in
    `pos`, twice (forces with `torch.autograd.grad(E, pos, create_graph=True)`, then a backward through them), with
    the same values bit for bit.  The torsion's gradient flows through the first minimal candidate; a zero-length edge,
    a collinear triplet's cross-product term, atan2(0, 0) and the self candidate (plane1 x plane1) pass nothing
    (DESIGN.md §6).  Otherwise the outputs do not require grad, as before."""
    if edge_index.dim() != 2 or edge_index.size(0) != 2:
        raise ValueError("edge_index must be [2, E]")
    e = edge_index.size(1)
    n = int(num_nodes)
    ops.check_int32_total(e, "edges")
    ei = edge_index.contiguous()
    j, i = ei[0], ei[1]
    if e and (int(ei.min()) < 0 or int(ei.max()) >= n):
        raise ValueError("xyz_to_dat: edge_index holds node ids outside [0, num_nodes)")
    want_grad = _knn_batch is None and pos.requires_grad and torch.is_grad_enabled()
    g = _xyz_to_dat_sorted(pos, ei, n, use_torsion, _knn_batch, want_grad)
    sorted_in = g is not None
    if not sorted_in:                                                   # arbitrary edge order
        perm = torch.sort(i * n + j, stable=True).indices              # sorted position -> caller's edge id
        g = _xyz_to_dat_sorted(pos, ei[:, perm].contiguous(), n, use_torsion, _knn_batch, want_grad)
        if g is None:
            raise RuntimeError("xyz_to_dat: internal error, sorted edge list rejected")
    if want_grad:
        geo = autograd_dd.geometry(pos, g, 3 if use_torsion else 2)
        dist, angle, torsion = geo[0], geo[1], (geo[2] if use_torsion else None)
    else:
        dist, angle, torsion = g.dist, g.angle, g.torsion
    if sorted_in:
        if use_torsion:
            return dist, angle, torsion, i, j, g.idx_kj64, g.idx_ji64
        return dist, angle, i, j, g.idx_kj64, g.idx_ji64
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(e, device=perm.device)                    # caller's edge id -> sorted position
    tp = g.trip_ptr.long()
    cnt = (tp[1:] - tp[:-1])[inv]                                      # triplets per edge, caller's order
    start = tp[:-1][inv]
    t = int(cnt.sum())
    first = torch.cumsum(cnt, 0) - cnt
    take = torch.repeat_interleave(start - first, cnt) + torch.arange(t, device=perm.device)
    idx_kj = perm[g.idx_kj64[take]]
    idx_ji = torch.repeat_interleave(torch.arange(e, device=perm.device), cnt)
    if use_torsion:
        return dist[inv], angle[take], torsion[take], i, j, idx_kj, idx_ji
    return dist[inv], angle[take], i, j, idx_kj, idx_ji
