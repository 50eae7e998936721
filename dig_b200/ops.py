"""Tensor-level wrappers over the C ABI (include/dig3d.h).

PyTorch is used for device memory (caching allocator) and streams only; every computation below
is a hand-written sm_90a kernel in libdig3d.so.  Inputs are validated here (dtype / device /
contiguity / alignment), the C side only returns codes.  Nothing in this module has a CPU path.
"""
import ctypes

import torch

from . import _lib
from ._lib import call

BASIS_IDS = {("dimenet", 7, 6): 0, ("dimenet", 3, 6): 1, ("gemnet", 2, 3): 2}


_RAW_STREAM = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream():
    """Raw handle of torch's current CUDA stream on the current device (every op is launched on it).  The private
    accessor is ~10x cheaper than building a torch.cuda.Stream object per launch; same value."""
    if _RAW_STREAM is not None:
        return ctypes.c_void_p(_RAW_STREAM(torch.cuda.current_device()))
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t, dtype=None, name="tensor", align=4):
    """Device pointer of a validated tensor (None -> NULL).  Called ~1500 times per training step: one combined test on
    the fast path, the specific diagnosis only when it fails."""
    if t is None:
        return None
    try:
        ptr = t.data_ptr()
        ok = t.is_cuda and t.is_contiguous() and (dtype is None or t.dtype == dtype) and not (ptr & (align - 1))
    except AttributeError:
        raise TypeError(f"{name}: expected a torch.Tensor, got {type(t)}") from None
    if ok:
        return ctypes.c_void_p(ptr)
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name}: expected a torch.Tensor, got {type(t)}")
    if not t.is_cuda:
        raise RuntimeError(f"{name}: dig_b200 ops run on CUDA tensors only (got device {t.device}); "
                           "there is no CPU fallback")
    if dtype is not None and t.dtype != dtype:
        raise TypeError(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name}: tensor must be contiguous")
    if t.numel() and ptr % align != 0:
        raise ValueError(f"{name}: storage must be {align}-byte aligned")
    return ctypes.c_void_p(ptr)                       # empty tensor with an odd (or null) pointer


class Graph3D:
    """Radius graph in CSR-by-target form plus the implicit triplet structure."""
    __slots__ = ("n_nodes", "n_graphs", "n_edges", "n_triplets", "cap", "graph_ptr", "batch",
                 "row_ptr", "src", "dst", "edge_index", "dist", "vec", "trip_ptr",
                 "angle", "torsion", "idx_kj", "idx_ji", "idx_kj64", "idx_ji64",
                 "out_ptr", "out_list", "pos_in",      # out-edge lists (CSR by source), None for graphs built without them
                 "comenet_refs")                       # ComENet's reference atoms (comenet_geometry)

    def __init__(self):
        for s in self.__slots__:
            setattr(self, s, None)


def build_graph(pos, batch, cutoff, num_graphs=None, max_num_neighbors=32, want_vec=False,
                want_edge_index=True, z=None, z_rows=0):
    """radius_graph(pos, r=cutoff, batch) (reference spherenet.py:304 etc.) + triplet offsets.

    One host<->device synchronisation: the edge and triplet totals (two ints) are read back to size
    the per-edge / per-triplet buffers (the reference path has >= 10 implicit syncs, SURVEY.md 3.2).
    The same read-back carries the index validation (batch ids inside [0, num_graphs) and sorted; with `z`,
    atomic numbers inside the `z_rows`-row embedding table): the reference's nn.Embedding / scatter raise a
    device-side assert for those, here they raise ValueError before any kernel indexes with them."""
    if pos.dim() != 2 or pos.size(1) != 3:
        raise ValueError(f"pos must be [N, 3], got {tuple(pos.shape)}")
    n = pos.size(0)
    if batch is None:
        batch = torch.zeros(n, dtype=torch.long, device=pos.device)
    if batch.shape != (n,):
        raise ValueError("batch must be [N]")
    pos = pos.detach()
    dev = pos.device
    st = _stream()
    if num_graphs is None:
        num_graphs = int(batch[-1].item()) + 1 if n else 0
    g = Graph3D()
    g.n_nodes, g.n_graphs, g.batch = n, int(num_graphs), batch
    cap = int(max_num_neighbors) + 1
    g.cap = cap
    g.graph_ptr = torch.empty(g.n_graphs + 1, dtype=torch.int32, device=dev)
    call("dig3d_graph_ptr", _p(batch, torch.int64, "batch"), n, g.n_graphs, _p(g.graph_ptr), st)
    nbr = torch.empty(max(n, 1) * cap, dtype=torch.int32, device=dev)
    deg = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    tcnt = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    zeroed = torch.zeros(4 + max(n, 1), dtype=torch.int32, device=dev)     # one fill: totals [4] + out-degree counters [n]
    totals, out_cnt = zeroed[:4], zeroed[4:]
    if z is not None and z.shape != (n,):
        raise ValueError("z must be [N]")
    call("dig3d_validate_nodes", _p(batch), _p(z, torch.int64, "z"), n, g.n_graphs, int(z_rows),
         ctypes.c_void_p(totals.data_ptr() + 8), st)
    call("dig3d_radius_neighbors", _p(pos, torch.float32, "pos"), _p(batch), _p(g.graph_ptr), n, g.n_graphs,
         float(cutoff), cap, _p(nbr), _p(deg), st)
    call("dig3d_triplet_count_out", _p(nbr), _p(deg), n, cap, _p(tcnt), _p(out_cnt), st)
    g.row_ptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
    node_trip_ptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
    g.out_ptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
    call("dig3d_scan_counts3", _p(deg), _p(tcnt), _p(out_cnt), n, _p(g.row_ptr), _p(node_trip_ptr), _p(g.out_ptr),
         _p(totals), st)
    tot = totals[:3].tolist()                      # the one sync of the forward pass
    if tot[2]:
        what = [msg for bit, msg in ((1, f"batch ids outside [0, {g.n_graphs})"), (2, "batch is not sorted ascending"),
                                     (4, f"atomic numbers outside the {z_rows}-row embedding table")) if tot[2] & bit]
        raise ValueError("invalid node indices: " + "; ".join(what))
    g.n_edges, g.n_triplets = int(tot[0]), int(tot[1])
    e = g.n_edges
    g.src = torch.empty(max(e, 1), dtype=torch.int32, device=dev)[:e]
    g.dst = torch.empty(max(e, 1), dtype=torch.int32, device=dev)[:e]
    g.dist = torch.empty(max(e, 1), dtype=torch.float32, device=dev)[:e]
    g.trip_ptr = (torch.empty if e else torch.zeros)(e + 1, dtype=torch.int32, device=dev)   # edge_fill writes all e + 1 entries
    g.edge_index = torch.empty(2, e, dtype=torch.int64, device=dev) if want_edge_index else None
    g.vec = torch.empty(e, 3, dtype=torch.float32, device=dev) if want_vec else None
    g.out_list = torch.empty(max(e, 1), dtype=torch.int32, device=dev)[:e]
    g.pos_in = torch.empty(max(e, 1), dtype=torch.int32, device=dev)[:e]
    if e:
        call("dig3d_edge_fill_out", _p(pos), _p(nbr), _p(deg), _p(g.row_ptr), _p(node_trip_ptr), n, cap, e,
             _p(g.edge_index) if want_edge_index else None, _p(g.src), _p(g.dst), _p(g.dist),
             _p(g.vec) if want_vec else None, _p(g.trip_ptr), _p(g.graph_ptr), _p(batch), _p(g.out_ptr), _p(g.out_list),
             _p(g.pos_in), st)
    return g


def radius_graph_dense(pos, batch, cutoff, num_graphs=None, max_num_neighbors=32, want_edge_index=True, z=None,
                       z_rows=0):
    """radius_graph(pos, r=cutoff, batch, max_num_neighbors) for ANY max_num_neighbors >= 0 (csrc/graph_dense.cu):
    the edges of `build_graph` -- same hits, same (target, source) order -- without its [N, max_num_neighbors + 1]
    neighbour table and its cap of 63.  Returns a Graph3D with src, dst, row_ptr, graph_ptr, batch, n_nodes, n_edges,
    n_graphs and, if asked, edge_index; no triplet offsets, distances or out-edge lists.

    One host synchronisation (the edge total, with the index validation of `build_graph`).  Raises ValueError for
    invalid batch ids / atomic numbers and for 2^31 edges or more, before any edge is written."""
    if pos.dim() != 2 or pos.size(1) != 3:
        raise ValueError(f"pos must be [N, 3], got {tuple(pos.shape)}")
    m = int(max_num_neighbors)
    if m < 0:
        raise ValueError(f"max_num_neighbors must be >= 0, got {m}")
    n = pos.size(0)
    if batch is None:
        batch = torch.zeros(n, dtype=torch.long, device=pos.device)
    if batch.shape != (n,):
        raise ValueError("batch must be [N]")
    if z is not None and z.shape != (n,):
        raise ValueError("z must be [N]")
    pos = pos.detach()
    dev = pos.device
    st = _stream()
    if num_graphs is None:
        num_graphs = int(batch[-1].item()) + 1 if n else 0
    g = Graph3D()
    g.n_nodes, g.n_graphs, g.batch = n, int(num_graphs), batch
    info = torch.zeros(2, dtype=torch.int64, device=dev)
    if n:
        g.graph_ptr = torch.empty(g.n_graphs + 1, dtype=torch.int32, device=dev)
        call("dig3d_graph_ptr", _p(batch, torch.int64, "batch"), n, g.n_graphs, _p(g.graph_ptr), st)
        call("dig3d_validate_nodes", _p(batch), _p(z, torch.int64, "z"), n, g.n_graphs, int(z_rows),
             ctypes.c_void_p(info.data_ptr() + 8), st)
    else:                                                  # no nodes: every graph is empty
        g.graph_ptr = torch.zeros(g.n_graphs + 1, dtype=torch.int32, device=dev)
    counts = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    g.row_ptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
    info_host = (ctypes.c_int64 * 2)()
    try:
        call("dig3d_radius_graph_dense_count", _p(pos, torch.float32, "pos"), _p(batch), _p(g.graph_ptr), n,
             g.n_graphs, float(cutoff), m, _p(counts), _p(g.row_ptr), _p(info), ctypes.byref(info_host), st)
        rejected = None
    except _lib.Dig3dError as exc:
        if exc.rc != -1:                                   # DIG3D_EINVAL: the input was rejected
            raise
        rejected = exc
    flags = int(info_host[1])
    if flags:
        what = [msg for bit, msg in ((1, f"batch ids outside [0, {g.n_graphs})"), (2, "batch is not sorted ascending"),
                                     (4, f"atomic numbers outside the {z_rows}-row embedding table")) if flags & bit]
        raise ValueError("invalid node indices: " + "; ".join(what))
    if rejected is not None:
        raise ValueError(str(rejected)) from None
    e = g.n_edges = int(info_host[0])
    g.src = torch.empty(max(e, 1), dtype=torch.int32, device=dev)[:e]
    g.dst = torch.empty(max(e, 1), dtype=torch.int32, device=dev)[:e]
    g.edge_index = torch.empty(2, e, dtype=torch.int64, device=dev) if want_edge_index else None
    call("dig3d_radius_graph_dense_fill", _p(pos), _p(batch), _p(g.graph_ptr), n, g.n_graphs, float(cutoff), m,
         _p(g.row_ptr), e, _p(g.edge_index) if want_edge_index else None, _p(g.src), _p(g.dst), st)
    return g


def check_int32_total(total, what):
    """Kernels index edges and triplets with int32: a total of 2^31 or more is refused before it is allocated."""
    if int(total) >= 1 << 31:
        raise ValueError(f"{int(total)} {what}: the kernels index them with int32, the limit is 2^31 - 1")


def triplet_geometry_any_degree(g, pos, use_torsion, n_heavy, nn=None):
    """xyz_to_dat's angle / torsion / idx_kj64 / idx_ji64 at any in-degree (dig3d_triplet_geometry_any_degree).
    use_torsion: 0, 1 (min over all candidates) or 2 (G-SphereNet's single reference atom; nn = [2, N] nearest
    neighbours from dig3d_knn2).  n_heavy: the edges whose source has in-degree > 64 (flags[1] of
    dig3d_edges_to_csr); n_heavy == n_edges runs every edge on the heavy-edge kernel."""
    dev = pos.device
    t = g.n_triplets
    g.angle = torch.empty(t, dtype=torch.float32, device=dev)
    g.torsion = torch.empty(t, dtype=torch.float32, device=dev) if use_torsion else None
    g.idx_kj64 = torch.empty(t, dtype=torch.int64, device=dev)
    g.idx_ji64 = torch.empty(t, dtype=torch.int64, device=dev)
    e = g.n_edges
    if e and t:
        ws = torch.empty(n_heavy + 1, dtype=torch.int32, device=dev) if 0 < n_heavy < e else None
        call("dig3d_triplet_geometry_any_degree", _p(pos.detach(), torch.float32, "pos"), _p(g.src), _p(g.dst),
             _p(g.row_ptr), _p(g.trip_ptr), e, int(n_heavy), int(use_torsion),
             _p(nn[0]) if nn is not None else None, _p(nn[1]) if nn is not None else None, _p(ws), _p(g.angle),
             _p(g.torsion) if use_torsion else None, _p(g.idx_kj64), _p(g.idx_ji64), _stream())
    return g


def _out_lists(g):
    """(out_ptr, out_list, pos_in) device addresses of a graph's out-edge lists, or three NULLs."""
    if getattr(g, "out_ptr", None) is None or g.out_list is None or g.pos_in is None:
        return None, None, None
    return g.out_ptr.data_ptr(), g.out_list.data_ptr(), g.pos_in.data_ptr()


def triplet_geometry(g, pos, use_torsion, want_idx=True, want_idx64=False):
    """xyz_to_dat's angle / torsion / idx_kj / idx_ji (reference utils/geometric_computing.py:43-75)."""
    dev = pos.device
    t = g.n_triplets
    g.angle = torch.empty(t, dtype=torch.float32, device=dev)
    g.torsion = torch.empty(t, dtype=torch.float32, device=dev) if use_torsion else None
    if want_idx:
        g.idx_kj = torch.empty(t, dtype=torch.int32, device=dev)
        g.idx_ji = torch.empty(t, dtype=torch.int32, device=dev)
    if want_idx64:
        g.idx_kj64 = torch.empty(t, dtype=torch.int64, device=dev)
        g.idx_ji64 = torch.empty(t, dtype=torch.int64, device=dev)
    if g.n_edges and t:
        call("dig3d_triplet_geometry", _p(pos.detach(), torch.float32, "pos"), _p(g.src), _p(g.dst),
             _p(g.row_ptr), _p(g.trip_ptr), g.n_edges, int(bool(use_torsion)), _p(g.angle),
             _p(g.torsion) if use_torsion else None,
             _p(g.idx_kj) if want_idx else None, _p(g.idx_ji) if want_idx else None,
             _p(g.idx_kj64) if want_idx64 else None, _p(g.idx_ji64) if want_idx64 else None, _stream())
    return g


def edge_basis(dist, cutoff, envelope_exponent, freq, basis_id, envelope_on_bessel, num_radial,
               n_bessel, want_rbf0=True, want_bessel=True):
    e = dist.numel()
    dev = dist.device
    rbf0 = torch.empty(e, num_radial, dtype=torch.float32, device=dev) if want_rbf0 else None
    bess = torch.empty(e, n_bessel, dtype=torch.float32, device=dev) if want_bessel else None
    if e:
        call("dig3d_edge_basis", _p(dist, torch.float32, "dist"), e, float(cutoff), int(envelope_exponent),
             _p(freq.detach(), torch.float32, "freq") if freq is not None else None, int(basis_id),
             int(bool(envelope_on_bessel)), _p(rbf0) if want_rbf0 else None,
             _p(bess) if want_bessel else None, _stream())
    return rbf0, bess


def triplet_basis(bess, angle, torsion, idx_kj, basis_id, ns, nr, want_tbf):
    """Materialised sbf [T, ns*nr] / tbf [T, ns*ns*nr] (API-parity / test path)."""
    t = angle.numel()
    dev = angle.device
    sbf = torch.empty(t, ns * nr, dtype=torch.float32, device=dev)
    tbf = torch.empty(t, ns * ns * nr, dtype=torch.float32, device=dev) if want_tbf else None
    if t:
        call("dig3d_triplet_basis", _p(bess, torch.float32), _p(angle, torch.float32),
             _p(torsion, torch.float32) if want_tbf else None, _p(idx_kj, torch.int32), t, int(basis_id),
             _p(sbf), _p(tbf) if want_tbf else None, _stream())
    return sbf, tbf


# "edge" (default): one warp per (k -> j) edge, persistent CTAs.  "node": one CTA per middle node of the triplets -- all
# threads busy in the harmonics phase and no repeated out-edge search, bit-identical output, but slower at the headline
# size on an earlier GPU (three CTA-wide barriers per pass and only ~15 in-edges to spread over the eight contraction
# warps; not measured on the H100); kept as the starting point for a version that keeps several nodes in flight per CTA.
PROJECT_MODE = ["edge"]

# Kernel behind the "edge" mode for the torsion models (dig3d_triplet_basis_project_set_mode, process-wide):
# "scalar" = round 1's kernel (reference-rounded closed-form harmonics, scalar FMA chains), "packed" = FFMA2 chains on
# pairs of outputs with the same closed forms, "recurrence" (default) = packed + harmonics from the Legendre / angle-addition
# recurrences (csrc/harmonics.cuh).
PROJECT_KERNELS = {"scalar": 0, "packed": 1, "recurrence": 2}


def set_project_kernel(name):
    call("dig3d_triplet_basis_project_set_mode", PROJECT_KERNELS[name])


def triplet_basis_project(g, bess, basis_id, w_sbf1_rows, w_t1_rows):
    """w_sbf1_rows: [32, ns*nr], w_t1_rows: [32, ns*ns*nr] or None.
    Returns sbf_p [4, T, 8], t_p [4, T, 8] | None (layer-major: layer l's rows are contiguous)."""
    t = g.n_triplets
    dev = bess.device
    sbf_p = torch.empty(4, max(t, 1), 8, dtype=torch.float32, device=dev)
    t_p = torch.empty(4, max(t, 1), 8, dtype=torch.float32, device=dev) if w_t1_rows is not None else None
    if t == 0:
        return sbf_p[:, :0], (t_p[:, :0] if t_p is not None else None)
    if t and g.n_edges and PROJECT_MODE[0] == "node":
        call("dig3d_triplet_basis_project_node", _p(bess, torch.float32), _p(g.angle),
             _p(g.torsion) if w_t1_rows is not None else None, _p(g.src), _p(g.row_ptr), _p(g.trip_ptr),
             _p(g.graph_ptr), _p(g.batch, torch.int64), g.n_nodes, t, g.cap, int(basis_id), 4, 8,
             _p(w_sbf1_rows, torch.float32, "w_sbf1"),
             _p(w_t1_rows, torch.float32, "w_t1") if w_t1_rows is not None else None,
             _p(sbf_p), _p(t_p) if t_p is not None else None, _stream())
    elif t and g.n_edges:
        call("dig3d_triplet_basis_project_lists", _p(bess, torch.float32), _p(g.angle),
             _p(g.torsion) if w_t1_rows is not None else None, _p(g.src), _p(g.dst), _p(g.row_ptr),
             _p(g.trip_ptr), _p(g.graph_ptr), _p(g.batch, torch.int64), g.n_edges, t, int(basis_id), 4, 8,
             _p(w_sbf1_rows, torch.float32, "w_sbf1"),
             _p(w_t1_rows, torch.float32, "w_t1") if w_t1_rows is not None else None,
             _p(sbf_p), _p(t_p) if t_p is not None else None, *_out_lists(g), _stream())
    return sbf_p, t_p


def segment_sum(x, ptr):
    """scatter(x, index, dim=0, reduce='sum') for a sorted index given as CSR pointers."""
    if x.dim() != 2:
        raise ValueError("segment_sum expects [rows, width]")
    s = ptr.numel() - 1
    if x.size(0) == 0:
        return torch.zeros(s, x.size(1), dtype=torch.float32, device=x.device)
    out = torch.empty(s, x.size(1), dtype=torch.float32, device=x.device)
    if s:
        call("dig3d_segment_sum", _p(x, torch.float32, "x", align=16 if x.size(1) % 4 == 0 else 4), _p(ptr, torch.int32, "ptr"), s, x.size(1),
             _p(out), _stream())
    return out


def graph_readout(v_all, graph_ptr, n_graphs, n_nodes):
    """v_all: [n_blocks, N, C] -> u [n_graphs, C] (sum over nodes of each graph, then over blocks)."""
    nb, _, c = v_all.shape
    u = torch.empty(n_graphs, c, dtype=torch.float32, device=v_all.device)
    if n_graphs:
        call("dig3d_graph_readout", _p(v_all, torch.float32, align=4), _p(graph_ptr, torch.int32), n_graphs,
             n_nodes, nb, c, _p(u, align=4), _stream())
    return u


# ----------------------------------------------------------------------------- SphereNet / DimeNet++
def _wp(t, name):
    return _p(t.detach(), torch.float32, name, align=16).value if t is not None else None


def pack_init_e(m):
    w = _lib.InitEWeights()
    w.emb = _wp(m.emb.weight, "emb")
    w.w_rbf0, w.b_rbf0 = _wp(m.lin_rbf_0.weight, "lin_rbf_0.w"), _wp(m.lin_rbf_0.bias, "lin_rbf_0.b")
    w.w_lin, w.b_lin = _wp(m.lin.weight, "lin.w"), _wp(m.lin.bias, "lin.b")
    w.w_rbf1 = _wp(m.lin_rbf_1.weight, "lin_rbf_1.w")
    return w


def pack_update_e(m, torsion):
    w = _lib.UpdateEWeights()
    w.w_rbf1, w.w_rbf2 = _wp(m.lin_rbf1.weight, "lin_rbf1"), _wp(m.lin_rbf2.weight, "lin_rbf2")
    w.w_sbf2 = _wp(m.lin_sbf2.weight, "lin_sbf2")
    w.w_t2 = _wp(m.lin_t2.weight, "lin_t2") if torsion else None
    w.w_rbf = _wp(m.lin_rbf.weight, "lin_rbf")
    w.w_kj, w.b_kj = _wp(m.lin_kj.weight, "lin_kj.w"), _wp(m.lin_kj.bias, "lin_kj.b")
    w.w_ji, w.b_ji = _wp(m.lin_ji.weight, "lin_ji.w"), _wp(m.lin_ji.bias, "lin_ji.b")
    w.w_down, w.w_up = _wp(m.lin_down.weight, "lin_down"), _wp(m.lin_up.weight, "lin_up")
    res = list(m.layers_before_skip) + list(m.layers_after_skip)
    for r, layer in enumerate(res):
        w.w_res[2 * r], w.b_res[2 * r] = _wp(layer.lin1.weight, "res.lin1.w"), _wp(layer.lin1.bias, "res.lin1.b")
        w.w_res[2 * r + 1], w.b_res[2 * r + 1] = _wp(layer.lin2.weight, "res.lin2.w"), _wp(layer.lin2.bias, "res.lin2.b")
    w.w_lin, w.b_lin = _wp(m.lin.weight, "lin.w"), _wp(m.lin.bias, "lin.b")
    return w


def pack_update_v(m):
    w = _lib.UpdateVWeights()
    w.w_up, w.b_up = _wp(m.lin_up.weight, "lin_up.w"), _wp(m.lin_up.bias, "lin_up.b")
    for l, lin in enumerate(m.lins):
        w.w_lins[l], w.b_lins[l] = _wp(lin.weight, "lins.w"), _wp(lin.bias, "lins.b")
    w.w_out = _wp(m.lin.weight, "lin.w")
    w.n_lins = len(m.lins)
    return w


def pack_update_v_array(holders):
    """UpdateVWeights[len(holders)]: the node-MLP weight structs of a forward, one per block."""
    return (_lib.UpdateVWeights * len(holders))(*[pack_update_v(h) for h in holders])


def sphere_init_e(z, g, rbf0, w, hidden, v_in=None):
    e1 = torch.empty(max(g.n_edges, 1), hidden, dtype=torch.float32, device=rbf0.device)[:g.n_edges]
    if v_in is None:
        v_in = torch.zeros(g.n_nodes, hidden, dtype=torch.float32, device=rbf0.device)
    if g.n_edges:
        call("dig3d_sphere_init_e", _p(z, torch.int64, "z"), _p(g.src), _p(g.dst), _p(rbf0), g.n_edges,
             ctypes.byref(w), _p(e1), _p(v_in), _stream())
    return e1, v_in


def sphere_update_e(e1, g, rbf0, sbf_p, t_p, col0, w, hidden, int_emb, v_in=None):
    """One update_e block (parts A + B).  sbf_p/t_p: [4, T, 8]; col0 // 8 selects the layer slice."""
    dev = e1.device
    e = g.n_edges
    x_ji = torch.empty(max(e, 1), hidden, dtype=torch.float32, device=dev)[:e]
    x_down = torch.empty(max(e, 1), int_emb, dtype=torch.float32, device=dev)[:e]
    e1_out = torch.empty(max(e, 1), hidden, dtype=torch.float32, device=dev)[:e]
    if v_in is None:
        v_in = torch.zeros(g.n_nodes, hidden, dtype=torch.float32, device=dev)
    if e:
        st = _stream()
        call("dig3d_sphere_update_e_a", _p(e1), _p(rbf0), e, ctypes.byref(w), _p(x_ji), _p(x_down), st)
        sp = ctypes.c_void_p(sbf_p[col0 // 8].data_ptr())
        tp = ctypes.c_void_p(t_p[col0 // 8].data_ptr()) if t_p is not None else None
        call("dig3d_sphere_update_e_b", _p(e1), _p(x_ji), _p(x_down), _p(rbf0), sp, tp, 8, _p(g.src),
             _p(g.dst), _p(g.row_ptr), _p(g.trip_ptr), e, ctypes.byref(w), _p(e1_out), _p(v_in), st)
    return e1_out, v_in


def sphere_update_v_batched(v_in_all, holders, out_channels, v_out_all):
    """All node MLPs of a forward in one launch.  v_in_all [NB, N, H], holders: NB update_v modules."""
    nb, n, _ = v_in_all.shape
    arr = pack_update_v_array(holders)
    if n:
        call("dig3d_sphere_update_v_batched", _p(v_in_all, torch.float32, "v_in_all", 16), n, nb, int(out_channels),
             arr, _p(v_out_all, align=4), _stream())
    return v_out_all


def sphere_update_v(v_in, w, out_channels, v_out):
    n = v_in.size(0)
    if n:
        call("dig3d_sphere_update_v", _p(v_in), n, int(out_channels), ctypes.byref(w), _p(v_out, align=4), _stream())
    return v_out


# ----------------------------------------------------------------------------- SchNet
def pack_schnet_block(ue, uv):
    w = _lib.SchnetBlockWeights()
    w.w_lin = _wp(ue.lin.weight, "update_e.lin")
    g = ue.mlp[0].weight.size(1)
    w0 = torch.nn.functional.pad(ue.mlp[0].weight.detach(), (0, 64 - g)).contiguous()   # zero-pad G -> 64
    w.w_mlp0, w.b_mlp0 = _wp(w0, "mlp.0.w"), _wp(ue.mlp[0].bias, "mlp.0.b")
    w.w_mlp2, w.b_mlp2 = _wp(ue.mlp[2].weight, "mlp.2.w"), _wp(ue.mlp[2].bias, "mlp.2.b")
    w.w_v1, w.b_v1 = _wp(uv.lin1.weight, "update_v.lin1.w"), _wp(uv.lin1.bias, "update_v.lin1.b")
    w.w_v2, w.b_v2 = _wp(uv.lin2.weight, "update_v.lin2.w"), _wp(uv.lin2.bias, "update_v.lin2.b")
    return w, w0          # keep the padded copy alive until the kernel has been enqueued


def schnet_block(v, g, offset, coeff, cutoff, hidden, filters, w):
    n = v.size(0)
    dev = v.device
    vlin = torch.empty(n, filters, dtype=torch.float32, device=dev)
    agg = torch.zeros(n, filters, dtype=torch.float32, device=dev)
    v_out = torch.empty(n, hidden, dtype=torch.float32, device=dev)
    call("dig3d_schnet_block", _p(v, torch.float32, "v", 16), n, _p(g.dist), _p(g.src), _p(g.dst), g.n_edges,
         _p(offset, torch.float32, "offset"), offset.numel(), float(coeff), float(cutoff), int(hidden),
         int(filters), ctypes.byref(w), _p(vlin), _p(agg), _p(v_out), _stream())
    return v_out


def schnet_readout(v, lin1, lin2, out_channels):
    n = v.size(0)
    node_out = torch.empty(n, out_channels, dtype=torch.float32, device=v.device)
    call("dig3d_schnet_readout", _p(v, torch.float32), n, v.size(1), _p(lin1.weight.detach(), torch.float32),
         _p(lin1.bias.detach(), torch.float32), _p(lin2.weight.detach(), torch.float32),
         _p(lin2.bias.detach(), torch.float32), int(out_channels), _p(node_out), _stream())
    return node_out


def radius_graph_pbc(pos, cell, natoms, radius, max_num_neighbors_threshold):
    """Periodic radius graph (ocpmodels' radius_graph_pbc, 2022): every periodic image of every atom of the same
    structure within `radius` of each target atom, the image range per axis being the batch maximum of
    ceil(radius / plane spacing); with max_num_neighbors_threshold > 0 each target keeps that many nearest (ties: first
    in enumeration order), <= 0 keeps all.  pos [N, 3] fp32, cell [B, 3, 3] (rows = lattice vectors), natoms [B].

    Returns (edge_index [2, E] int64 = (source j, target i), grouped by target, sources then image cells in the
    reference's enumeration order; cell_offsets [E, 3] fp32 integer image cells; neighbors [B] int64 edges per
    structure).  One host synchronisation (the edge total).  Raises ValueError for a cell of zero or non-finite volume,
    natoms that do not sum to N, or more than 2^31 - 1 edges."""
    if pos.dim() != 2 or pos.size(1) != 3:
        raise ValueError(f"pos must be [N, 3], got {tuple(pos.shape)}")
    if natoms.dim() != 1 or cell.shape != (natoms.numel(), 3, 3):
        raise ValueError(f"cell must be [B, 3, 3] and natoms [B], got {tuple(cell.shape)} and {tuple(natoms.shape)}")
    if not 0.0 < float(radius) < float("inf"):
        raise ValueError(f"radius must be positive and finite, got {radius}")
    pos = pos.detach()
    dev = pos.device
    n, nb = pos.size(0), natoms.numel()
    cell = cell.detach().to(device=dev, dtype=torch.float32).contiguous()
    natoms = natoms.to(device=dev, dtype=torch.int64).contiguous()
    thr = int(max_num_neighbors_threshold)
    st = _stream()
    graph_ptr = torch.empty(nb + 1, dtype=torch.int32, device=dev)
    counts = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    select = torch.empty(2 * max(n, 1), dtype=torch.int32, device=dev)
    row_ptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
    info = torch.empty(6, dtype=torch.int64, device=dev)
    n_edges = ctypes.c_int64(0)
    try:
        call("dig3d_radius_graph_pbc_count", _p(pos, torch.float32, "pos"), _p(cell), _p(natoms), n, nb, float(radius),
             thr, _p(graph_ptr), _p(counts), _p(select), _p(row_ptr), _p(info), ctypes.byref(n_edges), st)
    except _lib.Dig3dError as exc:
        if exc.rc == -1:                                   # DIG3D_EINVAL: the input was rejected
            raise ValueError(str(exc)) from None
        raise
    e = n_edges.value
    edge_index = torch.empty(2, e, dtype=torch.int64, device=dev)
    cell_offsets = torch.empty(e, 3, dtype=torch.float32, device=dev)
    neighbors = torch.empty(nb, dtype=torch.int64, device=dev)
    call("dig3d_radius_graph_pbc_fill", _p(pos), _p(cell), n, nb, float(radius), _p(graph_ptr), _p(select),
         _p(row_ptr), _p(info), e, _p(edge_index), _p(cell_offsets), _p(neighbors), st)
    return edge_index, cell_offsets, neighbors


# ----------------------------------------------------------------------------- ComENet
def comenet_geometry(g, pos, cutoff, want_angles=False):
    """-> (feature1 [E,12], feature2 [E,6], angles [E,3] or None).  The reference atoms it chose stay on the graph
    (g.comenet_refs) for the force kernels below."""
    dev = pos.device
    e, n = g.n_edges, g.n_nodes
    refs = torch.empty(4 * max(n, 1) + 2, dtype=torch.int32, device=dev)   # + the two batch-wide "empty segment" flags
    f1 = torch.empty(max(e, 1), 12, dtype=torch.float32, device=dev)[:e]
    f2 = torch.empty(max(e, 1), 6, dtype=torch.float32, device=dev)[:e]
    angles = torch.empty(e, 3, dtype=torch.float32, device=dev) if want_angles else None
    call("dig3d_comenet_geometry", _p(pos.detach(), torch.float32, "pos"), _p(g.dist), _p(g.src), _p(g.dst),
         _p(g.row_ptr), _p(g.graph_ptr), _p(g.batch, torch.int64), n, e, float(cutoff), _p(refs), _p(f1), _p(f2),
         _p(angles) if want_angles else None, _stream())
    g.comenet_refs = refs
    return f1, f2, angles


def _comenet_force_inputs(g, pos):
    if getattr(g, "comenet_refs", None) is None:
        raise ValueError("ComENet forces need the reference atoms of ops.comenet_geometry(g, pos, ...) on the graph")
    if g.out_ptr is None or g.out_list is None:
        raise ValueError("ComENet forces need the graph's out-edge lists (ops.build_graph)")
    return _p(pos.detach(), torch.float32, "pos")


def comenet_features_bwd(g, pos, cutoff, df1, df2):
    """dpos [N, 3] = d loss / d pos through comenet_geometry's feature1 / feature2 given their gradients df1 [E,12] /
    df2 [E,6].  Deterministic (no float atomics)."""
    p = _comenet_force_inputs(g, pos)
    e, n = g.n_edges, g.n_nodes
    dpos = torch.empty(n, 3, dtype=F32, device=pos.device)
    work = torch.empty(max(18 * e, 1), dtype=F32, device=pos.device)
    if n:
        call("dig3d_comenet_features_bwd", p, _p(g.dist), _p(g.src), _p(g.dst), _p(g.row_ptr), _p(g.out_ptr),
             _p(g.out_list), _p(g.comenet_refs), n, e, float(cutoff), _p(df1, F32, "df1"), _p(df2, F32, "df2"),
             _p(work), _p(dpos), _stream())
    return dpos


def comenet_features_tangent(g, pos, cutoff, cvec):
    """(feature1_dot [E,12], feature2_dot [E,6]) along the per-atom displacement cvec [N, 3]."""
    p = _comenet_force_inputs(g, pos)
    e, n = g.n_edges, g.n_nodes
    f1d = torch.empty(max(e, 1), 12, dtype=F32, device=pos.device)[:e]
    f2d = torch.empty(max(e, 1), 6, dtype=F32, device=pos.device)[:e]
    if e:
        call("dig3d_comenet_features_tangent", p, _p(g.dist), _p(g.src), _p(g.dst), _p(g.comenet_refs), n, e,
             float(cutoff), _p(cvec, F32, "cvec"), _p(f1d), _p(f2d), _stream())
    return f1d, f2d


def comenet_ocp_features_bwd(gv, cutoff, df1, df2):
    """ComENet-OCP: (dpos [N, 3], dvec [E, 3]) = d loss / d pos and d loss / d(distance vector) through the features of
    dig3d_comenet_geometry_edges, given their gradients df1 [E,12] / df2 [E,6] in the target-sorted edge order of the
    graph view `gv` (comenet_ocp.ComENet._edge_geometry: vec, dist, src, dst, row_ptr, out_ptr, out_list, refs in that
    order).  Deterministic (no float atomics)."""
    e, n = gv.n_edges, gv.n_nodes
    dev = gv.vec.device
    if e == 0:
        return torch.zeros(n, 3, dtype=F32, device=dev), torch.zeros(0, 3, dtype=F32, device=dev)
    dpos = torch.empty(n, 3, dtype=F32, device=dev)
    work = torch.empty(18 * e, dtype=F32, device=dev)
    if n:
        call("dig3d_comenet_features_bwd_vec", _p(gv.vec, F32, "vec"), _p(gv.dist), _p(gv.src), _p(gv.dst),
             _p(gv.row_ptr), _p(gv.out_ptr), _p(gv.out_list), _p(gv.refs), n, e, float(cutoff), _p(df1, F32, "df1"),
             _p(df2, F32, "df2"), _p(work), _p(dpos), _stream())
    return dpos, work[15 * e:18 * e].view(e, 3)


def comenet_ocp_features_tangent(gv, cutoff, cvec):
    """(feature1_dot [E,12], feature2_dot [E,6]) of ComENet-OCP along the per-atom displacement cvec [N, 3], the cell held
    fixed, in the graph view's target-sorted edge order."""
    e, n = gv.n_edges, gv.n_nodes
    dev = gv.vec.device
    f1d = torch.empty(max(e, 1), 12, dtype=F32, device=dev)[:e]
    f2d = torch.empty(max(e, 1), 6, dtype=F32, device=dev)[:e]
    if e:
        call("dig3d_comenet_features_tangent_vec", _p(gv.vec, F32, "vec"), _p(gv.dist), _p(gv.src), _p(gv.dst),
             _p(gv.refs), n, e, float(cutoff), _p(cvec, F32, "cvec"), _p(f1d), _p(f2d), _stream())
    return f1d, f2d


def pbc_cell_bwd(dvec, cell_offsets, row_ptr, graph_ptr, n_graphs):
    """dcell [G, 3, 3] = sum over each graph's edges of cell_offsets[e]^T dvec[e] (the cell term of get_pbc_distances'
    distance_vec = pos[row] - pos[col] + cell_offsets . cell); edges in target-sorted order, graph g's edges
    row_ptr[graph_ptr[g]] .. row_ptr[graph_ptr[g + 1]].  Deterministic (no float atomics)."""
    if dvec.numel() == 0:
        return torch.zeros(n_graphs, 3, 3, dtype=F32, device=dvec.device)
    dcell = torch.empty(n_graphs, 3, 3, dtype=F32, device=dvec.device)
    if n_graphs:
        call("dig3d_pbc_cell_bwd", _p(dvec, F32, "dvec"), _p(cell_offsets, F32, "cell_offsets"), _p(row_ptr),
             _p(graph_ptr), n_graphs, _p(dcell), _stream())
    return dcell


def comenet_embed(z, emb_weight):
    n = z.numel()
    x = torch.empty(n, emb_weight.size(1), dtype=torch.float32, device=emb_weight.device)
    call("dig3d_comenet_embed", _p(z, torch.int64, "z"), _p(emb_weight.detach(), torch.float32), n, _p(x), _stream())
    return x


def pack_comenet_block(m):
    w = _lib.ComenetBlockWeights()
    w.w_lin, w.b_lin = _wp(m.lin.weight, "lin.w"), _wp(m.lin.bias, "lin.b")
    w.w_f1a, w.w_f1b = _wp(m.lin_feature1.lin1.weight, "f1.lin1"), _wp(m.lin_feature1.lin2.weight, "f1.lin2")
    w.w_f2a, w.w_f2b = _wp(m.lin_feature2.lin1.weight, "f2.lin1"), _wp(m.lin_feature2.lin2.weight, "f2.lin2")
    w.w_rel1, w.b_rel1, w.w_root1 = (_wp(m.conv1.lin_rel.weight, "c1.rel.w"), _wp(m.conv1.lin_rel.bias, "c1.rel.b"),
                                     _wp(m.conv1.lin_root.weight, "c1.root"))
    w.w_rel2, w.b_rel2, w.w_root2 = (_wp(m.conv2.lin_rel.weight, "c2.rel.w"), _wp(m.conv2.lin_rel.bias, "c2.rel.b"),
                                     _wp(m.conv2.lin_root.weight, "c2.root"))
    w.w_lin1, w.b_lin1 = _wp(m.lin1.weight, "lin1.w"), _wp(m.lin1.bias, "lin1.b")
    w.w_lin2, w.b_lin2 = _wp(m.lin2.weight, "lin2.w"), _wp(m.lin2.bias, "lin2.b")
    w.w_cat, w.b_cat = _wp(m.lin_cat.weight, "lin_cat.w"), _wp(m.lin_cat.bias, "lin_cat.b")
    for l, lin in enumerate(m.lins):
        w.w_lins[l], w.b_lins[l] = _wp(lin.weight, "lins.w"), _wp(lin.bias, "lins.b")
    w.n_lins = len(m.lins)
    w.norm_w, w.norm_b, w.norm_ms = _wp(m.norm.weight, "norm.w"), _wp(m.norm.bias, "norm.b"), _wp(m.norm.mean_scale, "norm.ms")
    w.w_final, w.b_final = _wp(m.final.weight, "final.w"), _wp(m.final.bias, "final.b")
    return w


def pack_comenet_head(lins, lin_out):
    h = _lib.ComenetHeadWeights()
    for l, lin in enumerate(lins):
        h.w_lins[l], h.b_lins[l] = _wp(lin.weight, "head.lins.w"), _wp(lin.bias, "head.lins.b")
    h.n_lins = len(lins)
    if lin_out is not None:
        h.w_out, h.b_out = _wp(lin_out.weight, "lin_out.w"), _wp(lin_out.bias, "lin_out.b")
    return h


def comenet_block(x, f1, f2, g, w, head, out_channels, last):
    """One SimpleInteractionBlock; returns x_next [N,256], or node_out [N,out_channels] when `last`."""
    dev = x.device
    n, hch = x.shape
    xs = torch.empty(n, hch, dtype=torch.float32, device=dev)
    h = torch.empty(n, hch, dtype=torch.float32, device=dev)
    agg = torch.zeros(2, n, hch, dtype=torch.float32, device=dev)
    stats = torch.empty(2, max(g.n_graphs, 1), hch, dtype=torch.float32, device=dev)
    x_out = None if last else torch.empty(n, hch, dtype=torch.float32, device=dev)
    node_out = torch.empty(n, out_channels, dtype=torch.float32, device=dev) if last else None
    call("dig3d_comenet_block", _p(x, torch.float32, "x", 16), _p(f1), _p(f2), _p(g.src), _p(g.dst),
         _p(g.graph_ptr), _p(g.batch, torch.int64), n, g.n_edges, g.n_graphs, ctypes.byref(w), ctypes.byref(head),
         int(out_channels), _p(xs), _p(agg[0]), _p(agg[1]), _p(h), _p(stats), _p(x_out) if x_out is not None else None,
         _p(node_out) if node_out is not None else None, _stream())
    return node_out if last else x_out


def edge_weighted_sum(w, x, g):
    """agg[i] = sum_{e=(j->i)} w[e] * x[j]  (EdgeGraphConv, comenet.py:66-73); w [E, W] in the graph's CSR edge order."""
    out = torch.empty(g.n_nodes, x.size(1), dtype=torch.float32, device=x.device)
    if g.n_nodes:
        call("dig3d_edge_weighted_sum", _p(w, torch.float32, "w", 16), _p(x, torch.float32, "x", 16), _p(g.src),
             _p(g.row_ptr), g.n_nodes, x.size(1), _p(out, align=16), _stream())
    return out


def comenet_filter_sum(feat, weff_t, x, g):
    """agg[i] = sum_{e=(j->i)} (feat[e] @ weff_t) * x[j]: EdgeGraphConv aggregation with the TwoLayerLinear filter folded
    into one [Q, W] matrix (comenet.py:66-73, :87-112)."""
    out = torch.empty(g.n_nodes, x.size(1), dtype=torch.float32, device=x.device)
    if g.n_nodes:
        call("dig3d_comenet_filter_sum", _p(feat, torch.float32, "feat"), feat.size(1), _p(weff_t, torch.float32, "weff_t", 16),
             _p(x, torch.float32, "x", 16), _p(g.src), _p(g.row_ptr), g.n_nodes, x.size(1), _p(out, align=16), _stream())
    return out


# ----------------------------------------------------------------------------- wgmma update_e
_TC_MATS = ("lin_ji", "lin_kj", "lin_down", "lin_up", "lin")


# Generation counter of every packed-weight cache below.  Writes through `tensor.data` (EMA weight swaps,
# `reset_parameters`) do not bump `tensor._version`, so the model classes call invalidate_packed() from
# reset_parameters / load_state_dict / train(); user code that edits `.data` of an eval-mode model must call it too.
_PACK_GENERATION = [0]


def invalidate_packed():
    _PACK_GENERATION[0] += 1


# A parameter object that is REPLACED (module.weight = nn.Parameter(...)) is invisible to caches keyed on the old
# object's version / address: every parameter registration in the process bumps the generation (cheap; model
# construction bumps it a few hundred times, nothing is cached yet).
try:
    from torch.nn.modules.module import register_module_parameter_registration_hook as _reg_hook
    _reg_hook(lambda _module, _name, _param: invalidate_packed())
except ImportError:          # older torch: replaced parameters need an explicit model.invalidate_packed()
    pass


def plan_key(model, *extra):
    """(cached parameter list, key) of a model's inference plan: pack generation, sum of tensor._version, every parameter's
    storage address, plus `extra`.  The list is cached on the model and refreshed by plan_key_refresh() on a miss."""
    params = model.__dict__.get("_plan_params")
    if params is None:
        params = model.__dict__["_plan_params"] = list(model.parameters())
    return (_PACK_GENERATION[0], sum(p._version for p in params), tuple(p.data_ptr() for p in params)) + tuple(extra)


def plan_key_refresh(model, *extra):
    """On a plan miss: re-read the parameter list (parameters may have been replaced or moved) and return the key the new
    plan is stored under."""
    model.__dict__.pop("_plan_params", None)
    return plan_key(model, *extra)


def _pack_matrices(mats, kind):
    """One device buffer holding the packed copies of `mats` ([N, K] fp32 weights) + their byte offsets.
    kind 'tc': TF32 hi/lo planes (dig3d_tc_pack, 8*N*K bytes); kind 'h16': FP16 hi/lo slabs (dig3d_h16_pack, 4*N*K)."""
    dev = mats[0].device
    per = 8 if kind == "tc" else 4
    sizes = [per * w.size(0) * w.size(1) for w in mats]
    offs = [0]
    for sz in sizes:
        offs.append(offs[-1] + sz)
    buf = torch.empty(offs[-1], dtype=torch.uint8, device=dev)
    if buf.data_ptr() % 128:
        raise RuntimeError("packed weight buffer is not 128-byte aligned")
    for first in range(0, len(mats), 16):
        chunk = mats[first:first + 16]
        n = len(chunk)
        wp = (ctypes.c_void_p * n)(*[_p(w.detach(), torch.float32, "w", 16).value for w in chunk])
        op = (ctypes.c_void_p * n)(*[buf.data_ptr() + o for o in offs[first:first + n]])
        ns = (ctypes.c_int32 * n)(*[w.size(0) for w in chunk])
        ks = (ctypes.c_int32 * n)(*[w.size(1) for w in chunk])
        call("dig3d_tc_pack" if kind == "tc" else "dig3d_h16_pack", wp, ns, ks, op, n, _stream())
    return buf, offs


def tc_pack_update_e(m, torsion, cache, kind="tc"):
    """Packed (hi/lo split, UMMA layout) copies of the dense weights of one update_e block for the tensor-core
    chain `kind` ('tc' = 3xTF32, 'h16' = 3xFP16).  `cache` (a dict owned by the model) keeps them until a
    parameter changes (tensor._version) or the model invalidates it (`invalidate_packed()`: writes through
    `.data` do not bump `_version`)."""
    mats = [m.lin_ji.weight, m.lin_kj.weight, m.lin_down.weight, m.lin_up.weight]
    res = list(m.layers_before_skip) + list(m.layers_after_skip)
    for layer in res:
        mats += [layer.lin1.weight, layer.lin2.weight]
    mats.append(m.lin.weight)
    key = (_PACK_GENERATION[0],) + tuple((w.data_ptr(), w._version) for w in mats)
    hit = cache.get((id(m), kind))
    if hit is None or hit[0] != key:
        buf, offs = _pack_matrices(mats, kind)
        hit = (key, buf, offs)
        cache[(id(m), kind)] = hit
    _, buf, offs = hit
    base = buf.data_ptr()
    w = _lib.TcUpdateE()
    w.p_ji, w.p_kj, w.p_down, w.p_up = (base + offs[0], base + offs[1], base + offs[2], base + offs[3])
    for r in range(6):
        w.p_res[r] = base + offs[4 + r]
    w.p_lin = base + offs[10]
    w.b_ji, w.b_kj, w.b_lin = _wp(m.lin_ji.bias, "b_ji"), _wp(m.lin_kj.bias, "b_kj"), _wp(m.lin.bias, "b_lin")
    for r, layer in enumerate(res):
        w.b_res[2 * r], w.b_res[2 * r + 1] = _wp(layer.lin1.bias, "res.b1"), _wp(layer.lin2.bias, "res.b2")
    w.w_rbf1, w.w_rbf2, w.w_rbf = _wp(m.lin_rbf1.weight, "rbf1"), _wp(m.lin_rbf2.weight, "rbf2"), _wp(m.lin_rbf.weight, "rbf")
    w.w_sbf2 = _wp(m.lin_sbf2.weight, "sbf2")
    w.w_t2 = _wp(m.lin_t2.weight, "t2") if torsion else None
    return w


def tc_pack_matrix(weight, cache, key, kind="tc"):
    """Packed copy of one [N, K] weight (cached until the parameter changes).  The buffer is OWNED by `cache`:
    keep the dict alive until the kernels that read it have run (the model keeps it for its lifetime)."""
    k = (_PACK_GENERATION[0], weight.data_ptr(), weight._version)
    hit = cache.get((key, kind))
    if hit is None or hit[0] != k:
        buf, _ = _pack_matrices([weight], kind)
        hit = (k, buf)
        cache[(key, kind)] = hit
    return hit[1]


def sphere_init_e_tc(z, g, rbf0, w, packed_lin, hidden, v_in=None):
    e1 = torch.empty(max(g.n_edges, 1), hidden, dtype=torch.float32, device=rbf0.device)[:g.n_edges]
    if v_in is None:
        v_in = torch.zeros(g.n_nodes, hidden, dtype=torch.float32, device=rbf0.device)
    if g.n_edges:
        call("dig3d_sphere_init_e_tc", _p(z, torch.int64, "z"), _p(g.src), _p(g.dst), _p(rbf0), g.n_edges,
             ctypes.byref(w), _p(packed_lin), _p(e1), _p(v_in), _stream())
    return e1, v_in


def sphere_update_e_tc(e1, g, rbf0, sbf_p, t_p, col0, w, hidden, int_emb, v_in=None):
    """update_e (A + triplet gather + B) with the dense chain on wgmma."""
    dev = e1.device
    e = g.n_edges
    x_ji = torch.empty(max(e, 1), hidden, dtype=torch.float32, device=dev)[:e]
    x_down = torch.empty(max(e, 1), int_emb, dtype=torch.float32, device=dev)[:e]
    m_ws = torch.empty(max(e, 1), int_emb, dtype=torch.float32, device=dev)[:e]
    e1_out = torch.empty(max(e, 1), hidden, dtype=torch.float32, device=dev)[:e]
    if v_in is None:
        v_in = torch.zeros(g.n_nodes, hidden, dtype=torch.float32, device=dev)
    if e:
        st = _stream()
        call("dig3d_sphere_update_e_a_tc", _p(e1), _p(rbf0), e, ctypes.byref(w), _p(x_ji), _p(x_down), st)
        sp = ctypes.c_void_p(sbf_p[col0 // 8].data_ptr())
        tp = ctypes.c_void_p(t_p[col0 // 8].data_ptr()) if t_p is not None else None
        call("dig3d_sphere_triplet_gather", _p(x_down), sp, tp, 8, _p(g.src), _p(g.dst), _p(g.row_ptr),
             _p(g.trip_ptr), e, w.w_sbf2, w.w_t2, _p(m_ws), st)
        call("dig3d_sphere_update_e_b_tc", _p(m_ws), _p(e1), _p(x_ji), _p(rbf0), _p(g.dst), e, ctypes.byref(w),
             _p(e1_out), _p(v_in), st)
    return e1_out, v_in, x_ji, x_down


# "warp" (default): one warp per (source node, share) -- rows staged in the warp's own shared memory by one bulk copy, no
# CTA-wide barrier; "node": one CTA per source node (round 2's first node-centred kernel); "tc": the node organisation
# with the 8 -> 64 expansions on wgmma (3xFP16 operands); "edge": one warp per edge.  "warp" / "node" / "edge" are
# bit-identical.
GATHER_MODE = ["warp"]
# warps sharing one node in "warp" mode; None = by the average number of triplets per node
GATHER_SPLIT = [None]


def gather_split(g):
    if GATHER_SPLIT[0] is not None:
        return int(GATHER_SPLIT[0])
    per_node = g.n_triplets / max(g.n_nodes, 1)
    return max(1, min(8, int(per_node // 384) + 1))


def _ptr(x):
    """Device pointer argument: a raw address (int, workspace of the planned inference forward) or a validated tensor."""
    return x if type(x) is int else _p(x)


def triplet_gather(x_down, sp, tp, g, w_sbf2, w_t2, m_out, st):
    """m[e] = sum_t x_down[kj] * lin_sbf2(sbf_p) * lin_t2(t_p)  (spherenet.py:163-171); sp / tp are layer slices.
    x_down / m_out: tensors or raw device addresses."""
    mode = GATHER_MODE[0]
    if mode == "warp":
        call("dig3d_sphere_triplet_gather_warp", _ptr(x_down), sp, tp, 8, _p(g.src), _p(g.row_ptr), _p(g.trip_ptr),
             _p(g.graph_ptr), _p(g.batch, torch.int64), g.n_nodes, g.cap, gather_split(g), w_sbf2, w_t2, _ptr(m_out),
             *_out_lists(g), st)
    elif mode in ("node", "tc"):
        call("dig3d_sphere_triplet_gather_tc" if mode == "tc" else "dig3d_sphere_triplet_gather_node", _ptr(x_down), sp,
             tp, 8, _p(g.src), _p(g.row_ptr), _p(g.trip_ptr), _p(g.graph_ptr), _p(g.batch, torch.int64), g.n_nodes, g.cap,
             w_sbf2, w_t2, _ptr(m_out), st)
    else:
        call("dig3d_sphere_triplet_gather", _ptr(x_down), sp, tp, 8, _p(g.src), _p(g.dst), _p(g.row_ptr),
             _p(g.trip_ptr), g.n_edges, w_sbf2, w_t2, _ptr(m_out), st)


def init_e_tables(init_e, cache):
    """(tab_i, tab_j, packed rbf panel) of an init_e block for dig3d_sphere_init_e_h16_tab: the first two K = 128 panels of
    lin(cat[x_i, x_j, rbf0]) only depend on the atomic number, so they become two [emb rows, 128] tables (exact fp32
    FFMA GEMMs); the third panel is packed for the tensor engine.  Cached in `cache` per parameter version."""
    w, emb = init_e.lin.weight, init_e.emb.weight
    key = (_PACK_GENERATION[0], w.data_ptr(), w._version, emb.data_ptr(), emb._version)
    hit = cache.get("init_e.tables")
    if hit is None or hit[0] != key:
        wd, ed = w.detach(), emb.detach().contiguous()
        tab_i = linear(ed, wd[:, :128].contiguous())
        tab_j = linear(ed, wd[:, 128:256].contiguous())
        packed, _ = _pack_matrices([wd[:, 256:384].contiguous()], "h16")
        hit = (key, tab_i, tab_j, packed)
        cache["init_e.tables"] = hit
    return hit[1], hit[2], hit[3]


def sphere_init_e_h16(z, g, rbf0, w, packed_lin, hidden, v_in=None, tables=None):
    """tables = init_e_tables(...): the table form (one K = 128 job per tile); else three K = 128 panels of packed_lin."""
    e1 = torch.empty(max(g.n_edges, 1), hidden, dtype=torch.float32, device=rbf0.device)[:g.n_edges]
    if v_in is None:
        v_in = torch.zeros(g.n_nodes, hidden, dtype=torch.float32, device=rbf0.device)
    if g.n_edges and tables is not None:
        tab_i, tab_j, packed = tables
        call("dig3d_sphere_init_e_h16_tab", _p(z, torch.int64, "z"), _p(g.src), _p(g.dst), _p(rbf0), g.n_edges,
             ctypes.byref(w), _p(packed), _p(tab_i, torch.float32, "tab_i", 16), _p(tab_j, torch.float32, "tab_j", 16),
             _p(e1), _p(v_in), _stream())
    elif g.n_edges:
        call("dig3d_sphere_init_e_h16", _p(z, torch.int64, "z"), _p(g.src), _p(g.dst), _p(rbf0), g.n_edges,
             ctypes.byref(w), _p(packed_lin), _p(e1), _p(v_in), _stream())
    return e1, v_in


def sphere_update_e_h16(e1, g, rbf0, sbf_p, t_p, col0, w, hidden, int_emb, v_in=None):
    """update_e (A + triplet gather + B) with the dense chain on wgmma, register-accumulator engine (3xFP16)."""
    dev = e1.device
    e = g.n_edges
    x_ji = torch.empty(max(e, 1), hidden, dtype=torch.float32, device=dev)[:e]
    x_down = torch.empty(max(e, 1), int_emb, dtype=torch.float32, device=dev)[:e]
    m_ws = torch.empty(max(e, 1), int_emb, dtype=torch.float32, device=dev)[:e]
    e1_out = torch.empty(max(e, 1), hidden, dtype=torch.float32, device=dev)[:e]
    if v_in is None:
        v_in = torch.zeros(g.n_nodes, hidden, dtype=torch.float32, device=dev)
    if e:
        st = _stream()
        call("dig3d_sphere_update_e_a_h16", _p(e1), _p(rbf0), e, ctypes.byref(w), _p(x_ji), _p(x_down), st)
        sp = ctypes.c_void_p(sbf_p[col0 // 8].data_ptr())
        tp = ctypes.c_void_p(t_p[col0 // 8].data_ptr()) if t_p is not None else None
        triplet_gather(x_down, sp, tp, g, w.w_sbf2, w.w_t2, m_ws, st)
        call("dig3d_sphere_update_e_b_h16", _p(m_ws), _p(e1), _p(x_ji), _p(rbf0), _p(g.dst), e, ctypes.byref(w),
             _p(e1_out), _p(v_in), st)
    return e1_out, v_in, x_ji, x_down


def update_v_h16_supported(holder, out_channels):
    return bool(_lib.load().dig3d_sphere_update_v_h16_supported(
        holder.lin_up.weight.size(1), holder.lin_up.weight.size(0), int(out_channels), len(holder.lins)))


def pack_update_v_h16(holders, cache):
    """(packed-weight pointer array, UpdateVWeights array, n_lins) of the node MLPs for dig3d_sphere_update_v_h16; the
    packed buffers live in `cache` (same invalidation rules as tc_pack_update_e)."""
    n_lins = len(holders[0].lins)
    ptrs = []
    for h in holders:
        mats = [h.lin_up.weight] + [lin.weight for lin in h.lins]
        key = (_PACK_GENERATION[0],) + tuple((w.data_ptr(), w._version) for w in mats)
        hit = cache.get((id(h), "h16v"))
        if hit is None or hit[0] != key:
            halves = []
            for w in mats:                                   # output rows 0..127, then 128..255, back to back
                halves += [w.detach()[:128], w.detach()[128:]]
            buf, offs = _pack_matrices(halves, "h16")
            hit = (key, buf, offs)
            cache[(id(h), "h16v")] = hit
        _, buf, offs = hit
        ptrs += [buf.data_ptr() + offs[2 * l] for l in range(n_lins + 1)]
    parr = (ctypes.c_void_p * len(ptrs))(*ptrs)
    return parr, pack_update_v_array(holders), n_lins


def sphere_update_v_h16(v_in_all, holders, out_channels, v_out_all, cache):
    """All node MLPs of a forward in one launch on the register-accumulator engine (3xFP16 operands).
    v_in_all [NB, N, 128], holders: NB update_v modules (128 -> 256 -> ... -> out_channels)."""
    nb, n, _ = v_in_all.shape
    parr, arr, n_lins = pack_update_v_h16(holders, cache)
    if n:
        call("dig3d_sphere_update_v_h16", _p(v_in_all, torch.float32, "v_in_all", 16), n, nb, int(out_channels), n_lins,
             parr, arr, _p(v_out_all, align=4), _stream())
    return v_out_all


def h16_overflow(clear=True):
    """True if an operand of the 3xFP16 chain left the fp16 range (|activation| >= 8190) since the last clear.  Every
    3xFP16 entry point (init_e, update_e parts A / B / BA, update_v, linear_h16) raises it in the launch whose outputs
    the out-of-range operand turned into inf / NaN."""
    return bool(_lib.load().dig3d_h16_overflow(int(bool(clear))))


def h16_set_fast_swish(on):
    call("dig3d_h16_set_fast_swish", int(bool(on)))


def tc_set_fast_swish(on):
    call("dig3d_tc_set_fast_swish", int(bool(on)))


def tc_timeouts():
    """mbarrier waits that timed out in the tensor-core kernels (they trap, so a non-zero count is only ever seen
    together with a failed launch)."""
    lib = _lib.load()
    return lib.dig3d_tc_timeouts() + lib.dig3d_h16_timeouts() + lib.dig3d_wgrad_tc_timeouts()


def wgrad_set_mode(tensor_cores):
    """True (default): weight gradients of >= 64-wide layers on wgmma (3xTF32, csrc/train_tc.cu); False: FFMA kernel."""
    _lib.load().dig3d_wgrad_set_mode(1 if tensor_cores else 0)


# ---------------------------------------------------------------------------------------------------------------
# Training primitives (csrc/train_ops.cu); dig_b200/autograd.py wraps them in autograd Functions.
F32 = torch.float32


def _idx(t, name="index"):
    if t.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"{name}: expected an int32 or int64 index tensor, got {t.dtype}")
    return _p(t, None, name), int(t.dtype == torch.int64)


def linear(x, weight, bias=None, want_act=False):
    """y = x weight^T + bias for x [..., K] (nn.Linear); want_act: also swish(y) from the same kernel.
    Grouped form: weight [G, N, K] (3-D) with x [G, rows, K] and bias [G, N]: G independent linears in one launch."""
    groups = weight.size(0) if weight.dim() == 3 else 1
    k = x.size(-1)
    nout = weight.size(-2)
    if weight.dim() not in (2, 3) or weight.size(-1) != k:
        raise ValueError(f"linear: weight {tuple(weight.shape)} does not match input width {k}")
    if groups > 1 or weight.dim() == 3:
        if x.dim() != 3 or x.size(0) != groups or (bias is not None and tuple(bias.shape) != (groups, nout)):
            raise ValueError(f"grouped linear: x {tuple(x.shape)}, weight {tuple(weight.shape)} do not agree")
    if x.numel() == 0:                       # empty edge / triplet sets (isolated atoms): nothing to launch
        y = torch.zeros(x.shape[:-1] + (nout,), device=x.device, dtype=torch.float32)
        return (y, y.clone()) if want_act else y
    rows = x.numel() // k // groups
    y = torch.empty(x.shape[:-1] + (nout,), device=x.device, dtype=F32)
    act_out = torch.empty_like(y) if want_act else None
    call("dig3d_linear", _p(x, F32, "x"), rows, k, nout, _p(weight, F32, "weight"), _p(bias, F32, "bias"),
         _p(y), _p(act_out), groups, _stream())
    return (y, act_out) if want_act else y


def adam_step(param, grad, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, weight_decay, step):
    """One fused Adam update over flat fp32 buffers (parallel.FlatAdam)."""
    n = param.numel()
    if not (grad.numel() == exp_avg.numel() == exp_avg_sq.numel() == n):
        raise ValueError("adam_step: buffer sizes differ")
    call("dig3d_adam_step", _p(param, F32, "param", 16), _p(grad, F32, "grad", 16), _p(exp_avg, F32, "exp_avg", 16),
         _p(exp_avg_sq, F32, "exp_avg_sq", 16), n, lr, beta1, beta2, eps, weight_decay, int(step), _stream())


def wgrad(dy, x, weight_shape, want_bias):
    """(dW, db) of y = x W^T + b given dy; weight_shape (N, K) or, grouped, (G, N, K) with dy [G,rows,N], x [G,rows,K]."""
    groups = weight_shape[0] if len(weight_shape) == 3 else 1
    nout, k = weight_shape[-2], weight_shape[-1]
    lead = (groups,) if len(weight_shape) == 3 else ()
    dev = x.device
    buf = torch.zeros(groups * nout * k + (groups * nout if want_bias else 0), device=dev, dtype=F32)   # one fill
    dw = buf[:groups * nout * k].view(lead + (nout, k))
    db = buf[groups * nout * k:].view(lead + (nout,)) if want_bias else None
    if x.numel() == 0:
        return dw, db
    rows = x.numel() // k // groups
    call("dig3d_wgrad", _p(dy, F32, "dy"), _p(x, F32, "x"), rows, nout, k, _p(dw), _p(db), groups, _stream())
    return dw, db


def act(x, mode):
    if x.numel() == 0:
        return torch.empty_like(x)
    y = torch.empty_like(x)
    call("dig3d_act", _p(x, F32, "x"), x.numel(), mode, _p(y), _stream())
    return y


def act_bwd(x, dy, mode):
    if x.numel() == 0:
        return torch.empty_like(x)
    dx = torch.empty_like(x)
    call("dig3d_act_bwd", _p(x, F32, "x"), _p(dy, F32, "dy"), x.numel(), mode, _p(dx), _stream())
    return dx


def ewise(a, b, op):
    if a.shape != b.shape:
        raise ValueError(f"ewise: shapes differ {tuple(a.shape)} vs {tuple(b.shape)}")
    y = torch.empty_like(a)
    if a.numel() == 0:
        return y
    call("dig3d_ewise", _p(a, F32, "a"), _p(b, F32, "b"), a.numel(), op, _p(y), _stream())
    return y


def rowscale(a, s):
    if a.numel() == 0:
        return torch.empty_like(a)
    rows, width = a.size(0), a.numel() // max(a.size(0), 1)
    if s.numel() != rows:
        raise ValueError("rowscale: one scale per row expected")
    y = torch.empty_like(a)
    call("dig3d_rowscale", _p(a, F32, "a"), _p(s, F32, "s"), rows, width, _p(y), _stream())
    return y


def gather_rows(x, idx):
    if idx.numel() == 0:
        return torch.empty((0,) + tuple(x.shape[1:]), device=x.device, dtype=torch.float32)
    width = x.numel() // max(x.size(0), 1) if x.dim() > 1 else 1
    rows = idx.numel()
    y = torch.empty((rows,) + tuple(x.shape[1:]), device=x.device, dtype=F32)
    ip, i64 = _idx(idx)
    call("dig3d_gather_rows", _p(x, F32, "x"), ip, i64, rows, width, _p(y), _stream())
    return y


def scatter_add_rows(y, idx, n_rows):
    if idx.numel() == 0:
        return torch.zeros((n_rows,) + tuple(y.shape[1:]), device=y.device, dtype=torch.float32)
    width = y.numel() // max(y.size(0), 1) if y.dim() > 1 else 1
    out = torch.zeros((n_rows,) + tuple(y.shape[1:]), device=y.device, dtype=F32)
    ip, i64 = _idx(idx)
    call("dig3d_scatter_add_rows", _p(y, F32, "y"), ip, i64, idx.numel(), width, _p(out), _stream())
    return out


def transpose(w):
    rows, cols = w.shape
    out = torch.empty(cols, rows, device=w.device, dtype=F32)
    call("dig3d_transpose", _p(w, F32, "w"), rows, cols, _p(out), _stream())
    return out


def schnet_edge_features(dist, offset, coeff, cutoff):
    """(gaussian smearing [E, G], cosine cutoff [E]) of schnet.py:92-94 / :31, materialised for the training path."""
    e, ng = dist.numel(), offset.numel()
    gauss = torch.empty(e, ng, device=dist.device, dtype=F32)
    cut = torch.empty(e, device=dist.device, dtype=F32)
    if e == 0:
        return gauss, cut
    call("dig3d_schnet_edge_features", _p(dist, F32, "dist"), e, _p(offset, F32, "offset"), ng, float(coeff),
         float(cutoff), _p(gauss), _p(cut), _stream())
    return gauss, cut


def rbf_freq_grad(dist, cutoff, envelope_exponent, freq, drbf0):
    """d(loss)/d(dist_emb.freq) from d(loss)/d(rbf0)."""
    dfreq = torch.zeros_like(freq, dtype=F32)
    if dist.numel() == 0:
        return dfreq
    call("dig3d_rbf_freq_grad", _p(dist, F32, "dist"), dist.numel(), float(cutoff), int(envelope_exponent),
         _p(freq.detach(), F32, "freq"), freq.numel(), _p(drbf0, F32, "drbf0"), _p(dfreq), _stream())
    return dfreq


def sphere_triplet_gather(x_down, sbf_p, t_p, g, w_sbf2, w_t2):
    """m[E, 64] = sum over the triplets of each edge of x_down[kj] * lin_sbf2(sbf_p) * lin_t2(t_p)  (spherenet.py:163-171)."""
    e = g.n_edges
    if e == 0 or g.n_triplets == 0:
        return torch.zeros(e, x_down.size(1), device=x_down.device, dtype=F32)
    m = torch.empty(e, x_down.size(1), device=x_down.device, dtype=F32)
    if (x_down.size(1) == 64 and g.cap is not None and g.cap <= 64 and g.graph_ptr is not None and g.batch is not None
            and (x_down.data_ptr() & 15) == 0 and GATHER_MODE[0] != "edge"):
        # the inference organisation (warp per source node, out-edge lists): bit-identical to the edge-centred kernel
        triplet_gather(_p(x_down, F32, "x_down").value, _p(sbf_p, F32, "sbf_p"), _p(t_p, F32, "t_p"), g,
                       _p(w_sbf2, F32, "w_sbf2"), _p(w_t2, F32, "w_t2"), _p(m).value, _stream())
        return m
    call("dig3d_sphere_triplet_gather", _p(x_down, F32, "x_down"), _p(sbf_p, F32, "sbf_p"), _p(t_p, F32, "t_p"), 8,
         _p(g.src), _p(g.dst), _p(g.row_ptr), _p(g.trip_ptr), e, _p(w_sbf2, F32, "w_sbf2"), _p(w_t2, F32, "w_t2"),
         _p(m), _stream())
    return m


def sphere_triplet_gather_bwd(dm, x_down, sbf_p, t_p, g, w_sbf2, w_t2):
    """-> (dx_down, d_sbf_p, d_t_p | None, dw_sbf2, dw_t2 | None)."""
    dev = dm.device
    tors = t_p is not None
    dx = torch.zeros_like(x_down)
    d_s = torch.empty_like(sbf_p)
    d_t = torch.empty_like(t_p) if tors else None
    dws = torch.zeros_like(w_sbf2)
    dwt = torch.zeros_like(w_t2) if tors else None
    if g.n_edges == 0 or g.n_triplets == 0:
        return dx, d_s, d_t, dws, dwt
    call("dig3d_sphere_triplet_gather_bwd", _p(dm, F32, "dm"), _p(x_down, F32), _p(sbf_p, F32), _p(t_p, F32),
         _p(g.src), _p(g.dst), _p(g.row_ptr), _p(g.trip_ptr), g.n_edges, _p(w_sbf2, F32), _p(w_t2, F32), _p(dx),
         _p(d_s), _p(d_t), _p(dws), _p(dwt), _stream())
    return dx, d_s, d_t, dws, dwt


def triplet_basis_project_bwd(g, bess, basis_id, d_sbf_p, d_t_p, n_sbf, n_tbf):
    """d_sbf_p / d_t_p: lists (<= 4) of [T, 8] gradients or None -> dw_sbf1 [32, n_sbf], dw_t1 [32, n_tbf] | None."""
    dev = bess.device
    tors = d_t_p is not None
    dws = torch.zeros(32, n_sbf, device=dev, dtype=F32)
    dwt = torch.zeros(32, n_tbf, device=dev, dtype=F32) if tors else None
    arr = ctypes.c_void_p * 4

    def ptrs(lst):
        vals = [(_p(t, F32, "grad").value if t is not None else None) for t in lst] + [None] * (4 - len(lst))
        return arr(*vals)
    if g.n_edges == 0 or g.n_triplets == 0:
        return dws, dwt
    ps = ptrs(d_sbf_p)
    pt = ptrs(d_t_p) if tors else None
    call("dig3d_triplet_basis_project_bwd", _p(bess, F32), _p(g.angle), _p(g.torsion) if tors else None, _p(g.src),
         _p(g.dst), _p(g.row_ptr), _p(g.trip_ptr), _p(g.graph_ptr), _p(g.batch, torch.int64), g.n_edges, g.n_triplets,
         int(basis_id), ps, pt, _p(dws), _p(dwt), _stream())
    return dws, dwt


def graphnorm(h, graph_ptr, weight, bias, mean_scale, eps=1e-5):
    """-> (y, shift [G, W], std [G, W])"""
    g, wd = graph_ptr.numel() - 1, h.size(1)
    y = torch.empty_like(h)
    shift = torch.empty(g, wd, device=h.device, dtype=F32)
    std = torch.empty(g, wd, device=h.device, dtype=F32)
    call("dig3d_graphnorm", _p(h, F32, "h"), _p(graph_ptr, torch.int32), g, wd, _p(weight, F32), _p(bias, F32),
         _p(mean_scale, F32), float(eps), _p(y), _p(shift), _p(std), _stream())
    return y, shift, std


def graphnorm_bwd(h, dy, graph_ptr, weight, mean_scale, shift, std):
    g, wd = graph_ptr.numel() - 1, h.size(1)
    dx = torch.empty_like(h)
    dw = torch.zeros(wd, device=h.device, dtype=F32)
    db = torch.zeros(wd, device=h.device, dtype=F32)
    dms = torch.zeros(wd, device=h.device, dtype=F32)
    call("dig3d_graphnorm_bwd", _p(h, F32, "h"), _p(dy, F32, "dy"), _p(graph_ptr, torch.int32), g, wd, _p(weight, F32),
         _p(mean_scale, F32), _p(shift), _p(std), _p(dx), _p(dw), _p(db), _p(dms), _stream())
    return dx, dw, db, dms


def graphnorm_tangent(h, hd, graph_ptr, weight, mean_scale, shift, std):
    """y_dot of GraphNorm along h_dot, from graphnorm's shift / std."""
    g, wd = graph_ptr.numel() - 1, h.size(1)
    yd = torch.empty_like(h)
    call("dig3d_graphnorm_tangent", _p(h, F32, "h"), _p(hd, F32, "h_dot"), _p(graph_ptr, torch.int32), g, wd,
         _p(weight, F32), _p(mean_scale, F32), _p(shift), _p(std), _p(yd), _stream())
    return yd


def graphnorm_tangent_bwd(h, hd, dyd, graph_ptr, weight, mean_scale, shift, std):
    """-> (dh, dh_dot, dweight, dmean_scale) of graphnorm_tangent given dy_dot."""
    g, wd = graph_ptr.numel() - 1, h.size(1)
    dh = torch.empty_like(h)
    dhd = torch.empty_like(h)
    dw = torch.zeros(wd, device=h.device, dtype=F32)
    dms = torch.zeros(wd, device=h.device, dtype=F32)
    call("dig3d_graphnorm_tangent_bwd", _p(h, F32, "h"), _p(hd, F32, "h_dot"), _p(dyd, F32, "dy_dot"),
         _p(graph_ptr, torch.int32), g, wd, _p(weight, F32), _p(mean_scale, F32), _p(shift), _p(std), _p(dh), _p(dhd),
         _p(dw), _p(dms), _stream())
    return dh, dhd, dw, dms


# ---------------------------------------------------------------------------------------------------------------
# Position gradients (forces)
def edge_dist_bwd(pos, g, ddist, dpos):
    if g.n_edges == 0:
        return
    call("dig3d_edge_dist_bwd", _p(pos, F32, "pos"), _p(g.src), _p(g.dst), _p(g.dist), _p(ddist, F32, "ddist"), g.n_edges,
         _p(dpos), _stream())


def triplet_angle_bwd(pos, g, dangle, dpos):
    if g.n_edges == 0 or g.n_triplets == 0:
        return
    call("dig3d_triplet_angle_bwd", _p(pos, F32, "pos"), _p(g.src), _p(g.dst), _p(g.row_ptr), _p(g.trip_ptr),
         _p(dangle, F32, "dangle"), g.n_edges, _p(dpos), _stream())


def edge_basis_bwd(dist, cutoff, envelope_exponent, freq, basis_id, envelope_on_bessel, drbf0, n_bessel,
                   want_ddist=True, want_bess_dx=False):
    e = dist.numel()
    ddist = torch.zeros(e, device=dist.device, dtype=F32) if want_ddist else None
    bdx = torch.empty(e, n_bessel, device=dist.device, dtype=F32) if want_bess_dx else None
    if e == 0:
        return ddist, bdx
    call("dig3d_edge_basis_bwd", _p(dist, F32, "dist"), e, float(cutoff), int(envelope_exponent),
         _p(freq.detach(), F32, "freq") if freq is not None else None, int(basis_id), int(bool(envelope_on_bessel)),
         _p(drbf0, F32, "drbf0"), _p(ddist), _p(bdx), _stream())
    return ddist, bdx


def triplet_torsion_bwd(pos, g, dtorsion, dpos):
    if g.n_edges == 0 or g.n_triplets == 0:
        return
    call("dig3d_triplet_torsion_bwd", _p(pos, F32, "pos"), _p(g.src), _p(g.dst), _p(g.row_ptr), _p(g.trip_ptr),
         _p(dtorsion, F32, "dtorsion"), g.n_edges, _p(dpos), _stream())


def triplet_basis_project_bwd_geom(g, bess, bess_dx, basis_id, d_sbf_p, d_t_p, w_sbf1_rows, w_t1_rows, cutoff):
    """-> (ddist_kj [E], dangle [T], dtorsion [T] | None); d_t_p / w_t1_rows None = no torsion branch."""
    dev = bess.device
    tors = d_t_p is not None
    ddist = torch.zeros(g.n_edges, device=dev, dtype=F32)
    dangle = torch.zeros(g.n_triplets, device=dev, dtype=F32)
    dtors = torch.zeros(g.n_triplets, device=dev, dtype=F32) if tors else None
    arr = ctypes.c_void_p * 4

    def ptrs(lst):
        return arr(*([(_p(t, F32, "grad", align=16).value if t is not None else None) for t in lst]
                     + [None] * (4 - len(lst))))
    if g.n_edges == 0 or g.n_triplets == 0:
        return ddist, dangle, dtors
    call("dig3d_triplet_basis_project_bwd_geom", _p(bess, F32), _p(bess_dx, F32), _p(g.angle),
         _p(g.torsion) if tors else None, _p(g.src), _p(g.dst), _p(g.row_ptr), _p(g.trip_ptr), _p(g.graph_ptr),
         _p(g.batch, torch.int64), g.n_edges, g.n_triplets, int(basis_id), ptrs(d_sbf_p), ptrs(d_t_p) if tors else None,
         _p(w_sbf1_rows, F32), _p(w_t1_rows, F32) if tors else None, float(cutoff), _p(ddist), _p(dangle), _p(dtors),
         _stream())
    return ddist, dangle, dtors


def triplet_basis_bwd(g, bess, bess_dx, angle, torsion, basis_id, d_sbf, d_tbf, cutoff, want_dtorsion):
    """Reverse mode of `triplet_basis`: d_sbf [T, ns*nr] / d_tbf [T, ns*ns*nr] (either None = zero) ->
    (ddist [E], the k->j edge's share through bess; dangle [T]; dtorsion [T] | None).  bess_dx: `edge_basis_bwd`'s
    d(bess)/dx.  Needs the graph's out-edge lists (`build_graph` makes them)."""
    dev = bess.device
    e, t = g.n_edges, angle.numel()
    if g.out_ptr is None or g.out_list is None or g.pos_in is None:
        raise ValueError("triplet_basis_bwd: the graph carries no out-edge lists (build it with ops.build_graph)")
    ddist = torch.empty(e, device=dev, dtype=F32)
    dangle = torch.empty(t, device=dev, dtype=F32)
    dtors = torch.empty(t, device=dev, dtype=F32) if want_dtorsion else None
    if e == 0:
        return ddist, dangle, dtors
    call("dig3d_triplet_basis_bwd", _p(bess, F32, "bess"), _p(bess_dx, F32, "bess_dx"), _p(angle, F32, "angle"),
         _p(torsion, F32, "torsion") if (want_dtorsion or d_tbf is not None) else None, _p(g.dst), _p(g.row_ptr),
         _p(g.trip_ptr), _p(g.out_ptr), _p(g.out_list), _p(g.pos_in), e, t, int(basis_id), _p(d_sbf, F32, "d_sbf"),
         _p(d_tbf, F32, "d_tbf"), float(cutoff), _p(ddist), _p(dangle), _p(dtors), _stream())
    return ddist, dangle, dtors


def schnet_edge_features_bwd(dist, offset, coeff, cutoff, dgauss, dcut):
    ddist = torch.empty_like(dist)
    if dist.numel() == 0:
        return ddist
    call("dig3d_schnet_edge_features_bwd", _p(dist, F32, "dist"), dist.numel(), _p(offset, F32), offset.numel(),
         float(coeff), float(cutoff), _p(dgauss, F32), _p(dcut, F32), _p(ddist), _stream())
    return ddist


def rowdot(a, b):
    if a.numel() == 0:
        return torch.zeros(a.size(0), device=a.device, dtype=torch.float32)
    rows = a.size(0)
    out = torch.empty(rows, device=a.device, dtype=F32)
    call("dig3d_rowdot", _p(a, F32, "a"), _p(b, F32, "b"), rows, a.numel() // max(rows, 1), _p(out), _stream())
    return out


# ---------------------------------------------------------------------------------------------------------------
# wgmma linears of the training path
TC_LINEAR_MIN_ROWS = 512


def linear_tc_supported(k, nout):
    return (nout == 128 and k in (64, 128, 256, 384)) or (nout == 64 and k == 128)


def _packed_weight(weight, transposed):
    """TF32 hi/lo-split UMMA-layout copy of W (or W^T).  The copy lives ON the tensor object (attribute
    `_dig3d_packed`), so it dies with the parameter -- a cache keyed by address could hand a new tensor that reuses
    the storage the packed weights of a dead one -- and is re-packed when the tensor changes (tensor._version).
    Pass the parameter itself (not a .detach() view, which is a new object every time)."""
    store = weight.__dict__.setdefault("_dig3d_packed", {})
    hit = store.get(bool(transposed))
    tag = (_PACK_GENERATION[0], weight._version, weight.data_ptr(), tuple(weight.shape))
    if hit is not None and hit[0] == tag:
        return hit[1]
    n, k = (weight.size(1), weight.size(0)) if transposed else (weight.size(0), weight.size(1))
    buf = torch.empty(2 * n * k, dtype=F32, device=weight.device)
    one = ctypes.c_void_p * 1
    call("dig3d_tc_pack_t", one(_p(weight.detach(), F32, "w", 16).value), (ctypes.c_int32 * 1)(n), (ctypes.c_int32 * 1)(k),
         (ctypes.c_int32 * 1)(int(bool(transposed))), one(buf.data_ptr()), 1, _stream())
    store[bool(transposed)] = (tag, buf)
    return buf


def linear_tc(x, weight, bias=None, transposed=False, want_act=False):
    """y = x W^T + b (transposed=False) or y = x W (transposed=True: the input-gradient GEMM) on wgmma 3xTF32.
    want_act: also return swish(y)."""
    k = x.size(-1)
    nout = weight.size(1) if transposed else weight.size(0)
    rows = x.numel() // k
    packed = _packed_weight(weight, transposed)
    y = torch.empty(x.shape[:-1] + (nout,), device=x.device, dtype=F32)
    act_out = torch.empty_like(y) if want_act else None
    call("dig3d_linear_tc", _p(x, F32, "x", 16), rows, k, nout, _p(packed), _p(bias, F32, "bias"), _p(y), _p(act_out),
         _stream())
    return (y, act_out) if want_act else y


# ---------------------------------------------------------------------------------------------------------------
# training-path linears on the two-tile tensor engine (3xFP16 operands, csrc/spherenet_h16.cu)
H16_LINEAR_MIN_ROWS = 1024
_H16_REGISTRY = {}          # id(weight) -> [weakref, {transposed: (tag, buffer)}]


def linear_h16_supported(k, nout):
    return k in (64, 128, 256, 384) and 64 <= nout <= 512 and nout % 64 == 0      # == dig3d_linear_h16_supported


def _h16_tag(weight):
    return (_PACK_GENERATION[0], weight._version, weight.data_ptr(), tuple(weight.shape))


def _h16_slices(weight, transposed):
    """(source pointer offset in elements, N, K, trans) of the <= 128-row output slices of W (or W^T)."""
    n_out, k = (weight.size(1), weight.size(0)) if transposed else (weight.size(0), weight.size(1))
    out = []
    for c0 in range(0, n_out, 128):
        n = 128 if n_out - c0 >= 128 else 64
        # W [n_out, k] row-major: slice rows c0..c0+n (offset c0*k); W^T from W [k, n_out]: column slice (offset c0)
        out.append((c0 if transposed else c0 * k, n, k, n_out if transposed else 0))     # trans = source row stride
    return out


def _h16_pack_jobs(jobs):
    """jobs: (weight, transposed, buffer).  Packs every output slice, 16 slices per launch."""
    flat = []
    for w, tr, buf in jobs:
        off = 0
        for src_off, n, k, trans in _h16_slices(w, tr):
            flat.append((w.data_ptr() + 4 * src_off, n, k, trans, buf.data_ptr() + off))
            off += 4 * n * k
    for first in range(0, len(flat), 16):
        chunk = flat[first:first + 16]
        m = len(chunk)
        wp = (ctypes.c_void_p * m)(*[c[0] for c in chunk])
        ns = (ctypes.c_int32 * m)(*[c[1] for c in chunk])
        ks = (ctypes.c_int32 * m)(*[c[2] for c in chunk])
        ts = (ctypes.c_int32 * m)(*[c[3] for c in chunk])
        op = (ctypes.c_void_p * m)(*[c[4] for c in chunk])
        call("dig3d_h16_pack_t", wp, ns, ks, ts, op, m, _stream())


_H16_BATCHES = {"stamp": -1, "calls": []}      # cached ctypes argument arrays of repack_h16_all (rebuilt when the registry changes)
_H16_STAMP = [0]                                # bumps whenever an entry is added to / dropped from the registry


def _h16_packed(weight, transposed):
    """Packed 3xFP16 copy of W (or W^T) for dig3d_linear_h16, owned by a registry entry that dies with the tensor;
    repacked when the tensor changed (version / generation)."""
    import weakref
    ent = _H16_REGISTRY.get(id(weight))
    if ent is None or ent[0]() is not weight:
        def drop(_r, key=id(weight)):
            _H16_REGISTRY.pop(key, None)
            _H16_STAMP[0] += 1
        ent = [weakref.ref(weight, drop), {}]
        _H16_REGISTRY[id(weight)] = ent
    tr = bool(transposed)
    hit = ent[1].get(tr)
    if hit is not None:
        tag = hit[0]
        if tag[0] == _PACK_GENERATION[0] and tag[1] == weight._version and tag[2] == weight.data_ptr():
            return hit[1]
    tag = _h16_tag(weight)
    buf = hit[1] if hit is not None else torch.empty(4 * weight.numel(), dtype=torch.uint8, device=weight.device)
    _h16_pack_jobs([(weight.detach(), tr, buf)])
    if hit is None:
        _H16_STAMP[0] += 1
    ent[1][tr] = (tag, buf)
    return buf


def repack_h16_all():
    """Re-pack every registered weight (both orientations in use) in a few batched launches: called by the optimizer
    right after it changed the parameters, so the next step's linears find current copies.  The ctypes argument arrays
    are cached (parameter and buffer addresses do not move between steps), so a call costs ~len(registry)/16 launches."""
    cache = _H16_BATCHES
    if cache["stamp"] != _H16_STAMP[0]:
        flat, ents = [], []
        for key, ent in list(_H16_REGISTRY.items()):
            w = ent[0]()
            if w is None:
                continue
            for tr, (tag, buf) in ent[1].items():
                off = 0
                for src_off, n, k, trans in _h16_slices(w, tr):
                    flat.append((w.data_ptr() + 4 * src_off, n, k, trans, buf.data_ptr() + off))
                    off += 4 * n * k
                ents.append((ent, tr, w, buf))
        calls = []
        for first in range(0, len(flat), 16):
            chunk = flat[first:first + 16]
            m = len(chunk)
            calls.append(((ctypes.c_void_p * m)(*[c[0] for c in chunk]), (ctypes.c_int32 * m)(*[c[1] for c in chunk]),
                          (ctypes.c_int32 * m)(*[c[2] for c in chunk]), (ctypes.c_int32 * m)(*[c[3] for c in chunk]),
                          (ctypes.c_void_p * m)(*[c[4] for c in chunk]), m))
        cache.update(stamp=_H16_STAMP[0], calls=calls, ents=ents,
                     ptrs=[(w.data_ptr(), buf.data_ptr()) for _, _, w, buf in ents])
    ents = cache.get("ents", [])
    if not ents:
        return
    if any(w.data_ptr() != p[0] for (_, _, w, _), p in zip(ents, cache["ptrs"])):     # a parameter moved: rebuild
        cache["stamp"] = -1
        return repack_h16_all()
    st = _stream()
    for wp, ns, ks, ts, op, m in cache["calls"]:
        call("dig3d_h16_pack_t", wp, ns, ks, ts, op, m, st)
    gen = _PACK_GENERATION[0]
    for ent, tr, w, buf in ents:
        ent[1][tr] = ((gen, w._version, w.data_ptr(), tuple(w.shape)), buf)


def linear_h16(x, weight, bias=None, transposed=False, want_act=False, residual=None, act_only=False):
    """y = x W^T + b (transposed=False) or y = x W (transposed=True: the input-gradient GEMM) on the two-tile wgmma
    engine, 3xFP16 operands (fp32-level accuracy, |x| < 8190); want_act: also return swish(y).
    residual [rows, nout]: added in the epilogue to the last output (swish(y) + r with want_act, else y + r);
    act_only (with want_act): the pre-activation is not written and only swish(y) (+ r) is returned."""
    k = x.size(-1)
    nout = weight.size(1) if transposed else weight.size(0)
    rows = x.numel() // k
    packed = _h16_packed(weight, transposed)
    shape = x.shape[:-1] + (nout,)
    y = None if (want_act and act_only) else torch.empty(shape, device=x.device, dtype=F32)
    act_out = torch.empty(shape, device=x.device, dtype=F32) if want_act else None
    if residual is not None and tuple(residual.shape) != tuple(shape):
        raise ValueError(f"linear_h16: residual {tuple(residual.shape)} does not match the output {tuple(shape)}")
    call("dig3d_linear_h16", _p(x, F32, "x", 16), rows, k, nout, _p(packed), _p(bias, F32, "bias"), _p(y, align=16),
         _p(act_out, align=16), _p(residual, F32, "residual", 16), _stream())
    if want_act:
        return act_out if act_only else (y, act_out)
    return y


# ---------------------------------------------------------------------------------------------------------------
# second order (force training, SchNet)
def act_bwd2(x, dy, g, mode):
    out = torch.empty_like(x)
    if x.numel():
        call("dig3d_act_bwd2", _p(x, F32, "x"), _p(dy, F32, "dy"), _p(g, F32, "g"), x.numel(), mode, _p(out), _stream())
    return out


# ------------------------------------------------------------------ forward-mode kernels (force training, autograd_jvp.py)
def geometry_jvp(pos, cvec, g, want_angle=True, want_torsion=False):
    """Tangents of dist [E], angle [T], torsion [T] along the per-atom displacement cvec [N, 3]."""
    dev = pos.device
    d_dot = torch.zeros(g.n_edges, device=dev, dtype=F32)
    a_dot = torch.zeros(g.n_triplets, device=dev, dtype=F32) if want_angle else None
    t_dot = torch.zeros(g.n_triplets, device=dev, dtype=F32) if want_torsion else None
    if g.n_edges:
        call("dig3d_geometry_jvp", _p(pos, F32, "pos"), _p(cvec, F32, "cvec"), _p(g.src), _p(g.dst), _p(g.row_ptr),
             _p(g.trip_ptr), _p(g.dist), g.n_edges, _p(d_dot), _p(a_dot), _p(t_dot), _stream())
    return d_dot, a_dot, t_dot


def edge_basis_tangent(dist, dist_dot, cutoff, envelope_exponent, freq, basis_id, envelope_on_bessel, nr, n_bessel,
                       want_rbf0=True, want_bess=True):
    e = dist.numel()
    r_dot = torch.zeros(e, nr, device=dist.device, dtype=F32) if want_rbf0 else None
    b_dot = torch.zeros(e, n_bessel, device=dist.device, dtype=F32) if want_bess else None
    if e:
        call("dig3d_edge_basis_tangent", _p(dist, F32, "dist"), _p(dist_dot, F32, "dist_dot"), e, float(cutoff),
             int(envelope_exponent), _p(freq.detach(), F32, "freq") if freq is not None else None, int(basis_id),
             int(bool(envelope_on_bessel)), _p(r_dot), _p(b_dot), _stream())
    return r_dot, b_dot


def rbf_freq_grad_tangent(dist, dist_dot, cutoff, envelope_exponent, freq, g_dot):
    dfreq = torch.zeros_like(freq, dtype=F32)
    if dist.numel():
        call("dig3d_rbf_freq_grad_tangent", _p(dist, F32, "dist"), _p(dist_dot, F32, "dist_dot"), dist.numel(),
             float(cutoff), int(envelope_exponent), _p(freq.detach(), F32, "freq"), freq.numel(),
             _p(g_dot, F32, "g_dot"), _p(dfreq), _stream())
    return dfreq


def triplet_basis_tangent(bess, bess_dot, angle, angle_dot, torsion, torsion_dot, idx_kj, basis_id, ns, nr, want_tbf):
    t = angle.numel()
    dev = angle.device
    s_dot = torch.zeros(t, ns * nr, dtype=F32, device=dev)
    t_dot = torch.zeros(t, ns * ns * nr, dtype=F32, device=dev) if want_tbf else None
    if t:
        call("dig3d_triplet_basis_tangent", _p(bess, F32), _p(bess_dot, F32), _p(angle, F32), _p(angle_dot, F32),
             _p(torsion, F32) if want_tbf else None, _p(torsion_dot, F32) if want_tbf else None,
             _p(idx_kj, torch.int32), t, int(basis_id), _p(s_dot), _p(t_dot), _stream())
    return s_dot, t_dot


def edge_dist_bwd2(pos, g, ddist, g_dpos):
    """-> (d_ddist [E], d_pos [N,3]) of edge_dist_bwd given g_dpos = d(loss)/d(dpos)."""
    d_ddist = torch.zeros(g.n_edges, device=pos.device, dtype=F32)
    d_pos = torch.zeros_like(pos)
    if g.n_edges:
        call("dig3d_edge_dist_bwd2", _p(pos, F32, "pos"), _p(g.src), _p(g.dst), _p(g.dist), _p(ddist, F32, "ddist"),
             _p(g_dpos, F32, "g_dpos"), g.n_edges, _p(d_ddist), _p(d_pos), _stream())
    return d_ddist, d_pos


def schnet_edge_features_bwd2(dist, offset, coeff, cutoff, dgauss, dcut, g):
    """-> (d_dgauss [E,G], d_dcut [E], d_dist [E]) of schnet_edge_features_bwd given g = d(loss)/d(ddist)."""
    e, ng = dist.numel(), offset.numel()
    d_dg = torch.empty(e, ng, device=dist.device, dtype=F32)
    d_dc = torch.empty(e, device=dist.device, dtype=F32)
    d_d = torch.empty(e, device=dist.device, dtype=F32)
    if e:
        call("dig3d_schnet_edge_features_bwd2", _p(dist, F32, "dist"), e, _p(offset, F32), ng, float(coeff), float(cutoff),
             _p(dgauss, F32), _p(dcut, F32), _p(g, F32, "g"), _p(d_dg), _p(d_dc), _p(d_d), _stream())
    return d_dg, d_dc, d_d


# ---------------------------------------------------------------------------------------------------------------
# ProNet
def pronet_edge_features(g, pos_ca, pos_n, pos_c, level, cutoff, num_pos_emb, want_angles=False):
    """-> (feature0 [E,24], feature1 [E,12|36], pos_emb [E,P], dist [E], angles [E,5] | None); level 0 = aminoacid,
    1 = backbone / allatom."""
    e = g.n_edges
    dev = pos_ca.device
    n_ang = 1 if level == 0 else 3
    f0 = torch.empty(e, 24, device=dev, dtype=F32)
    f1 = torch.empty(e, 12 * n_ang, device=dev, dtype=F32)
    pe = torch.empty(e, num_pos_emb, device=dev, dtype=F32)
    dist = torch.empty(e, device=dev, dtype=F32)
    ang = torch.empty(e, 5, device=dev, dtype=F32) if want_angles else None
    if e:
        call("dig3d_pronet_edge_features", _p(pos_ca, F32, "coords_ca"), _p(pos_n, F32, "coords_n"),
             _p(pos_c, F32, "coords_c"), _p(g.src), _p(g.dst), e, g.n_nodes, int(level), float(cutoff), int(num_pos_emb),
             _p(dist), _p(f0), _p(f1), _p(pe), _p(ang), _stream())
    return f0, f1, pe, dist, ang


def linear_set_config(cfg):
    """Tile configuration of the 128 -> 128 training linear (0 / 1 / 2, see include/dig3d.h); experiments only."""
    call("dig3d_linear_set_config", int(cfg))


# ----------------------------------------------------------------------------- G-SphereNet generation (csrc/gsphere.cu)
I64 = torch.int64
F64 = torch.float64


def gsphere_edge_flags(g):
    """int32 [E]: 1 for the edges listed in cat(idx_ji, idx_kj) (G-SphereNet spherenet.py:170); needs g.idx_kj64."""
    e, t = g.n_edges, g.n_triplets
    flag = torch.zeros(max(e, 1), dtype=torch.int32, device=g.dist.device)[:e]
    if e:
        call("dig3d_gsphere_edge_flags", _p(g.trip_ptr, torch.int32, "trip_ptr"),
             _p(g.idx_kj64, I64, "idx_kj") if t else None, e, t, _p(flag), _stream())
    return flag


def gsphere_keep_rows(x, flag=None, ptr=None, fallback=None, fallback_idx=None):
    """In place: rows r of x [R, W] with flag[r] != 0 (or a non-empty CSR segment ptr[r]..ptr[r+1]) keep their value
    (as fallback + (x - fallback)), the others become fallback[fallback_idx[r] or r] or 0.  Returns x."""
    rows = x.size(0)
    width = x.numel() // max(rows, 1)
    if rows and width:
        call("dig3d_gsphere_keep_rows", _p(flag, torch.int32, "flag"), _p(ptr, torch.int32, "ptr"), _p(x, F32, "x"),
             _p(fallback, F32, "fallback"), _p(fallback_idx, I64, "fallback_idx"), rows, width, _stream())
    return x


def gsphere_attention(q, kv, n_keys, n_heads, k_off, v_off, d_k=32):
    """Multi-head attention pooling with one query per molecule over that molecule's n_keys consecutive key rows; heads
    of d_k channels (d_k = 32: dig3d_gsphere_attention, any other width: dig3d_gsphere_attention_dk)."""
    w = d_k * n_heads
    out = torch.empty(q.size(0), w, dtype=F32, device=q.device)
    if q.size(1) != w:
        raise ValueError(f"gsphere_attention: query width {q.size(1)} != {d_k} * {n_heads} heads")
    if kv.size(0) != q.size(0) * n_keys:
        raise ValueError("gsphere_attention: key rows != queries * n_keys")
    if q.size(0):
        args = (_p(q, F32, "q"), _p(kv, F32, "kv"), kv.size(1), int(k_off), int(v_off), q.size(0), int(n_keys),
                int(n_heads))
        if d_k == 32:
            call("dig3d_gsphere_attention", *args, _p(out), _stream())
        else:
            call("dig3d_gsphere_attention_dk", *args, int(d_k), _p(out), _stream())
    return out


def gsphere_tanh(x):
    y = torch.empty_like(x)
    if x.numel():
        call("dig3d_gsphere_tanh", _p(x, F32, "x"), x.numel(), _p(y), _stream())
    return y


def gsphere_flow_reverse(st, rescale, latent):
    """latent [G, D] in place through the ST_Net_Exp layers, last first; st [G, L, 2D], rescale [L]."""
    rows, dim = latent.shape
    n_layers = rescale.numel()
    if tuple(st.shape) != (rows, n_layers, 2 * dim):
        raise ValueError(f"gsphere_flow_reverse: st {tuple(st.shape)} vs latent {tuple(latent.shape)}")
    if rows:
        call("dig3d_gsphere_flow_reverse", _p(st, F32, "st"), _p(rescale, F32, "rescale"), rows, dim, n_layers,
             _p(latent, F32, "latent"), _stream())
    return latent


def gsphere_focus_select(logit, z, n_mols, n_atoms, focus_th, emit):
    """-> (score [G, n], can_focus [G, n] (first `continuing` rows valid), cont_src [G], emit_src [G], counts [2])."""
    dev = logit.device
    score = torch.empty(n_mols, n_atoms, dtype=F32, device=dev)
    can = torch.empty(n_mols, n_atoms, dtype=F32, device=dev)
    idx = torch.empty(2 * n_mols + 2, dtype=torch.int32, device=dev)
    cont_src, emit_src, counts = idx[:n_mols], idx[n_mols:2 * n_mols], idx[2 * n_mols:]
    call("dig3d_gsphere_focus_select", _p(logit, F32, "logit"), _p(z, I64, "z"), n_mols, n_atoms, z.size(1),
         float(focus_th), int(bool(emit)), _p(score), _p(can), _p(cont_src), _p(emit_src), _p(counts), _stream())
    return score, can, cont_src, emit_src, counts


def gsphere_compact(src, n_atoms, ld_out, z, pos, focus):
    """Rows src of the molecule state (z [G, ld], pos [G, ld, 3], focus [G, ld]) into new [R, ld_out] buffers."""
    rows, dev = src.numel(), z.device
    z2 = torch.empty(rows, ld_out, dtype=I64, device=dev)
    pos2 = torch.empty(rows, ld_out, 3, dtype=F32, device=dev)
    f2 = torch.empty(rows, ld_out, dtype=I64, device=dev)
    if rows:
        call("dig3d_gsphere_compact", _p(src, torch.int32, "src"), rows, n_atoms, z.size(1), ld_out, _p(z, I64, "z"),
             _p(pos, F32, "pos"), _p(focus, I64, "focus"), _p(z2), _p(pos2), _p(f2), _stream())
    return z2, pos2, f2


def gsphere_neighbors(pos, n_atoms, focus_id, want_c2):
    g = focus_id.numel()
    c = torch.empty(2, g, dtype=I64, device=pos.device)
    if g:
        call("dig3d_gsphere_neighbors", _p(pos, F32, "pos"), pos.size(1), g, n_atoms, _p(focus_id, I64, "focus_id"),
             _p(c[0]), _p(c[1]) if want_c2 else None, _stream())
    return c[0], (c[1] if want_c2 else None)


def gsphere_place(n_atoms, focus_id, c1, c2, dist, angle, torsion, type_id, z, pos, focus):
    g = focus_id.numel()
    if g:
        call("dig3d_gsphere_place", g, n_atoms, z.size(1), _p(focus_id, I64, "focus_id"), _p(c1, I64, "c1"),
             _p(c2, I64, "c2"), _p(dist, F32, "dist"), _p(angle, F32, "angle"), _p(torsion, F32, "torsion"),
             _p(type_id, I64, "type_id"), _p(z, I64, "z"), _p(pos, F32, "pos"), _p(focus, I64, "focus"), _stream())


def gsphere_gather_local(feat, n_mols, n_atoms, ids):
    """cat_j feat[g * n_atoms + ids[j][g]] -> [G, len(ids) * W]."""
    width = feat.size(1)
    out = torch.empty(n_mols, len(ids) * width, dtype=F32, device=feat.device)
    idp = [_p(t, I64, "ids") for t in ids] + [None] * (3 - len(ids))
    if n_mols:
        call("dig3d_gsphere_gather_local", _p(feat, F32, "feat"), n_mols, n_atoms, width, *idp, len(ids), _p(out),
             _stream())
    return out


def gsphere_type_scale(latent, emb, feat, n_mols, n_atoms):
    """(type [G] = argmax latent, feat [G*n, W] * emb[type] per molecule)."""
    width = feat.size(1)
    type_id = torch.empty(n_mols, dtype=I64, device=feat.device)
    out = torch.empty_like(feat)
    if n_mols:
        call("dig3d_gsphere_type_scale", _p(latent, F32, "latent"), latent.size(1), _p(emb, F32, "emb"),
             _p(feat, F32, "feat"), n_mols, n_atoms, width, _p(type_id), _p(out), _stream())
    return type_id, out


# ---- G-SphereNet training (csrc/gsphere_train.cu) ------------------------------------------------------------------
def _att_check(q, qgraph, graph_ptr, k, v, n_heads, d_k):
    w = d_k * n_heads
    if q.dim() != 2 or q.size(1) != w or k.shape != v.shape or k.dim() != 2 or k.size(1) != w:
        raise ValueError(f"gsphere attention: q {tuple(q.shape)}, k {tuple(k.shape)}, v {tuple(v.shape)} for "
                         f"{n_heads} heads of {d_k}")
    if qgraph.shape != (q.size(0),):
        raise ValueError("gsphere attention: one graph id per query expected")
    if graph_ptr.dim() != 1 or graph_ptr.numel() < 1:
        raise ValueError("gsphere attention: graph_ptr must be [n_graphs + 1]")


def gsphere_att_fwd(q, qgraph, graph_ptr, k, v, n_heads, d_k=32):
    """Attention pooling of query j over the rows graph_ptr[qgraph[j]] .. graph_ptr[qgraph[j] + 1] of k / v (att.py:18-35
    with at most one query per graph) -> (out [Q, d_k n_heads], stat [Q, n_heads, 2] = (max, denominator)).  d_k = 32
    runs dig3d_gsphere_att_fwd, any other head width dig3d_gsphere_att_fwd_dk."""
    _att_check(q, qgraph, graph_ptr, k, v, n_heads, d_k)
    n_q = q.size(0)
    out = torch.empty(n_q, d_k * n_heads, dtype=F32, device=q.device)
    stat = torch.empty(n_q, n_heads, 2, dtype=F32, device=q.device)
    if n_q:
        args = (_p(q, F32, "q"), _p(qgraph, I64, "qgraph"), _p(graph_ptr, torch.int32, "graph_ptr"), _p(k, F32, "k"),
                _p(v, F32, "v"), n_q, n_heads)
        if d_k == 32:
            call("dig3d_gsphere_att_fwd", *args, _p(out), _p(stat), _stream())
        else:
            call("dig3d_gsphere_att_fwd_dk", *args, int(d_k), _p(out), _p(stat), _stream())
    return out, stat


def gsphere_att_bwd(dout, q, qgraph, graph_ptr, k, v, stat, n_heads, d_k=32):
    """(dq, dk, dv) of gsphere_att_fwd; key rows of graphs without a query get 0."""
    _att_check(q, qgraph, graph_ptr, k, v, n_heads, d_k)
    dq = torch.empty_like(q)
    dkv = torch.zeros((2,) + tuple(k.shape), dtype=F32, device=k.device)      # one fill
    if q.size(0):
        args = (_p(dout, F32, "dout"), _p(q, F32, "q"), _p(qgraph, I64, "qgraph"),
                _p(graph_ptr, torch.int32, "graph_ptr"), _p(k, F32, "k"), _p(v, F32, "v"), _p(stat, F32, "stat"),
                q.size(0), n_heads)
        if d_k == 32:
            call("dig3d_gsphere_att_bwd", *args, _p(dq), _p(dkv[0]), _p(dkv[1]), _stream())
        else:
            call("dig3d_gsphere_att_bwd_dk", *args, int(d_k), _p(dq), _p(dkv[0]), _p(dkv[1]), _stream())
    return dq, dkv[0], dkv[1]


def _flow_check(st, rescale, x):
    if x.dim() != 2 or x.dtype not in (F32, F64):
        raise ValueError(f"gsphere flow: x must be a float32 or float64 [rows, dim] tensor, got {x.dtype} "
                         f"{tuple(x.shape)}")
    rows, dim = x.shape
    if tuple(st.shape) != (rescale.numel(), rows, 2 * dim):
        raise ValueError(f"gsphere flow: st {tuple(st.shape)} vs {rescale.numel()} layers and x {tuple(x.shape)}")
    return rows, dim, rescale.numel(), int(x.dtype == F64)


def gsphere_flow_fwd(st, rescale, x):
    """flow_forward (net_utils.py:83-93): st [L, rows, 2D] of the L layers, rescale [L], x [rows, D] (float32 or float64)
    -> (latent [rows, D] in x's dtype, log_jac [rows, D] float32)."""
    rows, dim, n_layers, f64 = _flow_check(st, rescale, x)
    out = torch.empty_like(x)
    log_jac = torch.empty(rows, dim, dtype=F32, device=x.device)
    if rows:
        call("dig3d_gsphere_flow_fwd", _p(st, F32, "st"), _p(rescale, F32, "rescale"), _p(x, x.dtype, "x"), f64, rows,
             dim, n_layers, _p(out), _p(log_jac), _stream())
    return out, log_jac


def gsphere_flow_bwd(st, rescale, x, dlatent, dlog_jac):
    """(dst [L, rows, 2D], drescale [L]) of gsphere_flow_fwd."""
    rows, dim, n_layers, f64 = _flow_check(st, rescale, x)
    dst = torch.empty_like(st)
    drescale = torch.empty(n_layers, dtype=F32, device=st.device)
    part = torch.empty(max(n_layers * rows * dim, 1), dtype=F32, device=st.device)
    call("dig3d_gsphere_flow_bwd", _p(st, F32, "st"), _p(rescale, F32, "rescale"), _p(x, x.dtype, "x"), f64,
         _p(dlatent, x.dtype, "dlatent"), _p(dlog_jac, F32, "dlog_jac"), rows, dim, n_layers, _p(dst), _p(part),
         _p(drescale), _stream())
    return dst, drescale


def gsphere_sigmoid(x):
    y = torch.empty_like(x)
    if x.numel():
        call("dig3d_gsphere_sigmoid", _p(x, F32, "x"), x.numel(), _p(y), _stream())
    return y


GSPHERE_TANH, GSPHERE_SIGMOID = 0, 1


def gsphere_unary_bwd(y, dy, mode):
    """dx from the forward output y: dy (1 - y^2) for GSPHERE_TANH, dy y (1 - y) for GSPHERE_SIGMOID."""
    if y.shape != dy.shape:
        raise ValueError(f"gsphere_unary_bwd: shapes differ {tuple(y.shape)} vs {tuple(dy.shape)}")
    dx = torch.empty_like(y)
    if y.numel():
        call("dig3d_gsphere_unary_bwd", _p(y, F32, "y"), _p(dy, F32, "dy"), y.numel(), mode, _p(dx), _stream())
    return dx


def gsphere_keep_rows_bwd(dy, flag=None, ptr=None, want_dx=True, want_dfb=True):
    """(dx, dfb) of gsphere_keep_rows with a row-aligned fallback: kept rows pass dy to x, the others to the fallback."""
    rows = dy.size(0)
    width = dy.numel() // max(rows, 1)
    dx = torch.empty_like(dy) if want_dx else None
    dfb = torch.empty_like(dy) if want_dfb else None
    if rows and width:
        call("dig3d_gsphere_keep_rows_bwd", _p(flag, torch.int32, "flag"), _p(ptr, torch.int32, "ptr"),
             _p(dy, F32, "dy"), rows, width, _p(dx), _p(dfb), _stream())
    return dx, dfb


# ---- bond-length MMD (csrc/mmd.cu) -------------------------------------------------------------------------------------
_MMD_CTAS_PER_SM = 4          # the pair kernel's occupancy (256 threads, 62 registers): one wave of persistent CTAs


def mmd_terms(source, target, kernel_mul=2.0, kernel_num=5, fix_sigma=None):
    """(bandwidth, XX, YY, XY) of compute_mmd (eval_bond_mmd_utils.py:44-97) as a 4-element fp64 tensor on the device.

    source / target: 1-D float32 or float64 tensors, concatenated and cast to fp64 here (the reference's torch.cat
    promotes a float32 + float64 pair the same way; two float32 inputs are computed in fp64 too).  CPU tensors are copied
    to the current CUDA device.  fix_sigma: None or 0 selects the data bandwidth.  One launch sequence on the current
    stream, no host synchronisation."""
    for name, t in (("source", source), ("target", target)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"mmd_terms: {name} must be a torch.Tensor, got {type(t)}")
        if t.dim() != 1 or t.dtype not in (torch.float32, torch.float64):
            raise TypeError(f"mmd_terms: {name} must be a 1-D float32 / float64 tensor, got {t.dtype} {tuple(t.shape)}")
    if not torch.cuda.is_available():
        raise RuntimeError("mmd_terms needs a CUDA device (sm_90a); there is no CPU fallback")
    devs = {t.device for t in (source, target) if t.is_cuda}
    if len(devs) > 1:
        raise ValueError(f"mmd_terms: source and target are on different devices {sorted(map(str, devs))}")
    dev = devs.pop() if devs else torch.device("cuda", torch.cuda.current_device())
    kernel_num = int(kernel_num)
    with torch.cuda.device(dev):
        v = torch.cat([source.to(dev, F64), target.to(dev, F64)]).contiguous()
        ctas = _MMD_CTAS_PER_SM * torch.cuda.get_device_properties(dev).multi_processor_count
        ws = torch.empty(3 * ctas, dtype=F64, device=dev)
        out = torch.empty(4, dtype=F64, device=dev)
        call("dig3d_mmd_terms", _p(v, F64, "v", align=8), source.numel(), target.numel(), float(kernel_mul), kernel_num,
             float(fix_sigma) if fix_sigma else 0.0, _p(ws), ws.numel(), _p(out), _stream())
    return out


# ---- xyz2mol (csrc/xyz2mol.cu) -----------------------------------------------------------------------------------------
XYZ2MOL_MAX_ATOMS = 64        # AC rows are uint64 masks in csrc/xyz2mol.cuh


def xyz2mol(z, pos):
    """Bond-order matrices and validity flags of G molecules with n atoms each (xyz2mol with use_graph=True, reference
    eval_validity_utils.py:382-405), on the device.

    z: [G, n] tensor of an integer dtype (atomic numbers; any value is accepted, elements outside H, C, N, O, F bond to
    nothing and make a molecule invalid, as in the reference).  pos: [G, n, 3] float32 / float64 tensor, converted to
    fp64 exactly.  CPU tensors are copied to the current CUDA device.  1 <= n <= 64 (ValueError otherwise).
    Returns (bo [G, n, n] int8, valid [G] int8) on the device: one launch on the current stream, no host
    synchronisation.  valid is 1 / 0; -1 marks an internal capacity overflow of the matching (see xyz2mol.cuh)."""
    for name, t in (("z", z), ("pos", pos)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"xyz2mol: {name} must be a torch.Tensor, got {type(t)}")
    if z.dtype.is_floating_point or z.dtype.is_complex or z.dtype == torch.bool:
        raise TypeError(f"xyz2mol: z must have an integer dtype, got {z.dtype}")
    if pos.dtype not in (torch.float32, torch.float64):
        raise TypeError(f"xyz2mol: pos must be float32 / float64, got {pos.dtype}")
    if z.dim() != 2 or pos.dim() != 3 or pos.size(2) != 3 or tuple(pos.shape[:2]) != tuple(z.shape):
        raise ValueError(f"xyz2mol: expected z [G, n] and pos [G, n, 3], got {tuple(z.shape)} and {tuple(pos.shape)}")
    g, n = z.shape
    if not 1 <= n <= XYZ2MOL_MAX_ATOMS:
        raise ValueError(f"xyz2mol: molecules need 1 to {XYZ2MOL_MAX_ATOMS} atoms, got {n}")
    if not torch.cuda.is_available():
        raise RuntimeError("xyz2mol needs a CUDA device (sm_90a); there is no CPU fallback")
    devs = {t.device for t in (z, pos) if t.is_cuda}
    if len(devs) > 1:
        raise ValueError(f"xyz2mol: z and pos are on different devices {sorted(map(str, devs))}")
    dev = devs.pop() if devs else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        zd = z.to(dev, I64).contiguous()
        pd = pos.to(dev, F64).contiguous()
        bo = torch.empty((g, n, n), dtype=torch.int8, device=dev)
        valid = torch.empty(g, dtype=torch.int8, device=dev)
        call("dig3d_xyz2mol", _p(zd, I64, "z", align=8), _p(pd, F64, "pos", align=8), g, n, _p(bo), _p(valid),
             _stream())
    return bo, valid


# ---- G-SphereNet trajectories (csrc/gen_traj.cu) -----------------------------------------------------------------------
GEN_TRAJ_MAX_ATOMS = 32       # one warp per molecule, one lane per atom
GEN_TRAJ_FIELDS = ("atom_type", "position", "batch", "cannot_focus", "focus", "c1_focus", "c2_c1_focus",
                   "new_atom_type", "new_dist", "new_angle", "new_torsion")


def gen_traj_ptr(n_atoms):
    """[6, M + 1] int64 exclusive prefix sums of dig3d_gen_traj (atoms, n^2, rows, steps, angles, torsions) for the
    atom counts n_atoms [M] (host int64 tensor)."""
    n = n_atoms.to(I64)
    counts = torch.stack([n, n * n, n * (n - 1) // 2, n - 1, (n - 2).clamp_min(0), (n - 3).clamp_min(0)])
    ptr = torch.zeros((6, n.numel() + 1), dtype=I64)
    torch.cumsum(counts, dim=1, out=ptr[:, 1:])
    return ptr


def gen_traj(atom_type, pos, con, n_atoms, device=None):
    """Every field of QM93DGEN.get (reference ggraph3D_dataset.py:192-302) for M molecules, on the device.

    atom_type [N] integer, pos [N, 3] float32 and con [sum n^2] integer (each molecule's n x n bond matrix, row-major,
    back to back) are the molecules concatenated; n_atoms [M] their atom counts, 2 <= n <= 32 (ValueError otherwise).
    Positions must be finite.  Host tensors are copied to `device` (default: the current CUDA device).
    Returns (out, ptr, status): out maps each name of GEN_TRAJ_FIELDS to one device tensor holding all molecules' rows
    (get()'s dtypes; c1_focus [., 2], c2_c1_focus [., 3], the others 1-D); ptr = gen_traj_ptr(n_atoms) on the host, whose
    rows 2..5 index the row / step / angle / torsion fields; status [M] int32 on the device (1: the molecule's spanning
    tree has no edge, all its atoms coincide).  One launch on the current stream, no host synchronisation."""
    for name, t in (("atom_type", atom_type), ("pos", pos), ("con", con), ("n_atoms", n_atoms)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"gen_traj: {name} must be a torch.Tensor, got {type(t)}")
    for name, t in (("atom_type", atom_type), ("con", con), ("n_atoms", n_atoms)):
        if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
            raise TypeError(f"gen_traj: {name} must have an integer dtype, got {t.dtype}")
    if pos.dtype != torch.float32:
        raise TypeError(f"gen_traj: pos must be float32, got {pos.dtype}")
    n_cpu = n_atoms.detach().to("cpu", I64).reshape(-1)
    if n_cpu.numel() and (int(n_cpu.min()) < 2 or int(n_cpu.max()) > GEN_TRAJ_MAX_ATOMS):
        raise ValueError(f"gen_traj: molecules need 2 to {GEN_TRAJ_MAX_ATOMS} atoms, got "
                         f"{int(n_cpu.min())} .. {int(n_cpu.max())}")
    ptr = gen_traj_ptr(n_cpu)
    tot = ptr[:, -1].tolist()
    if (atom_type.dim() != 1 or atom_type.numel() != tot[0] or tuple(pos.shape) != (tot[0], 3)
            or con.dim() != 1 or con.numel() != tot[1]):
        raise ValueError(f"gen_traj: expected atom_type [{tot[0]}], pos [{tot[0]}, 3] and con [{tot[1]}], got "
                         f"{tuple(atom_type.shape)}, {tuple(pos.shape)} and {tuple(con.shape)}")
    if not bool(torch.isfinite(pos).all()):
        raise ValueError("gen_traj: positions must be finite")
    if not torch.cuda.is_available():
        raise RuntimeError("gen_traj needs a CUDA device (sm_90a); there is no CPU fallback")
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    rows, steps, angles, torsions = tot[2:]
    with torch.cuda.device(dev):
        z = atom_type.to(dev, I64).contiguous()
        p = pos.to(dev).contiguous()
        c = con.to(dev, I64).contiguous()
        ptr_d = ptr.to(dev)
        # at least one element each, so that no pointer is NULL when a field is empty (e.g. only 2-atom molecules)
        e = lambda r, *w, dtype=I64: torch.empty((max(r, 1),) + w, dtype=dtype, device=dev)[:r]
        out = dict(atom_type=e(rows), position=e(rows, 3, dtype=torch.float32), batch=e(rows),
                   cannot_focus=e(rows, dtype=torch.float32), focus=e(steps), c1_focus=e(angles, 2),
                   c2_c1_focus=e(torsions, 3), new_atom_type=e(steps), new_dist=e(steps, dtype=F64),
                   new_angle=e(angles, dtype=F64), new_torsion=e(torsions, dtype=F64))
        status = e(n_cpu.numel(), dtype=torch.int32)
        call("dig3d_gen_traj", _p(z, I64, "atom_type", align=8), _p(p, torch.float32, "pos"), _p(c, I64, "con", align=8),
             _p(ptr_d), n_cpu.numel(), *(_p(out[k]) for k in ("atom_type", "position", "batch", "cannot_focus", "focus",
                                                               "c1_focus", "c2_c1_focus", "new_atom_type", "new_dist",
                                                               "new_angle", "new_torsion")),
             _p(status), _stream())
    return out, ptr, status
