"""Shared test utilities (test infrastructure; may import oracle/)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")

from oracle.gen_golden import CASES  # noqa: E402  (case table only; no reference import)
from oracle.weights import formula_state_dict  # noqa: E402


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def case_inputs(name, device="cpu"):
    g = load_golden(name)
    z = torch.from_numpy(g["z"]).to(device)
    pos = torch.from_numpy(g["pos"]).to(device)
    batch = torch.from_numpy(g["batch"]).to(device)
    return g, z, pos, batch


def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def sphere_forward_op_by_op(model, data):
    """SphereNet / DimeNet++ 3xFP16 inference issued op by op through the tensor wrappers, with separate launches: init_e
    alone, then part A, the triplet gather and part B of every block, then update_v (the 3xFP16 engine, or the exact-fp32
    FFMA engine for shapes it does not support) and the readout.  The planned model forward (init_e fused with part A of
    block 0, part B fused with the next block's part A) must equal it bit for bit."""
    from dig_b200 import ops
    m = model
    z, pos = data.z, data.pos
    g = ops.build_graph(pos, data.batch, m.cutoff, num_graphs=getattr(data, "num_graphs", None), z=z,
                        z_rows=m.init_e.emb.num_embeddings)
    ops.triplet_geometry(g, pos, use_torsion=m._torsion, want_idx=False)
    ns, nr, L, H = m.num_spherical, m.num_radial, m.num_layers, m.hidden_channels
    rbf0, bess = ops.edge_basis(g.dist, m.cutoff, m.envelope_exponent, m.emb.dist_emb.freq, m._basis_id,
                                envelope_on_bessel=not m._torsion, num_radial=nr, n_bessel=ns * nr)
    proj = [ops.triplet_basis_project(g, bess, m._basis_id, *m._projection_rows(first, min(4, L - first)))
            for first in range(0, L, 4)]
    v_in_all = torch.zeros(L + 1, g.n_nodes, H, dtype=torch.float32, device=pos.device)
    v_all = torch.empty(L + 1, g.n_nodes, m.out_channels, dtype=torch.float32, device=pos.device)
    cache = {}                  # owns the packed weights: kept until the kernels below have run
    tables = ops.init_e_tables(m.init_e, cache) if os.environ.get("DIG3D_INIT_TABLES", "1") != "0" else None
    packed = ops.tc_pack_matrix(m.init_e.lin.weight, cache, "init_e.lin", kind="h16")
    e1, _ = ops.sphere_init_e_h16(z, g, rbf0, ops.pack_init_e(m.init_e), packed, H, v_in=v_in_all[0], tables=tables)
    for l in range(L):
        sbf_p, t_p = proj[l // 4]
        w = ops.tc_pack_update_e(m.update_es[l], m._torsion, cache, kind="h16")
        e1, _, _, _ = ops.sphere_update_e_h16(e1, g, rbf0, sbf_p, t_p, 8 * (l % 4), w, H, m.int_emb_size,
                                              v_in=v_in_all[l + 1])
    holders = [m.init_v] + list(m.update_vs)
    if ops.update_v_h16_supported(m.init_v, m.out_channels):
        ops.sphere_update_v_h16(v_in_all, holders, m.out_channels, v_all, cache)
    else:
        ops.sphere_update_v_batched(v_in_all, holders, m.out_channels, v_all)
    u = ops.graph_readout(v_all, g.graph_ptr, g.n_graphs, g.n_nodes)
    torch.cuda.synchronize()
    return u


def comenet_forward_op_by_op(model, data, record=None):
    """ComENet 3xFP16 inference issued op by op through the tensor wrappers: every hidden x hidden linear as
    `ops.linear_h16` (swish and residuals fused as in the planned forward), the EdgeGraphConv aggregations as
    `ops.comenet_filter_sum`.  The planned model forward must equal it bit for bit.  `record` (a dict): filled with the
    graph, the features and every intermediate, keyed "emb", "<block>.x1", "<block>.filt<c>", "<block>.agg<c>",
    "<block>.root<c>", "<block>.conv<c>", "<block>.h<c>", "<block>.t", "<block>.cat", "<block>.lins<l>", "<block>.norm",
    "<block>.shift", "<block>.std", "<block>.final", "head<l>", "out", "energy"."""
    from dig_b200 import ops
    rec = record if record is not None else {}
    m = model
    z, pos = data.z.long(), data.pos
    g = ops.build_graph(pos, data.batch, m.cutoff, num_graphs=getattr(data, "num_graphs", None), want_edge_index=False,
                        z=z, z_rows=m.emb.emb.num_embeddings)
    f1, f2, _ = ops.comenet_geometry(g, pos, m.cutoff)
    rec.update(graph=g, z=z, f1=f1, f2=f2)
    lin = ops.linear_h16
    x = rec["emb"] = ops.comenet_embed(z, m.emb.emb.weight)                    # swish(emb[z])
    for b, blk in enumerate(m.interaction_blocks):
        x = rec[f"{b}.x1"] = lin(x, blk.lin.weight, blk.lin.bias, want_act=True, act_only=True)
        hs = []
        for c, (conv, lf, l, feat) in enumerate(((blk.conv1, blk.lin_feature1, blk.lin1, f1),
                                                 (blk.conv2, blk.lin_feature2, blk.lin2, f2)), 1):
            filt = rec[f"{b}.filt{c}"] = m._filter_t(lf)
            agg = rec[f"{b}.agg{c}"] = ops.comenet_filter_sum(feat, filt, x, g)
            # GraphConv: lin_rel(agg) + lin_root(x) -- the second GEMM adds the first in its epilogue
            root = rec[f"{b}.root{c}"] = lin(x, conv.lin_root.weight, None)
            h = rec[f"{b}.conv{c}"] = lin(agg, conv.lin_rel.weight, conv.lin_rel.bias, residual=root)
            hs.append(lin(h, l.weight, l.bias, want_act=True, act_only=True))
            rec[f"{b}.h{c}"] = hs[-1]
        wa, wb = m._cat_halves(blk)
        # lin_cat(cat[h1, h2]) + x = h1 Wa^T + b + (h2 Wb^T + x)
        t = rec[f"{b}.t"] = lin(hs[1], wb, None, residual=x)
        h = rec[f"{b}.cat"] = lin(hs[0], wa, blk.lin_cat.bias, residual=t)
        for i, l in enumerate(blk.lins):
            h = rec[f"{b}.lins{i}"] = lin(h, l.weight, l.bias, want_act=True, act_only=True, residual=h)   # swish(l(h)) + h
        h, rec[f"{b}.shift"], rec[f"{b}.std"] = ops.graphnorm(h, g.graph_ptr, blk.norm.weight.detach(),
                                                               blk.norm.bias.detach(), blk.norm.mean_scale.detach(),
                                                               blk.norm.eps)
        rec[f"{b}.norm"] = h
        x = rec[f"{b}.final"] = lin(h, blk.final.weight, blk.final.bias)
    for i, l in enumerate(m.lins):
        x = rec[f"head{i}"] = lin(x, l.weight, l.bias, want_act=True, act_only=True)
    x = rec["out"] = ops.linear(x, m.lin_out.weight.detach(), m.lin_out.bias.detach())
    rec["energy"] = ops.segment_sum(x, g.graph_ptr)
    return rec["energy"]
