"""ctypes binding of libdig3d.so (the C ABI declared in include/dig3d.h).

The library is built in-tree by `__graft_entry__.build()` / `python -m dig_b200.build`.
There is NO fallback: if the shared object is missing or a symbol is absent, importing the
ops raises, and every op raises unless its tensors live on a CUDA device.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdig3d.so")

P = c_void_p


class InitEWeights(Structure):
    _fields_ = [(n, P) for n in ("emb", "w_rbf0", "b_rbf0", "w_lin", "b_lin", "w_rbf1")]


class UpdateEWeights(Structure):
    _fields_ = ([(n, P) for n in ("w_rbf1", "w_rbf2", "w_sbf2", "w_t2", "w_rbf",
                                  "w_kj", "b_kj", "w_ji", "b_ji", "w_down", "w_up")]
                + [("w_res", P * 6), ("b_res", P * 6), ("w_lin", P), ("b_lin", P)])


class SchnetBlockWeights(Structure):
    _fields_ = [(n, P) for n in ("w_lin", "w_mlp0", "b_mlp0", "w_mlp2", "b_mlp2", "w_v1", "b_v1", "w_v2", "b_v2")]


class ComenetBlockWeights(Structure):
    _fields_ = ([(n, P) for n in ("w_lin", "b_lin", "w_f1a", "w_f1b", "w_f2a", "w_f2b", "w_rel1", "b_rel1",
                                  "w_root1", "w_rel2", "b_rel2", "w_root2", "w_lin1", "b_lin1", "w_lin2",
                                  "b_lin2", "w_cat", "b_cat")]
                + [("w_lins", P * 8), ("b_lins", P * 8)]
                + [(n, P) for n in ("norm_w", "norm_b", "norm_ms", "w_final", "b_final")]
                + [("n_lins", c_int32)])


class ComenetHeadWeights(Structure):
    _fields_ = [("w_lins", P * 8), ("b_lins", P * 8), ("w_out", P), ("b_out", P), ("n_lins", c_int32)]


class TcUpdateE(Structure):
    _fields_ = ([(n, P) for n in ("p_ji", "b_ji", "p_kj", "b_kj", "p_down", "p_up")]
                + [("p_res", P * 6), ("b_res", P * 6)]
                + [(n, P) for n in ("p_lin", "b_lin", "w_rbf1", "w_rbf2", "w_rbf", "w_sbf2", "w_t2")])


class UpdateVWeights(Structure):
    _fields_ = [("w_up", P), ("b_up", P), ("w_lins", P * 8), ("b_lins", P * 8), ("w_out", P),
                ("n_lins", c_int32)]


# name -> argtypes (restype is int unless listed in _RESTYPES); mirrors include/dig3d.h
SIGNATURES = {
    "dig3d_last_error": [],
    "dig3d_abi_version": [],
    "dig3d_graph_ptr": [P, c_int64, c_int64, P, P],
    "dig3d_radius_neighbors": [P, P, P, c_int64, c_int64, c_double, c_int32, P, P, P],
    "dig3d_validate_nodes": [P, P, c_int64, c_int64, c_int32, P, P],
    "dig3d_knn2": [P, P, P, c_int64, c_int64, P, P, P],
    "dig3d_triplet_geometry_knn": [P, P, P, P, P, c_int64, P, P, P, P, P, P, P],
    "dig3d_triplet_count_out": [P, P, c_int64, c_int32, P, P, P],
    "dig3d_scan_counts3": [P, P, P, c_int64, P, P, P, P, P],
    "dig3d_edge_fill_out": [P, P, P, P, P, c_int64, c_int32, c_int64, P, P, P, P, P, P, P, P, P, P, P, P],
    "dig3d_edges_to_csr": [P, P, c_int64, c_int64, P, P, P, P, P, P, P, P],
    "dig3d_triplet_geometry": [P, P, P, P, P, c_int64, c_int32, P, P, P, P, P, P, P],
    "dig3d_triplet_geometry_any_degree": [P, P, P, P, P, c_int64, c_int64, c_int32, P, P, P, P, P, P, P, P],
    "dig3d_triplet_geometry_any_degree_arg": [P, P, P, P, P, c_int64, c_int64, P, P, P, P, P, P, P],
    "dig3d_triplet_torsion_bwd_arg": [P, P, P, P, P, P, P, c_int64, P, P],
    "dig3d_triplet_geometry_bwd2": [P, P, P, P, P, P, P, P, P, c_int64, P, P, P, P],
    "dig3d_radius_graph_dense_count": [P, P, P, c_int64, c_int64, c_double, c_int64, P, P, P, P, P],
    "dig3d_radius_graph_dense_fill": [P, P, P, c_int64, c_int64, c_double, c_int64, P, c_int64, P, P, P, P],
    "dig3d_edge_basis": [P, c_int64, c_double, c_int32, P, c_int32, c_int32, P, P, P],
    "dig3d_triplet_basis": [P, P, P, P, c_int64, c_int32, P, P, P],
    "dig3d_triplet_basis_project_lists": [P, P, P, P, P, P, P, P, P, c_int64, c_int64, c_int32, c_int32,
                                    c_int32, P, P, P, P, P, P, P, P],
    "dig3d_segment_sum": [P, P, c_int64, c_int64, P, P],
    "dig3d_sphere_init_e": [P, P, P, P, c_int64, POINTER(InitEWeights), P, P, P],
    "dig3d_sphere_update_e_a": [P, P, c_int64, POINTER(UpdateEWeights), P, P, P],
    "dig3d_sphere_update_e_b": [P, P, P, P, P, P, c_int32, P, P, P, P, c_int64,
                                POINTER(UpdateEWeights), P, P, P],
    "dig3d_sphere_update_v": [P, c_int64, c_int32, POINTER(UpdateVWeights), P, P],
    "dig3d_sphere_update_v_batched": [P, c_int64, c_int32, c_int32, P, P, P],
    "dig3d_graph_readout": [P, P, c_int64, c_int64, c_int32, c_int32, P, P],
    "dig3d_tc_pack": [P, P, P, P, c_int32, P],
    "dig3d_tc_timeouts": [],
    "dig3d_sphere_init_e_tc": [P, P, P, P, c_int64, POINTER(InitEWeights), P, P, P, P],
    "dig3d_sphere_update_e_a_tc": [P, P, c_int64, POINTER(TcUpdateE), P, P, P],
    "dig3d_sphere_triplet_gather": [P, P, P, c_int32, P, P, P, P, c_int64, P, P, P, P],
    "dig3d_sphere_triplet_gather_warp": [P, P, P, c_int32, P, P, P, P, P, c_int64, c_int32, c_int32, P, P, P, P, P,
                                         P, P],
    "dig3d_sphere_update_e_b_tc": [P, P, P, P, P, c_int64, POINTER(TcUpdateE), P, P, P],
    "dig3d_tc_set_fast_swish": [c_int32],
    "dig3d_h16_pack": [P, P, P, P, c_int32, P],
    "dig3d_sphere_init_e_h16": [P, P, P, P, c_int64, POINTER(InitEWeights), P, P, P, P],
    "dig3d_sphere_init_e_h16_tab": [P, P, P, P, c_int64, POINTER(InitEWeights), P, P, P, P, P, P],
    "dig3d_sphere_update_e_a_h16": [P, P, c_int64, POINTER(TcUpdateE), P, P, P],
    "dig3d_sphere_update_e_b_h16": [P, P, P, P, P, c_int64, POINTER(TcUpdateE), P, P, P],
    "dig3d_sphere_update_e_ba_h16": [P, P, P, P, P, c_int64, POINTER(TcUpdateE), POINTER(TcUpdateE), P, P, P, P, P],
    "dig3d_sphere_init_update_e_a_h16": [P, P, P, P, c_int64, POINTER(InitEWeights), P, P, P, POINTER(TcUpdateE), P, P,
                                         P, P, P],
    "dig3d_sphere_update_v_h16_supported": [c_int32, c_int32, c_int32, c_int32],
    "dig3d_sphere_update_v_h16": [P, c_int64, c_int32, c_int32, c_int32, P, P, P, P],
    "dig3d_h16_pack_t": [P, P, P, P, P, c_int32, P],
    "dig3d_linear_h16_supported": [c_int32, c_int32],
    "dig3d_linear_h16": [P, c_int64, c_int32, c_int32, P, P, P, P, P, P],
    "dig3d_h16_overflow": [c_int32],
    "dig3d_h16_timeouts": [],
    "dig3d_h16_trace": [c_int32, P],
    "dig3d_h16_set_fast_swish": [c_int32],
    "dig3d_tc_trace": [c_int32, P],
    "dig3d_schnet_block": [P, c_int64, P, P, P, c_int64, P, c_int32, c_double, c_double, c_int32, c_int32,
                           POINTER(SchnetBlockWeights), P, P, P, P],
    "dig3d_schnet_readout": [P, c_int64, c_int32, P, P, P, P, c_int32, P, P],
    "dig3d_comenet_geometry": [P, P, P, P, P, P, P, c_int64, c_int64, c_double, P, P, P, P, P],
    "dig3d_comenet_features_bwd": [P, P, P, P, P, P, P, P, c_int64, c_int64, c_double, P, P, P, P, P],
    "dig3d_comenet_features_tangent": [P, P, P, P, P, c_int64, c_int64, c_double, P, P, P, P],
    "dig3d_comenet_features_tangent_bwd": [P, P, P, P, P, P, P, P, c_int64, c_int64, c_double, P, P, P, P, P, P],
    "dig3d_comenet_embed": [P, P, c_int64, P, P],
    "dig3d_pbc_edge_vectors": [P, P, P, P, P, c_int64, P, P, P],
    "dig3d_comenet_geometry_edges": [P, P, P, P, P, c_int64, c_int64, c_double, P, P, P, P, P, P],
    "dig3d_comenet_features_bwd_vec": [P, P, P, P, P, P, P, P, c_int64, c_int64, c_double, P, P, P, P, P],
    "dig3d_comenet_features_tangent_vec": [P, P, P, P, P, c_int64, c_int64, c_double, P, P, P, P],
    "dig3d_comenet_features_tangent_bwd_vec": [P, P, P, P, P, P, P, P, c_int64, c_int64, c_double, P, P, P, P, P, P],
    "dig3d_pbc_cell_bwd": [P, P, P, P, c_int64, P, P],
    "dig3d_radius_graph_pbc_count": [P, P, P, c_int64, c_int64, c_double, c_int32, P, P, P, P, P, P, P],
    "dig3d_radius_graph_pbc_fill": [P, P, c_int64, c_int64, c_double, P, P, P, P, c_int64, P, P, P, P],
    "dig3d_comenet_block": [P, P, P, P, P, P, P, c_int64, c_int64, c_int64, POINTER(ComenetBlockWeights),
                            POINTER(ComenetHeadWeights), c_int32, P, P, P, P, P, P, P, P],
    "dig3d_edge_weighted_sum": [P, P, P, P, c_int64, c_int32, P, P],
    "dig3d_comenet_filter_sum": [P, c_int32, P, P, P, P, c_int64, c_int32, P, P],
    "dig3d_linear": [P, c_int64, c_int32, c_int32, P, P, P, P, c_int32, P],
    "dig3d_wgrad": [P, P, c_int64, c_int32, c_int32, P, P, c_int32, P],
    "dig3d_wgrad_tc": [P, P, c_int64, c_int32, c_int32, P, P, c_int32, P],
    "dig3d_wgrad_tc_supported": [c_int64, c_int32, c_int32],
    "dig3d_wgrad_set_mode": [c_int32],
    "dig3d_wgrad_tc_timeouts": [],
    "dig3d_act": [P, c_int64, c_int32, P, P],
    "dig3d_act_bwd": [P, P, c_int64, c_int32, P, P],
    "dig3d_adam_step": [P, P, P, P, c_int64, c_double, c_double, c_double, c_double, c_double, c_int64, P],
    "dig3d_ewise": [P, P, c_int64, c_int32, P, P],
    "dig3d_rowscale": [P, P, c_int64, c_int32, P, P],
    "dig3d_gather_rows": [P, P, c_int32, c_int64, c_int32, P, P],
    "dig3d_scatter_add_rows": [P, P, c_int32, c_int64, c_int32, P, P],
    "dig3d_rbf_freq_grad": [P, c_int64, c_double, c_int32, P, c_int32, P, P, P],
    "dig3d_triplet_basis_project_bwd": [P, P, P, P, P, P, P, P, P, c_int64, c_int64, c_int32, P, P, P, P, P],
    "dig3d_sphere_triplet_gather_bwd": [P, P, P, P, P, P, P, P, c_int64, P, P, P, P, P, P, P, P],
    "dig3d_graphnorm": [P, P, c_int64, c_int32, P, P, P, c_double, P, P, P, P],
    "dig3d_graphnorm_bwd": [P, P, P, c_int64, c_int32, P, P, P, P, P, P, P, P, P],
    "dig3d_graphnorm_tangent": [P, P, P, c_int64, c_int32, P, P, P, P, P, P],
    "dig3d_graphnorm_tangent_bwd": [P, P, P, P, c_int64, c_int32, P, P, P, P, P, P, P, P, P],
    "dig3d_edge_dist_bwd": [P, P, P, P, P, c_int64, P, P],
    "dig3d_triplet_angle_bwd": [P, P, P, P, P, P, c_int64, P, P],
    "dig3d_edge_basis_bwd": [P, c_int64, c_double, c_int32, P, c_int32, c_int32, P, P, P, P],
    "dig3d_triplet_basis_project_bwd_geom": [P, P, P, P, P, P, P, P, P, P, c_int64, c_int64, c_int32, P, P, P, P,
                                             c_double, P, P, P, P],
    "dig3d_triplet_basis_bwd": [P, P, P, P, P, P, P, P, P, P, c_int64, c_int64, c_int32, P, P, c_double, P, P, P, P],
    "dig3d_triplet_torsion_bwd": [P, P, P, P, P, P, c_int64, P, P],
    "dig3d_schnet_edge_features_bwd": [P, c_int64, P, c_int32, c_double, c_double, P, P, P, P],
    "dig3d_rowdot": [P, P, c_int64, c_int32, P, P],
    "dig3d_tc_pack_t": [P, P, P, P, P, c_int32, P],
    "dig3d_linear_tc_supported": [c_int32, c_int32],
    "dig3d_linear_tc": [P, c_int64, c_int32, c_int32, P, P, P, P, P],
    "dig3d_act_bwd2": [P, P, P, c_int64, c_int32, P, P],
    "dig3d_geometry_jvp": [P, P, P, P, P, P, P, c_int64, P, P, P, P],
    "dig3d_edge_basis_tangent": [P, P, c_int64, c_double, c_int32, P, c_int32, c_int32, P, P, P],
    "dig3d_rbf_freq_grad_tangent": [P, P, c_int64, c_double, c_int32, P, c_int32, P, P, P],
    "dig3d_edge_basis_tangent_bwd": [P, P, c_int64, c_double, c_int32, P, c_int32, c_int32, P, P, P, P, P],
    "dig3d_triplet_basis_tangent_bwd": [P, P, P, P, P, P, P, P, P, P, P, P, P, P, c_int64, c_int64, c_int32, P, P,
                                        c_double, P, P, P, P, P, P, P],
    "dig3d_triplet_basis_tangent": [P, P, P, P, P, P, P, c_int64, c_int32, P, P, P],
    "dig3d_edge_dist_bwd2": [P, P, P, P, P, P, c_int64, P, P, P],
    "dig3d_schnet_edge_features_bwd2": [P, c_int64, P, c_int32, c_double, c_double, P, P, P, P, P, P, P],
    "dig3d_pronet_edge_features": [P, P, P, P, P, c_int64, c_int64, c_int32, c_double, c_int32, P, P, P, P, P, P],
    "dig3d_linear_set_config": [c_int32],
    "dig3d_transpose": [P, c_int32, c_int32, P, P],
    "dig3d_schnet_edge_features": [P, c_int64, P, c_int32, c_double, c_double, P, P, P],
    "dig3d_gsphere_edge_flags": [P, P, c_int64, c_int64, P, P],
    "dig3d_gsphere_keep_rows": [P, P, P, P, P, c_int64, c_int32, P],
    "dig3d_gsphere_attention": [P, P, c_int32, c_int32, c_int32, c_int64, c_int32, c_int32, P, P],
    "dig3d_gsphere_attention_dk": [P, P, c_int32, c_int32, c_int32, c_int64, c_int32, c_int32, c_int32, P, P],
    "dig3d_gsphere_tanh": [P, c_int64, P, P],
    "dig3d_gsphere_flow_reverse": [P, P, c_int64, c_int32, c_int32, P, P],
    "dig3d_gsphere_focus_select": [P, P, c_int64, c_int32, c_int32, c_double, c_int32, P, P, P, P, P, P],
    "dig3d_gsphere_compact": [P, c_int64, c_int32, c_int32, c_int32, P, P, P, P, P, P, P],
    "dig3d_gsphere_neighbors": [P, c_int32, c_int64, c_int32, P, P, P, P],
    "dig3d_gsphere_place": [c_int64, c_int32, c_int32, P, P, P, P, P, P, P, P, P, P, P],
    "dig3d_gsphere_gather_local": [P, c_int64, c_int32, c_int32, P, P, P, c_int32, P, P],
    "dig3d_gsphere_type_scale": [P, c_int32, P, P, c_int64, c_int32, c_int32, P, P, P],
    "dig3d_gsphere_att_fwd": [P, P, P, P, P, c_int64, c_int32, P, P, P],
    "dig3d_gsphere_att_bwd": [P, P, P, P, P, P, P, c_int64, c_int32, P, P, P, P],
    "dig3d_gsphere_att_fwd_dk": [P, P, P, P, P, c_int64, c_int32, c_int32, P, P, P],
    "dig3d_gsphere_att_bwd_dk": [P, P, P, P, P, P, P, c_int64, c_int32, c_int32, P, P, P, P],
    "dig3d_gsphere_flow_fwd": [P, P, P, c_int32, c_int64, c_int32, c_int32, P, P, P],
    "dig3d_gsphere_flow_bwd": [P, P, P, c_int32, P, P, c_int64, c_int32, c_int32, P, P, P, P],
    "dig3d_gsphere_sigmoid": [P, c_int64, P, P],
    "dig3d_gsphere_unary_bwd": [P, P, c_int64, c_int32, P, P],
    "dig3d_gsphere_keep_rows_bwd": [P, P, P, c_int64, c_int32, P, P, P],
    "dig3d_mmd_terms": [P, c_int64, c_int64, c_double, c_int32, c_double, P, c_int64, P, P],
    "dig3d_xyz2mol": [P, P, c_int64, c_int32, P, P, P],
    "dig3d_gen_traj": [P, P, P, P, c_int64, P, P, P, P, P, P, P, P, P, P, P, P, P],
    "dig3d_fire_step": [P, P, P, P, c_int32, P, P, P, c_int64, P, P, P, P, P, P, P, P, P, c_double, c_int32,
                        c_double, c_double, P],
    "dig3d_relax_compact": [P, P, c_int64, P, P, P, P, P, P],
}
_RESTYPES = {"dig3d_last_error": c_char_p}

_lib = None


class Dig3dError(RuntimeError):
    """A non-zero return code of the library; `rc` holds it (DIG3D_EINVAL = -1: the arguments were rejected)."""
    rc = None


def load():
    """Load libdig3d.so and bind every declared symbol (raises if anything is missing)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Dig3dError(
            f"{LIB_PATH} not found: build it with `python -m dig_b200.build` "
            "(nvcc -gencode arch=compute_90a,code=sm_90a). There is no CPU/PyTorch fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as exc:
            raise Dig3dError(f"libdig3d.so does not export {name}") from exc
        fn.argtypes = argtypes
        fn.restype = _RESTYPES.get(name, ctypes.c_int)
    _lib = lib
    return lib


# Launch accounting (bench.py's `gpu_launches`) and optional per-kernel CUDA-event timing
# (bench.py's roofline pass).  Every entry point except scan/ptr helpers, dig3d_mmd_terms (three kernels) and
# dig3d_relax_compact (two) launches exactly one kernel.
launch_count = 0
_timing = None            # None, or dict name -> list of (start_event, stop_event)


def start_timing():
    global _timing
    _timing = {}


def stop_timing():
    """Returns {entry point: [ms, ...]} for the calls made since start_timing() (synchronises)."""
    global _timing
    import torch
    torch.cuda.synchronize()
    out = {k: [a.elapsed_time(b) for a, b in v] for k, v in (_timing or {}).items()}
    _timing = None
    return out


def call(name, *args):
    global launch_count
    lib = load()
    if _timing is not None:
        import torch
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        rc = getattr(lib, name)(*args)
        b.record()
        _timing.setdefault(name, []).append((a, b))
    else:
        rc = getattr(lib, name)(*args)
    launch_count += 1
    if rc != 0:
        msg = lib.dig3d_last_error()
        err = Dig3dError(f"{name} failed (rc={rc}): {msg.decode() if msg else ''}")
        err.rc = rc
        raise err
