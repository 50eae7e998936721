/* dig3d.h -- C ABI of libdig3d.so, the sm_90a (H100) implementation of DIG's 3D-graph
 * message-passing hot path (dig.threedgraph.method.{SchNet,SphereNet,DimeNetPP,ComENet}).
 *
 * The reference has NO native/FFI boundary for this path (SURVEY.md 8b): every device op is a
 * third-party wheel or ATen kernel launched from Python.  Each entry point below therefore cites
 * the reference Python call site(s) whose device work it replaces.
 *
 * Conventions (all entry points):
 *   - plain pointers + sizes, no torch types; all pointers are DEVICE pointers unless named *_host;
 *   - caller owns every buffer (no allocation, no synchronisation inside except the one read-back of
 *     dig3d_radius_graph_pbc_count and dig3d_radius_graph_dense_count; the only process-wide state are the
 *     experiment switches dig3d_tc_set_fast_swish / dig3d_tc_trace / dig3d_linear_set_config and a thread-local
 *     error string);
 *   - `stream` is a cudaStream_t passed as void*;
 *   - returns 0 on success, a negative DIG3D_E* code otherwise; dig3d_last_error() returns a
 *     thread-local message for the last failing call;
 *   - fp32 everywhere; indices are int32 inside kernels, int64 at the reference-facing API
 *     (edge_index / idx_kj / idx_ji outputs).
 */
#ifndef DIG3D_H
#define DIG3D_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define DIG3D_OK 0
#define DIG3D_EINVAL (-1)
#define DIG3D_ECUDA (-2)
#define DIG3D_EUNSUPPORTED (-3)

const char* dig3d_last_error(void);
int dig3d_abi_version(void);

/* ------------------------------------------------------------------ graph construction
 * radius_graph(pos, r, batch)            schnet.py:156 dimenetpp.py:277 spherenet.py:304 comenet.py:294
 * (torch_cluster 1.6.0 CUDA semantics: per-graph brute force, strict d2 < r*r, first
 *  max_num_neighbors+1 hits in ascending source index incl. self, self removed afterwards)
 * + SparseTensor / repeat_interleave triplet enumeration   utils/geometric_computing.py:27-41
 */

/* G-SphereNet's private geometry (reference dig/ggraph3D/method/G_SphereNet/model/geometric_computing.py:12-19,54-104):
 * dig3d_knn2 = the two nearest neighbours of every node inside its graph (torch_cluster knn semantics; -1 where the
 * graph is too small); dig3d_triplet_geometry_knn = angles as dig3d_triplet_geometry plus the single-reference torsion
 * (reference atom = nearest neighbour of j, or the second nearest when the nearest is i), mapped to (0, 2 pi]. */
int dig3d_knn2(const float* pos, const int64_t* batch, const int32_t* graph_ptr, int64_t n_nodes, int64_t n_graphs,
               int32_t* nn1, int32_t* nn2, void* stream);
int dig3d_triplet_geometry_knn(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                               const int32_t* trip_ptr, int64_t n_edges, const int32_t* nn1, const int32_t* nn2,
                               float* angle, float* torsion, int64_t* idx_kj64, int64_t* idx_ji64, void* stream);

/* ptr[g] = first node of graph g, ptr[n_graphs] = n_nodes (batch is sorted ascending). */
int dig3d_graph_ptr(const int64_t* batch, int64_t n_nodes, int64_t n_graphs, int32_t* ptr, void* stream);

/* nbr[n*cap + s] = s-th in-neighbour (ascending) of node n, deg[n] = count (self excluded);
 * cap = max_num_neighbors + 1. */
int dig3d_radius_neighbors(const float* pos, const int64_t* batch, const int32_t* ptr, int64_t n_nodes,
                           int64_t n_graphs, double cutoff, int32_t cap, int32_t* nbr, int32_t* deg, void* stream);

/* Radius graph for any max_num_neighbors, without the nbr[N][cap] table (csrc/graph_dense.cu): the semantics of
 * dig3d_radius_neighbors + dig3d_edge_fill_out at cap = max_num_neighbors + 1, in two passes.
 * _count: counts[n_nodes] (workspace), row_ptr[n_nodes+1]; info [2] int64 on the device, zeroed by the caller, whose
 * info[1] may carry dig3d_validate_nodes' flags (int32 at byte offset 8).  The stream is synchronised once and
 * info_host[0] = E, info_host[1] = those flags; E >= 2^31 returns DIG3D_EINVAL (info_host still written).
 * _fill: src / dst [E] int32 and edge_index [2,E] int64 (nullable), sorted by (target, source). */
int dig3d_radius_graph_dense_count(const float* pos, const int64_t* batch, const int32_t* graph_ptr, int64_t n_nodes,
                                   int64_t n_graphs, double cutoff, int64_t max_num_neighbors, int32_t* counts,
                                   int32_t* row_ptr, int64_t* info, int64_t* info_host, void* stream);
int dig3d_radius_graph_dense_fill(const float* pos, const int64_t* batch, const int32_t* graph_ptr, int64_t n_nodes,
                                  int64_t n_graphs, double cutoff, int64_t max_num_neighbors, const int32_t* row_ptr,
                                  int64_t n_edges, int64_t* edge_index, int32_t* src, int32_t* dst, void* stream);

/* Index validation (the reference's nn.Embedding / scatter raise a device-side assert for these; e.g.
 * spherenet.py:86 `self.emb(x)`): ORs into *flags (caller-zeroed) bit 0 = a batch id outside [0, n_graphs),
 * bit 1 = batch not sorted ascending, bit 2 = an atomic number outside [0, z_rows) (z nullable). */
int dig3d_validate_nodes(const int64_t* batch, const int64_t* z, int64_t n_nodes, int64_t n_graphs, int32_t z_rows,
                         int32_t* flags, void* stream);

/* tcnt[i] = number of triplets (k->j->i, k != i) over the in-edges of node i; also counts the OUT-degree of every node
 * into out_cnt[n_nodes] (zero-initialised by the caller, nullable): the radius graph caps the in-degree only, so the
 * out-degree is not the in-degree. */
int dig3d_triplet_count_out(const int32_t* nbr, const int32_t* deg, int64_t n_nodes, int32_t cap, int32_t* tcnt,
                            int32_t* out_cnt, void* stream);

/* Exclusive scans: row_ptr[0..n] of deg, node_trip_ptr[0..n] of tcnt; totals[0]=E, totals[1]=T; out_ptr[0..n] of
 * out_cnt (both nullable together). */
int dig3d_scan_counts3(const int32_t* deg, const int32_t* tcnt, const int32_t* out_cnt, int64_t n_nodes,
                       int32_t* row_ptr, int32_t* node_trip_ptr, int32_t* out_ptr, int32_t* totals, void* stream);

/* Per-edge arrays, edges sorted by (target i, source j):
 *   edge_index[2,E] int64 (row 0 = source j, row 1 = target i), src/dst int32, dist[E],
 *   vec[E,3] = pos[j]-pos[i] (nullable), trip_ptr[E+1] (first triplet of each edge).
 *   dist = sqrt(sum((pos_i-pos_j)^2)) with ATen-CUDA rounding (geometric_computing.py:25).
 * And the OUT-edge lists (CSR by source; out_list, out_ptr and pos_in nullable together, graph_ptr and batch needed
 * with them): out_list[out_ptr[j] .. out_ptr[j+1]) = the edges (j -> i) in ascending i, pos_in[e] for e = (j -> i) =
 * position of i among j's own in-neighbours (deg[j] if i is not one).  The triplet kernels (projection: per (k -> j) edge; gather: per node and
 * layer) read them instead of searching the nodes of j's graph for j's out-edges. */
int dig3d_edge_fill_out(const float* pos, const int32_t* nbr, const int32_t* deg, const int32_t* row_ptr,
                        const int32_t* node_trip_ptr, int64_t n_nodes, int32_t cap, int64_t n_edges,
                        int64_t* edge_index, int32_t* src, int32_t* dst, float* dist, float* vec,
                        int32_t* trip_ptr, const int32_t* graph_ptr, const int64_t* batch, const int32_t* out_ptr,
                        int32_t* out_list, int32_t* pos_in, void* stream);

/* CSR / triplet offsets / distances for a CALLER-SUPPLIED edge_index [2,E] int64 sorted by (target, source)
 * (the entry of xyz_to_dat(pos, edge_index, num_nodes, ...), utils/geometric_computing.py:12).
 * cnt_ws: [2E+2] int32 workspace; flags: [6] int32, 8-byte aligned, written afterwards as
 * flags[0] != 0 => edge_index unsorted or out of range; flags[1] = heavy edges (source in-degree > 64);
 * flags[2] = E; flags[3] = number of triplets T as int32; flags[4..5] = T as int64 (T >= 2^31 wraps flags[3] and
 * trip_ptr: the caller must refuse it before any triplet kernel runs). */
int dig3d_edges_to_csr(const float* pos, const int64_t* edge_index, int64_t n_edges, int64_t n_nodes, int32_t* src,
                       int32_t* dst, int32_t* row_ptr, int32_t* cnt_ws, int32_t* trip_ptr, float* dist,
                       int32_t* flags, void* stream);

/* ------------------------------------------------------------------ geometry
 * xyz_to_dat(pos, edge_index, N, use_torsion)     utils/geometric_computing.py:43-75
 * angle[T], torsion[T] (nullable), idx_kj/idx_ji int32 (nullable) and int64 (nullable).
 * Triplets ordered by (edge ji ascending, k ascending); torsion = min over k_n != i of the
 * dihedral in (0, 2pi], the k_n == k self candidate included, cross products in ATen's
 * fma(a,b,-rn(c*d)) form (SURVEY.md 5.9a). */
int dig3d_triplet_geometry(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                           const int32_t* trip_ptr, int64_t n_edges, int32_t use_torsion, float* angle,
                           float* torsion, int32_t* idx_kj, int32_t* idx_ji, int64_t* idx_kj64,
                           int64_t* idx_ji64, void* stream);

/* dig3d_triplet_geometry (use_torsion 0 / 1) and dig3d_triplet_geometry_knn (use_torsion 2, nn1 / nn2 of dig3d_knn2)
 * at ANY in-degree, with the int64 indices.  The edges whose source has in-degree <= 64 run the warp-per-edge kernel of
 * those entry points; the n_heavy others (flags[1] of dig3d_edges_to_csr) run a CTA-per-edge kernel that folds the
 * torsion min across shared-memory tiles of planes.  Both call the same per-triplet device code, so a triplet's bits
 * do not depend on which kernel computed it.  0 < n_heavy < n_edges: the heavy edges are compacted on the device into
 * heavy_ws [n_heavy + 1]; n_heavy == n_edges runs every edge on the heavy kernel (no list, heavy_ws unused). */
int dig3d_triplet_geometry_any_degree(const float* pos, const int32_t* src, const int32_t* dst,
                                      const int32_t* row_ptr, const int32_t* trip_ptr, int64_t n_edges,
                                      int64_t n_heavy, int32_t use_torsion, const int32_t* nn1, const int32_t* nn2,
                                      int32_t* heavy_ws, float* angle, float* torsion, int64_t* idx_kj64,
                                      int64_t* idx_ji64, void* stream);

/* dig3d_triplet_geometry_any_degree with use_torsion 1 (same kernels, same angle / torsion / index bits) that also writes
 * tors_arg[T]: the slot s of the winning torsion candidate among j's in-edges (c = src[row_ptr[j] + s]), the first slot
 * among exactly equal minima, -1 when no candidate is finite.  The derivative kernels dig3d_triplet_torsion_bwd_arg and
 * dig3d_triplet_geometry_bwd2 read it instead of searching again. */
int dig3d_triplet_geometry_any_degree_arg(const float* pos, const int32_t* src, const int32_t* dst,
                                          const int32_t* row_ptr, const int32_t* trip_ptr, int64_t n_edges,
                                          int64_t n_heavy, int32_t* heavy_ws, float* angle, float* torsion,
                                          int64_t* idx_kj64, int64_t* idx_ji64, int32_t* tors_arg, void* stream);

/* ------------------------------------------------------------------ basis
 * dist_emb / angle_emb / torsion_emb      spherenet/features.py:167-263, dimenetpp/features.py:149-220
 * basis_id: 0 = dimenet flavour ns=7 nr=6, 1 = dimenet ns=3 nr=6, 2 = gemnet ns=2 nr=3 (ComENet).
 */
/* rbf0[E,nr] = env(d/c) * sin(freq*d/c); bess[E,ns*nr] = j~_ln(d/c) (times env(d/c) if envelope_on_bessel,
 * the DimeNet++ angle_emb variant, dimenetpp/features.py:214). */
int dig3d_edge_basis(const float* dist, int64_t n_edges, double cutoff, int32_t envelope_exponent,
                     const float* freq, int32_t basis_id, int32_t envelope_on_bessel, float* rbf0,
                     float* bess, void* stream);

/* Materialise sbf[T, ns*nr] and (nullable) tbf[T, ns*ns*nr] exactly as the reference's angle_emb /
 * torsion_emb do (test / API-parity path; the fused model path never materialises them). */
int dig3d_triplet_basis(const float* bess, const float* angle, const float* torsion, const int32_t* idx_kj,
                        int64_t n_triplets, int32_t basis_id, float* sbf, float* tbf, void* stream);

/* Fused basis evaluation + first basis projection for ALL layers:
 *   sbf_p[L, T, B] = lin_sbf1_l(sbf),  t_p[L, T, B] = lin_t1_l(tbf) (nullable => DimeNet++), layer-major
 * w_sbf1: [L][B][ns*nr], w_t1: [L][B][ns*ns*nr] (PyTorch [out,in] per layer, layers concatenated).
 * Requires L*B == 32.                                     spherenet.py:163,167  dimenetpp.py:146
 * out_ptr / out_list / pos_in: the out-edge lists of dig3d_edge_fill_out (nullable together: the out-edges are then
 * searched among the nodes of each graph; read by the torsion models' kernel).  The torsion models' harmonics come from
 * the recurrences the reference derives its closed forms from (features.py:74-148; csrc/harmonics.cuh); DimeNet++
 * (no torsion) uses the reference-rounded closed forms. */
int dig3d_triplet_basis_project_lists(const float* bess, const float* angle, const float* torsion,
                                      const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                                      const int32_t* trip_ptr, const int32_t* graph_ptr, const int64_t* batch,
                                      int64_t n_edges, int64_t n_triplets, int32_t basis_id, int32_t n_layers,
                                      int32_t basis_emb, const float* w_sbf1, const float* w_t1, float* sbf_p,
                                      float* t_p, const int32_t* out_ptr, const int32_t* out_list,
                                      const int32_t* pos_in, void* stream);

/* ------------------------------------------------------------------ segmented reductions
 * scatter(src, index, dim=0, dim_size, reduce='sum') with a SORTED index given as CSR pointers
 * (spherenet.py:211,224 schnet.py:55,81 comenet.py:398): out[s, :] = sum_{r in [ptr[s], ptr[s+1])} x[r, :].
 * No atomics, deterministic. */
int dig3d_segment_sum(const float* x, const int32_t* ptr, int64_t n_segments, int64_t width, float* out,
                      void* stream);

/* ------------------------------------------------------------------ SphereNet / DimeNet++ blocks
 * All weights are PyTorch nn.Linear layout [out, in] row-major fp32; null bias pointer = no bias.
 * H = hidden_channels (128), I = int_emb_size (64), B = basis_emb (8), nr = num_radial (6),
 * O = out_emb_channels (256).  Only these sizes are compiled in round 1. */
typedef struct {
  const float* emb;        /* [95, H]   init_e.emb.weight */
  const float* w_rbf0;     /* [H, nr]   init_e.lin_rbf_0.weight */
  const float* b_rbf0;     /* [H] */
  const float* w_lin;      /* [H, 3H]   init_e.lin.weight */
  const float* b_lin;      /* [H] */
  const float* w_rbf1;     /* [H, nr]   init_e.lin_rbf_1.weight */
} dig3d_init_e_weights;

typedef struct {
  const float *w_rbf1, *w_rbf2;   /* [B, nr], [H, B] */
  const float *w_sbf2, *w_t2;     /* [I, B], [I, B] (w_t2 null => DimeNet++) */
  const float *w_rbf;             /* [H, nr] */
  const float *w_kj, *b_kj, *w_ji, *b_ji;   /* [H, H], [H] */
  const float *w_down, *w_up;     /* [I, H], [H, I] */
  const float *w_res[6], *b_res[6]; /* before_skip.0.{lin1,lin2}, after_skip.{0,1}.{lin1,lin2}: [H,H],[H] */
  const float *w_lin, *b_lin;     /* [H, H], [H] */
} dig3d_update_e_weights;

typedef struct {
  const float *w_up, *b_up;       /* [O, H], [O] */
  const float *w_lins[8], *b_lins[8]; /* [O, O], [O]; first n_lins used */
  const float *w_out;             /* [out_channels, O] */
  int32_t n_lins;                 /* num_output_layers */
} dig3d_update_v_weights;

/* init.forward (spherenet.py:79-91, dimenetpp.py:71-78) fused with the edge->node scatter of
 * update_v (spherenet.py:211): writes e1[E,H] and ACCUMULATES e2 into v_in[N,H] (caller zeroes). */
int dig3d_sphere_init_e(const int64_t* z, const int32_t* src, const int32_t* dst, const float* rbf0,
                        int64_t n_edges, const dig3d_init_e_weights* w, float* e1, float* v_in,
                        void* stream);

/* update_e.forward part A (spherenet.py:154-161): x_ji[E,H], x_kj_down[E,I]. */
int dig3d_sphere_update_e_a(const float* e1, const float* rbf0, int64_t n_edges,
                            const dig3d_update_e_weights* w, float* x_ji, float* x_down, void* stream);

/* update_e.forward part B (spherenet.py:163-180) fused with update_v's scatter (spherenet.py:211):
 * triplet gather * basis, segmented sum over idx_ji, lin_up, residual stack; writes e1_out[E,H]
 * and ACCUMULATES e2 into v_in[N,H].  sbf_p/t_p are the layer's [T, ld_p] slices (col offset
 * applied by the caller), t_p null => DimeNet++. */
int dig3d_sphere_update_e_b(const float* e1_in, const float* x_ji, const float* x_down, const float* rbf0,
                            const float* sbf_p, const float* t_p, int32_t ld_p, const int32_t* src,
                            const int32_t* dst, const int32_t* row_ptr, const int32_t* trip_ptr,
                            int64_t n_edges, const dig3d_update_e_weights* w, float* e1_out, float* v_in,
                            void* stream);

/* update_v.forward after the scatter (spherenet.py:212-215): v_out[N, out_channels]. */
int dig3d_sphere_update_v(const float* v_in, int64_t n_nodes, int32_t out_channels,
                          const dig3d_update_v_weights* w, float* v_out, void* stream);

/* All n_blocks (= num_layers + 1 <= 8) node MLPs in one launch: v_in_all [n_blocks, N, H], w[n_blocks],
 * v_out_all [n_blocks, N, out_channels]. */
int dig3d_sphere_update_v_batched(const float* v_in_all, int64_t n_nodes, int32_t n_blocks, int32_t out_channels,
                                  const dig3d_update_v_weights* w, float* v_out_all, void* stream);

/* update_u over all blocks (spherenet.py:223-225,313-318): u[g, c] = sum_l sum_{n in g} v[l][n][c],
 * v: [n_blocks, N, C] contiguous. */
int dig3d_graph_readout(const float* v, const int32_t* graph_ptr, int64_t n_graphs, int64_t n_nodes,
                        int32_t n_blocks, int32_t channels, float* u, void* stream);

/* ------------------------------------------------------------------ update_e on the tensor cores (wgmma)
 * Same math as dig3d_sphere_update_e_a/_b with the dense chain on wgmma tf32 (3xTF32 split, one K-chunk per
 * tensor-core accumulation, chunks summed in fp32).  Weights are pre-split / pre-arranged once per parameter update:
 *   dig3d_tc_pack: W [N,K] (nn.Linear layout) -> [K/32][hi|lo][8][N][4] floats (2*N*K floats per matrix). */
int dig3d_tc_pack(const float* const* weights, const int32_t* n, const int32_t* k, float* const* outs,
                  int32_t count, void* stream);
/* number of mbarrier waits that hit the bounded-spin limit since library load (0 = healthy) */
int dig3d_tc_timeouts(void);

typedef struct {
  const float *p_ji, *b_ji, *p_kj, *b_kj;     /* packed lin_ji / lin_kj [128,128] + fp32 biases */
  const float *p_down, *p_up;                 /* packed lin_down [64,128], lin_up [128,64] */
  const float *p_res[6], *b_res[6];           /* packed residual linears, order as dig3d_update_e_weights */
  const float *p_lin, *b_lin;
  const float *w_rbf1, *w_rbf2, *w_rbf;       /* small fp32 matrices, nn.Linear layout */
  const float *w_sbf2, *w_t2;                 /* [64,8] (w_t2 null => DimeNet++) */
} dig3d_tc_update_e;

/* init.forward on wgmma; packed_lin = dig3d_tc_pack of init_e.lin.weight [128, 384] (one matrix, K = 384). */
int dig3d_sphere_init_e_tc(const int64_t* z, const int32_t* src, const int32_t* dst, const float* rbf0,
                           int64_t n_edges, const dig3d_init_e_weights* w, const float* packed_lin, float* e1,
                           float* v_in, void* stream);
int dig3d_sphere_update_e_a_tc(const float* e1, const float* rbf0, int64_t n_edges, const dig3d_tc_update_e* w,
                               float* x_ji, float* x_down, void* stream);
/* m[e] = sum over the triplets of edge e of x_down[kj] * lin_sbf2(sbf_p) * lin_t2(t_p)   (spherenet.py:163-171);
 * SIMT, one warp per edge, register accumulation over the contiguous triplet range (no atomics). */
int dig3d_sphere_triplet_gather(const float* x_down, const float* sbf_p, const float* t_p, int32_t ld_p,
                                const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                                const int32_t* trip_ptr, int64_t n_edges, const float* w_sbf2, const float* w_t2,
                                float* m, void* stream);
/* The same sums (bit-identical) organised around the SOURCE node, one WARP per (source node j, share): the warp stages
 * the x_down rows of j's in-edges (contiguous in the target-sorted edge list, <= cap x 256 B) in its own shared memory
 * with one cp.async.bulk (own mbarrier) and serves every out-edge (j -> i) of its share from it; in-neighbour positions
 * by ballot, no CTA-wide barrier.  Every edge that has a source is written (all of m[E, 64]).  split >= 1 warps share
 * a node (out-edge r of the node goes to share r % split); cap = max in-degree + 1 <= 64.  out_ptr / out_list / pos_in: the out-edge lists of dig3d_edge_fill_out
 * (nullable together: without them the warp searches the nodes of the graph). */
int dig3d_sphere_triplet_gather_warp(const float* x_down, const float* sbf_p, const float* t_p, int32_t ld_p,
                                     const int32_t* src, const int32_t* row_ptr, const int32_t* trip_ptr,
                                     const int32_t* graph_ptr, const int64_t* batch, int64_t n_nodes, int32_t cap,
                                     int32_t split, const float* w_sbf2, const float* w_t2, float* m,
                                     const int32_t* out_ptr, const int32_t* out_list, const int32_t* pos_in,
                                     void* stream);
/* lin_up + residual stack + lin (spherenet.py:172-180) on wgmma; writes e1_out, ACCUMULATES e2 into v_in. */
int dig3d_sphere_update_e_b_tc(const float* m, const float* e1_in, const float* x_ji, const float* rbf0,
                               const int32_t* dst, int64_t n_edges, const dig3d_tc_update_e* w, float* e1_out,
                               float* v_in, void* stream);
/* debugging probe: enable / read the clock64() timeline CTA 0 of the tensor kernels records (host buffer, 64 x i64) */
int dig3d_tc_trace(int32_t on, long long* out64);
/* 1: MUFU-only swish in the tensor-path epilogues (faster, ~1e-6 less accurate); default 0. */
int dig3d_tc_set_fast_swish(int32_t on);

/* ---- second-generation dense chain: two 128-edge tiles in flight per CTA, fp16 x3 split operands on wgmma
 * (csrc/spherenet_h16.cu).  Same arithmetic contract as the *_tc entry points above (update_e.forward
 * spherenet.py:150-182, init.forward spherenet.py:79-91); `w` is a dig3d_tc_update_e whose p_* members point to
 * dig3d_h16_pack output (4*N*K bytes per matrix: K/32 slabs of [hi|lo][4][N][8 halves], w*64 = hi + lo).
 * Activations must stay below 8190 in magnitude: larger values poison the affected energies with inf/NaN and
 * raise the flag returned by dig3d_h16_overflow -- every 3xFP16 entry point (init_e, update_e parts A / B / BA,
 * update_v, linear_h16) raises it in the launch whose outputs became non-finite (the *_tc chain has fp32 range and
 * is the fallback). */
int dig3d_h16_pack(const float* const* weights, const int32_t* n, const int32_t* k, void* const* outs, int32_t count,
                   void* stream);
int dig3d_sphere_init_e_h16(const int64_t* z, const int32_t* src, const int32_t* dst, const float* rbf0,
                            int64_t n_edges, const dig3d_init_e_weights* w, const void* packed_lin, float* e1,
                            float* v_in, void* stream);
/* The same with the embedding panels folded into two tables: lin(cat[x_i, x_j, rbf0]) = tab_i[z_i] + tab_j[z_j] +
 * W[:, 256:384] rbf0 + b, tab_i = emb W[:, 0:128]^T, tab_j = emb W[:, 128:256]^T ([emb rows, 128] fp32, computed once per
 * parameter version with dig3d_linear); packed_rbf_panel: dig3d_h16_pack of W[:, 256:384].  One K = 128 job per tile
 * instead of three.                                                          spherenet.py:86-90 */
int dig3d_sphere_init_e_h16_tab(const int64_t* z, const int32_t* src, const int32_t* dst, const float* rbf0,
                                int64_t n_edges, const dig3d_init_e_weights* w, const void* packed_rbf_panel,
                                const float* tab_i, const float* tab_j, float* e1, float* v_in, void* stream);
/* update_e part A (x_ji, x_down) and part B (e1_out, edge -> node sums added into v_in, which the caller zeroes) on
 * the register-accumulator engine: persistent CTAs, two consumer warpgroups with one 64-edge unit each, activations
 * kept in wgmma register fragments between layers.                               spherenet.py:150-182, 211 */
int dig3d_sphere_update_e_a_h16(const float* e1, const float* rbf0, int64_t n_edges, const dig3d_tc_update_e* w,
                                float* x_ji, float* x_down, void* stream);
int dig3d_sphere_update_e_b_h16(const float* m, const float* e1_in, const float* x_ji, const float* rbf0,
                                const int32_t* dst, int64_t n_edges, const dig3d_tc_update_e* w, float* e1_out,
                                float* v_in, void* stream);
/* dig3d_sphere_update_e_b_h16 of block l with part A of block l + 1 (dig3d_sphere_update_e_a_h16 on the e1 this kernel
 * produces) appended to the same unit chain: one launch, one set-up and one read of e1 less per block; bit-identical to
 * the two separate launches.  w_next: the next block's weights; x_ji_next [E, 128] (must not alias x_ji), x_down_next
 * [E, 64]: its part-A outputs.                                                  spherenet.py:150-182 */
int dig3d_sphere_update_e_ba_h16(const float* m, const float* e1_in, const float* x_ji, const float* rbf0,
                                 const int32_t* dst, int64_t n_edges, const dig3d_tc_update_e* w,
                                 const dig3d_tc_update_e* w_next, float* e1_out, float* v_in, float* x_ji_next,
                                 float* x_down_next, void* stream);
/* init_e (dig3d_sphere_init_e_h16_tab with tab_i / tab_j and packed_init = the rbf panel, or dig3d_sphere_init_e_h16 with
 * both tables null and packed_init = the packed lin) with part A of block 0 (dig3d_sphere_update_e_a_h16, weights w) on
 * the e1 fragment in registers: one launch and one read of e1 less; bit-identical to the two launches.  Writes e1,
 * adds the edge -> node sums into v_in (zeroed by the caller), writes x_ji [E, 128] and x_down [E, 64].
 *                                                                          spherenet.py:79-91, 150-161 */
int dig3d_sphere_init_update_e_a_h16(const int64_t* z, const int32_t* src, const int32_t* dst, const float* rbf0,
                                     int64_t n_edges, const dig3d_init_e_weights* w_init, const void* packed_init,
                                     const float* tab_i, const float* tab_j, const dig3d_tc_update_e* w, float* e1,
                                     float* v_in, float* x_ji, float* x_down, void* stream);
/* update_v.forward after the scatter (spherenet.py:212-215) for ALL blocks of a forward on the register-accumulator
 * engine's roles (64-node units, operands in per-consumer fp16 planes, every 256-wide layer as two 128-column halves,
 * unit pairs of one block dealt over the grid); H = 128, O = 256,
 * out_channels <= 4.  packed[b * (n_lins + 1) + l] = dig3d_h16_pack of block b's lin_up (l = 0) / lins[l - 1]
 * as TWO [128, K] matrices back to back (output rows 0..127, then 128..255). */
int dig3d_sphere_update_v_h16_supported(int32_t hidden, int32_t out_emb, int32_t out_channels, int32_t n_lins);
int dig3d_sphere_update_v_h16(const float* v_in_all, int64_t n_nodes, int32_t n_blocks, int32_t out_channels,
                              int32_t n_lins, const void* const* packed, const dig3d_update_v_weights* w,
                              float* v_out_all, void* stream);
/* Training-path linears on the same engine: y[rows, nout] = x[rows, k] W^T + bias, optionally also swish(y);
 * dig3d_h16_pack_t: trans[i] = 0 packs weights[i] as a row-major [n, k] matrix; trans[i] = ld > 0 packs the TRANSPOSE of
 * a [k, n] block whose rows are ld floats apart (a column slice of W for the input-gradient GEMM dX = dY W). */
int dig3d_h16_pack_t(const float* const* weights, const int32_t* n, const int32_t* k, const int32_t* trans,
                     void* const* outs, int32_t count, void* stream);
int dig3d_linear_h16_supported(int32_t k, int32_t nout);
/* y (pre-activation) and act_out (swish(y)) may each be NULL (not both); residual [rows, nout] (nullable) is added to the
 * last output written (act_out if given, else y): swish(x W^T + b) + r is a residual layer in one launch, x W^T + b + r the
 * sum of two linears.  All 128-column slices of a wide layer run in one launch; small row counts use one tile per CTA. */
int dig3d_linear_h16(const float* x, int64_t rows, int32_t k, int32_t nout, const void* packed, const float* bias,
                     float* y, float* act_out, const float* residual, void* stream);
/* 1 if an operand left the fp16 range since the flag was last cleared (synchronises the device). */
int dig3d_h16_overflow(int32_t clear);
int dig3d_h16_timeouts(void);
/* debugging probe: enable / read the clock64() timeline CTA 0 of update_e part B records (host buffer, 128 x i64) */
int dig3d_h16_trace(int32_t on, long long* out128);
int dig3d_h16_set_fast_swish(int32_t on);

/* ------------------------------------------------------------------ SchNet
 * One interaction (update_e + update_v, schnet.py:29-35,53-59) for hidden_channels == num_filters in
 * {32, 64, 128}:  vlin = lin(v);  agg[i] = sum_{j->i} vlin[j] * mlp(gauss(d)) * C(d);
 *                 v_out = v + lin2(ssp(lin1(agg))).   agg must be zeroed by the caller.
 * w_mlp0 is [F, 64]: mlp.0.weight zero padded from num_gaussians to 64 columns. */
typedef struct {
  const float *w_lin;                 /* [F, H]  update_es.l.lin.weight (no bias) */
  const float *w_mlp0, *b_mlp0;       /* [F, 64 (padded G)], [F] */
  const float *w_mlp2, *b_mlp2;       /* [F, F], [F] */
  const float *w_v1, *b_v1;           /* [H, F], [H]   update_vs.l.lin1 */
  const float *w_v2, *b_v2;           /* [H, H], [H]   update_vs.l.lin2 */
} dig3d_schnet_block_weights;

int dig3d_schnet_block(const float* v, int64_t n_nodes, const float* dist, const int32_t* src,
                       const int32_t* dst, int64_t n_edges, const float* offset, int32_t n_gauss, double coeff,
                       double cutoff, int32_t hidden, int32_t filters, const dig3d_schnet_block_weights* w,
                       float* vlin, float* agg, float* v_out, void* stream);

/* update_u before the graph scatter (schnet.py:78-80): node_out[N, out_channels] = lin2(ssp(lin1(v))). */
int dig3d_schnet_readout(const float* v, int64_t n_nodes, int32_t hidden, const float* w1, const float* b1,
                         const float* w2, const float* b2, int32_t out_channels, float* node_out, void* stream);

/* ------------------------------------------------------------------ ComENet (hidden 256, middle 64, nr=3, ns=2)
 * dig3d_comenet_geometry: reference atoms (4x scatter_min, comenet.py:304-327), theta/phi/tau
 * (comenet.py:365-385) and the basis features feature1[E,12] / feature2[E,6]
 * (comenet/features.py:289-295,340-348).  refs: [4 * N + 2] int32 workspace (nearest / second-nearest
 * in-edge, nearest / second-nearest out-edge of every node, then two batch-wide flags "some node has no in-edge /
 * no out-edge": the reference penalises edge 0 in that case, comenet.py:305-308); angles: nullable [E,3]. */
int dig3d_comenet_geometry(const float* pos, const float* dist, const int32_t* src, const int32_t* dst,
                           const int32_t* row_ptr, const int32_t* graph_ptr, const int64_t* batch,
                           int64_t n_nodes, int64_t n_edges, double cutoff, int32_t* refs, float* feature1,
                           float* feature2, float* angles, void* stream);
/* Forces through the geometry above (refs: the buffer dig3d_comenet_geometry filled for the same pos and graph).
 * features_bwd: dpos[N,3] (every row written) = d loss / d pos given dfeature1 [E,12] / dfeature2 [E,6], with ATen's
 * conventions at singular points (a zero vector's norm and atan2(0, 0) pass no gradient) and no float atomics: three
 * passes (per edge: the five edge-vector gradients into work[0, 15E); per edge: their sum, in edge order, into
 * work[15E, 18E); per node: out-edges minus in-edges).  work: [18 * E] floats; out_ptr / out_list: the out-edge lists
 * of dig3d_edge_fill_out.  features_tangent: feature1_dot [E,12] / feature2_dot [E,6] along the per-atom displacement
 * cvec [N,3], the transpose of features_bwd. */
int dig3d_comenet_features_bwd(const float* pos, const float* dist, const int32_t* src, const int32_t* dst,
                               const int32_t* row_ptr, const int32_t* out_ptr, const int32_t* out_list,
                               const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                               const float* dfeature1, const float* dfeature2, float* work, float* dpos,
                               void* stream);
int dig3d_comenet_features_tangent(const float* pos, const float* dist, const int32_t* src, const int32_t* dst,
                                   const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                                   const float* cvec, float* feature1_dot, float* feature2_dot, void* stream);
/* Hessian-vector products through the geometry above.  features_tangent_bwd: dpos[N,3] (every row written) =
 * d/dpos of sum(g1 * feature1_dot + g2 * feature2_dot), feature*_dot = features_tangent(cvec) with cvec held constant,
 * i.e. sum over edges and features of g_k (d2 feature_k / dpos2) cvec.  g1 [E,12], g2 [E,6]; work: [18 * E] floats, the
 * three passes of features_bwd with the first evaluated on dual numbers along cvec.  Same conventions (an aliased
 * cross product is constant, a zero norm or atan2(0, 0) passes nothing) and no float atomics. */
int dig3d_comenet_features_tangent_bwd(const float* pos, const float* dist, const int32_t* src, const int32_t* dst,
                                       const int32_t* row_ptr, const int32_t* out_ptr, const int32_t* out_list,
                                       const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                                       const float* cvec, const float* g1, const float* g2, float* work, float* dpos,
                                       void* stream);

/* ComENet-OCP (reference dig/threedgraph/method/comenet/ocp/comenet-ocp.py:343-474): the graph arrives as an arbitrary
 * edge list with periodic images.  dig3d_pbc_edge_vectors = ocpmodels' get_pbc_distances (distance_vec = pos[row] -
 * pos[col] + cell_offsets . cell, called at :352-359; edge_graph[e] = graph of edge e).  dig3d_comenet_geometry_edges =
 * the four scatter_min / argmin over the UNSORTED target / source index (:374-399, 64-bit atomicMin of (distance, edge
 * id): ties resolve to the first edge like torch_scatter), then theta / phi / tau and the two basis features from the
 * distance vectors.  src / dst = int32 copies of edge_index[0] / [1]; refs [4 * N + 2] int32 and keys [2 * N] u64 are
 * workspaces. */
int dig3d_pbc_edge_vectors(const float* pos, const int64_t* edge_index, const float* cell, const float* cell_offsets,
                           const int32_t* edge_graph, int64_t n_edges, float* vec, float* dist, void* stream);
int dig3d_comenet_geometry_edges(const float* vec, const float* dist, const int64_t* edge_index, const int32_t* src,
                                 const int32_t* dst, int64_t n_nodes, int64_t n_edges, double cutoff, int32_t* refs,
                                 unsigned long long* keys, float* feature1, float* feature2, float* angles,
                                 void* stream);
/* Forces and cell gradients through the geometry above.  The gather and node passes of dig3d_comenet_features_bwd need
 * CSR edge order, so these run on the edges sorted by target: vec [E,3] / dist [E] / src / dst permuted, row_ptr over
 * the targets, out_ptr / out_list the out-edge lists by source in that order, refs [4 * N] the refs of
 * dig3d_comenet_geometry_edges with every edge id mapped to its sorted position (the flags are not read).
 * features_bwd_vec: dig3d_comenet_features_bwd with the edge vectors read from vec: work[15E, 18E) = dvec [E,3] =
 * d loss / d vec, dpos [N,3] = sum over out-edges - sum over in-edges of dvec (a self-image edge cancels).  Besides one
 * edge read twice, a cross product of two self-image edges of one atom with exactly parallel vectors (its images at +a
 * and -a) is aliased too: identically zero as a function of the cell, derivative zero.
 * features_tangent_vec: feature1_dot [E,12] / feature2_dot [E,6] along the per-atom displacement cvec [N,3], the cell
 * held fixed (vec_dot[e] = cvec[src] - cvec[dst]); the transpose of features_bwd_vec's dpos.
 * pbc_cell_bwd: dcell [G,3,3], dcell[g][a][b] = sum over the edges of graph g of cell_offsets[e][a] * dvec[e][b]; graph
 * g's edges are [row_ptr[graph_ptr[g]], row_ptr[graph_ptr[g + 1]]) (edges grouped by the graph of their target).  One
 * CTA per graph, a fixed-shape reduction and no float atomics: the same bits run to run. */
int dig3d_comenet_features_bwd_vec(const float* vec, const float* dist, const int32_t* src, const int32_t* dst,
                                   const int32_t* row_ptr, const int32_t* out_ptr, const int32_t* out_list,
                                   const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                                   const float* dfeature1, const float* dfeature2, float* work, float* dpos,
                                   void* stream);
int dig3d_comenet_features_tangent_vec(const float* vec, const float* dist, const int32_t* src, const int32_t* dst,
                                       const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                                       const float* cvec, float* feature1_dot, float* feature2_dot, void* stream);
/* features_tangent_bwd_vec: dig3d_comenet_features_tangent_bwd on the sorted edges with the edge vectors read from vec
 * and their tangent cvec[src] - cvec[dst] (the cell held fixed): the Hessian-vector products in pos. */
int dig3d_comenet_features_tangent_bwd_vec(const float* vec, const float* dist, const int32_t* src,
                                           const int32_t* dst, const int32_t* row_ptr, const int32_t* out_ptr,
                                           const int32_t* out_list, const int32_t* refs, int64_t n_nodes,
                                           int64_t n_edges, double cutoff, const float* cvec, const float* g1,
                                           const float* g2, float* work, float* dpos, void* stream);
int dig3d_pbc_cell_bwd(const float* dvec, const float* cell_offsets, const int32_t* row_ptr, const int32_t* graph_ptr,
                       int64_t n_graphs, float* dcell, void* stream);

/* Periodic radius graph = ocpmodels' radius_graph_pbc(data, radius, max_num_neighbors) (2022), called by ComENet-OCP
 * with otf_graph=True (comenet-ocp.py:343-350).  pos [N,3], cell [B,3,3] (rows = lattice vectors), natoms [B] int64.
 * Image range per axis = ceil(radius * |a_k x a_l| / vol), maximum over the batch; candidates per target i: source j
 * of the same structure, then image cell (cartesian product, last axis fastest); kept when d2 <= fp32(radius^2) and
 * d2 > 1e-4; with max_num_neighbors > 0 each target keeps its max_num_neighbors smallest d2 (ties: first enumerated).
 * Count pass: graph_ptr [B+1], counts [N], select [2N] and row_ptr [N+1] int32 and info [6] int64 are written
 * (device); the stream is synchronised once and *n_edges_host receives E.  Returns DIG3D_EINVAL for a cell with
 * zero or non-finite volume, natoms that do not sum to N, an image range above 2^31 candidates per atom, or E >= 2^31.
 * Fill pass (after a successful count, same buffers): edge_index [2,E] int64 = (j, i) grouped by target in
 * enumeration order, cell_offsets [E,3] fp32 = integer image cell, neighbors [B] int64 = edges per structure. */
int dig3d_radius_graph_pbc_count(const float* pos, const float* cell, const int64_t* natoms, int64_t n_atoms,
                                 int64_t n_graphs, double radius, int32_t max_num_neighbors, int32_t* graph_ptr,
                                 int32_t* counts, uint32_t* select, int32_t* row_ptr, int64_t* info,
                                 int64_t* n_edges_host, void* stream);
int dig3d_radius_graph_pbc_fill(const float* pos, const float* cell, int64_t n_atoms, int64_t n_graphs, double radius,
                                const int32_t* graph_ptr, const uint32_t* select, const int32_t* row_ptr,
                                const int64_t* info, int64_t n_edges, int64_t* edge_index, float* cell_offsets,
                                int64_t* neighbors, void* stream);

/* x = act(emb(z))   EmbeddingBlock.forward, comenet.py:125-127 */
int dig3d_comenet_embed(const int64_t* z, const float* emb, int64_t n_nodes, float* x, void* stream);

typedef struct {
  const float *w_lin, *b_lin;                 /* [256,256],[256]  interaction_blocks.b.lin */
  const float *w_f1a, *w_f1b;                 /* lin_feature1.lin1 [64,12], .lin2 [256,64] (no bias) */
  const float *w_f2a, *w_f2b;                 /* lin_feature2.lin1 [64,6],  .lin2 [256,64] */
  const float *w_rel1, *b_rel1, *w_root1;     /* conv1.lin_rel (+bias), conv1.lin_root */
  const float *w_rel2, *b_rel2, *w_root2;     /* conv2 */
  const float *w_lin1, *b_lin1, *w_lin2, *b_lin2;
  const float *w_cat, *b_cat;                 /* [256,512],[256] */
  const float *w_lins[8], *b_lins[8];         /* lins.{l} */
  const float *norm_w, *norm_b, *norm_ms;     /* GraphNorm weight, bias, mean_scale */
  const float *w_final, *b_final;
  int32_t n_lins;
} dig3d_comenet_block_weights;

typedef struct {                               /* output head, comenet.py:394-396 (n_lins == 0: no head) */
  const float *w_lins[8], *b_lins[8];
  const float *w_out, *b_out;                  /* [out_channels,256],[out_channels] */
  int32_t n_lins;
} dig3d_comenet_head_weights;

/* One SimpleInteractionBlock (comenet.py:195-215): 5 kernels (entry lin, both edge convolutions with
 * the edge->node scatter fused, node block, GraphNorm statistics, norm + final).  When head->n_lins > 0
 * the output head is fused behind `final` and node_out[N,out_channels] is written instead of x_out.
 * Workspaces: xs, h [N,256]; agg1, agg2 [N,256] ZEROED by the caller; stats [2, n_graphs, 256]. */
int dig3d_comenet_block(const float* x_in, const float* feature1, const float* feature2, const int32_t* src,
                        const int32_t* dst, const int32_t* graph_ptr, const int64_t* batch, int64_t n_nodes,
                        int64_t n_edges, int64_t n_graphs, const dig3d_comenet_block_weights* w,
                        const dig3d_comenet_head_weights* head, int32_t out_channels, float* xs, float* agg1,
                        float* agg2, float* h, float* stats, float* x_out, float* node_out, void* stream);
/* EdgeGraphConv aggregation for the tensor-engine forward: agg[i] = sum over the in-edges e = (j -> i) of w[e] * x[j]
 * (comenet.py:66-73), w [E, width] in CSR (target-sorted) edge order, width 128 or 256; every row of agg is written. */
int dig3d_edge_weighted_sum(const float* w, const float* x, const int32_t* src, const int32_t* row_ptr, int64_t n_nodes,
                            int32_t width, float* out, void* stream);
/* The same with the bias-free, activation-free TwoLayerLinear edge filter folded in (W_eff = W2 W1, weff_t = W_eff^T
 * [q, width]): agg[i][c] = sum_e (sum_q weff_t[q][c] feat[e][q]) * x[src e][c]; q = 12 or 6; every row written. */
int dig3d_comenet_filter_sum(const float* feat, int32_t q, const float* weff_t, const float* x, const int32_t* src,
                             const int32_t* row_ptr, int64_t n_nodes, int32_t width, float* out, void* stream);

/* ------------------------------------------------------------------ training primitives (csrc/train_ops.cu)
 * Forward/backward building blocks of the training path (reference run.py:103-135 = forward + loss.backward();
 * the reference gets its backward from torch.autograd over ATen ops -- here each primitive has a hand-written
 * kernel and torch.autograd only records the tape, see dig_b200/autograd.py).  All fp32, row-major.
 *   linear:  y[rows,nout] = x[rows,k] w[nout,k]^T (+ bias)           nn.Linear (torch F.linear)
 *   wgrad:   dw[nout,k] += dy^T x ; db[nout] += colsum(dy) (db nullable); dw/db must be initialised by caller
 *   act:     mode 0 swish (spherenet.py:14), mode 1 shifted softplus (schnet.py:97-103), mode 2 relu (pronet.py:340);
 *            act_bwd: dx = dy*act'(x)
 *   ewise:   op 0 y = a*b, op 1 y = a+b ; rowscale: y[r,:] = a[r,:] * s[r]
 *   gather_rows: y[r,:] = x[idx[r],:] ; scatter_add_rows: out[idx[r],:] += y[r,:] (atomics; out initialised) */
/* groups >= 1: that many independent problems of the same shape stacked along a leading dimension (x [G,rows,k],
 * w [G,nout,k], bias [G,nout], y [G,rows,nout], dw [G,nout,k], db [G,nout]) in ONE launch -- the five node MLPs of a
 * SphereNet / DimeNet++ forward are small (2304 rows) and latency-bound one at a time. */
int dig3d_linear(const float* x, int64_t rows, int32_t k, int32_t nout, const float* w, const float* bias, float* y,
                 float* act_out /* nullable: also receives swish(y) */, int32_t groups, void* stream);
int dig3d_wgrad(const float* dy, const float* x, int64_t rows, int32_t nout, int32_t k, float* dw, float* db,
                int32_t groups, void* stream);
/* The same contract on the tensor cores (csrc/train_tc.cu): 3xTF32 wgmma with the transposed operand tiles built on
 * the fly, one row chunk per tensor-core accumulation summed in fp32 registers, coalesced red.global of the partial tiles.  dig3d_wgrad routes here when
 * dig3d_wgrad_tc_supported (nout >= 64, k >= 64, rows >= 1024 and mode 1); dig3d_wgrad_set_mode(0) forces the FFMA kernel. */
int dig3d_wgrad_tc(const float* dy, const float* x, int64_t rows, int32_t nout, int32_t k, float* dw, float* db,
                   int32_t groups, void* stream);
int dig3d_wgrad_tc_supported(int64_t rows, int32_t nout, int32_t k);
int dig3d_wgrad_set_mode(int32_t mode);
int dig3d_wgrad_tc_timeouts(void);
/* tile configuration of the 128 -> 128 linear (tuning / experiments): 0 = 64-row tiles, 1 = 64-row tiles with two CTAs
 * per SM (default), 2 = 128-row tiles */
int dig3d_linear_set_config(int32_t cfg);
int dig3d_act(const float* x, int64_t n, int32_t mode, float* y, void* stream);
int dig3d_act_bwd(const float* x, const float* dy, int64_t n, int32_t mode, float* dx, void* stream);
/* Fused Adam step over FLAT fp32 buffers (run.py:49 `Adam(model.parameters(), lr, weight_decay)`; torch.optim.Adam
 * semantics, amsgrad off): step = 1-based count of this update. */
int dig3d_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, double lr,
                    double beta1, double beta2, double eps, double weight_decay, int64_t step, void* stream);
int dig3d_ewise(const float* a, const float* b, int64_t n, int32_t op, float* y, void* stream);
int dig3d_rowscale(const float* a, const float* s, int64_t rows, int32_t width, float* y, void* stream);
int dig3d_gather_rows(const float* x, const void* idx, int32_t idx_is_64, int64_t rows, int32_t width, float* y,
                      void* stream);
int dig3d_scatter_add_rows(const float* y, const void* idx, int32_t idx_is_64, int64_t rows, int32_t width,
                           float* out, void* stream);
/* dfreq[num_radial] += d(loss)/d(dist_emb.freq) given drbf0[E, num_radial] (rbf0 = envelope * sin(freq * d/cutoff),
 * spherenet/features.py:180-182); dfreq initialised by the caller. */
int dig3d_rbf_freq_grad(const float* dist, int64_t n_edges, double cutoff, int32_t envelope_exponent,
                        const float* freq, int32_t num_radial, const float* drbf0, float* dfreq, void* stream);
/* Backward of dig3d_triplet_basis_project_lists w.r.t. the projection weights: dw_sbf1[32, ns*nr] / dw_t1[32, ns*ns*nr]
 * (rows = layer*8 + basis row, same row order as the forward's w_sbf1 / w_t1; zero-initialised by the caller) from
 * the per-layer gradients d_sbf_p[l] / d_t_p[l] ([T, 8] each, HOST arrays of 4 device pointers, entries may be NULL).
 * The [T, ns*ns*nr] basis is recomputed on chip, never materialised.  dw_t1 NULL = no torsion (DimeNet++). */
int dig3d_triplet_basis_project_bwd(const float* bess, const float* angle, const float* torsion, const int32_t* src,
                                    const int32_t* dst, const int32_t* row_ptr, const int32_t* trip_ptr,
                                    const int32_t* graph_ptr, const int64_t* batch, int64_t n_edges, int64_t n_triplets,
                                    int32_t basis_id, const float* const* d_sbf_p, const float* const* d_t_p,
                                    float* dw_sbf1, float* dw_t1, void* stream);
/* Backward of dig3d_sphere_triplet_gather (spherenet.py:163-171): from dm[E, 64] computes dx_down[E, 64] (atomics, zeroed
 * by the caller), d_sbf_p / d_t_p [T, 8] (every row written) and dw_sbf2 / dw_t2 [64, 8] (zeroed by the caller). */
int dig3d_sphere_triplet_gather_bwd(const float* dm, const float* x_down, const float* sbf_p, const float* t_p,
                                    const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                                    const int32_t* trip_ptr, int64_t n_edges, const float* w_sbf2, const float* w_t2,
                                    float* dx_down, float* d_sbf_p, float* d_t_p, float* dw_sbf2, float* dw_t2,
                                    void* stream);
/* GraphNorm (torch_geometric.nn.GraphNorm as used at comenet.py:160,213) for the training path:
 * y = weight * (h - mean*mean_scale) / sqrt(mean((h - mean*mean_scale)^2) + eps) + bias per graph and channel;
 * shift / stdv [n_graphs, width] are kept for the backward.  bwd: dx every row written; dweight / dbias /
 * dmean_scale [width] accumulated with atomics (zeroed by the caller). */
int dig3d_graphnorm(const float* h, const int32_t* graph_ptr, int64_t n_graphs, int32_t width, const float* weight,
                    const float* bias, const float* mean_scale, double eps, float* y, float* shift, float* stdv,
                    void* stream);
int dig3d_graphnorm_bwd(const float* h, const float* dy, const int32_t* graph_ptr, int64_t n_graphs, int32_t width,
                        const float* weight, const float* mean_scale, const float* shift, const float* stdv, float* dx,
                        float* dweight, float* dbias, float* dmean_scale, void* stream);
/* GraphNorm's forward mode (force training) from the forward's shift / stdv: with o = h - shift,
 * y_dot = weight * (o_dot / std - o * std_dot / std^2), o_dot = h_dot - mean_scale * mean(h_dot),
 * std_dot = mean(o * o_dot) / std; every row of y_dot written.  tangent_bwd: the gradients of y_dot given dy_dot;
 * dh / dh_dot every row written, dweight / dmean_scale [width] accumulated with atomics (zeroed by the caller). */
int dig3d_graphnorm_tangent(const float* h, const float* h_dot, const int32_t* graph_ptr, int64_t n_graphs,
                            int32_t width, const float* weight, const float* mean_scale, const float* shift,
                            const float* stdv, float* y_dot, void* stream);
int dig3d_graphnorm_tangent_bwd(const float* h, const float* h_dot, const float* dy_dot, const int32_t* graph_ptr,
                                int64_t n_graphs, int32_t width, const float* weight, const float* mean_scale,
                                const float* shift, const float* stdv, float* dh, float* dh_dot, float* dweight,
                                float* dmean_scale, void* stream);
/* ---- position gradients (forces = -dE/dpos; reference run.py:126,165 takes them with torch.autograd.grad) ----
 * edge_dist_bwd: dpos[N,3] += d|pos_i - pos_j| (atomics; dpos initialised by the caller).
 * triplet_angle_bwd: dpos += d angle[t] for angle = atan2(|ji x jk|, ji.jk) (geometric_computing.py:43-48).
 * edge_basis_bwd: ddist[E] = drbf0 . d rbf0/d dist (written, 0 when drbf0 is NULL) and bess_dx[E, ns*nr] = d/dx of the
 *   (enveloped, when envelope_on_bessel) Bessel basis of dig3d_edge_basis; either output may be NULL.
 * triplet_torsion_bwd: dpos += d torsion[t] through the minimising candidate (geometric_computing.py:53-75).
 * triplet_basis_project_bwd_geom: dangle[T], ddist_kj[E] (and dtorsion[T] when the torsion arguments are given; every
 *   row written) of dig3d_triplet_basis_project_lists given d_sbf_p / d_t_p (host arrays of 4 device pointers, NULL
 *   entries allowed) and the forward's w_sbf1 / w_t1 rows.
 * triplet_basis_bwd: reverse mode of dig3d_triplet_basis (materialised sbf [T, ns*nr] / tbf [T, ns*ns*nr]) given
 *   d_sbf / d_tbf (either NULL = zero): dangle[T], dtorsion[T] (NULL: skip) and ddist[E], the k->j edge's share through
 *   bess, with bess_dx from dig3d_edge_basis_bwd.  Every row of every output written (0 for an edge that is no
 *   triplet's k->j edge); one warp per k->j edge over the out-edge lists of dig3d_edge_fill_out, deterministic.
 * schnet_edge_features_bwd: ddist[E] from dgauss[E,G] / dcut[E] (either may be NULL).  rowdot: out[r] = a[r,:].b[r,:]. */
int dig3d_edge_dist_bwd(const float* pos, const int32_t* src, const int32_t* dst, const float* dist, const float* ddist,
                        int64_t n_edges, float* dpos, void* stream);
int dig3d_triplet_angle_bwd(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                            const int32_t* trip_ptr, const float* dangle, int64_t n_edges, float* dpos, void* stream);
int dig3d_edge_basis_bwd(const float* dist, int64_t n_edges, double cutoff, int32_t envelope_exponent, const float* freq,
                         int32_t basis_id, int32_t envelope_on_bessel, const float* drbf0, float* ddist, float* bess_dx,
                         void* stream);
int dig3d_triplet_basis_project_bwd_geom(const float* bess, const float* bess_dx, const float* angle,
                                         const float* torsion, const int32_t* src, const int32_t* dst,
                                         const int32_t* row_ptr, const int32_t* trip_ptr, const int32_t* graph_ptr,
                                         const int64_t* batch, int64_t n_edges, int64_t n_triplets, int32_t basis_id,
                                         const float* const* d_sbf_p, const float* const* d_t_p, const float* w_sbf1,
                                         const float* w_t1, double cutoff, float* ddist, float* dangle, float* dtorsion,
                                         void* stream);
int dig3d_triplet_basis_bwd(const float* bess, const float* bess_dx, const float* angle, const float* torsion,
                            const int32_t* dst, const int32_t* row_ptr, const int32_t* trip_ptr, const int32_t* out_ptr,
                            const int32_t* out_list, const int32_t* pos_in, int64_t n_edges, int64_t n_triplets,
                            int32_t basis_id, const float* d_sbf, const float* d_tbf, double cutoff, float* ddist,
                            float* dangle, float* dtorsion, void* stream);
int dig3d_triplet_torsion_bwd(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                              const int32_t* trip_ptr, const float* dtorsion, int64_t n_edges, float* dpos, void* stream);
/* ---- forward-mode (tangent) kernels of the force-TRAINING path (reference run.py:110-123; dig_b200/autograd_jvp.py) ----
 * d/d(theta) of  c . dE/dpos  (c = d loss / d force, fixed) is the parameter gradient of the directional derivative of E
 * along c, so the second-order path of DimeNet++ / SphereNet needs only FIRST-order tangents of the geometry and bases:
 * geometry_jvp: dist_dot[E], angle_dot[T] (NULL: skip), torsion_dot[T] (NULL: skip) along cvec[N,3]; every row written.
 * edge_basis_tangent: rbf0_dot[E,nr] / bess_dot[E,ns*nr] (either may be NULL) for dist_dot.
 * rbf_freq_grad_tangent: dfreq[nr] += d(loss)/d(freq) through rbf0_dot given g_dot = d(loss)/d(rbf0_dot).
 * triplet_basis_tangent: tangents of dig3d_triplet_basis' sbf [T, ns*nr] / tbf [T, ns*ns*nr] (same layouts). */
int dig3d_geometry_jvp(const float* pos, const float* cvec, const int32_t* src, const int32_t* dst,
                       const int32_t* row_ptr, const int32_t* trip_ptr, const float* dist, int64_t n_edges,
                       float* dist_dot, float* angle_dot, float* torsion_dot, void* stream);
int dig3d_edge_basis_tangent(const float* dist, const float* dist_dot, int64_t n_edges, double cutoff,
                             int32_t envelope_exponent, const float* freq, int32_t basis_id, int32_t envelope_on_bessel,
                             float* rbf0_dot, float* bess_dot, void* stream);
int dig3d_rbf_freq_grad_tangent(const float* dist, const float* dist_dot, int64_t n_edges, double cutoff,
                                int32_t envelope_exponent, const float* freq, int32_t nr, const float* g_dot,
                                float* dfreq, void* stream);
int dig3d_triplet_basis_tangent(const float* bess, const float* bess_dot, const float* angle, const float* angle_dot,
                                const float* torsion, const float* torsion_dot, const int32_t* idx_kj,
                                int64_t n_triplets, int32_t basis_id, float* sbf_dot, float* tbf_dot, void* stream);
/* Reverse mode of the tangents in their value inputs (Hessian-vector products of DimeNet++ / SphereNet):
 * edge_basis_tangent_bwd: given g_rbf0_dot = d(loss)/d(rbf0_dot) [E,nr] (nullable), d_dist [E] (through d2 rbf0/dx2)
 *   and d_dist_dot [E] (through d rbf0/dx); and, when bess_dxx is non-NULL, bess_dxx [E,ns*nr] = d2(bess)/dx2 (x = dist /
 *   cutoff, enveloped like the forward's bess when envelope_on_bessel).  Every output is written, none accumulated.
 * triplet_basis_tangent_bwd: reverse of triplet_basis_tangent with bess_dot = bess_dx * dist_dot / cutoff folded in,
 *   given g_sbf [T, ns*nr] / g_tbf [T, ns*ns*nr] (either NULL = zero): d_dist / d_dist_dot [E] (the k->j edge's share,
 *   summed by one warp per edge, no atomics) and d_angle / d_angle_dot / d_torsion / d_torsion_dot [T] (the torsion
 *   pair nullable).  bess_dx from dig3d_edge_basis_bwd, bess_dxx from dig3d_edge_basis_tangent_bwd; needs the graph's
 *   out-edge lists, like dig3d_triplet_basis_bwd. */
int dig3d_edge_basis_tangent_bwd(const float* dist, const float* dist_dot, int64_t n_edges, double cutoff,
                                 int32_t envelope_exponent, const float* freq, int32_t basis_id,
                                 int32_t envelope_on_bessel, const float* g_rbf0_dot, float* d_dist, float* d_dist_dot,
                                 float* bess_dxx, void* stream);
int dig3d_triplet_basis_tangent_bwd(const float* bess, const float* bess_dx, const float* bess_dxx,
                                    const float* dist_dot, const float* angle, const float* angle_dot,
                                    const float* torsion, const float* torsion_dot, const int32_t* dst,
                                    const int32_t* row_ptr, const int32_t* trip_ptr, const int32_t* out_ptr,
                                    const int32_t* out_list, const int32_t* pos_in, int64_t n_edges,
                                    int64_t n_triplets, int32_t basis_id, const float* g_sbf, const float* g_tbf,
                                    double cutoff, float* d_dist, float* d_dist_dot, float* d_angle,
                                    float* d_angle_dot, float* d_torsion, float* d_torsion_dot, void* stream);
int dig3d_schnet_edge_features_bwd(const float* dist, int64_t n_edges, const float* offset, int32_t n_gauss,
                                   double coeff, double cutoff, const float* dgauss, const float* dcut, float* ddist,
                                   void* stream);
int dig3d_rowdot(const float* a, const float* b, int64_t rows, int32_t width, float* out, void* stream);
/* Generic linear on wgmma (3xTF32 split, fp32-accurate; same machinery as the fused update_e chain): y = x W^T + bias
 * for the shapes dig3d_linear_tc_supported() reports (K in {64,128,256,384} -> 128, 128 -> 64); act_out (nullable)
 * additionally receives swish(y).  `packed` = dig3d_tc_pack / dig3d_tc_pack_t output for W; tc_pack_t packs W^T when
 * trans[i] != 0 (the source is then read as [K, N]), which gives the input-gradient GEMM dx = dy W. */
int dig3d_tc_pack_t(const float* const* weights, const int32_t* n, const int32_t* k, const int32_t* trans,
                    float* const* outs, int32_t count, void* stream);
int dig3d_linear_tc_supported(int32_t k, int32_t nout);
int dig3d_linear_tc(const float* x, int64_t rows, int32_t k, int32_t nout, const float* packed, const float* bias,
                    float* y, float* act_out, void* stream);
/* ---- second order, for training ON forces (run.py:110-123: loss.backward() through forces taken with create_graph=True);
 * built for the ops SchNet uses.  act_bwd2: out = g * dy * act''(x).  edge_dist_bwd2 / schnet_edge_features_bwd2: the
 * backward of the corresponding *_bwd entry points w.r.t. all their inputs (d_pos accumulated with atomics into a
 * caller-initialised buffer; d_dgauss / d_dcut / dgauss / dcut nullable). */
int dig3d_act_bwd2(const float* x, const float* dy, const float* g, int64_t n, int32_t mode, float* out, void* stream);
int dig3d_edge_dist_bwd2(const float* pos, const int32_t* src, const int32_t* dst, const float* dist, const float* ddist,
                         const float* g_dpos, int64_t n_edges, float* d_ddist, float* d_pos, void* stream);
int dig3d_schnet_edge_features_bwd2(const float* dist, int64_t n_edges, const float* offset, int32_t n_gauss,
                                    double coeff, double cutoff, const float* dgauss, const float* dcut, const float* g,
                                    float* d_dgauss, float* d_dcut, float* d_dist, void* stream);
/* ---- xyz_to_dat's derivatives at any in-degree (tors_arg from dig3d_triplet_geometry_any_degree_arg; n_edges < 2^26).
 * triplet_torsion_bwd_arg: dpos += d torsion[t] through candidate tors_arg[t] (one warp per edge, no search, no shared
 *   memory); the self candidate c = k, tors_arg = -1, |ji| = 0 and atan2(0, 0) pass nothing.
 * triplet_geometry_bwd2: the backward of dig3d_triplet_angle_bwd + dig3d_triplet_torsion_bwd_arg given
 *   g_dpos = d(loss)/d(dpos): d_dangle[t] = <grad angle_t, g_dpos>, d_dtorsion[t] = <grad torsion_t, g_dpos> (every row
 *   written when non-NULL) and d_pos += dangle_t H_angle_t g_dpos + dtorsion_t H_torsion_t g_dpos (atomics into a
 *   caller-initialised buffer).  dangle / dtorsion NULL = zero; tors_arg may be NULL when dtorsion and d_dtorsion are. */
int dig3d_triplet_torsion_bwd_arg(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                                  const int32_t* trip_ptr, const int32_t* tors_arg, const float* dtorsion,
                                  int64_t n_edges, float* dpos, void* stream);
int dig3d_triplet_geometry_bwd2(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                                const int32_t* trip_ptr, const int32_t* tors_arg, const float* dangle,
                                const float* dtorsion, const float* g_dpos, int64_t n_edges, float* d_dangle,
                                float* d_dtorsion, float* d_pos, void* stream);
/* ProNet (pronet.py:352-449, pronet/features.py:253-344): per-edge geometry from the C-alpha chain (sequence-neighbour
 * references), level 0 = aminoacid (feature1[E,12] from tau), level 1 = backbone / allatom (feature1[E,36] from the three
 * Euler angles of the N-CA-C frames; needs pos_n / pos_c); feature0[E,24] = d_theta_phi_emb, pos_emb[E,num_pos_emb];
 * dist[E] and angles[E,5] = (theta, phi, a1, a2, a3) are optional outputs (nullable). */
int dig3d_pronet_edge_features(const float* pos_ca, const float* pos_n, const float* pos_c, const int32_t* src,
                               const int32_t* dst, int64_t n_edges, int64_t n_nodes, int32_t level, double cutoff,
                               int32_t num_pos_emb, float* dist, float* feature0, float* feature1, float* pos_emb,
                               float* angles, void* stream);
/* out[cols, rows] = in[rows, cols]^T (weights for the input-gradient GEMM dx = dy W) */
int dig3d_transpose(const float* in, int32_t rows, int32_t cols, float* out, void* stream);
/* SchNet training path: gaussian smearing gauss[E, n_gauss] (schnet.py:92-94) and cosine cutoff cut[E]
 * (schnet.py:31) materialised (the fused inference kernel keeps them on chip). */
int dig3d_schnet_edge_features(const float* dist, int64_t n_edges, const float* offset, int32_t n_gauss, double coeff,
                               double cutoff, float* gauss, float* cut, void* stream);

/* ------------------------------------------------------------------ G-SphereNet generation (csrc/gsphere.cu)
 * reference dig/ggraph3D/method/G_SphereNet/model/{sphgen.py:82-204, spherenet.py, att.py, net_utils.py}.
 * Generation state is padded per molecule: z[G, ld] int64, pos[G, ld, 3], focus[G, ld] int64; at a step every active
 * molecule has n_atoms atoms, rows g*n_atoms .. of the flattened node arrays.
 *
 * SphereNet copy (spherenet.py:170-172,205,297): edge_flags marks the edges listed in cat(idx_ji, idx_kj) (flag zeroed
 * by the caller); keep_rows keeps x[r] where flag[r] != 0 (or, flag NULL, where the CSR segment ptr[r]..ptr[r+1] is not
 * empty) and writes fallback[fallback_idx ? fallback_idx[r] : r] (or 0 without fallback) elsewhere, in place. */
int dig3d_gsphere_edge_flags(const int32_t* trip_ptr, const int64_t* idx_kj, int64_t n_edges, int64_t n_triplets,
                             int32_t* flag, void* stream);
int dig3d_gsphere_keep_rows(const int32_t* flag, const int32_t* ptr, float* x, const float* fallback,
                            const int64_t* fallback_idx, int64_t rows, int32_t width, void* stream);
/* MH_ATT with one query per molecule (att.py:18-35): q[n_queries, 32*n_heads] projected queries; keys / values of query g
 * are rows g*n_keys .. of kv[*, ld_kv] at columns k_off / v_off; out = softmax-weighted value sum (d_k = 32). */
int dig3d_gsphere_attention(const float* q, const float* kv, int32_t ld_kv, int32_t k_off, int32_t v_off,
                            int64_t n_queries, int32_t n_keys, int32_t n_heads, float* out, void* stream);
/* The same at any head width d_k >= 1: q[n_queries, n_heads*d_k], scores divided by sqrt(d_k) computed in fp64 and
 * rounded to fp32 (att.py); equal to dig3d_gsphere_attention at d_k = 32. */
int dig3d_gsphere_attention_dk(const float* q, const float* kv, int32_t ld_kv, int32_t k_off, int32_t v_off,
                               int64_t n_queries, int32_t n_keys, int32_t n_heads, int32_t d_k, float* out,
                               void* stream);
/* Flow reverse (net_utils.py:28-37,75-80): y = tanh(x); flow_reverse applies the n_layers ST_Net_Exp affine maps, last
 * layer first, to latent[rows, dim] in place, st[g, l, :] = linear2 output (2*dim wide) of layer l, rescale[l] = its
 * Rescale weight. */
int dig3d_gsphere_tanh(const float* x, int64_t n, float* y, void* stream);
int dig3d_gsphere_flow_reverse(const float* st, const float* rescale, int64_t rows, int32_t dim, int32_t n_layers,
                               float* latent, void* stream);
/* Focus decision and compaction (sphgen.py:116-142), one CTA: score = sigmoid(logit[G, n_atoms]); can_focus rows of the
 * continuing molecules in order, cont_src / emit_src = their source rows, counts = (continuing, emitted). */
int dig3d_gsphere_focus_select(const float* logit, const int64_t* z, int64_t n_mols, int32_t n_atoms, int32_t ld,
                               double focus_th, int32_t emit, float* score, float* can_focus, int32_t* cont_src,
                               int32_t* emit_src, int32_t* counts, void* stream);
/* out row k = in row src[k] (first n_atoms columns of z / pos, n_atoms - 1 of focus). */
int dig3d_gsphere_compact(const int32_t* src, int64_t rows, int32_t n_atoms, int32_t ld_in, int32_t ld_out,
                          const int64_t* z, const float* pos, const int64_t* focus, int64_t* z_out, float* pos_out,
                          int64_t* focus_out, void* stream);
/* c1 = nearest atom to the focus, c2 (nullable) = nearest atom to c1 among the rest (sphgen.py:165-169,185-189). */
int dig3d_gsphere_neighbors(const float* pos, int32_t ld, int64_t n_mols, int32_t n_atoms, const int64_t* focus_id,
                            int64_t* c1, int64_t* c2, void* stream);
/* The new atom: type, position (sphgen.py:162-197, dattoxyz geometric_computing.py:107-122) and focus, written at
 * column n_atoms of z / pos and n_atoms - 1 of focus. */
int dig3d_gsphere_place(int64_t n_mols, int32_t n_atoms, int32_t ld, const int64_t* focus_id, const int64_t* c1,
                        const int64_t* c2, const float* dist, const float* angle, const float* torsion,
                        const int64_t* type_id, int64_t* z, float* pos, int64_t* focus, void* stream);
/* out[g] = cat_j feat[g*n_atoms + id_j[g]] for j < n_ids (<= 3): the local query features. */
int dig3d_gsphere_gather_local(const float* feat, int64_t n_mols, int32_t n_atoms, int32_t width, const int64_t* id0,
                               const int64_t* id1, const int64_t* id2, int32_t n_ids, float* out, void* stream);
/* type[g] = argmax latent[g, :dim]; out = feat * emb[type[g]] over the molecule's atoms (sphgen.py:151-153). */
int dig3d_gsphere_type_scale(const float* latent, int32_t dim, const float* emb, const float* feat, int64_t n_mols,
                             int32_t n_atoms, int32_t width, int64_t* type_out, float* out, void* stream);

/* ------------------------------------------------------------------ G-SphereNet training (csrc/gsphere_train.cu)
 * SphGen.forward (sphgen.py:44-79) and its backward; no atomics anywhere.
 * att_fwd: MH_ATT over ragged step graphs (att.py:18-35): query j [32*n_heads] attends to the rows
 * graph_ptr[qgraph[j]] .. graph_ptr[qgraph[j] + 1] of k / v; stat[j, h] = (segment maximum, denominator).
 * att_bwd: dq, and dk / dv of the key rows of every queried graph (each graph has at most one query; the caller
 * zeroes dk / dv for the others). */
int dig3d_gsphere_att_fwd(const float* q, const int64_t* qgraph, const int32_t* graph_ptr, const float* k,
                          const float* v, int64_t n_queries, int32_t n_heads, float* out, float* stat, void* stream);
int dig3d_gsphere_att_bwd(const float* dout, const float* q, const int64_t* qgraph, const int32_t* graph_ptr,
                          const float* k, const float* v, const float* stat, int64_t n_queries, int32_t n_heads,
                          float* dq, float* dk, float* dv, void* stream);
/* att_fwd / att_bwd at any head width d_k >= 1 (rows n_heads*d_k wide, scale sqrt(d_k) in fp64 rounded to fp32);
 * equal to the two above at d_k = 32. */
int dig3d_gsphere_att_fwd_dk(const float* q, const int64_t* qgraph, const int32_t* graph_ptr, const float* k,
                             const float* v, int64_t n_queries, int32_t n_heads, int32_t d_k, float* out, float* stat,
                             void* stream);
int dig3d_gsphere_att_bwd_dk(const float* dout, const float* q, const int64_t* qgraph, const int32_t* graph_ptr,
                             const float* k, const float* v, const float* stat, int64_t n_queries, int32_t n_heads,
                             int32_t d_k, float* dq, float* dk, float* dv, void* stream);
/* Flow forward (net_utils.py:83-93): st[l, rows, 2*dim] = linear2 output of layer l, rescale[l] its Rescale weight;
 * x = (x + t) * exp(exp(w_l) tanh(s)) over the layers in order, in float64 when x_f64 (x0 / x_out are double) else
 * float; log_jac[rows, dim] (float) = sum_l log(|s_l| + 1e-20).
 * flow_bwd: dst [n_layers, rows, 2*dim] and drescale [n_layers] from d x_out and d log_jac; part is scratch of
 * n_layers * rows * dim floats (per-element shares of d exp(w_l), reduced in a fixed order). */
int dig3d_gsphere_flow_fwd(const float* st, const float* rescale, const void* x0, int32_t x_f64, int64_t rows,
                           int32_t dim, int32_t n_layers, void* x_out, float* log_jac, void* stream);
int dig3d_gsphere_flow_bwd(const float* st, const float* rescale, const void* x0, int32_t x_f64, const void* dx_out,
                           const float* dlog_jac, int64_t rows, int32_t dim, int32_t n_layers, float* dst, float* part,
                           float* drescale, void* stream);
/* y = 1 / (1 + exp(-x)) (the focus classifier's Sigmoid); unary_bwd: dx = dy (1 - y^2) (mode 0, tanh) or
 * dy y (1 - y) (mode 1, sigmoid) from the forward output y. */
int dig3d_gsphere_sigmoid(const float* x, int64_t n, float* y, void* stream);
int dig3d_gsphere_unary_bwd(const float* y, const float* dy, int64_t n, int32_t mode, float* dx, void* stream);
/* Backward of gsphere_keep_rows: dx = dy on kept rows, 0 elsewhere; dfb = dy on the other rows, 0 on kept ones (either
 * output nullable). */
int dig3d_gsphere_keep_rows_bwd(const int32_t* flag, const int32_t* ptr, const float* dy, int64_t rows, int32_t width,
                                float* dx, float* dfb, void* stream);

/* ------------------------------------------------------------------ bond-length MMD (csrc/mmd.cu)
 * compute_mmd, reference dig/ggraph3D/utils/eval_bond_mmd_utils.py:44-97, in fp64: v[n_source + n_target] = [source;
 * target].  out[0] = bandwidth b (fix_sigma if non-zero, else sum_ij (v_i - v_j)^2 / (n^2 - n) from a two-pass centred
 * sum), out[1..3] = XX / n_s^2, YY / n_t^2, XY / (n_s n_t), the sums over S x S, T x T, S x T (diagonals included) of
 * sum_k exp(-d^2 / b_k), b_k = b / kernel_mul^(kernel_num / 2) * kernel_mul^k, 1 <= kernel_num <= 64.  Three launches;
 * workspace[workspace_len] (>= 3 doubles) takes 3 partials per CTA of the persistent pair grid (workspace_len / 3 CTAs),
 * reduced in a fixed order: the result is deterministic for a given workspace_len.  Empty or constant input gives NaN
 * terms, as in the reference. */
int dig3d_mmd_terms(const double* v, int64_t n_source, int64_t n_target, double kernel_mul, int32_t kernel_num,
                    double fix_sigma, double* workspace, int64_t workspace_len, double* out, void* stream);

/* ------------------------------------------------------------------ xyz2mol (csrc/xyz2mol.cu, csrc/xyz2mol.cuh)
 * xyz2mol(use_graph=True), reference dig/ggraph3D/utils/eval_validity_utils.py:382-405, for n_mols molecules of n_atoms
 * atoms each (1 <= n_atoms <= 64): z[n_mols * n_atoms] atomic numbers (any value; elements other than H, C, N, O, F
 * bond to nothing and make the molecule invalid), pos[n_mols * n_atoms * 3] fp64 coordinates.  Writes the bond-order
 * matrix bo[n_mols * n_atoms * n_atoms] (row-major per molecule) and valid[n_mols] (1 / 0; -1 would mark an internal
 * capacity overflow of the matching, which the bounds in xyz2mol.cuh rule out).  One launch, one thread per molecule. */
int dig3d_xyz2mol(const int64_t* z, const double* pos, int64_t n_mols, int32_t n_atoms, int8_t* bo, int8_t* valid,
                  void* stream);

/* ------------------------------------------------------------------ G-SphereNet trajectories (csrc/gen_traj.cu)
 * QM93DGEN.get, reference dig/ggraph3D/dataset/ggraph3D_dataset.py:192-302, for n_mols molecules of 2 to 32 atoms, one
 * warp per molecule.  Inputs: atom_type [N] int64, pos [N, 3] fp32, con = the molecules' n x n bond matrices back to
 * back (int64).  ptr [6, n_mols + 1] int64 holds exclusive prefix sums per molecule of, in this order: n (atoms), n^2
 * (con), n(n-1)/2 (trajectory rows), n-1 (steps), max(n-2, 0) (angles), max(n-3, 0) (torsions).  Writes every field of
 * get() at the molecule's offsets: out_type / out_pos [rows, 3] / out_batch / out_cannot_focus per trajectory row,
 * out_focus / out_new_type / out_dist per step, out_c1 [angles, 2], out_angle per angle step, out_c2 [torsions, 3],
 * out_torsion per torsion step; atom indices are offset as get() offsets them.  status[m] = 0, or 1 where the
 * spanning tree has no edge (one atom, or all atoms at one position; that molecule's outputs are not written). */
int dig3d_gen_traj(const int64_t* atom_type, const float* pos, const int64_t* con, const int64_t* ptr, int64_t n_mols,
                   int64_t* out_type, float* out_pos, int64_t* out_batch, float* out_cannot_focus, int64_t* out_focus,
                   int64_t* out_c1, int64_t* out_c2, int64_t* out_new_type, double* out_dist, double* out_angle,
                   double* out_torsion, int32_t* status, void* stream);

/* ------------------------------------------------------------------ FIRE relaxation (csrc/relax.cu)
 * One FIRE step (N_min 5, f_inc 1.1, f_dec 0.5, alpha_start 0.1, f_alpha 0.99) for n_active structures, one CTA each.
 * Structure a of the active list is batch structure s = active[a], atoms graph_ptr[s] .. graph_ptr[s + 1] of
 * pos / vel [N, 3] fp32 (batch order, updated in place); grad [sum n_a, 3] = dE/dpos of the active structures back to
 * back, structure a at sub_ptr[a] (the force is -grad); energy [n_active, n_out] (nullable) their model outputs.
 * fixed [N] (nullable, 0 / 1): fixed atoms feel no force, count in no reduction and are never written.  Per batch
 * structure, fp64 dt / alpha and int32 n_pos / steps hold the FIRE state; the step writes fmax_out[s] = max over free
 * atoms of |F_i| (fp64), energy_out[s] = the row sum of energy, force_out (nullable) the structure's forces with zero
 * rows on fixed atoms, and status[s] = 1 if fmax_out < fmax (no free atom: converged), else 2 if steps >= max_steps
 * (neither moves), else 0 and the structure takes its step: the power check (skipped while steps = 0), velocity mixing
 * or reset, v += dt F, dr = dt v clipped to |dr| <= max_step over the structure, steps += 1.  Every reduction is fp64 in
 * a fixed order that depends only on the structure's atom count: bit-identical between runs and batch compositions. */
int dig3d_fire_step(float* pos, float* vel, const float* grad, const float* energy, int32_t n_out,
                    const int32_t* graph_ptr, const int32_t* active, const int32_t* sub_ptr, int64_t n_active,
                    const uint8_t* fixed, double* dt, double* alpha, int32_t* n_pos, int32_t* steps, int32_t* status,
                    double* fmax_out, float* energy_out, float* force_out, double fmax, int32_t max_steps,
                    double dt_max, double max_step, void* stream);
/* The structures of a batch with status[s] == 0, in batch order: active[A], new_ptr[A + 1] (their graph_ptr in the
 * sub-batch), atom_map[M] (sub-batch atom -> batch atom), new_batch[M] int64 (sub-batch structure of each atom) and
 * counts[2] = (A, M).  Buffers are sized for every structure (n_graphs, n_graphs + 1, N, N); only the first A / A + 1 /
 * M entries are written.  Two launches: one CTA scans, then one warp per active structure fills. */
int dig3d_relax_compact(const int32_t* status, const int32_t* graph_ptr, int64_t n_graphs, int32_t* active,
                        int32_t* new_ptr, int32_t* atom_map, int64_t* new_batch, int32_t* counts, void* stream);

#ifdef __cplusplus
}
#endif
#endif
