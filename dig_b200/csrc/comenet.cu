// ComENet on sm_90a, fp32.
//
//   reference atoms + theta / phi / tau     comenet.py:295-385  (4x scatter_min + ~60 elementwise launches)
//   angle_emb / torsion_emb (gemnet basis)  comenet/features.py:257-348
//   SimpleInteractionBlock.forward          comenet.py:195-215
//   EdgeGraphConv (PyG GraphConv)           comenet.py:130-133
//   GraphNorm                               torch_geometric.nn.GraphNorm, used comenet.py:160,213
//   output head                             comenet.py:394-398
//
// Everything is per edge or per node (no triplets).  Edge kernels own 64 target-sorted edges, node
// kernels 32 nodes; the [E, 256] edge filters and messages of the two convolutions never reach HBM
// (the reference materialises both, 31 MB each per 16 structures).
#include "dense.cuh"
#include "generated/basis_gemnet_2_3.cuh"

namespace dig3d {

constexpr int CH = 256;          // hidden_channels
constexpr int CM = 64;           // middle_channels
constexpr int CTN = 32;          // nodes per CTA
constexpr int CLD = CH + 4;
constexpr int NF1 = 12, NF2 = 6; // num_radial * num_spherical^2, num_radial * num_spherical (nr=3, ns=2)

// ------------------------------------------------------------------ reference atoms
// a0_in/a1_in: nearest / second-nearest IN-edge of each node (scatter_min over the target index);
// a0_out/a1_out: the same over the OUT-edges (scatter_min over the source index).  Ties keep the
// first edge id; nodes without edges get 0 (argmin >= E -> 0, comenet.py:305).
// Reference quirk reproduced (comenet.py:305-308,318-322): the +cutoff penalty of the second pass is written with
// `add[argmin0] = cutoff` AFTER the empty segments were mapped to edge 0, so whenever ANY node of the batch has no
// in-edge (resp. out-edge -- routine under the 32-neighbour cap), edge 0 is penalised too, which can change the
// second-nearest reference atom of dst[0] (resp. src[0]).  PASS 0 finds the nearest edges and raises the two
// batch-wide flags; PASS 1 (a second launch) finds the second-nearest ones.
template <int PASS>
__global__ void comenet_refs_kernel(const float* __restrict__ dist, const int32_t* __restrict__ src,
                                    const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ graph_ptr,
                                    const int64_t* __restrict__ batch, int n_nodes, float cutoff,
                                    int32_t* __restrict__ a0_in, int32_t* __restrict__ a1_in,
                                    int32_t* __restrict__ a0_out, int32_t* __restrict__ a1_out,
                                    int32_t* __restrict__ flags /* [2]: some node has no in-edge / no out-edge */) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_nodes) return;
  const float INF = __int_as_float(0x7f800000);
  {
    const int b = row_ptr[n], e = row_ptr[n + 1];
    if (PASS == 0) {
      int best = -1; float bv = INF;
      for (int k = b; k < e; ++k) { const float d = dist[k]; if (d < bv) { bv = d; best = k; } }
      a0_in[n] = best < 0 ? 0 : best;
      if (best < 0) atomicOr(flags, 1);
    } else {
      const int best = a0_in[n];
      const bool pen0 = flags[0] != 0;
      int sec = -1; float sv = INF;
      for (int k = b; k < e; ++k) {
        const float d = (k == best || (pen0 && k == 0)) ? __fadd_rn(dist[k], cutoff) : dist[k];
        if (d < sv) { sv = d; sec = k; }
      }
      a1_in[n] = sec < 0 ? 0 : sec;
    }
  }
  {
    const int g = (int)batch[n];
    const int lo = graph_ptr[g], hi = graph_ptr[g + 1];
    const int best0 = PASS == 0 ? -1 : a0_out[n];
    const bool pen0 = PASS == 1 && flags[1] != 0;
    int best = -1; float bv = INF;
    for (int i = lo; i < hi; ++i) {
      if (i == n) continue;
      const int ib = row_ptr[i], di = row_ptr[i + 1] - ib;
      int a = 0, b = di;
      while (a < b) { int mid = (a + b) >> 1; if (src[ib + mid] < n) a = mid + 1; else b = mid; }
      if (a < di && src[ib + a] == n) {
        const int e = ib + a;
        const float d = (PASS == 1 && (e == best0 || (pen0 && e == 0))) ? __fadd_rn(dist[e], cutoff) : dist[e];
        if (d < bv) { bv = d; best = e; }
      }
    }
    if (PASS == 0) {
      a0_out[n] = best < 0 ? 0 : best;
      if (best < 0) atomicOr(flags + 1, 1);
    } else {
      a1_out[n] = best < 0 ? 0 : best;
    }
  }
}

// vecs = pos[j] - pos[i] (comenet.py:297), or -- FROM_VEC, the OCP variant with periodic images -- the precomputed
// distance vectors of get_pbc_distances (comenet-ocp.py:352-365), passed in `pos` as [E, 3].
template <bool FROM_VEC = false>
__device__ __forceinline__ f3 edge_vec(const float* __restrict__ pos, const int32_t* __restrict__ src,
                                       const int32_t* __restrict__ dst, int e) {
  if (FROM_VEC) return load3(pos, e);
  return sub3(load3(pos, src[e]), load3(pos, dst[e]));
}
__device__ __forceinline__ f3 neg3(const f3 a) { return {-a.x, -a.y, -a.z}; }
__device__ __forceinline__ float fold_pi(float t) { return t < 0.f ? __fadd_rn(t, 3.14159274101257324f) : t; }

// theta / phi / tau and the two basis features of every edge
template <bool FROM_VEC>
__global__ void comenet_edge_features_kernel(const float* __restrict__ pos, const float* __restrict__ dist,
                                             const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                             const int32_t* __restrict__ a0_in, const int32_t* __restrict__ a1_in,
                                             const int32_t* __restrict__ a0_out, const int32_t* __restrict__ a1_out,
                                             int n_edges, float inv_cutoff, float* __restrict__ f1,
                                             float* __restrict__ f2, float* __restrict__ angles) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const int j = src[e], i = dst[e];
  const int e0i = a0_in[i], e1i = a1_in[i], e0j = a0_out[j], e1j = a1_out[j];
  const int n0 = src[e0i], n0_j = dst[e0j];
  const int idx_iref = (n0 == j) ? e1i : e0i;                            // comenet.py:344-348
  const int idx_jref = (n0_j == i) ? e1j : e0j;                          // comenet.py:350-354
  const f3 pos_ji = edge_vec<FROM_VEC>(pos, src, dst, e);
  const f3 pos_in0 = edge_vec<FROM_VEC>(pos, src, dst, e0i), pos_in1 = edge_vec<FROM_VEC>(pos, src, dst, e1i);
  const f3 pos_iref = edge_vec<FROM_VEC>(pos, src, dst, idx_iref), pos_jref = edge_vec<FROM_VEC>(pos, src, dst, idx_jref);
  const f3 mji = neg3(pos_ji);
  // theta                                                                comenet.py:365-368
  const f3 pl1 = cross_aten(mji, pos_in0);
  const float theta = fold_pi(atan2f(norm3_aten(pl1), sum3_aten(mul3(mji, pos_in0))));
  // phi                                                                  comenet.py:371-377
  const float dist_ji = norm3_aten(pos_ji);
  const f3 pl2 = cross_aten(mji, pos_in1);
  const float phi = fold_pi(atan2f(__fdiv_rn(sum3_aten(mul3(cross_aten(pl1, pl2), pos_ji)), dist_ji),
                                   sum3_aten(mul3(pl1, pl2))));
  // tau                                                                  comenet.py:380-385
  const f3 q1 = cross_aten(pos_ji, pos_jref), q2 = cross_aten(pos_ji, pos_iref);
  const float tau = fold_pi(atan2f(__fdiv_rn(sum3_aten(mul3(cross_aten(q1, q2), pos_ji)), dist_ji),
                                   sum3_aten(mul3(q1, q2))));
  if (angles) { angles[3 * (size_t)e] = theta; angles[3 * (size_t)e + 1] = phi; angles[3 * (size_t)e + 2] = tau; }
  // features                                                             comenet/features.py:289-295,340-348
  const float x = __fmul_rn(dist[e], inv_cutoff);
  float rb[6], y0[2], ylm[4];
  basis_gemnet_2_3::bessel(x, rb);
  basis_gemnet_2_3::yl0(tau, y0);
  basis_gemnet_2_3::ylm(theta, phi, ylm);
#pragma unroll
  for (int l = 0; l < 2; ++l)
#pragma unroll
    for (int r = 0; r < 3; ++r) f2[(size_t)e * NF2 + l * 3 + r] = __fmul_rn(rb[l * 3 + r], y0[l]);
#pragma unroll
  for (int h = 0; h < 4; ++h)
#pragma unroll
    for (int r = 0; r < 3; ++r) f1[(size_t)e * NF1 + h * 3 + r] = __fmul_rn(rb[(h == 0 ? 0 : 1) * 3 + r], ylm[h]);
}

// ------------------------------------------------------------------ OCP variant: arbitrary edge lists, periodic images
// distance_vec = pos[row] - pos[col] + cell_offsets . cell[graph of the edge]      (ocpmodels get_pbc_distances, called
// at comenet-ocp.py:352-359; row = edge_index[0] = source j, col = edge_index[1] = target i)
__global__ void pbc_edge_vectors_kernel(const float* __restrict__ pos, const int64_t* __restrict__ edge_index,
                                        const float* __restrict__ cell, const float* __restrict__ cell_offsets,
                                        const int32_t* __restrict__ edge_graph, int n_edges,
                                        float* __restrict__ vec, float* __restrict__ dist) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const int64_t j = edge_index[e], i = edge_index[(size_t)n_edges + e];
  const float* c = cell + (size_t)edge_graph[e] * 9;
  const float o0 = cell_offsets[3 * (size_t)e], o1 = cell_offsets[3 * (size_t)e + 1], o2 = cell_offsets[3 * (size_t)e + 2];
  f3 v = sub3(load3(pos, (int)j), load3(pos, (int)i));
  // offsets = cell_offsets[1x3] . cell[3x3] (bmm), accumulated over the cell rows in order
  v.x = __fadd_rn(v.x, __fmaf_rn(o2, c[6], __fmaf_rn(o1, c[3], __fmul_rn(o0, c[0]))));
  v.y = __fadd_rn(v.y, __fmaf_rn(o2, c[7], __fmaf_rn(o1, c[4], __fmul_rn(o0, c[1]))));
  v.z = __fadd_rn(v.z, __fmaf_rn(o2, c[8], __fmaf_rn(o1, c[5], __fmul_rn(o0, c[2]))));
  vec[3 * (size_t)e] = v.x; vec[3 * (size_t)e + 1] = v.y; vec[3 * (size_t)e + 2] = v.z;
  dist[e] = norm3_aten(v);
}

// scatter_min + argmin over an UNSORTED index (comenet-ocp.py:374-399) as a 64-bit atomicMin of
// (distance bits << 32 | edge id): distances are positive, so their bit patterns order like the values, and the
// edge id breaks ties towards the first occurrence exactly like torch_scatter's CPU argmin.
// pass 0: nearest edges; pass 1: second nearest (the nearest edge of the node, and edge 0 when some node of the batch
// has no edge -- the reference's `add[argmin0] = cutoff` quirk -- are penalised by +cutoff).
template <int PASS>
__global__ void refs_atomic_edges_kernel(const float* __restrict__ dist, const int64_t* __restrict__ edge_index,
                                         int n_edges, float cutoff, const int32_t* __restrict__ a0_in,
                                         const int32_t* __restrict__ a0_out, const int32_t* __restrict__ flags,
                                         unsigned long long* __restrict__ key_in,
                                         unsigned long long* __restrict__ key_out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const int j = (int)edge_index[e], i = (int)edge_index[(size_t)n_edges + e];
  float di = dist[e], dj = di;
  if (PASS == 1) {
    if (e == a0_in[i] || (flags[0] && e == 0)) di = __fadd_rn(di, cutoff);
    if (e == a0_out[j] || (flags[1] && e == 0)) dj = __fadd_rn(dj, cutoff);
  }
  atomicMin(key_in + i, ((unsigned long long)__float_as_uint(di) << 32) | (unsigned)e);
  atomicMin(key_out + j, ((unsigned long long)__float_as_uint(dj) << 32) | (unsigned)e);
}
template <int PASS>
__global__ void refs_atomic_nodes_kernel(const unsigned long long* __restrict__ key_in,
                                         const unsigned long long* __restrict__ key_out, int n_nodes,
                                         int32_t* __restrict__ a_in, int32_t* __restrict__ a_out,
                                         int32_t* __restrict__ flags) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_nodes) return;
  const unsigned long long ki = key_in[n], ko = key_out[n];
  const bool ei = ki == ~0ull, eo = ko == ~0ull;
  a_in[n] = ei ? 0 : (int)(ki & 0xffffffffull);           // argmin >= E -> 0      comenet-ocp.py:375
  a_out[n] = eo ? 0 : (int)(ko & 0xffffffffull);
  if (PASS == 0) {
    if (ei) atomicOr(flags, 1);
    if (eo) atomicOr(flags + 1, 1);
  }
}

// ------------------------------------------------------------------ node linear: y = act?(x W^T + b)
struct NodeSmem2 {
  float a[CTN * CLD];
  float b[CTN * CLD];
  float ws[2 * CH * LDW];
};

// mode 0: y = swish(x W^T + b)                 (block entry lin, comenet.py:196)
// mode 1: x gathered from an embedding table:  y = swish(emb[z])  handled by comenet_embed_kernel
__global__ void __launch_bounds__(DT, 1)
comenet_node_lin_kernel(const float* __restrict__ x, int n_nodes, const float* __restrict__ w,
                        const float* __restrict__ bias, float* __restrict__ y) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  NodeSmem2& s = *reinterpret_cast<NodeSmem2*>(smem_raw);
  const int n0 = blockIdx.x * CTN, rows = min(CTN, n_nodes - n0);
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  tile_load<CH>(s.a, CLD, x + (size_t)n0 * CH, CH, rows);
  for (int id = threadIdx.x; id < (CTN - rows) * CH; id += DT) s.a[(rows + id / CH) * CLD + id % CH] = 0.f;
  __syncthreads();
  float acc[2][16];
  zero_acc(acc);
  gemm_tile<CTN, CH, CH>(s.a, CLD, w, CH, s.ws, acc);
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int c = tx + 16 * q;
      s.b[(ty * 2 + p) * CLD + c] = swish(acc[p][q] + __ldg(bias + c));
    }
  __syncthreads();
  tile_store<CH>(y + (size_t)n0 * CH, CH, s.b, CLD, rows);
}

__global__ void comenet_embed_kernel(const int64_t* __restrict__ z, const float* __restrict__ emb, int n_nodes,
                                     float* __restrict__ x) {
  const int id = blockIdx.x * blockDim.x + threadIdx.x;   // x = act(emb(z))     comenet.py:125-127
  if (id >= n_nodes * CH) return;
  x[id] = swish(__ldg(emb + (size_t)z[id / CH] * CH + id % CH));
}

// ------------------------------------------------------------------ edge convolutions
// agg_c[i] += sum_{j->i} lin_feature_c(feature_c)[e] * x[j]   for c = 1, 2     comenet.py:198-199,203-204
struct ConvSmem {
  float msg[64 * CLD];
  float mid[64 * (CM + 4)];
  float ws[2 * CH * LDW];
  float feat[64 * NF1];
  int src[64];
  int dst[64];
};

__global__ void __launch_bounds__(DT, 1)
comenet_conv_kernel(const float* __restrict__ x, const float* __restrict__ f1, const float* __restrict__ f2,
                    const int32_t* __restrict__ src, const int32_t* __restrict__ dst, int n_edges,
                    dig3d_comenet_block_weights W, float* __restrict__ agg1, float* __restrict__ agg2) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ConvSmem& s = *reinterpret_cast<ConvSmem*>(smem_raw);
  const int e0 = blockIdx.x * 64, rows = min(64, n_edges - e0);
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  for (int r = threadIdx.x; r < 64; r += DT) {
    s.src[r] = (r < rows) ? src[e0 + r] : -1;
    s.dst[r] = (r < rows) ? dst[e0 + r] : -1;
  }
  for (int c = 0; c < 2; ++c) {
    const int nf = c == 0 ? NF1 : NF2;
    const float* feat = c == 0 ? f1 : f2;
    const float* w1 = c == 0 ? W.w_f1a : W.w_f2a;   // [CM, nf]
    const float* w2 = c == 0 ? W.w_f1b : W.w_f2b;   // [CH, CM]
    __syncthreads();
    for (int id = threadIdx.x; id < 64 * nf; id += DT)
      s.feat[id] = (id / nf < rows) ? __ldg(feat + (size_t)e0 * nf + id) : 0.f;
    __syncthreads();
    for (int id = threadIdx.x; id < 64 * CM; id += DT) {   // lin1: K = nf (12 or 6), no bias
      const int r = id / CM, m = id % CM;
      float a = 0.f;
      for (int k = 0; k < nf; ++k) a = fmaf(s.feat[r * nf + k], __ldg(w1 + m * nf + k), a);
      s.mid[r * (CM + 4) + m] = a;
    }
    __syncthreads();
    float acc[4][16];
    zero_acc(acc);
    gemm_tile<64, CH, CM>(s.mid, CM + 4, w2, CM, s.ws, acc);   // lin2: [64 x 64] x [64 x 256]
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int r = ty * 4 + p;
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        const int col = tx + 16 * q;
        const float xj = (r < rows) ? __ldg(x + (size_t)s.src[r] * CH + col) : 0.f;
        s.msg[r * CLD + col] = __fmul_rn(acc[p][q], xj);        // edge_weight * x_j   comenet.py:133
      }
    }
    __syncthreads();
    tile_segment_accumulate(s.msg, CLD, s.dst, rows, c == 0 ? agg1 : agg2, CH);
  }
}

// ------------------------------------------------------------------ node part of the block
struct NodeSmem4 {
  float xs[CTN * CLD];
  float a1[CTN * CLD];
  float a2[CTN * CLD];
  float t[CTN * CLD];
  float ws[2 * CH * LDW];
};

template <bool ACT>
__device__ __forceinline__ void store_tile(float* dstbuf, const float (&acc)[2][16], const float* __restrict__ bias,
                                           const float* addbuf) {
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int c = tx + 16 * q, r = ty * 2 + p;
      float v = acc[p][q] + (bias ? __ldg(bias + c) : 0.f);
      if (ACT) v = swish(v);
      if (addbuf) v = v + addbuf[r * CLD + c];
      dstbuf[r * CLD + c] = v;
    }
}

// h = lin_cat([act(lin1(conv1)), act(lin2(conv2))]) + x;  h = act(lin(h)) + h (x n_lins)   comenet.py:199-212
__global__ void __launch_bounds__(DT, 1)
comenet_node_block_kernel(const float* __restrict__ x, const float* __restrict__ agg1,
                          const float* __restrict__ agg2, int n_nodes, dig3d_comenet_block_weights W,
                          float* __restrict__ h_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  NodeSmem4& s = *reinterpret_cast<NodeSmem4*>(smem_raw);
  const int n0 = blockIdx.x * CTN, rows = min(CTN, n_nodes - n0);
  tile_load<CH>(s.xs, CLD, x + (size_t)n0 * CH, CH, rows);
  tile_load<CH>(s.a1, CLD, agg1 + (size_t)n0 * CH, CH, rows);
  tile_load<CH>(s.a2, CLD, agg2 + (size_t)n0 * CH, CH, rows);
  for (int id = threadIdx.x; id < (CTN - rows) * CH; id += DT) {
    const int o = (rows + id / CH) * CLD + id % CH;
    s.xs[o] = 0.f; s.a1[o] = 0.f; s.a2[o] = 0.f;
  }
  __syncthreads();
  float acc[2][16];
  // conv1: lin_rel(agg1) + b + lin_root(x)   (PyG GraphConv)
  zero_acc(acc);
  gemm_tile<CTN, CH, CH>(s.a1, CLD, W.w_rel1, CH, s.ws, acc);
  gemm_tile<CTN, CH, CH>(s.xs, CLD, W.w_root1, CH, s.ws, acc);
  store_tile<false>(s.a1, acc, W.b_rel1, nullptr);
  __syncthreads();
  zero_acc(acc);
  gemm_tile<CTN, CH, CH>(s.a1, CLD, W.w_lin1, CH, s.ws, acc);
  store_tile<true>(s.t, acc, W.b_lin1, nullptr);                  // h1
  __syncthreads();
  zero_acc(acc);
  gemm_tile<CTN, CH, CH>(s.a2, CLD, W.w_rel2, CH, s.ws, acc);
  gemm_tile<CTN, CH, CH>(s.xs, CLD, W.w_root2, CH, s.ws, acc);
  store_tile<false>(s.a2, acc, W.b_rel2, nullptr);
  __syncthreads();
  zero_acc(acc);
  gemm_tile<CTN, CH, CH>(s.a2, CLD, W.w_lin2, CH, s.ws, acc);
  store_tile<true>(s.a1, acc, W.b_lin2, nullptr);                 // h2
  __syncthreads();
  // lin_cat(cat[h1, h2]) + x
  zero_acc(acc);
  gemm_tile<CTN, CH, CH>(s.t, CLD, W.w_cat, 2 * CH, s.ws, acc);
  gemm_tile<CTN, CH, CH>(s.a1, CLD, W.w_cat + CH, 2 * CH, s.ws, acc);
  store_tile<false>(s.a2, acc, W.b_cat, s.xs);
  __syncthreads();
  float* cur = s.a2;
  float* nxt = s.t;
  for (int l = 0; l < W.n_lins; ++l) {
    zero_acc(acc);
    gemm_tile<CTN, CH, CH>(cur, CLD, W.w_lins[l], CH, s.ws, acc);
    store_tile<true>(nxt, acc, W.b_lins[l], cur);                 // act(lin(h)) + h
    __syncthreads();
    float* tmp = cur; cur = nxt; nxt = tmp;
  }
  tile_store<CH>(h_out + (size_t)n0 * CH, CH, cur, CLD, rows);
}

// ------------------------------------------------------------------ GraphNorm statistics
// shift[g, c] = mean_g[c] * mean_scale[c];  istd[g, c] = sqrt(mean_g((h - shift)^2) + eps)
__global__ void __launch_bounds__(CH)
comenet_graphnorm_stats_kernel(const float* __restrict__ h, const int32_t* __restrict__ graph_ptr,
                               const float* __restrict__ mean_scale, float eps, float* __restrict__ shift,
                               float* __restrict__ stdv) {
  const int g = blockIdx.x, c = threadIdx.x;
  const int n0 = graph_ptr[g], n1 = graph_ptr[g + 1];
  const float cnt = (float)max(n1 - n0, 1);
  float sum = 0.f;
  for (int n = n0; n < n1; ++n) sum += h[(size_t)n * CH + c];
  const float sh = __fmul_rn(__fdiv_rn(sum, cnt), __ldg(mean_scale + c));
  float sq = 0.f;
  for (int n = n0; n < n1; ++n) { const float o = __fsub_rn(h[(size_t)n * CH + c], sh); sq += __fmul_rn(o, o); }
  shift[(size_t)g * CH + c] = sh;
  stdv[(size_t)g * CH + c] = __fsqrt_rn(__fadd_rn(__fdiv_rn(sq, cnt), eps));
}

// x_next = final( weight * (h - shift) / std + bias )                     comenet.py:213-214
// head (last block only, n_head > 0): x = act(lin(x)) x n_head; out = lin_out(x)   comenet.py:394-396
__global__ void __launch_bounds__(DT, 1)
comenet_norm_final_kernel(const float* __restrict__ h, const int64_t* __restrict__ batch, int n_nodes,
                          const float* __restrict__ shift, const float* __restrict__ stdv,
                          dig3d_comenet_block_weights W, dig3d_comenet_head_weights HW, int out_channels,
                          float* __restrict__ x_next, float* __restrict__ node_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  NodeSmem2& s = *reinterpret_cast<NodeSmem2*>(smem_raw);
  const int n0 = blockIdx.x * CTN, rows = min(CTN, n_nodes - n0);
  for (int id = threadIdx.x; id < CTN * CH; id += DT) {
    const int r = id / CH, c = id % CH;
    float v = 0.f;
    if (r < rows) {
      const int g = (int)batch[n0 + r];
      const float o = __fsub_rn(__ldg(h + (size_t)(n0 + r) * CH + c), __ldg(shift + (size_t)g * CH + c));
      v = __fadd_rn(__fdiv_rn(__fmul_rn(__ldg(W.norm_w + c), o), __ldg(stdv + (size_t)g * CH + c)),
                    __ldg(W.norm_b + c));
    }
    s.a[r * CLD + c] = v;
  }
  __syncthreads();
  float acc[2][16];
  zero_acc(acc);
  gemm_tile<CTN, CH, CH>(s.a, CLD, W.w_final, CH, s.ws, acc);
  store_tile<false>(s.b, acc, W.b_final, nullptr);
  __syncthreads();
  float* cur = s.b;
  float* nxt = s.a;
  if (!node_out) {
    tile_store<CH>(x_next + (size_t)n0 * CH, CH, cur, CLD, rows);
    return;
  }
  for (int l = 0; l < HW.n_lins; ++l) {
    zero_acc(acc);
    gemm_tile<CTN, CH, CH>(cur, CLD, HW.w_lins[l], CH, s.ws, acc);
    store_tile<true>(nxt, acc, HW.b_lins[l], nullptr);
    __syncthreads();
    float* tmp = cur; cur = nxt; nxt = tmp;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = warp; r < rows; r += DT / 32)
    for (int oc = 0; oc < out_channels; ++oc) {
      float part = 0.f;
      for (int c = lane; c < CH; c += 32) part = fmaf(cur[r * CLD + c], __ldg(HW.w_out + (size_t)oc * CH + c), part);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
      if (lane == 0) node_out[(size_t)(n0 + r) * out_channels + oc] = part + __ldg(HW.b_out + oc);
    }
}

template <class K>
static int smem_attr(K kernel, size_t bytes) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(%zu bytes): %s", bytes, cudaGetErrorString(e));
    return DIG3D_ECUDA;
  }
  return DIG3D_OK;
}

// ---------------------------------------------------------------------------------- EdgeGraphConv aggregation
// agg[i][c] = sum_{e = (j -> i)} w[e][c] * x[j][c]       (comenet.py:66-73: message x_j * edge_weight, aggr = 'add')
// for an edge filter that is already materialised: w = lin_feature(feat) comes out of a GEMM on the dense engine as an
// [E, W] matrix; one warp per target node streams its (contiguous, CSR-sorted) rows of w and gathers the source rows of x
// from L2; lanes own float4 columns, the sum stays in registers, one coalesced row store.  No atomics, no zero fill.
template <int W4>
__global__ void __launch_bounds__(256)
edge_weighted_sum_kernel(const float* __restrict__ w, const float* __restrict__ x, const int32_t* __restrict__ src,
                         const int32_t* __restrict__ row_ptr, int n_nodes, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n_nodes) return;
  constexpr int PER = W4 / 32;                      // float4 columns per lane
  float4 acc[PER];
#pragma unroll
  for (int p = 0; p < PER; ++p) acc[p] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
  for (int e = e0; e < e1; ++e) {
    const float4* wr = reinterpret_cast<const float4*>(w + (size_t)e * (W4 * 4));
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)__ldg(src + e) * (W4 * 4));
#pragma unroll
    for (int p = 0; p < PER; ++p) {
      const float4 a = __ldg(wr + lane + 32 * p), b = __ldg(xr + lane + 32 * p);
      acc[p].x = fmaf(a.x, b.x, acc[p].x); acc[p].y = fmaf(a.y, b.y, acc[p].y);
      acc[p].z = fmaf(a.z, b.z, acc[p].z); acc[p].w = fmaf(a.w, b.w, acc[p].w);
    }
  }
  float4* o = reinterpret_cast<float4*>(out + (size_t)i * (W4 * 4));
#pragma unroll
  for (int p = 0; p < PER; ++p) o[lane + 32 * p] = acc[p];
}

// The same aggregation with the edge filter folded in: TwoLayerLinear(bias=False, act=False) is ONE linear map
// W_eff = W2 W1 [W, Q] (comenet.py:87-112 without bias / activation), so
//   agg[i][c] = sum_{e=(j->i)} ( sum_q W_eff[c][q] feat[e][q] ) * x[j][c]
// costs Q + 1 FMAs per edge and channel instead of 64 + 1 and never materialises an [E, W] filter.  weff_t = W_eff^T
// [Q, W] (host side: one tiny GEMM per parameter version).  One warp per (node, 128-channel half): a lane keeps its four
// channels' Q filter coefficients in registers, streams the node's CSR rows of feat (broadcast loads) and gathers x rows.
template <int Q>
__global__ void __launch_bounds__(256)
comenet_filter_sum_kernel(const float* __restrict__ feat, const float* __restrict__ weff_t, const float* __restrict__ x,
                          const int32_t* __restrict__ src, const int32_t* __restrict__ row_ptr, int n_nodes, int width,
                          float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int halves = width / 128;
  const int i = wid / halves, c0 = (wid % halves) * 128 + lane * 4;
  if (i >= n_nodes) return;
  float4 wq[Q];
#pragma unroll
  for (int q = 0; q < Q; ++q) wq[q] = __ldg(reinterpret_cast<const float4*>(weff_t + (size_t)q * width + c0));
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
  for (int e = e0; e < e1; ++e) {
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (size_t)__ldg(src + e) * width + c0));
    const float* f = feat + (size_t)e * Q;
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      const float fq = __ldg(f + q);
      w.x = fmaf(wq[q].x, fq, w.x); w.y = fmaf(wq[q].y, fq, w.y); w.z = fmaf(wq[q].z, fq, w.z); w.w = fmaf(wq[q].w, fq, w.w);
    }
    acc.x = fmaf(w.x, xv.x, acc.x); acc.y = fmaf(w.y, xv.y, acc.y); acc.z = fmaf(w.z, xv.z, acc.z); acc.w = fmaf(w.w, xv.w, acc.w);
  }
  *reinterpret_cast<float4*>(out + (size_t)i * width + c0) = acc;
}

}  // namespace dig3d

using namespace dig3d;

extern "C" {

int dig3d_comenet_geometry(const float* pos, const float* dist, const int32_t* src, const int32_t* dst,
                           const int32_t* row_ptr, const int32_t* graph_ptr, const int64_t* batch,
                           int64_t n_nodes, int64_t n_edges, double cutoff, int32_t* refs /*[4 * N + 2]*/,
                           float* feature1, float* feature2, float* angles, void* stream) {
  DIG3D_REQUIRE(pos && dist && src && dst && row_ptr && graph_ptr && batch && refs && feature1 && feature2,
                "comenet_geometry: null pointer");
  if (n_nodes == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* a0i = refs; int32_t* a1i = refs + n_nodes; int32_t* a0o = refs + 2 * n_nodes; int32_t* a1o = refs + 3 * n_nodes;
  int32_t* flags = refs + 4 * n_nodes;
  cudaMemsetAsync(flags, 0, 2 * sizeof(int32_t), st);
  comenet_refs_kernel<0><<<ceil_div(n_nodes, 128), 128, 0, st>>>(dist, src, row_ptr, graph_ptr, batch, (int)n_nodes,
                                                               (float)cutoff, a0i, a1i, a0o, a1o, flags);
  comenet_refs_kernel<1><<<ceil_div(n_nodes, 128), 128, 0, st>>>(dist, src, row_ptr, graph_ptr, batch, (int)n_nodes,
                                                               (float)cutoff, a0i, a1i, a0o, a1o, flags);
  DIG3D_LAUNCH_CHECK();
  if (n_edges) {
    comenet_edge_features_kernel<false><<<ceil_div(n_edges, 128), 128, 0, st>>>(
        pos, dist, src, dst, a0i, a1i, a0o, a1o, (int)n_edges, 1.0f / (float)cutoff, feature1, feature2, angles);
    DIG3D_LAUNCH_CHECK();
  }
  return DIG3D_OK;
}

int dig3d_pbc_edge_vectors(const float* pos, const int64_t* edge_index, const float* cell, const float* cell_offsets,
                           const int32_t* edge_graph, int64_t n_edges, float* vec, float* dist, void* stream) {
  DIG3D_REQUIRE(pos && edge_index && cell && cell_offsets && edge_graph && vec && dist, "pbc_edge_vectors: null pointer");
  if (n_edges == 0) return DIG3D_OK;
  pbc_edge_vectors_kernel<<<ceil_div(n_edges, 256), 256, 0, (cudaStream_t)stream>>>(
      pos, edge_index, cell, cell_offsets, edge_graph, (int)n_edges, vec, dist);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_comenet_geometry_edges(const float* vec, const float* dist, const int64_t* edge_index, const int32_t* src,
                                 const int32_t* dst, int64_t n_nodes, int64_t n_edges, double cutoff,
                                 int32_t* refs /*[4 * N + 2]*/, unsigned long long* keys /*[2 * N]*/,
                                 float* feature1, float* feature2, float* angles, void* stream) {
  DIG3D_REQUIRE(vec && dist && edge_index && src && dst && refs && keys && feature1 && feature2,
                "comenet_geometry_edges: null pointer");
  if (n_nodes == 0 || n_edges == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* a0i = refs; int32_t* a1i = refs + n_nodes; int32_t* a0o = refs + 2 * n_nodes; int32_t* a1o = refs + 3 * n_nodes;
  int32_t* flags = refs + 4 * n_nodes;
  unsigned long long* ki = keys; unsigned long long* ko = keys + n_nodes;
  const int ge = ceil_div(n_edges, 256), gn = ceil_div(n_nodes, 256);
  cudaMemsetAsync(flags, 0, 2 * sizeof(int32_t), st);
  cudaMemsetAsync(keys, 0xff, 2 * n_nodes * sizeof(unsigned long long), st);
  refs_atomic_edges_kernel<0><<<ge, 256, 0, st>>>(dist, edge_index, (int)n_edges, (float)cutoff, a0i, a0o, flags, ki, ko);
  refs_atomic_nodes_kernel<0><<<gn, 256, 0, st>>>(ki, ko, (int)n_nodes, a0i, a0o, flags);
  cudaMemsetAsync(keys, 0xff, 2 * n_nodes * sizeof(unsigned long long), st);
  refs_atomic_edges_kernel<1><<<ge, 256, 0, st>>>(dist, edge_index, (int)n_edges, (float)cutoff, a0i, a0o, flags, ki, ko);
  refs_atomic_nodes_kernel<1><<<gn, 256, 0, st>>>(ki, ko, (int)n_nodes, a1i, a1o, flags);
  DIG3D_LAUNCH_CHECK();
  comenet_edge_features_kernel<true><<<ceil_div(n_edges, 128), 128, 0, st>>>(
      vec, dist, src, dst, a0i, a1i, a0o, a1o, (int)n_edges, 1.0f / (float)cutoff, feature1, feature2, angles);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_comenet_embed(const int64_t* z, const float* emb, int64_t n_nodes, float* x, void* stream) {
  DIG3D_REQUIRE(z && emb && x, "comenet_embed: null pointer");
  if (n_nodes == 0) return DIG3D_OK;
  comenet_embed_kernel<<<ceil_div(n_nodes * CH, 256), 256, 0, (cudaStream_t)stream>>>(z, emb, (int)n_nodes, x);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_comenet_block(const float* x_in, const float* feature1, const float* feature2, const int32_t* src,
                        const int32_t* dst, const int32_t* graph_ptr, const int64_t* batch, int64_t n_nodes,
                        int64_t n_edges, int64_t n_graphs, const dig3d_comenet_block_weights* w,
                        const dig3d_comenet_head_weights* head, int32_t out_channels, float* xs, float* agg1,
                        float* agg2, float* h, float* stats /*[2, B, 256]*/, float* x_out, float* node_out,
                        void* stream) {
  DIG3D_REQUIRE(x_in && feature1 && feature2 && src && dst && graph_ptr && batch && w && head && xs && agg1 &&
                    agg2 && h && stats, "comenet_block: null pointer");
  DIG3D_REQUIRE(w->n_lins >= 0 && w->n_lins <= 8 && head->n_lins >= 0 && head->n_lins <= 8,
                "comenet_block: n_lins outside [0,8]");
  DIG3D_REQUIRE(!node_out || (head->w_out && head->b_out), "comenet_block: node_out needs the head's lin_out");
  DIG3D_REQUIRE(node_out || x_out, "comenet_block: no output buffer");
  if (n_nodes == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if ((rc = smem_attr(comenet_node_lin_kernel, sizeof(NodeSmem2)))) return rc;
  if ((rc = smem_attr(comenet_conv_kernel, sizeof(ConvSmem)))) return rc;
  if ((rc = smem_attr(comenet_node_block_kernel, sizeof(NodeSmem4)))) return rc;
  if ((rc = smem_attr(comenet_norm_final_kernel, sizeof(NodeSmem2)))) return rc;
  const int ngrid = ceil_div(n_nodes, CTN);
  comenet_node_lin_kernel<<<ngrid, DT, sizeof(NodeSmem2), st>>>(x_in, (int)n_nodes, w->w_lin, w->b_lin, xs);
  DIG3D_LAUNCH_CHECK();
  if (n_edges) {
    comenet_conv_kernel<<<ceil_div(n_edges, 64), DT, sizeof(ConvSmem), st>>>(xs, feature1, feature2, src, dst,
                                                                           (int)n_edges, *w, agg1, agg2);
    DIG3D_LAUNCH_CHECK();
  }
  comenet_node_block_kernel<<<ngrid, DT, sizeof(NodeSmem4), st>>>(xs, agg1, agg2, (int)n_nodes, *w, h);
  DIG3D_LAUNCH_CHECK();
  float* shift = stats;
  float* stdv = stats + n_graphs * CH;
  comenet_graphnorm_stats_kernel<<<(int)n_graphs, CH, 0, st>>>(h, graph_ptr, w->norm_ms, 1e-5f, shift, stdv);
  DIG3D_LAUNCH_CHECK();
  comenet_norm_final_kernel<<<ngrid, DT, sizeof(NodeSmem2), st>>>(h, batch, (int)n_nodes, shift, stdv, *w, *head,
                                                                out_channels, x_out, node_out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_edge_weighted_sum(const float* w, const float* x, const int32_t* src, const int32_t* row_ptr, int64_t n_nodes,
                            int32_t width, float* out, void* stream) {
  DIG3D_REQUIRE(w && x && src && row_ptr && out, "edge_weighted_sum: null pointer");
  DIG3D_REQUIRE(width == 128 || width == 256, "edge_weighted_sum: width %d is not compiled (128, 256)", width);
  DIG3D_REQUIRE((((uintptr_t)w | (uintptr_t)x | (uintptr_t)out) & 15) == 0, "edge_weighted_sum: 16-byte alignment");
  if (n_nodes == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ceil_div(n_nodes * 32, 256);
  if (width == 256) edge_weighted_sum_kernel<64><<<grid, 256, 0, st>>>(w, x, src, row_ptr, (int)n_nodes, out);
  else edge_weighted_sum_kernel<32><<<grid, 256, 0, st>>>(w, x, src, row_ptr, (int)n_nodes, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_comenet_filter_sum(const float* feat, int32_t q, const float* weff_t, const float* x, const int32_t* src,
                             const int32_t* row_ptr, int64_t n_nodes, int32_t width, float* out, void* stream) {
  DIG3D_REQUIRE(feat && weff_t && x && src && row_ptr && out, "comenet_filter_sum: null pointer");
  DIG3D_REQUIRE(width % 128 == 0 && width >= 128 && width <= 1024, "comenet_filter_sum: width %d must be a multiple of 128", width);
  DIG3D_REQUIRE(q == 12 || q == 6, "comenet_filter_sum: feature width %d is not compiled (12 = num_radial*num_spherical^2, 6)", q);
  DIG3D_REQUIRE((((uintptr_t)weff_t | (uintptr_t)x | (uintptr_t)out) & 15) == 0, "comenet_filter_sum: 16-byte alignment");
  if (n_nodes == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ceil_div(n_nodes * (width / 128) * 32, 256);
  if (q == 12) comenet_filter_sum_kernel<12><<<grid, 256, 0, st>>>(feat, weff_t, x, src, row_ptr, (int)n_nodes, width, out);
  else comenet_filter_sum_kernel<6><<<grid, 256, 0, st>>>(feat, weff_t, x, src, row_ptr, (int)n_nodes, width, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
