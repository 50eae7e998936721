// Graph construction + geometry for the 3D-graph path (sm_90a).
//
//   radius_graph                 reference call sites schnet.py:156, dimenetpp.py:277,
//                                spherenet.py:304, comenet.py:294 (torch_cluster 1.6.0 CUDA semantics)
//   triplet enumeration          utils/geometric_computing.py:27-41 (SparseTensor row-select)
//   dist / angle / torsion       utils/geometric_computing.py:25,43-75
//
// Data layout: in-neighbour lists are built once into nbr[N][cap]; edges are the CSR over
// TARGET nodes (row_ptr), so edge e = row_ptr[i] + s is (source nbr[i][s] -> target i) and the
// edge list is sorted by (i, j) exactly like the reference's edge_index.  Triplets of edge
// e = (j->i) are the in-edges (k->j) of j with k != i, in ascending k: they are implicit in the
// CSR and only their start offset trip_ptr[e] is stored.
#include <stdarg.h>
#include "common.cuh"

namespace dig3d {

constexpr int GEO_MAXDEG = 64;  // the capped builder's cap, and the in-degree the warp-per-edge geometry kernel handles

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// ------------------------------------------------------------------ graph_ptr
__global__ void graph_ptr_kernel(const int64_t* __restrict__ batch, int n_nodes, int n_graphs,
                                 int32_t* __restrict__ ptr) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n > n_nodes) return;
  // node n opens every graph in (batch[n-1], batch[n]]; n == n_nodes closes the tail.
  int64_t prev = (n == 0) ? -1 : batch[n - 1];
  int64_t cur = (n == n_nodes) ? (int64_t)n_graphs : batch[n];
  for (int64_t g = prev < -1 ? 0 : prev + 1; g <= cur && g <= n_graphs; ++g) ptr[g] = n;   // invalid ids: see validate_nodes
}

// ------------------------------------------------------------------ radius neighbours
// One thread per query node, ascending scan of the nodes of its own graph, like
// torch_cluster's radius_kernel: d2 accumulated as fma(diff, diff, d2), strict '<', at most
// `cap` hits counted INCLUDING the query itself, which is then dropped.
__global__ void radius_neighbors_kernel(const float* __restrict__ pos, const int64_t* __restrict__ batch,
                                        const int32_t* __restrict__ ptr, int n_nodes, int n_graphs, float r2, int cap,
                                        int32_t* __restrict__ nbr, int32_t* __restrict__ deg) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_nodes) return;
  const int64_t gb = batch[n];
  if (gb < 0 || gb >= n_graphs) { deg[n] = 0; return; }   // reported by validate_nodes_kernel; never index ptr[] with it
  int g = (int)gb;
  int lo = ptr[g], hi = ptr[g + 1];
  f3 q = load3(pos, n);
  int hits = 0, m = 0;
  int32_t* out = nbr + (size_t)n * cap;
  for (int c = lo; c < hi; ++c) {
    f3 p = load3(pos, c);
    float dx = __fsub_rn(p.x, q.x), dy = __fsub_rn(p.y, q.y), dz = __fsub_rn(p.z, q.z);
    float d2 = __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
    if (d2 < r2) {
      if (c != n) out[m++] = c;
      if (++hits >= cap) break;
    }
  }
  deg[n] = m;
}

// Index validation (the reference's nn.Embedding / scatter raise a device-side assert for these): bit 0 = a batch
// id outside [0, n_graphs), bit 1 = batch not sorted ascending, bit 2 = an atomic number outside [0, z_rows).
__global__ void validate_nodes_kernel(const int64_t* __restrict__ batch, const int64_t* __restrict__ z, int n_nodes,
                                      int n_graphs, int z_rows, int32_t* __restrict__ flags) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_nodes) return;
  int bad = 0;
  const int64_t b = batch[n];
  if (b < 0 || b >= n_graphs) bad |= 1;
  if (n > 0 && batch[n - 1] > b) bad |= 2;
  if (z) { const int64_t zz = z[n]; if (zz < 0 || zz >= z_rows) bad |= 4; }
  if (bad) atomicOr(flags, bad);
}

// Two nearest neighbours of every node inside its graph, torch_cluster.knn (CUDA) semantics as used by
// knn_graph(pos, 1 / 2, batch) at ggraph3D/.../geometric_computing.py:14,16: candidates scanned in ascending index,
// squared distance accumulated as fma(diff, diff, acc), the three best kept by strict-`>` insertion (self included,
// ties keep the lower index in front), then self is dropped.  nn1 / nn2 = -1 where the graph is too small.
__global__ void knn2_kernel(const float* __restrict__ pos, const int64_t* __restrict__ batch,
                            const int32_t* __restrict__ ptr, int n_nodes, int n_graphs,
                            int32_t* __restrict__ nn1, int32_t* __restrict__ nn2) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_nodes) return;
  const int64_t gb = batch[n];
  if (gb < 0 || gb >= n_graphs) { nn1[n] = nn2[n] = -1; return; }
  const int lo = ptr[gb], hi = ptr[gb + 1];
  const f3 q = load3(pos, n);
  const float INF = __int_as_float(0x7f800000);
  float bd[3] = {INF, INF, INF};
  int bi[3] = {-1, -1, -1};
  for (int c = lo; c < hi; ++c) {
    const f3 p = load3(pos, c);
    const float dx = __fsub_rn(p.x, q.x), dy = __fsub_rn(p.y, q.y), dz = __fsub_rn(p.z, q.z);
    const float d2 = __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      if (bd[e] > d2) {
#pragma unroll
        for (int m = 2; m > e; --m) { bd[m] = bd[m - 1]; bi[m] = bi[m - 1]; }
        bd[e] = d2; bi[e] = c;
        break;
      }
    }
  }
  int out[2] = {-1, -1}, k = 0;
#pragma unroll
  for (int e = 0; e < 3; ++e)
    if (bi[e] >= 0 && bi[e] != n && k < 2) out[k++] = bi[e];
  nn1[n] = out[0];
  nn2[n] = out[1];
}

__device__ __forceinline__ int find_sorted(const int32_t* __restrict__ list, int len, int key) {
  // position of key in ascending list, or -1
  int lo = 0, hi = len;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    int v = list[mid];
    if (v < key) lo = mid + 1; else hi = mid;
  }
  return (lo < len && list[lo] == key) ? lo : -1;
}

// ------------------------------------------------------------------ triplet count per node
// One WARP per node, lane = in-neighbour slot: the per-neighbour binary searches (six dependent L2 round trips each) run
// side by side instead of one after the other in a single thread (round 1: one thread per node, 23 us at 2 304 nodes --
// pure latency).
__global__ void triplet_count_kernel(const int32_t* __restrict__ nbr, const int32_t* __restrict__ deg,
                                     int n_nodes, int cap, int32_t* __restrict__ tcnt, int32_t* __restrict__ out_cnt) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n_nodes) return;
  const int d = deg[i];
  int cnt = 0;
  for (int s = lane; s < d; s += 32) {
    const int j = nbr[(size_t)i * cap + s];
    const int dj = deg[j];
    cnt += dj - (find_sorted(nbr + (size_t)j * cap, dj, i) >= 0 ? 1 : 0);
    if (out_cnt) atomicAdd(out_cnt + j, 1);           // out-degree of the source (zero-initialised by the caller)
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) tcnt[i] = cnt;
}

// ------------------------------------------------------------------ single-CTA dual exclusive scan
__global__ void __launch_bounds__(1024) scan_counts_kernel(const int32_t* __restrict__ a,
                                                          const int32_t* __restrict__ b,
                                                          const int32_t* __restrict__ c3, int n,
                                                          int32_t* __restrict__ pa, int32_t* __restrict__ pb,
                                                          int32_t* __restrict__ pc, int32_t* __restrict__ totals) {
  __shared__ int3 warp_tot[32];
  __shared__ int3 carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) carry = make_int3(0, 0, 0);
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    int idx = base + tid;
    int3 v = (idx < n) ? make_int3(a[idx], b[idx], c3 ? c3[idx] : 0) : make_int3(0, 0, 0);
    int3 s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int tx = __shfl_up_sync(0xffffffffu, s.x, o), ty = __shfl_up_sync(0xffffffffu, s.y, o),
          tz = __shfl_up_sync(0xffffffffu, s.z, o);
      if (lane >= o) { s.x += tx; s.y += ty; s.z += tz; }
    }
    if (lane == 31) warp_tot[wid] = s;
    __syncthreads();
    if (wid == 0) {
      int3 w = warp_tot[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int tx = __shfl_up_sync(0xffffffffu, w.x, o), ty = __shfl_up_sync(0xffffffffu, w.y, o),
            tz = __shfl_up_sync(0xffffffffu, w.z, o);
        if (lane >= o) { w.x += tx; w.y += ty; w.z += tz; }
      }
      warp_tot[lane] = w;
    }
    __syncthreads();
    int3 c = carry;
    int3 wofs = (wid == 0) ? make_int3(0, 0, 0) : warp_tot[wid - 1];
    if (idx < n) {
      pa[idx] = c.x + wofs.x + s.x - v.x;
      pb[idx] = c.y + wofs.y + s.y - v.y;
      if (pc) pc[idx] = c.z + wofs.z + s.z - v.z;
    }
    __syncthreads();
    if (tid == 0) { carry.x = c.x + warp_tot[31].x; carry.y = c.y + warp_tot[31].y; carry.z = c.z + warp_tot[31].z; }
    __syncthreads();
  }
  if (tid == 0) {
    pa[n] = carry.x; pb[n] = carry.y;
    if (pc) pc[n] = carry.z;
    totals[0] = carry.x; totals[1] = carry.y;
  }
}

// ------------------------------------------------------------------ edge fill
// One WARP per target node, lane = in-neighbour slot (round 1: one thread per node walking its <= 33 edges, 28 us of
// dependent loads).  The triplet offsets of the node's edges are a warp prefix sum of the per-edge counts.
__global__ void edge_fill_kernel(const float* __restrict__ pos, const int32_t* __restrict__ nbr,
                                 const int32_t* __restrict__ deg, const int32_t* __restrict__ row_ptr,
                                 const int32_t* __restrict__ node_trip_ptr, int n_nodes, int cap,
                                 int64_t n_edges, int64_t* __restrict__ edge_index, int32_t* __restrict__ src,
                                 int32_t* __restrict__ dst, float* __restrict__ dist, float* __restrict__ vec,
                                 int32_t* __restrict__ trip_ptr, const int32_t* __restrict__ graph_ptr,
                                 const int64_t* __restrict__ batch, const int32_t* __restrict__ out_ptr,
                                 int32_t* __restrict__ out_list, int32_t* __restrict__ pos_in) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n_nodes) return;
  if (out_list) {
    // Node i as a SOURCE: its out-edges (i -> c), c ascending over the nodes of its graph, with the position of c
    // among i's own in-neighbours (deg[i] if absent).  The triplet kernels used to rediscover this list -- one binary
    // search per candidate node -- once per in-edge (projection) and once per layer (gather).
    const int g = (int)batch[i];
    const int lo = graph_ptr[g], hi = graph_ptr[g + 1], di = deg[i];
    int w = out_ptr[i];
    for (int c0 = lo; c0 < hi; c0 += 32) {
      const int c = c0 + lane;
      int e = -1, p = 0;
      if (c < hi && c != i) {
        const int dc = deg[c];
        const int q = find_sorted(nbr + (size_t)c * cap, dc, i);       // slot of i among c's in-neighbours
        if (q >= 0) {
          e = row_ptr[c] + q;
          const int r = find_sorted(nbr + (size_t)i * cap, di, c);
          p = r >= 0 ? r : di;
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, e >= 0);
      if (e >= 0) {
        out_list[w + __popc(m & ((1u << lane) - 1))] = e;
        pos_in[e] = p;
      }
      w += __popc(m);
    }
  }
  const int d = deg[i], e0 = row_ptr[i];
  int t = node_trip_ptr[i];
  const f3 pi = load3(pos, i);
  for (int s0 = 0; s0 < d; s0 += 32) {
    const int s = s0 + lane;
    int c = 0;
    if (s < d) {
      const int j = nbr[(size_t)i * cap + s];
      const int e = e0 + s;
      src[e] = j; dst[e] = i;
      if (edge_index) { edge_index[e] = j; edge_index[n_edges + e] = i; }
      const f3 pj = load3(pos, j);
      // (pos[i]-pos[j]).pow(2).sum(-1).sqrt()   geometric_computing.py:25
      dist[e] = norm3_aten(sub3(pi, pj));
      if (vec) {  // vecs = pos[j] - pos[i]       comenet.py:297
        const f3 v = sub3(pj, pi);
        vec[3 * (size_t)e] = v.x; vec[3 * (size_t)e + 1] = v.y; vec[3 * (size_t)e + 2] = v.z;
      }
      const int dj = deg[j];
      c = dj - (find_sorted(nbr + (size_t)j * cap, dj, i) >= 0 ? 1 : 0);
    }
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    if (s < d) trip_ptr[e0 + s] = t + incl - c;
    t += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (i == n_nodes - 1 && lane == 0) trip_ptr[n_edges] = t;
}

// ------------------------------------------------------------------ CSR from a caller-supplied edge_index
// xyz_to_dat(pos, edge_index, ...) (utils/geometric_computing.py:12) takes any edge list; the kernels need
// it sorted by (target, source) -- what radius_graph produces.  flag[0] |= 1 if it is not.
__global__ void edges_prepare_kernel(const int64_t* __restrict__ edge_index, int64_t n_edges, int n_nodes,
                                     int32_t* __restrict__ src, int32_t* __restrict__ dst,
                                     int32_t* __restrict__ flag) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const int64_t j = edge_index[e], i = edge_index[n_edges + e];
  src[e] = (int32_t)j; dst[e] = (int32_t)i;
  bool bad = j < 0 || i < 0 || j >= n_nodes || i >= n_nodes;
  if (e > 0) {
    const int64_t pj = edge_index[e - 1], pi = edge_index[n_edges + e - 1];
    bad |= (pi > i) || (pi == i && pj >= j);
  }
  if (bad) atomicOr(flag, 1);
}

__global__ void csr_from_sorted_kernel(const int32_t* __restrict__ dst, int n_edges, int n_nodes,
                                       int32_t* __restrict__ row_ptr) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n > n_nodes) return;
  int lo = 0, hi = n_edges;                   // first edge with dst >= n
  while (lo < hi) { int mid = (lo + hi) >> 1; if (dst[mid] < n) lo = mid + 1; else hi = mid; }
  row_ptr[n] = lo;
}

// cnt[e] = triplets of edge e = (j -> i), dist[e]; flag[1] += edges whose source has more than max_deg in-edges (the
// heavy edges, only they pay an atomic), *t64 += the triplet total in 64 bits (one atomic per CTA): the int32 scan of
// cnt wraps at 2^31.
constexpr int COUNT_THREADS = 256;

__global__ void __launch_bounds__(COUNT_THREADS)
edge_triplet_count_kernel(const float* __restrict__ pos, const int32_t* __restrict__ src,
                          const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr, int n_edges,
                          int max_deg, int32_t* __restrict__ cnt, float* __restrict__ dist,
                          int32_t* __restrict__ flag, unsigned long long* __restrict__ t64) {
  __shared__ unsigned long long warp_sum[COUNT_THREADS / 32];
  const int e = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned long long c64 = 0;
  if (e < n_edges) {
    const int j = src[e], i = dst[e];
    const int b = row_ptr[j], d = row_ptr[j + 1] - b;
    if (d > max_deg) atomicAdd(flag + 1, 1);
    const int c = d - (find_sorted(src + b, d, i) >= 0 ? 1 : 0);
    cnt[e] = c;
    c64 = (unsigned long long)c;
    dist[e] = norm3_aten(sub3(load3(pos, i), load3(pos, j)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c64 += __shfl_xor_sync(0xffffffffu, c64, o);
  if (lane == 0) warp_sum[w] = c64;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long tot = 0;
#pragma unroll
    for (int k = 0; k < COUNT_THREADS / 32; ++k) tot += warp_sum[k];
    if (tot) atomicAdd(t64, tot);
  }
}

// ------------------------------------------------------------------ triplet geometry
// plane_s = cross(pos_ji, pos_k - pos_j) is both the angle's cross product and the torsion's plane1 / plane2, so it is
// computed once per in-edge s of j.  The per-triplet arithmetic lives in the two device functions below, which both
// geometry kernels call: whatever the in-degree, a triplet gets the same op sequence.

// One torsion candidate k_n of the triplet with plane p1: atan2(((p1 x p2) . ji) / |ji|, p1 . p2), <= 0 -> +2pi
//                                                              geometric_computing.py:53-75
__device__ __forceinline__ float torsion_candidate(const f3 p1, const f3 p2, const f3 pos_ji, const float dist_ji) {
  const float ta = sum3_aten(mul3(p1, p2));
  const float tb = __fdiv_rn(sum3_aten(mul3(cross_aten(p1, p2), pos_ji)), dist_ji);
  float tor = atan2f(tb, ta);
  if (tor <= 0.0f) tor = __fadd_rn(tor, 6.2831855f);
  return tor;
}

// best folded with fminf over the candidates planes[c], c in [0, n), c != skip (the slot of i).  fminf is exact and
// order-independent, so a min folded tile by tile equals the min over all candidates at once.
__device__ __forceinline__ float torsion_min_fold(float best, const f3 p1, const float (*planes)[3], int n, int skip,
                                                  const f3 pos_ji, const float dist_ji) {
  for (int c = 0; c < n; ++c) {
    if (c == skip) continue;
    const f3 p2 = {planes[c][0], planes[c][1], planes[c][2]};
    best = fminf(best, torsion_candidate(p1, p2, pos_ji, dist_ji));
  }
  return best;
}

// The same fold, also recording the slot of the winner: strict `<` in ascending slot order keeps the first slot among
// exactly equal minima (torch_scatter's CPU scatter_min arg rule); a tile folded after an earlier one passes slot0, its
// first slot.  The kept value is the one fminf would keep: candidates are NaN or in (0, 2 pi], and fminf skips NaN too.
__device__ __forceinline__ float torsion_min_fold_arg(float best, int& arg, const f3 p1, const float (*planes)[3],
                                                      int n, int skip, const f3 pos_ji, const float dist_ji,
                                                      int slot0) {
  for (int c = 0; c < n; ++c) {
    if (c == skip) continue;
    const f3 p2 = {planes[c][0], planes[c][1], planes[c][2]};
    const float tor = torsion_candidate(p1, p2, pos_ji, dist_ji);
    if (tor < best) { best = tor; arg = slot0 + c; }
  }
  return best;
}

// Outputs of triplet t = (k -> j -> i) with k the in-edge kj of j and plane p1: the angle, the indices and the torsion
// (use_torsion 1: `tor_min`, the min over all candidates folded by the caller; 2: G-SphereNet's single reference atom).
__device__ __forceinline__ void triplet_emit(const float* __restrict__ pos, const f3 pj, const f3 pos_ji,
                                             const float dist_ji, int k, const f3 p1, int t, int kj, int e, int j,
                                             int i, int use_torsion, float tor_min, float* __restrict__ angle,
                                             float* __restrict__ torsion, int32_t* __restrict__ idx_kj,
                                             int32_t* __restrict__ idx_ji, int64_t* __restrict__ idx_kj64,
                                             int64_t* __restrict__ idx_ji64, const int32_t* __restrict__ nn1,
                                             const int32_t* __restrict__ nn2) {
  // angle = atan2(|ji x jk|, ji . jk)       geometric_computing.py:44-48
  const f3 pos_jk = sub3(load3(pos, k), pj);
  const float a = sum3_aten(mul3(pos_ji, pos_jk));
  const float b = norm3_aten(p1);
  angle[t] = atan2f(b, a);
  if (idx_kj) idx_kj[t] = kj;
  if (idx_ji) idx_ji[t] = e;
  if (idx_kj64) idx_kj64[t] = kj;
  if (idx_ji64) idx_ji64[t] = e;
  if (use_torsion == 2) {
    // G-SphereNet's variant (ggraph3D/.../geometric_computing.py:87-103): ONE reference atom, the nearest
    // neighbour of j in its graph, or the second nearest when the nearest is i
    const int k_n = (nn1[j] == i) ? nn2[j] : nn1[j];
    const f3 p2 = cross_aten(pos_ji, sub3(load3(pos, k_n), pj));
    torsion[t] = torsion_candidate(p1, p2, pos_ji, dist_ji);
  } else if (use_torsion) {
    torsion[t] = tor_min;
  }
}

// One warp per edge e = (j -> i) whose source j has at most max_deg <= GEO_MAXDEG in-edges (heavier edges are left to
// triplet_geometry_heavy_kernel).  Lane s owns in-edge s of j (k = src[row_ptr[j]+s]), parks its plane in shared
// memory and every lane then scans all candidates k_n.
// ARG (use_torsion 1 only): also write tors_arg[t], the slot of the winning candidate among j's in-edges (-1 when no
// candidate is finite).  tors_arg is the last parameter, so the ARG = false instantiations keep their parameter layout.
constexpr int GEO_WARPS = 8;

template <bool ARG = false>
__global__ void __launch_bounds__(GEO_WARPS * 32)
triplet_geometry_kernel(const float* __restrict__ pos, const int32_t* __restrict__ src,
                        const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                        const int32_t* __restrict__ trip_ptr, int n_edges, int max_deg, int use_torsion,
                        float* __restrict__ angle, float* __restrict__ torsion, int32_t* __restrict__ idx_kj,
                        int32_t* __restrict__ idx_ji, int64_t* __restrict__ idx_kj64,
                        int64_t* __restrict__ idx_ji64, const int32_t* __restrict__ nn1 = nullptr,
                        const int32_t* __restrict__ nn2 = nullptr, int32_t* __restrict__ tors_arg = nullptr) {
  __shared__ float planes[GEO_WARPS][GEO_MAXDEG][3];
  __shared__ int32_t ks[GEO_WARPS][GEO_MAXDEG];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int e = blockIdx.x * GEO_WARPS + w;
  if (e >= n_edges) return;
  const int j = src[e], i = dst[e];
  const int base = row_ptr[j], d = row_ptr[j + 1] - base;
  if (d > max_deg) return;
  const f3 pj = load3(pos, j);
  const f3 pos_ji = sub3(load3(pos, i), pj);
  const float dist_ji = norm3_aten(pos_ji);
  // pass 1: planes
  for (int s = lane; s < d; s += 32) {
    int k = src[base + s];
    ks[w][s] = k;
    f3 pl = cross_aten(pos_ji, sub3(load3(pos, k), pj));
    planes[w][s][0] = pl.x; planes[w][s][1] = pl.y; planes[w][s][2] = pl.z;
  }
  __syncwarp();
  // position of i among j's in-neighbours (or d if absent): triplet slot s maps to
  // t = trip_ptr[e] + s - (s > p_i)
  int p_i = d;
  for (int s = 0; s < d; ++s) if (ks[w][s] == i) p_i = s;
  const int t0 = trip_ptr[e];
  for (int s = lane; s < d; s += 32) {
    if (s == p_i) continue;
    const f3 p1 = {planes[w][s][0], planes[w][s][1], planes[w][s][2]};
    float best = __int_as_float(0x7f800000);
    if constexpr (ARG) {
      int arg = -1;
      best = torsion_min_fold_arg(best, arg, p1, planes[w], d, p_i, pos_ji, dist_ji, 0);
      tors_arg[t0 + s - (s > p_i ? 1 : 0)] = arg;
    } else {
      if (use_torsion == 1) best = torsion_min_fold(best, p1, planes[w], d, p_i, pos_ji, dist_ji);
    }
    triplet_emit(pos, pj, pos_ji, dist_ji, ks[w][s], p1, t0 + s - (s > p_i ? 1 : 0), base + s, e, j, i, use_torsion,
                 best, angle, torsion, idx_kj, idx_ji, idx_kj64, idx_ji64, nn1, nn2);
  }
}

// One CTA per heavy edge e = (j -> i) (heavy[h], or h itself when heavy is null), any in-degree d of j.  Thread x owns
// the triplet slots s = x, x + HEAVY_THREADS, ...; for the full-candidate torsion the CTA walks j's in-edges in tiles
// of HEAVY_THREADS planes parked in shared memory and every thread folds its min across the tiles.  Shared memory stays
// at one tile whatever d is; the planes of a tile are recomputed once per slot pass (d / HEAVY_THREADS passes), which
// is small next to the d^2 torsion candidates per edge.
constexpr int HEAVY_THREADS = 128;

template <bool ARG = false>
__global__ void __launch_bounds__(HEAVY_THREADS)
triplet_geometry_heavy_kernel(const float* __restrict__ pos, const int32_t* __restrict__ src,
                              const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                              const int32_t* __restrict__ trip_ptr, const int32_t* __restrict__ heavy,
                              int use_torsion, float* __restrict__ angle, float* __restrict__ torsion,
                              int64_t* __restrict__ idx_kj64, int64_t* __restrict__ idx_ji64,
                              const int32_t* __restrict__ nn1, const int32_t* __restrict__ nn2,
                              int32_t* __restrict__ tors_arg = nullptr) {
  __shared__ float planes[HEAVY_THREADS][3];
  const int x = threadIdx.x;
  const int e = heavy ? heavy[blockIdx.x] : (int)blockIdx.x;
  const int j = src[e], i = dst[e];
  const int base = row_ptr[j], d = row_ptr[j + 1] - base;
  const f3 pj = load3(pos, j);
  const f3 pos_ji = sub3(load3(pos, i), pj);
  const float dist_ji = norm3_aten(pos_ji);
  int p_i = find_sorted(src + base, d, i);                 // j's in-neighbours ascend: the edges are sorted
  if (p_i < 0) p_i = d;
  const int t0 = trip_ptr[e];
  for (int s0 = 0; s0 < d; s0 += HEAVY_THREADS) {           // uniform across the CTA: every thread reaches the barriers
    const int s = s0 + x;
    int k = 0;
    f3 p1 = {0.f, 0.f, 0.f};
    if (s < d) {
      k = src[base + s];
      p1 = cross_aten(pos_ji, sub3(load3(pos, k), pj));
    }
    float best = __int_as_float(0x7f800000);
    int arg = -1;
    if (use_torsion == 1) {
      for (int c0 = 0; c0 < d; c0 += HEAVY_THREADS) {
        __syncthreads();                                    // the previous tile has been read
        const int c = c0 + x;
        if (c < d) {
          const f3 pl = cross_aten(pos_ji, sub3(load3(pos, src[base + c]), pj));
          planes[x][0] = pl.x; planes[x][1] = pl.y; planes[x][2] = pl.z;
        }
        __syncthreads();
        if (s < d && s != p_i) {
          if constexpr (ARG)
            best = torsion_min_fold_arg(best, arg, p1, planes, min(HEAVY_THREADS, d - c0), p_i - c0, pos_ji, dist_ji,
                                        c0);
          else
            best = torsion_min_fold(best, p1, planes, min(HEAVY_THREADS, d - c0), p_i - c0, pos_ji, dist_ji);
        }
      }
    }
    if constexpr (ARG)
      if (s < d && s != p_i) tors_arg[t0 + s - (s > p_i ? 1 : 0)] = arg;
    if (s < d && s != p_i)
      triplet_emit(pos, pj, pos_ji, dist_ji, k, p1, t0 + s - (s > p_i ? 1 : 0), base + s, e, j, i, use_torsion, best,
                   angle, torsion, nullptr, nullptr, idx_kj64, idx_ji64, nn1, nn2);
  }
}

// heavy[1 + h] = the edges whose source has more than max_deg in-edges (any order), heavy[0] = their number
// (zeroed by the dispatcher).  One atomic per warp that has a heavy edge.
__global__ void heavy_edges_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ row_ptr, int n_edges,
                                   int max_deg, int32_t* __restrict__ heavy) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
  bool h = false;
  if (e < n_edges) {
    const int j = src[e];
    h = row_ptr[j + 1] - row_ptr[j] > max_deg;
  }
  const unsigned m = __ballot_sync(0xffffffffu, h);
  if (!m) return;
  int base = 0;
  if (lane == 0) base = atomicAdd(heavy, __popc(m));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (h) heavy[1 + base + __popc(m & ((1u << lane) - 1))] = e;
}

// ------------------------------------------------------------------ segment sum (sorted index as CSR)
// out[s, c] = sum_{r in [ptr[s], ptr[s+1])} x[r, c]; one warp per (segment, 128-column strip),
// float4 lanes, rows added in ascending order (deterministic).
__global__ void segment_sum_kernel(const float* __restrict__ x, const int32_t* __restrict__ ptr,
                                   int n_segments, int width, float* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int strips = (width + 127) / 128;
  const int s = warp / strips, strip = warp % strips;
  if (s >= n_segments) return;
  const int r0 = ptr[s], r1 = ptr[s + 1];
  const int c = strip * 128 + lane * 4;
  if ((width & 3) == 0) {
    if (c >= width) return;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int r = r0;
    for (; r + 1 < r1; r += 2) {  // two independent loads in flight
      float4 v0 = __ldg(reinterpret_cast<const float4*>(x + (size_t)r * width + c));
      float4 v1 = __ldg(reinterpret_cast<const float4*>(x + (size_t)(r + 1) * width + c));
      acc.x += v0.x; acc.y += v0.y; acc.z += v0.z; acc.w += v0.w;
      acc.x += v1.x; acc.y += v1.y; acc.z += v1.z; acc.w += v1.w;
    }
    if (r < r1) {
      float4 v0 = __ldg(reinterpret_cast<const float4*>(x + (size_t)r * width + c));
      acc.x += v0.x; acc.y += v0.y; acc.z += v0.z; acc.w += v0.w;
    }
    *reinterpret_cast<float4*>(out + (size_t)s * width + c) = acc;
  } else {
    for (int cc = strip * 128 + lane; cc < min(width, strip * 128 + 128); cc += 32) {
      float acc = 0.f;
      for (int r = r0; r < r1; ++r) acc += __ldg(x + (size_t)r * width + cc);
      out[(size_t)s * width + cc] = acc;
    }
  }
}

// u[g, c] = sum_l sum_{n in graph g} v[l, n, c]   (small: one warp per (g, c))
__global__ void graph_readout_kernel(const float* __restrict__ v, const int32_t* __restrict__ gptr,
                                     int n_graphs, int n_nodes, int n_blocks, int channels,
                                     float* __restrict__ u) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_graphs * channels) return;
  const int g = warp / channels, c = warp % channels;
  const int n0 = gptr[g], n1 = gptr[g + 1];
  float total = 0.f;
  for (int l = 0; l < n_blocks; ++l) {  // u += scatter(v_l, batch): block by block, like the reference
    float part = 0.f;
    for (int n = n0 + lane; n < n1; n += 32) part += v[((size_t)l * n_nodes + n) * channels + c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    total += part;
  }
  if (lane == 0) u[(size_t)g * channels + c] = total;
}

}  // namespace dig3d

using namespace dig3d;

extern "C" {

const char* dig3d_last_error(void) { return g_err; }
int dig3d_abi_version(void) { return 2; }

int dig3d_graph_ptr(const int64_t* batch, int64_t n_nodes, int64_t n_graphs, int32_t* ptr, void* stream) {
  DIG3D_REQUIRE(batch && ptr && n_nodes >= 0 && n_graphs >= 0, "graph_ptr: bad arguments");
  graph_ptr_kernel<<<ceil_div(n_nodes + 1, 256), 256, 0, (cudaStream_t)stream>>>(batch, (int)n_nodes,
                                                                              (int)n_graphs, ptr);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_validate_nodes(const int64_t* batch, const int64_t* z, int64_t n_nodes, int64_t n_graphs, int32_t z_rows,
                         int32_t* flags, void* stream) {
  DIG3D_REQUIRE(batch && flags, "validate_nodes: null pointer");
  if (n_nodes == 0) return DIG3D_OK;
  validate_nodes_kernel<<<ceil_div(n_nodes, 256), 256, 0, (cudaStream_t)stream>>>(batch, z, (int)n_nodes,
                                                                                (int)n_graphs, z_rows, flags);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_radius_neighbors(const float* pos, const int64_t* batch, const int32_t* ptr, int64_t n_nodes,
                           int64_t n_graphs, double cutoff, int32_t cap, int32_t* nbr, int32_t* deg, void* stream) {
  DIG3D_REQUIRE(pos && batch && ptr && nbr && deg, "radius_neighbors: null pointer");
  DIG3D_REQUIRE(cap >= 1 && cap <= GEO_MAXDEG, "radius_neighbors: cap=%d outside [1,%d]", cap, GEO_MAXDEG);
  if (n_nodes == 0) return DIG3D_OK;
  const float r2 = (float)(cutoff * cutoff);
  radius_neighbors_kernel<<<ceil_div(n_nodes, 128), 128, 0, (cudaStream_t)stream>>>(
      pos, batch, ptr, (int)n_nodes, (int)n_graphs, r2, cap, nbr, deg);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_count_out(const int32_t* nbr, const int32_t* deg, int64_t n_nodes, int32_t cap, int32_t* tcnt,
                            int32_t* out_cnt, void* stream) {
  DIG3D_REQUIRE(nbr && deg && tcnt, "triplet_count: null pointer");
  if (n_nodes == 0) return DIG3D_OK;
  triplet_count_kernel<<<ceil_div(n_nodes * 32, 128), 128, 0, (cudaStream_t)stream>>>(nbr, deg, (int)n_nodes, cap,
                                                                                   tcnt, out_cnt);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_scan_counts3(const int32_t* deg, const int32_t* tcnt, const int32_t* out_cnt, int64_t n_nodes,
                       int32_t* row_ptr, int32_t* node_trip_ptr, int32_t* out_ptr, int32_t* totals, void* stream) {
  DIG3D_REQUIRE(deg && tcnt && row_ptr && node_trip_ptr && totals, "scan_counts: null pointer");
  DIG3D_REQUIRE((out_cnt != nullptr) == (out_ptr != nullptr), "scan_counts: out_cnt and out_ptr must agree");
  scan_counts_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(deg, tcnt, out_cnt, (int)n_nodes, row_ptr, node_trip_ptr,
                                                         out_ptr, totals);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_edge_fill_out(const float* pos, const int32_t* nbr, const int32_t* deg, const int32_t* row_ptr,
                        const int32_t* node_trip_ptr, int64_t n_nodes, int32_t cap, int64_t n_edges,
                        int64_t* edge_index, int32_t* src, int32_t* dst, float* dist, float* vec,
                        int32_t* trip_ptr, const int32_t* graph_ptr, const int64_t* batch, const int32_t* out_ptr,
                        int32_t* out_list, int32_t* pos_in, void* stream) {
  DIG3D_REQUIRE(pos && nbr && deg && row_ptr && node_trip_ptr && src && dst && dist && trip_ptr,
                "edge_fill: null pointer");
  DIG3D_REQUIRE(!out_list || (graph_ptr && batch && out_ptr && pos_in),
                "edge_fill: the out-edge lists need graph_ptr, batch, out_ptr and pos_in");
  if (n_nodes == 0) return DIG3D_OK;
  edge_fill_kernel<<<ceil_div(n_nodes * 32, 128), 128, 0, (cudaStream_t)stream>>>(
      pos, nbr, deg, row_ptr, node_trip_ptr, (int)n_nodes, cap, n_edges, edge_index, src, dst, dist, vec,
      trip_ptr, graph_ptr, batch, out_ptr, out_list, pos_in);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_geometry(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                           const int32_t* trip_ptr, int64_t n_edges, int32_t use_torsion, float* angle,
                           float* torsion, int32_t* idx_kj, int32_t* idx_ji, int64_t* idx_kj64,
                           int64_t* idx_ji64, void* stream) {
  DIG3D_REQUIRE(pos && src && dst && row_ptr && trip_ptr && angle, "triplet_geometry: null pointer");
  DIG3D_REQUIRE(!use_torsion || torsion, "triplet_geometry: torsion requested without output buffer");
  if (n_edges == 0) return DIG3D_OK;
  triplet_geometry_kernel<<<ceil_div(n_edges, GEO_WARPS), GEO_WARPS * 32, 0, (cudaStream_t)stream>>>(
      pos, src, dst, row_ptr, trip_ptr, (int)n_edges, GEO_MAXDEG, use_torsion, angle, torsion, idx_kj, idx_ji,
      idx_kj64, idx_ji64);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"

// The any-degree dispatcher, shared by dig3d_triplet_geometry_any_degree (ARG = false) and its _arg variant (ARG = true,
// use_torsion 1, also writes tors_arg).
template <bool ARG>
static int triplet_geometry_any_degree_impl(const float* pos, const int32_t* src, const int32_t* dst,
                                            const int32_t* row_ptr, const int32_t* trip_ptr, int64_t n_edges,
                                            int64_t n_heavy, int32_t use_torsion, const int32_t* nn1,
                                            const int32_t* nn2, int32_t* heavy_ws, float* angle, float* torsion,
                                            int64_t* idx_kj64, int64_t* idx_ji64, int32_t* tors_arg, void* stream) {
  DIG3D_REQUIRE(pos && src && dst && row_ptr && trip_ptr && angle && idx_kj64 && idx_ji64,
                "triplet_geometry_any_degree: null pointer");
  DIG3D_REQUIRE(use_torsion >= 0 && use_torsion <= 2, "triplet_geometry_any_degree: use_torsion=%d", use_torsion);
  DIG3D_REQUIRE(!use_torsion || torsion, "triplet_geometry_any_degree: torsion requested without output buffer");
  DIG3D_REQUIRE(use_torsion != 2 || (nn1 && nn2), "triplet_geometry_any_degree: the kNN torsion needs nn1 and nn2");
  DIG3D_REQUIRE(!ARG || (use_torsion == 1 && tors_arg), "triplet_geometry_any_degree_arg: null tors_arg");
  DIG3D_REQUIRE(n_heavy >= 0 && n_heavy <= n_edges && n_edges < (1ll << 31),
                "triplet_geometry_any_degree: %lld heavy edges of %lld", (long long)n_heavy, (long long)n_edges);
  DIG3D_REQUIRE(n_heavy == 0 || n_heavy == n_edges || heavy_ws,
                "triplet_geometry_any_degree: the heavy-edge list needs a workspace");
  if (n_edges == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (n_heavy < n_edges) {
    triplet_geometry_kernel<ARG><<<ceil_div(n_edges, GEO_WARPS), GEO_WARPS * 32, 0, st>>>(
        pos, src, dst, row_ptr, trip_ptr, (int)n_edges, GEO_MAXDEG, use_torsion, angle, torsion, nullptr, nullptr,
        idx_kj64, idx_ji64, nn1, nn2, tors_arg);
    DIG3D_LAUNCH_CHECK();
  }
  if (n_heavy == 0) return DIG3D_OK;
  const int32_t* heavy = nullptr;                           // n_heavy == n_edges: every edge, no list needed
  if (n_heavy < n_edges) {
    cudaMemsetAsync(heavy_ws, 0, sizeof(int32_t), st);
    heavy_edges_kernel<<<ceil_div(n_edges, 256), 256, 0, st>>>(src, row_ptr, (int)n_edges, GEO_MAXDEG, heavy_ws);
    DIG3D_LAUNCH_CHECK();
    heavy = heavy_ws + 1;
  }
  triplet_geometry_heavy_kernel<ARG><<<(unsigned)n_heavy, HEAVY_THREADS, 0, st>>>(
      pos, src, dst, row_ptr, trip_ptr, heavy, use_torsion, angle, torsion, idx_kj64, idx_ji64, nn1, nn2, tors_arg);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

extern "C" {

int dig3d_triplet_geometry_any_degree(const float* pos, const int32_t* src, const int32_t* dst,
                                      const int32_t* row_ptr, const int32_t* trip_ptr, int64_t n_edges,
                                      int64_t n_heavy, int32_t use_torsion, const int32_t* nn1, const int32_t* nn2,
                                      int32_t* heavy_ws, float* angle, float* torsion, int64_t* idx_kj64,
                                      int64_t* idx_ji64, void* stream) {
  return triplet_geometry_any_degree_impl<false>(pos, src, dst, row_ptr, trip_ptr, n_edges, n_heavy, use_torsion, nn1,
                                                 nn2, heavy_ws, angle, torsion, idx_kj64, idx_ji64, nullptr, stream);
}

int dig3d_triplet_geometry_any_degree_arg(const float* pos, const int32_t* src, const int32_t* dst,
                                          const int32_t* row_ptr, const int32_t* trip_ptr, int64_t n_edges,
                                          int64_t n_heavy, int32_t* heavy_ws, float* angle, float* torsion,
                                          int64_t* idx_kj64, int64_t* idx_ji64, int32_t* tors_arg, void* stream) {
  return triplet_geometry_any_degree_impl<true>(pos, src, dst, row_ptr, trip_ptr, n_edges, n_heavy, 1, nullptr,
                                                nullptr, heavy_ws, angle, torsion, idx_kj64, idx_ji64, tors_arg,
                                                stream);
}

int dig3d_knn2(const float* pos, const int64_t* batch, const int32_t* graph_ptr, int64_t n_nodes, int64_t n_graphs,
               int32_t* nn1, int32_t* nn2, void* stream) {
  DIG3D_REQUIRE(pos && batch && graph_ptr && nn1 && nn2, "knn2: null pointer");
  if (n_nodes == 0) return DIG3D_OK;
  knn2_kernel<<<ceil_div(n_nodes, 128), 128, 0, (cudaStream_t)stream>>>(pos, batch, graph_ptr, (int)n_nodes,
                                                                       (int)n_graphs, nn1, nn2);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_geometry_knn(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                               const int32_t* trip_ptr, int64_t n_edges, const int32_t* nn1, const int32_t* nn2,
                               float* angle, float* torsion, int64_t* idx_kj64, int64_t* idx_ji64, void* stream) {
  DIG3D_REQUIRE(pos && src && dst && row_ptr && trip_ptr && nn1 && nn2 && angle && torsion,
                "triplet_geometry_knn: null pointer");
  if (n_edges == 0) return DIG3D_OK;
  triplet_geometry_kernel<<<ceil_div(n_edges, GEO_WARPS), GEO_WARPS * 32, 0, (cudaStream_t)stream>>>(
      pos, src, dst, row_ptr, trip_ptr, (int)n_edges, GEO_MAXDEG, 2, angle, torsion, nullptr, nullptr, idx_kj64,
      idx_ji64, nn1, nn2);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_edges_to_csr(const float* pos, const int64_t* edge_index, int64_t n_edges, int64_t n_nodes, int32_t* src,
                       int32_t* dst, int32_t* row_ptr, int32_t* cnt_ws, int32_t* trip_ptr, float* dist,
                       int32_t* flags /*[6]: see include/dig3d.h*/, void* stream) {
  DIG3D_REQUIRE(pos && edge_index && src && dst && row_ptr && cnt_ws && trip_ptr && dist && flags,
                "edges_to_csr: null pointer");
  DIG3D_REQUIRE(((uintptr_t)flags & 7) == 0, "edges_to_csr: flags must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(flags, 0, 6 * sizeof(int32_t), st);
  if (n_edges) {
    edges_prepare_kernel<<<ceil_div(n_edges, 256), 256, 0, st>>>(edge_index, n_edges, (int)n_nodes, src, dst, flags);
    DIG3D_LAUNCH_CHECK();
  }
  csr_from_sorted_kernel<<<ceil_div(n_nodes + 1, 256), 256, 0, st>>>(dst, (int)n_edges, (int)n_nodes, row_ptr);
  DIG3D_LAUNCH_CHECK();
  if (n_edges) {
    edge_triplet_count_kernel<<<ceil_div(n_edges, COUNT_THREADS), COUNT_THREADS, 0, st>>>(
        pos, src, dst, row_ptr, (int)n_edges, GEO_MAXDEG, cnt_ws, dist, flags,
        reinterpret_cast<unsigned long long*>(flags + 4));
    DIG3D_LAUNCH_CHECK();
  }
  scan_counts_kernel<<<1, 1024, 0, st>>>(cnt_ws, cnt_ws, nullptr, (int)n_edges, trip_ptr, cnt_ws + n_edges + 1, nullptr,
                                         flags + 2);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_segment_sum(const float* x, const int32_t* ptr, int64_t n_segments, int64_t width, float* out,
                      void* stream) {
  DIG3D_REQUIRE(x && ptr && out && width > 0, "segment_sum: bad arguments");
  if (n_segments == 0) return DIG3D_OK;
  const int strips = (int)((width + 127) / 128);
  const int64_t warps = n_segments * strips;
  segment_sum_kernel<<<ceil_div(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, ptr, (int)n_segments,
                                                                               (int)width, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_graph_readout(const float* v, const int32_t* graph_ptr, int64_t n_graphs, int64_t n_nodes,
                        int32_t n_blocks, int32_t channels, float* u, void* stream) {
  DIG3D_REQUIRE(v && graph_ptr && u && channels > 0 && n_blocks > 0, "graph_readout: bad arguments");
  if (n_graphs == 0) return DIG3D_OK;
  graph_readout_kernel<<<ceil_div(n_graphs * channels * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      v, graph_ptr, (int)n_graphs, (int)n_nodes, n_blocks, channels, u);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
