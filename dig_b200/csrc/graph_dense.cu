// Radius graph without a neighbour table (sm_90a): torch_cluster.radius_graph(x, r, batch, max_num_neighbors=m) for
// any m, as called by users of the reference's utilities (utils/geometric_computing.py) and by ProNet
// (pronet.py:386) with their own max_num_neighbors.
//
// The capped builder (graph.cu) parks the neighbours of every node in an nbr[N][cap] table, cap <= 64.  Here the
// edges are built in two passes over the same scan: a count pass, an exclusive scan into row_ptr, then a fill pass
// that writes each target's edges at row_ptr[i], so memory is O(N + E) whatever m is.  Both passes run the same
// warp-per-query scan, so they agree on every hit:
//   - candidates c in ascending index inside the query's graph, 32 per step (lane = c - c0);
//   - d2 = fma(dz, dz, fma(dy, dy, dx * dx)) on __fsub_rn differences, a hit when d2 < r2 (strict);
//   - the first cap = m + 1 hits counted with the query itself, which is then dropped.
// The "first hits in index order" rule is a ballot plus a prefix count over the lanes: no atomics, so the result is
// the one of the capped builder's one-thread-per-query loop (radius_neighbors_kernel) hit for hit.
#include "common.cuh"

namespace dig3d {

constexpr int DENSE_WARPS = 4;

// Runs the scan of query n (one warp) and calls emit(c, slot) for every kept neighbour c != n, slot = its rank among
// them; returns their number.
template <class Emit>
__device__ __forceinline__ int radius_scan(const float* __restrict__ pos, const int64_t* __restrict__ batch,
                                           const int32_t* __restrict__ ptr, int n, int n_graphs, float r2, int cap,
                                           Emit emit) {
  const int lane = threadIdx.x & 31;
  const int64_t gb = batch[n];
  if (gb < 0 || gb >= n_graphs) return 0;                  // reported by validate_nodes_kernel; never index ptr[]
  const int lo = ptr[gb], hi = ptr[gb + 1];
  const f3 q = load3(pos, n);
  const unsigned below = (1u << lane) - 1;
  int hits = 0, kept = 0;
  for (int c0 = lo; c0 < hi && hits < cap; c0 += 32) {
    const int c = c0 + lane;
    bool hit = false;
    if (c < hi) {
      const f3 p = load3(pos, c);
      const float dx = __fsub_rn(p.x, q.x), dy = __fsub_rn(p.y, q.y), dz = __fsub_rn(p.z, q.z);
      const float d2 = __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
      hit = d2 < r2;
    }
    const unsigned hb = __ballot_sync(0xffffffffu, hit);
    const bool in_cap = hit && hits + __popc(hb & below) < cap;   // this hit is among the first cap
    const bool keep = in_cap && c != n;
    const unsigned kb = __ballot_sync(0xffffffffu, keep);
    if (keep) emit(c, kept + __popc(kb & below));
    hits += __popc(__ballot_sync(0xffffffffu, in_cap));
    kept += __popc(kb);
  }
  return kept;
}

__global__ void __launch_bounds__(DENSE_WARPS * 32)
radius_dense_count_kernel(const float* __restrict__ pos, const int64_t* __restrict__ batch,
                          const int32_t* __restrict__ ptr, int n_nodes, int n_graphs, float r2, int cap,
                          int32_t* __restrict__ counts) {
  const int n = blockIdx.x * DENSE_WARPS + (threadIdx.x >> 5);
  if (n >= n_nodes) return;
  const int m = radius_scan(pos, batch, ptr, n, n_graphs, r2, cap, [](int, int) {});
  if ((threadIdx.x & 31) == 0) counts[n] = m;
}

__global__ void __launch_bounds__(DENSE_WARPS * 32)
radius_dense_fill_kernel(const float* __restrict__ pos, const int64_t* __restrict__ batch,
                         const int32_t* __restrict__ ptr, int n_nodes, int n_graphs, float r2, int cap,
                         const int32_t* __restrict__ row_ptr, int64_t n_edges, int64_t* __restrict__ edge_index,
                         int32_t* __restrict__ src, int32_t* __restrict__ dst) {
  const int n = blockIdx.x * DENSE_WARPS + (threadIdx.x >> 5);
  if (n >= n_nodes) return;
  const int64_t e0 = row_ptr[n];
  radius_scan(pos, batch, ptr, n, n_graphs, r2, cap, [&](int c, int slot) {
    const int64_t e = e0 + slot;
    src[e] = c;
    dst[e] = n;
    if (edge_index) { edge_index[e] = c; edge_index[n_edges + e] = n; }
  });
}

// Single-CTA exclusive scan of the per-node counts: row_ptr[0..n] (int32; meaningful while the total is below 2^31)
// and *total in 64 bits.
__global__ void __launch_bounds__(1024) radius_dense_scan_kernel(const int32_t* __restrict__ counts, int n,
                                                                int32_t* __restrict__ row_ptr,
                                                                int64_t* __restrict__ total) {
  __shared__ long long warp_tot[32];
  __shared__ long long carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int idx = base + tid;
    const long long v = idx < n ? counts[idx] : 0;
    long long s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long t = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += t;
    }
    if (lane == 31) warp_tot[wid] = s;
    __syncthreads();
    if (wid == 0) {
      long long w = warp_tot[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long t = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += t;
      }
      warp_tot[lane] = w;
    }
    __syncthreads();
    if (idx < n) row_ptr[idx] = (int32_t)(carry + (wid == 0 ? 0 : warp_tot[wid - 1]) + s - v);
    __syncthreads();
    if (tid == 0) carry += warp_tot[31];
    __syncthreads();
  }
  if (tid == 0) {
    row_ptr[n] = (int32_t)carry;
    *total = carry;
  }
}

static inline int dense_cap(int64_t max_num_neighbors, int64_t n_nodes) {
  // hits never exceed the graph's size, so any cap above n_nodes is the same as n_nodes + 1
  return (int)(max_num_neighbors < n_nodes ? max_num_neighbors + 1 : n_nodes + 1);
}

}  // namespace dig3d

using namespace dig3d;

extern "C" {

int dig3d_radius_graph_dense_count(const float* pos, const int64_t* batch, const int32_t* graph_ptr, int64_t n_nodes,
                                   int64_t n_graphs, double cutoff, int64_t max_num_neighbors, int32_t* counts,
                                   int32_t* row_ptr, int64_t* info, int64_t* info_host, void* stream) {
  DIG3D_REQUIRE((pos || n_nodes == 0) && (batch || n_nodes == 0) && graph_ptr && counts && row_ptr && info &&
                info_host, "radius_graph_dense_count: null pointer");
  DIG3D_REQUIRE(n_nodes >= 0 && n_nodes < (1ll << 31) - 1 && n_graphs >= 0 && n_graphs < (1ll << 31),
                "radius_graph_dense_count: %lld nodes in %lld graphs", (long long)n_nodes, (long long)n_graphs);
  DIG3D_REQUIRE(max_num_neighbors >= 0, "radius_graph_dense_count: max_num_neighbors=%lld",
                (long long)max_num_neighbors);
  cudaStream_t st = (cudaStream_t)stream;
  const float r2 = (float)(cutoff * cutoff);
  if (n_nodes) {
    radius_dense_count_kernel<<<ceil_div(n_nodes, DENSE_WARPS), DENSE_WARPS * 32, 0, st>>>(
        pos, batch, graph_ptr, (int)n_nodes, (int)n_graphs, r2, dense_cap(max_num_neighbors, n_nodes), counts);
    DIG3D_LAUNCH_CHECK();
  }
  radius_dense_scan_kernel<<<1, 1024, 0, st>>>(counts, (int)n_nodes, row_ptr, info);
  DIG3D_LAUNCH_CHECK();
  cudaError_t err = cudaMemcpyAsync(info_host, info, 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, st);
  if (err == cudaSuccess) err = cudaStreamSynchronize(st);               // the one host read: E and the node checks
  if (err != cudaSuccess) {
    set_error("radius_graph_dense_count: %s", cudaGetErrorString(err));
    return DIG3D_ECUDA;
  }
  DIG3D_REQUIRE(info_host[0] < (1ll << 31), "radius_graph_dense: %lld edges, the limit is 2^31 - 1",
                (long long)info_host[0]);
  return DIG3D_OK;
}

int dig3d_radius_graph_dense_fill(const float* pos, const int64_t* batch, const int32_t* graph_ptr, int64_t n_nodes,
                                  int64_t n_graphs, double cutoff, int64_t max_num_neighbors, const int32_t* row_ptr,
                                  int64_t n_edges, int64_t* edge_index, int32_t* src, int32_t* dst, void* stream) {
  DIG3D_REQUIRE(graph_ptr && row_ptr, "radius_graph_dense_fill: null pointer");
  DIG3D_REQUIRE(n_edges >= 0 && n_edges < (1ll << 31), "radius_graph_dense_fill: %lld edges", (long long)n_edges);
  DIG3D_REQUIRE(n_edges == 0 || (pos && batch && src && dst), "radius_graph_dense_fill: null output");
  DIG3D_REQUIRE(max_num_neighbors >= 0 && n_nodes >= 0 && n_nodes < (1ll << 31) - 1,
                "radius_graph_dense_fill: bad arguments");
  if (n_edges == 0) return DIG3D_OK;
  const float r2 = (float)(cutoff * cutoff);
  radius_dense_fill_kernel<<<ceil_div(n_nodes, DENSE_WARPS), DENSE_WARPS * 32, 0, (cudaStream_t)stream>>>(
      pos, batch, graph_ptr, (int)n_nodes, (int)n_graphs, r2, dense_cap(max_num_neighbors, n_nodes), row_ptr,
      n_edges, edge_index, src, dst);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
