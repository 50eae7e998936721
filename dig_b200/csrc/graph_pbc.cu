// Periodic radius graph on sm_90a: ocpmodels' radius_graph_pbc + get_max_neighbors_mask (Open-Catalyst-Project/ocp,
// 2022), which ComENet-OCP calls with otf_graph=True (reference comenet-ocp.py:343-350).
//
// The reference builds every (target i, source j, image cell c) candidate of the batch as one dense array, masks it,
// then sorts a padded [N, max_neighbours] distance table to apply the cap.  Here nothing of size N^2 * cells exists:
//
//   setup   one CTA: graph_ptr = exclusive cumsum(natoms), the image range of every structure, its batch maximum
//           and the input checks (zero / non-finite cell volume, natoms that do not sum to N, image range too wide)
//   count   one warp per target atom enumerates its candidates in the reference's order (source j, then image cell,
//           last cell axis fastest), counts those inside the radius and, when the cap binds, finds the cap-th
//           smallest squared distance by a 4 x 8-bit radix select over re-enumerations (no candidate is stored)
//   scan    one CTA: row_ptr = exclusive scan of the kept counts
//   fill    one warp per target atom re-enumerates and writes its kept edges at row_ptr[i], in enumeration order
//
// Rounding follows the reference's fp32 torch ops: the image range with the ATen forms of torch.cross / sum / norm
// (common.cuh), the image offset cell^T . c in bmm's order (fma over the cell rows, as pbc_edge_vectors_kernel), the
// squared distance as (dx*dx + dy*dy) + dz*dz, kept when d2 <= fp32(radius^2) and d2 > fp32(1e-4).
// Cap ties: among equal d2 the candidate enumerated first is kept (the reference's torch.sort is unstable there).
#include "common.cuh"

namespace dig3d {

constexpr int PBC_WARPS = 8;                 // warps (= target atoms) per CTA in the count / fill kernels
constexpr int PBC_MAX_REP = 1 << 16;         // image range per axis beyond which the input is rejected
// info[] (int64, device): image range, error flags, edge total, largest structure
enum { PBC_R1 = 0, PBC_R2 = 1, PBC_R3 = 2, PBC_FLAGS = 3, PBC_EDGES = 4, PBC_NMAX = 5, PBC_INFO_LEN = 6 };
enum { PBC_BAD_VOLUME = 1, PBC_BAD_NATOMS = 2, PBC_TOO_WIDE = 4 };

__device__ __forceinline__ f3 div3s(const f3 a, float s) {
  return {__fdiv_rn(a.x, s), __fdiv_rn(a.y, s), __fdiv_rn(a.z, s)};
}

// rep = ceil(radius * |cross / vol|)                          (radius_graph_pbc: rep_a1 / rep_a2 / rep_a3)
__device__ __forceinline__ float pbc_rep(const f3 cross, float vol, float radius) {
  return ceilf(__fmul_rn(radius, norm3_aten(div3s(cross, vol))));
}

// ------------------------------------------------------------------ setup (single CTA)
__global__ void __launch_bounds__(1024) pbc_setup_kernel(const float* __restrict__ cell,
                                                         const int64_t* __restrict__ natoms, int n_graphs,
                                                         int64_t n_atoms, float radius, int32_t* __restrict__ graph_ptr,
                                                         int64_t* __restrict__ info) {
  __shared__ long long warp_tot[32];
  __shared__ long long carry;
  __shared__ unsigned long long nmax;
  __shared__ int rmax[3], flags;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) { carry = 0; nmax = 0; rmax[0] = rmax[1] = rmax[2] = 0; flags = 0; }
  __syncthreads();
  for (int base = 0; base < n_graphs; base += 1024) {
    const int g = base + tid;
    long long v = 0;
    if (g < n_graphs) {
      v = natoms[g];
      if (v < 0) { atomicOr(&flags, PBC_BAD_NATOMS); v = 0; }
      atomicMax(&nmax, (unsigned long long)v);
      const float* c = cell + 9 * (size_t)g;
      const f3 a1 = {c[0], c[1], c[2]}, a2 = {c[3], c[4], c[5]}, a3 = {c[6], c[7], c[8]};
      const f3 x23 = cross_aten(a2, a3);
      const float vol = sum3_aten(mul3(a1, x23));
      if (!isfinite(vol) || vol == 0.f) {
        atomicOr(&flags, PBC_BAD_VOLUME);
      } else {
        const float r[3] = {pbc_rep(x23, vol, radius), pbc_rep(cross_aten(a3, a1), vol, radius),
                            pbc_rep(cross_aten(a1, a2), vol, radius)};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          if (!(r[k] <= (float)PBC_MAX_REP)) atomicOr(&flags, PBC_TOO_WIDE);   // also NaN
          else atomicMax(&rmax[k], max(0, (int)r[k]));
        }
      }
    }
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
    const long long start = carry + (wid == 0 ? 0 : warp_tot[wid - 1]) + s - v;
    if (g < n_graphs) graph_ptr[g] = (int32_t)min(start, (long long)n_atoms);
    __syncthreads();
    if (tid == 0) carry += warp_tot[31];
    __syncthreads();
  }
  if (tid == 0) {
    int f = flags;
    if (carry != n_atoms) f |= PBC_BAD_NATOMS;
    graph_ptr[n_graphs] = (int32_t)n_atoms;
    long long cells = 1;
    for (int k = 0; k < 3; ++k) cells *= 2 * rmax[k] + 1;
    if (!f && (long long)nmax * cells >= (1ll << 31)) f |= PBC_TOO_WIDE;   // candidates per target must fit int32
    info[PBC_R1] = rmax[0]; info[PBC_R2] = rmax[1]; info[PBC_R3] = rmax[2];
    info[PBC_FLAGS] = f;
    info[PBC_EDGES] = 0;
    info[PBC_NMAX] = (long long)nmax;
  }
}

// ------------------------------------------------------------------ per-target candidate enumeration
struct PbcTarget {
  int i, start, n_src;            // target atom, first atom of its structure, atoms in it
  unsigned total;                 // candidates = n_src * cells
  int r1, r2, r3, n3, n23, cells;
  f3 pi;
  float c[9];                     // cell of the structure, row-major (rows = lattice vectors)
};

__device__ __forceinline__ bool pbc_target(const float* __restrict__ pos, const float* __restrict__ cell,
                                           const int32_t* __restrict__ graph_ptr, int n_graphs,
                                           const int64_t* __restrict__ info, int i, PbcTarget& t) {
  if (info[PBC_FLAGS]) return false;
  int lo = 0, hi = n_graphs;      // the structure of atom i: largest g with graph_ptr[g] <= i (graph_ptr[B] = N > i)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (graph_ptr[mid] <= i) lo = mid; else hi = mid - 1;
  }
  t.i = i;
  t.start = graph_ptr[lo];
  t.n_src = graph_ptr[lo + 1] - t.start;
  t.r1 = (int)info[PBC_R1]; t.r2 = (int)info[PBC_R2]; t.r3 = (int)info[PBC_R3];
  t.n3 = 2 * t.r3 + 1;
  t.n23 = (2 * t.r2 + 1) * t.n3;
  t.cells = (2 * t.r1 + 1) * t.n23;
  t.total = (unsigned)t.n_src * (unsigned)t.cells;
  t.pi = load3(pos, i);
#pragma unroll
  for (int k = 0; k < 9; ++k) t.c[k] = __ldg(cell + 9 * (size_t)lo + k);
  return true;
}

struct PbcCand {
  int j;                          // source atom (global id)
  int a1, a2, a3;                 // image cell
  float d2;
};

// candidate q of the target: source j = start + q / cells, cell = cartesian_prod(...)[q % cells]
__device__ __forceinline__ PbcCand pbc_candidate(const float* __restrict__ pos, const PbcTarget& t, unsigned q) {
  PbcCand r;
  const unsigned jl = q / (unsigned)t.cells;
  const int cc = (int)(q - jl * (unsigned)t.cells);
  const int u1 = cc / t.n23, rem = cc - u1 * t.n23;
  const int u2 = rem / t.n3, u3 = rem - u2 * t.n3;
  r.j = t.start + (int)jl;
  r.a1 = u1 - t.r1; r.a2 = u2 - t.r2; r.a3 = u3 - t.r3;
  const float o1 = (float)r.a1, o2 = (float)r.a2, o3 = (float)r.a3;
  // pbc_offsets = bmm(cell^T, unit_cell): offset[k] = sum over the cell rows r of cell[r][k] * c[r]
  const float ox = __fmaf_rn(o3, t.c[6], __fmaf_rn(o2, t.c[3], __fmul_rn(o1, t.c[0])));
  const float oy = __fmaf_rn(o3, t.c[7], __fmaf_rn(o2, t.c[4], __fmul_rn(o1, t.c[1])));
  const float oz = __fmaf_rn(o3, t.c[8], __fmaf_rn(o2, t.c[5], __fmul_rn(o1, t.c[2])));
  const f3 pj = load3(pos, r.j);
  const f3 d = sub3(t.pi, {__fadd_rn(pj.x, ox), __fadd_rn(pj.y, oy), __fadd_rn(pj.z, oz)});
  r.d2 = __fadd_rn(__fadd_rn(__fmul_rn(d.x, d.x), __fmul_rn(d.y, d.y)), __fmul_rn(d.z, d.z));
  return r;
}

__device__ __forceinline__ bool pbc_inside(float d2, float r2) { return d2 <= r2 && d2 > 1e-4f; }

// ------------------------------------------------------------------ count + cap threshold
// select[2i] = bits of the largest kept d2 (0xffffffff: every candidate inside the radius is kept),
// select[2i+1] = how many candidates with exactly that d2 are kept, first ones in enumeration order.
// Squared distances are positive, so their fp32 bit patterns order like the values.
__global__ void __launch_bounds__(PBC_WARPS * 32)
pbc_count_kernel(const float* __restrict__ pos, const float* __restrict__ cell, const int32_t* __restrict__ graph_ptr,
                 int n_atoms, int n_graphs, float r2, int cap, int64_t* __restrict__ info,
                 int32_t* __restrict__ counts, uint32_t* __restrict__ select) {
  __shared__ int hist[PBC_WARPS][256];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int i = blockIdx.x * PBC_WARPS + w;
  PbcTarget t;
  if (i >= n_atoms || !pbc_target(pos, cell, graph_ptr, n_graphs, info, i, t)) return;
  int* h = hist[w];
  int cnt = 0;
  for (unsigned q0 = 0; q0 < t.total; q0 += 32) {
    const unsigned q = q0 + lane;
    const bool in = q < t.total && pbc_inside(pbc_candidate(pos, t, q).d2, r2);
    cnt += __popc(__ballot_sync(0xffffffffu, in));
  }
  uint32_t thr = 0xffffffffu, ties = 0;
  int kept = cnt;
  if (cap > 0 && cnt > cap) {
    // radix select of the cap-th smallest d2, most significant byte first
    unsigned prefix = 0, pmask = 0;
    int k = cap;                                 // rank still to find among the candidates matching the prefix
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int b = lane; b < 256; b += 32) h[b] = 0;
      __syncwarp();
      for (unsigned q0 = 0; q0 < t.total; q0 += 32) {
        const unsigned q = q0 + lane;
        if (q < t.total) {
          const float d2 = pbc_candidate(pos, t, q).d2;
          const unsigned bits = __float_as_uint(d2);
          if (pbc_inside(d2, r2) && (bits & pmask) == prefix) atomicAdd(&h[(bits >> shift) & 255], 1);
        }
      }
      __syncwarp();
      int loc[8], s = 0;
#pragma unroll
      for (int b = 0; b < 8; ++b) { loc[b] = h[8 * lane + b]; s += loc[b]; }
      int incl = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int up = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += up;
      }
      const int excl = incl - s;
      const int owner = __ffs(__ballot_sync(0xffffffffu, excl < k && k <= incl)) - 1;
      int digit = 0, left = k;
      if (lane == owner) {
        int acc = excl;
        bool found = false;
#pragma unroll
        for (int b = 0; b < 8; ++b) {
          if (!found && acc + loc[b] >= k) { digit = 8 * lane + b; left = k - acc; found = true; }
          acc += loc[b];
        }
      }
      digit = __shfl_sync(0xffffffffu, digit, owner);
      k = __shfl_sync(0xffffffffu, left, owner);
      prefix |= (unsigned)digit << shift;
      pmask |= 0xffu << shift;
      __syncwarp();
    }
    thr = prefix;
    ties = (uint32_t)k;
    kept = cap;
  }
  if (lane == 0) {
    counts[i] = kept;
    select[2 * (size_t)i] = thr;
    select[2 * (size_t)i + 1] = ties;
    atomicAdd(reinterpret_cast<unsigned long long*>(info + PBC_EDGES), (unsigned long long)kept);
  }
}

// ------------------------------------------------------------------ exclusive scan (single CTA)
__global__ void __launch_bounds__(1024) pbc_scan_kernel(const int32_t* __restrict__ counts, int n,
                                                        int32_t* __restrict__ row_ptr) {
  __shared__ unsigned warp_tot[32];
  __shared__ unsigned carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int idx = base + tid;
    const unsigned v = idx < n ? (unsigned)counts[idx] : 0u;
    unsigned s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned t = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += t;
    }
    if (lane == 31) warp_tot[wid] = s;
    __syncthreads();
    if (wid == 0) {
      unsigned w = warp_tot[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += t;
      }
      warp_tot[lane] = w;
    }
    __syncthreads();
    if (idx < n) row_ptr[idx] = (int32_t)(carry + (wid == 0 ? 0u : warp_tot[wid - 1]) + s - v);
    __syncthreads();
    if (tid == 0) carry += warp_tot[31];
    __syncthreads();
  }
  if (tid == 0) row_ptr[n] = (int32_t)carry;
}

// ------------------------------------------------------------------ fill
__global__ void __launch_bounds__(PBC_WARPS * 32)
pbc_fill_kernel(const float* __restrict__ pos, const float* __restrict__ cell, const int32_t* __restrict__ graph_ptr,
                int n_atoms, int n_graphs, float r2, const int64_t* __restrict__ info,
                const uint32_t* __restrict__ select, const int32_t* __restrict__ row_ptr, int64_t n_edges,
                int64_t* __restrict__ edge_index, float* __restrict__ cell_offsets) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int i = blockIdx.x * PBC_WARPS + w;
  PbcTarget t;
  if (i >= n_atoms || !pbc_target(pos, cell, graph_ptr, n_graphs, info, i, t)) return;
  const uint32_t thr = select[2 * (size_t)i], ties = select[2 * (size_t)i + 1];
  const unsigned below = (1u << lane) - 1;
  int e = row_ptr[i], end = row_ptr[i + 1];
  unsigned tie_seen = 0;
  for (unsigned q0 = 0; q0 < t.total && e < end; q0 += 32) {
    const unsigned q = q0 + lane;
    PbcCand c{};
    bool in = false;
    if (q < t.total) { c = pbc_candidate(pos, t, q); in = pbc_inside(c.d2, r2); }
    const unsigned bits = __float_as_uint(c.d2);
    const bool eq = in && bits == thr;
    const unsigned beq = __ballot_sync(0xffffffffu, eq);
    const bool keep = in && (bits < thr || (eq && tie_seen + __popc(beq & below) < ties));
    const unsigned bk = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const int64_t o = e + __popc(bk & below);
      edge_index[o] = c.j;
      edge_index[n_edges + o] = i;
      cell_offsets[3 * o] = (float)c.a1;
      cell_offsets[3 * o + 1] = (float)c.a2;
      cell_offsets[3 * o + 2] = (float)c.a3;
    }
    e += __popc(bk);
    tie_seen += __popc(beq);
  }
}

// neighbors[g] = kept edges of structure g
__global__ void pbc_neighbors_kernel(const int32_t* __restrict__ graph_ptr, const int32_t* __restrict__ row_ptr,
                                     int n_graphs, int64_t* __restrict__ neighbors) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_graphs) return;
  neighbors[g] = (int64_t)row_ptr[graph_ptr[g + 1]] - row_ptr[graph_ptr[g]];
}

}  // namespace dig3d

using namespace dig3d;

extern "C" {

int dig3d_radius_graph_pbc_count(const float* pos, const float* cell, const int64_t* natoms, int64_t n_atoms,
                                 int64_t n_graphs, double radius, int32_t max_num_neighbors, int32_t* graph_ptr,
                                 int32_t* counts, uint32_t* select, int32_t* row_ptr, int64_t* info,
                                 int64_t* n_edges_host, void* stream) {
  DIG3D_REQUIRE((pos || n_atoms == 0) && ((cell && natoms) || n_graphs == 0) && graph_ptr && counts && select &&
                row_ptr && info && n_edges_host, "radius_graph_pbc_count: null pointer");
  DIG3D_REQUIRE(n_atoms >= 0 && n_atoms < (1ll << 31) && n_graphs >= 0 && n_graphs < (1ll << 31),
                "radius_graph_pbc_count: %lld atoms in %lld structures", (long long)n_atoms, (long long)n_graphs);
  DIG3D_REQUIRE(radius > 0.0 && radius < 1e18, "radius_graph_pbc_count: radius must be positive and finite, got %g",
                radius);
  cudaStream_t st = (cudaStream_t)stream;
  *n_edges_host = 0;
  if (n_graphs == 0) {
    DIG3D_REQUIRE(n_atoms == 0, "radius_graph_pbc: natoms sums to 0, but there are %lld atoms", (long long)n_atoms);
    cudaMemsetAsync(row_ptr, 0, sizeof(int32_t), st);
    DIG3D_LAUNCH_CHECK();
    return DIG3D_OK;
  }
  pbc_setup_kernel<<<1, 1024, 0, st>>>(cell, natoms, (int)n_graphs, n_atoms, (float)radius, graph_ptr, info);
  DIG3D_LAUNCH_CHECK();
  const float r2 = (float)(radius * radius);
  if (n_atoms) {
    pbc_count_kernel<<<ceil_div(n_atoms, PBC_WARPS), PBC_WARPS * 32, 0, st>>>(
        pos, cell, graph_ptr, (int)n_atoms, (int)n_graphs, r2, max_num_neighbors, info, counts, select);
    DIG3D_LAUNCH_CHECK();
  }
  pbc_scan_kernel<<<1, 1024, 0, st>>>(counts, (int)n_atoms, row_ptr);
  DIG3D_LAUNCH_CHECK();
  int64_t h[PBC_INFO_LEN];
  cudaError_t err = cudaMemcpyAsync(h, info, sizeof(h), cudaMemcpyDeviceToHost, st);
  if (err == cudaSuccess) err = cudaStreamSynchronize(st);               // the one host read: E and the input checks
  if (err != cudaSuccess) {
    set_error("radius_graph_pbc_count: %s", cudaGetErrorString(err));
    return DIG3D_ECUDA;
  }
  const long long f = h[PBC_FLAGS];
  DIG3D_REQUIRE(!(f & PBC_BAD_VOLUME), "radius_graph_pbc: a cell has zero or non-finite volume");
  DIG3D_REQUIRE(!(f & PBC_BAD_NATOMS), "radius_graph_pbc: natoms must be non-negative and sum to the %lld atoms of pos",
                (long long)n_atoms);
  DIG3D_REQUIRE(!(f & PBC_TOO_WIDE), "radius_graph_pbc: the image range (radius over the cell's plane spacing) is too "
                "wide: more than 2^31 candidates per atom");
  DIG3D_REQUIRE(h[PBC_EDGES] < (1ll << 31), "radius_graph_pbc: %lld edges, the limit is 2^31 - 1",
                (long long)h[PBC_EDGES]);
  *n_edges_host = h[PBC_EDGES];
  return DIG3D_OK;
}

int dig3d_radius_graph_pbc_fill(const float* pos, const float* cell, int64_t n_atoms, int64_t n_graphs, double radius,
                                const int32_t* graph_ptr, const uint32_t* select, const int32_t* row_ptr,
                                const int64_t* info, int64_t n_edges, int64_t* edge_index, float* cell_offsets,
                                int64_t* neighbors, void* stream) {
  DIG3D_REQUIRE((pos || n_atoms == 0) && ((cell && neighbors) || n_graphs == 0) && graph_ptr && select && row_ptr &&
                info, "radius_graph_pbc_fill: null pointer");
  DIG3D_REQUIRE(n_edges == 0 || (edge_index && cell_offsets), "radius_graph_pbc_fill: null output");
  if (n_graphs == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const float r2 = (float)(radius * radius);
  if (n_atoms && n_edges) {
    pbc_fill_kernel<<<ceil_div(n_atoms, PBC_WARPS), PBC_WARPS * 32, 0, st>>>(
        pos, cell, graph_ptr, (int)n_atoms, (int)n_graphs, r2, info, select, row_ptr, n_edges, edge_index,
        cell_offsets);
    DIG3D_LAUNCH_CHECK();
  }
  pbc_neighbors_kernel<<<ceil_div(n_graphs, 256), 256, 0, st>>>(graph_ptr, row_ptr, (int)n_graphs, neighbors);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
