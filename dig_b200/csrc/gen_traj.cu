// G-SphereNet's training trajectories (reference dig/ggraph3D/dataset/ggraph3D_dataset.py:192-302, QM93DGEN.get) for a
// ragged batch of molecules, one warp per molecule, lane j = atom j (n <= 32).  A trajectory depends on the molecule
// alone, so the dataset computes all of them once instead of once per molecule per epoch.
//
//  * Generation order: Prim's minimum spanning tree over the squared distances as networkx's prim_mst_edges walks it
//    (nx.from_numpy_array: an entry of 0 is no edge; start at node 0; the heap pops the smallest weight, ties by push
//    order = tree position of the tree-side node, then ascending index of the new node).  Lane w keeps the best
//    (weight, tree position) over the tree for its node; ties keep the earlier tree node.
//  * Arithmetic is the reference's op sequence as CPU ATen runs it: 3-element sums (((0 + x) + y) + z), norms
//    sqrt(fma(z, z, fma(y, y, x * x))), cross products fma(a, b, -rn(c * d)), each op rounded once.  atan2 is the
//    correctly rounded fp32 value (fp64 atan2, rounded once), where CPU torch calls the C library's atan2f.
//  * No atomics: every output element is written by one lane, so results are deterministic.
#include "common.cuh"

using namespace dig3d;

namespace {

constexpr int kWarps = 4;
constexpr double kTwoPi = 6.283185307179586;   // 2 * math.pi

// CPU ATen's sum starts from +0: a sum of negative zeros is +0 (the sign decides atan2(0, a) = 0 or pi)
__device__ __forceinline__ float sum3_cpu(const f3 v) { return __fadd_rn(__fadd_rn(__fadd_rn(0.f, v.x), v.y), v.z); }
__device__ __forceinline__ float norm3_cpu(const f3 v) {
  return __fsqrt_rn(__fmaf_rn(v.z, v.z, __fmaf_rn(v.y, v.y, __fmul_rn(v.x, v.x))));
}
__device__ __forceinline__ float sq_dist(const f3 a, const f3 b) {
  const f3 d = sub3(a, b);
  return sum3_cpu(mul3(d, d));
}
__device__ __forceinline__ float atan2_rn(float y, float x) { return (float)atan2((double)y, (double)x); }
__device__ __forceinline__ f3 shfl3(const f3 v, int src) {
  return {__shfl_sync(0xffffffffu, v.x, src), __shfl_sync(0xffffffffu, v.y, src), __shfl_sync(0xffffffffu, v.z, src)};
}
__device__ __forceinline__ unsigned long long warp_min(unsigned long long k) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, k, o);
    k = other < k ? other : k;
  }
  return k;
}
// (squared distance, index) as one ordered key: non-negative floats order as their bit patterns.
__device__ __forceinline__ unsigned long long dist_key(float d, int idx) {
  return ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)idx;
}

__global__ void __launch_bounds__(32 * kWarps) gen_traj_kernel(
    const int64_t* __restrict__ atom_type, const float* __restrict__ pos, const int64_t* __restrict__ con,
    const int64_t* __restrict__ ptr, int64_t n_mols, int64_t* __restrict__ out_type, float* __restrict__ out_pos,
    int64_t* __restrict__ out_batch, float* __restrict__ out_cannot_focus, int64_t* __restrict__ out_focus,
    int64_t* __restrict__ out_c1, int64_t* __restrict__ out_c2, int64_t* __restrict__ out_new_type,
    double* __restrict__ out_dist, double* __restrict__ out_angle, double* __restrict__ out_torsion,
    int32_t* __restrict__ status) {
  const int64_t m = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (m >= n_mols) return;
  const int lane = threadIdx.x & 31;
  const int64_t* atoms_ptr = ptr;
  const int64_t* mat_ptr = ptr + (n_mols + 1);
  const int64_t* row_ptr = ptr + 2 * (n_mols + 1);
  const int64_t* step_ptr = ptr + 3 * (n_mols + 1);
  const int64_t* angle_ptr = ptr + 4 * (n_mols + 1);
  const int64_t* torsion_ptr = ptr + 5 * (n_mols + 1);
  const int64_t a0 = atoms_ptr[m];
  const int n = (int)(atoms_ptr[m + 1] - a0);
  const bool active = lane < n;

  f3 p = {0.f, 0.f, 0.f};
  if (active) p = load3(pos + 3 * a0, lane);

  // ---- Prim's tree: the generation order, and the tree position of each new node's focus
  const unsigned long long kNone = ~0ull;
  bool in_tree = lane == 0;
  float key_w = 0.f;
  int key_t = -1;                       // tree position of the best tree node, -1: no edge yet
  int my_node = 0, my_focus = 0;        // lane t: node added at tree position t, and its focus's tree position
  int v = 0;
  for (int t = 1; t < n; ++t) {
    const f3 pv = shfl3(p, v);
    if (active && !in_tree) {
      const float s = sq_dist(pv, p);
      if (s != 0.f && (key_t < 0 || s < key_w)) {
        key_w = s;
        key_t = t - 1;
      }
    }
    const unsigned long long cand = (active && !in_tree && key_t >= 0)
        ? ((unsigned long long)__float_as_uint(key_w) << 32) | ((unsigned)key_t << 5) | (unsigned)lane
        : kNone;
    const unsigned long long best = warp_min(cand);
    if (best == kNone) {                // the graph has no edge out of the tree: all atoms coincide
      if (lane == 0) status[m] = 1;
      return;
    }
    v = (int)(best & 31);
    if (lane == v) in_tree = true;
    if (lane == t) {
      my_node = v;
      my_focus = (int)((best >> 5) & 31);
    }
  }
  if (n < 2) {                          // one atom: no tree edge, as the reference's zip(*edges) fails
    if (lane == 0) status[m] = 1;
    return;
  }
  if (lane == 0) status[m] = 0;

  // ---- lane j now holds the atom at generation position j
  const int node = my_node;
  const f3 q = shfl3(p, node);
  p = q;
  int64_t type = 0, valency = 0;
  const int64_t* con_row = con + mat_ptr[m] + (int64_t)node * n;
  if (active) {
    type = atom_type[a0 + node];
    for (int k = 0; k < n; ++k) valency += con_row[k];
  }
  int64_t partial = 0;

  const int64_t r0 = row_ptr[m], s0 = step_ptr[m], g0 = angle_ptr[m], h0 = torsion_ptr[m];
  for (int i = 0; i < n - 1; ++i) {
    const int node_i = __shfl_sync(0xffffffffu, node, i);
    if (active) partial += con_row[node_i];
    const int64_t off = (int64_t)i * (i + 1) / 2;
    if (lane <= i) {
      const int64_t r = r0 + off + lane;
      out_type[r] = type;
      out_pos[3 * r] = p.x;
      out_pos[3 * r + 1] = p.y;
      out_pos[3 * r + 2] = p.z;
      out_batch[r] = i;
      out_cannot_focus[r] = partial == valency ? 1.f : 0.f;
    }
    const int f = __shfl_sync(0xffffffffu, my_focus, i + 1);
    const f3 pf = shfl3(p, f), pn = shfl3(p, i + 1);
    const int64_t type_new = __shfl_sync(0xffffffffu, type, i + 1);
    if (lane == 0) {
      out_focus[s0 + i] = f + off;
      out_new_type[s0 + i] = type_new;
      out_dist[s0 + i] = (double)norm3_cpu(sub3(pn, pf));
    }
    if (i == 0) continue;
    // c1: first atom k <= i, k != f, of least squared distance to the focus (torch.argmin over the masked row)
    const unsigned long long k1 = (lane <= i && lane != f) ? dist_key(sq_dist(pf, p), lane) : kNone;
    const int c1 = (int)(warp_min(k1) & 31);
    const f3 pc1 = shfl3(p, c1);
    if (lane == 0) {
      out_c1[2 * (g0 + i - 1)] = c1 + off;
      out_c1[2 * (g0 + i - 1) + 1] = f + off;
      const f3 u = sub3(pc1, pf), w = sub3(pn, pf);
      const float a = sum3_cpu(mul3(u, w));
      const float b = norm3_cpu(cross_aten(u, w));
      out_angle[g0 + i - 1] = (double)atan2_rn(b, a);
    }
    if (i == 1) continue;
    const unsigned long long k2 = (lane <= i && lane != f && lane != c1) ? dist_key(sq_dist(pc1, p), lane) : kNone;
    const int c2 = (int)(warp_min(k2) & 31);
    const f3 pc2 = shfl3(p, c2);
    if (lane == 0) {
      const int64_t row = 3 * (h0 + i - 2);
      out_c2[row] = c2 + off;
      out_c2[row + 1] = c1 + off;
      out_c2[row + 2] = f + off;
      const f3 fc = sub3(pf, pc1);
      const f3 plane1 = cross_aten(fc, sub3(pn, pc1));
      const f3 plane2 = cross_aten(fc, sub3(pc2, pc1));
      const float a = sum3_cpu(mul3(plane1, plane2));
      const float b = __fdiv_rn(sum3_cpu(mul3(cross_aten(plane1, plane2), fc)), norm3_cpu(fc));
      double t = (double)atan2_rn(b, a);
      if (t <= 0.0) t += kTwoPi;        // the float64 steps_torsion tensor: the shift is an fp64 add
      out_torsion[h0 + i - 2] = t;
    }
  }
}

}  // namespace

extern "C" {

int dig3d_gen_traj(const int64_t* atom_type, const float* pos, const int64_t* con, const int64_t* ptr, int64_t n_mols,
                   int64_t* out_type, float* out_pos, int64_t* out_batch, float* out_cannot_focus, int64_t* out_focus,
                   int64_t* out_c1, int64_t* out_c2, int64_t* out_new_type, double* out_dist, double* out_angle,
                   double* out_torsion, int32_t* status, void* stream) {
  DIG3D_REQUIRE(n_mols >= 0 && (n_mols == 0 || (atom_type && pos && con && ptr && out_type && out_pos && out_batch &&
                                                 out_cannot_focus && out_focus && out_c1 && out_c2 && out_new_type &&
                                                 out_dist && out_angle && out_torsion && status)),
                "gen_traj: bad arguments (n_mols >= 0, every pointer set)");
  DIG3D_REQUIRE((n_mols + kWarps - 1) / kWarps < (1ll << 31), "gen_traj: too many molecules (%lld)",
                (long long)n_mols);
  if (n_mols == 0) return DIG3D_OK;
  gen_traj_kernel<<<ceil_div(n_mols, kWarps), 32 * kWarps, 0, (cudaStream_t)stream>>>(
      atom_type, pos, con, ptr, n_mols, out_type, out_pos, out_batch, out_cannot_focus, out_focus, out_c1, out_c2,
      out_new_type, out_dist, out_angle, out_torsion, status);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
