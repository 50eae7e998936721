// Position gradients (forces = -dE/dpos, reference run.py:126,165: torch.autograd.grad(out, pos)) for the geometry
// the models read: edge lengths (all models) and triplet angles (DimeNet++ / SphereNet), plus the SchNet edge features.
//
//   edge_dist_bwd        dist[e] = |pos_i - pos_j|                         schnet.py:158, geometric_computing.py:23
//   triplet_angle_bwd    angle[t] = atan2(|ji x jk|, ji . jk)              geometric_computing.py:43-48
//   schnet_edge_features_bwd / rowdot                                        schnet.py:24-33,92-94
//
//   triplet_torsion_bwd  torsion[t] = min_c dihedral(k, j->i, c)              geometric_computing.py:53-75
#include "common.cuh"
#include "dual.cuh"

namespace dig3d {

__device__ __forceinline__ f3 scale3(const f3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ f3 add3(const f3 a, const f3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ f3 cross3(const f3 a, const f3 b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
__device__ __forceinline__ void atomic_add3(float* __restrict__ p, int n, const f3 v) {
  atomicAdd(p + 3 * n, v.x);
  atomicAdd(p + 3 * n + 1, v.y);
  atomicAdd(p + 3 * n + 2, v.z);
}
__device__ __forceinline__ f3 warp_sum3(f3 v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
    v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
    v.z += __shfl_xor_sync(0xffffffffu, v.z, o);
  }
  return v;
}

// dpos[i] += ddist * (pos_i - pos_j) / dist ; dpos[j] -= the same.  Edges are sorted by target, so a warp's 32 edges
// mostly share the target: atomics on 3 floats per endpoint (E is small next to T).
__global__ void edge_dist_bwd_kernel(const float* __restrict__ pos, const int32_t* __restrict__ src,
                                     const int32_t* __restrict__ dst, const float* __restrict__ dist,
                                     const float* __restrict__ ddist, int n_edges, float* __restrict__ dpos) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const float d = dist[e];
  if (d == 0.f) return;                              // norm backward at 0: zero subgradient (torch)
  const int j = src[e], i = dst[e];
  const f3 u = scale3(sub3(load3(pos, i), load3(pos, j)), ddist[e] / d);
  atomic_add3(dpos, i, u);
  atomic_add3(dpos, j, scale3(u, -1.f));
}

// One warp per (j -> i) edge, lanes over the in-neighbours k of j (same enumeration as triplet_geometry_kernel).
// With u = pos_i - pos_j, v = pos_k - pos_j, a = u.v, w = u x v, b = |w|:  theta = atan2(b, a),
//   dtheta/da = -b / (a^2 + b^2),  dtheta/db = a / (a^2 + b^2),  db/du = v x w_hat,  db/dv = w_hat x u.
// The contributions to i and j are reduced over the warp (one atomic triple per edge), k gets its own atomics.
__global__ void __launch_bounds__(256)
triplet_angle_bwd_kernel(const float* __restrict__ pos, const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                         const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ trip_ptr,
                         const float* __restrict__ dangle, int n_edges, float* __restrict__ dpos) {
  const int lane = threadIdx.x & 31;
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (e >= n_edges) return;
  const int j = src[e], i = dst[e];
  const int base = row_ptr[j], d = row_ptr[j + 1] - base;
  int p_i = d;
  for (int s0 = 0; s0 < d; s0 += 32) {
    const int sl = s0 + lane;
    const unsigned hit = __ballot_sync(0xffffffffu, sl < d && src[base + sl] == i);
    if (hit) p_i = s0 + __ffs(hit) - 1;
  }
  const f3 pj = load3(pos, j);
  const f3 u = sub3(load3(pos, i), pj);
  const int t0 = trip_ptr[e];
  f3 gi = {0.f, 0.f, 0.f};
  for (int s = lane; s < d; s += 32) {
    if (s == p_i) continue;
    const int k = src[base + s];
    const float g = dangle[t0 + s - (s > p_i ? 1 : 0)];
    const f3 v = sub3(load3(pos, k), pj);
    const float a = u.x * v.x + u.y * v.y + u.z * v.z;
    const f3 w = cross3(u, v);
    const float b = sqrtf(w.x * w.x + w.y * w.y + w.z * w.z);
    const float den = a * a + b * b;
    if (den == 0.f) continue;
    const float ga = -b / den * g, gb = a / den * g;
    f3 gu = scale3(v, ga), gv = scale3(u, ga);
    if (b > 0.f) {
      const f3 wh = scale3(w, 1.0f / b);
      gu = add3(gu, scale3(cross3(v, wh), gb));
      gv = add3(gv, scale3(cross3(wh, u), gb));
    }
    gi = add3(gi, gu);
    atomic_add3(dpos, k, gv);
    atomic_add3(dpos, j, scale3(add3(gu, gv), -1.f));
  }
  gi = warp_sum3(gi);
  if (lane == 0) atomic_add3(dpos, i, gi);
}


// torsion[t] = min over the in-neighbours c != i of j of atan2(((p1 x p2) . u) / |u|, p1 . p2) (<= 0 -> + 2 pi), with
// u = pos_i - pos_j, p1 = u x (pos_k - pos_j), p2 = u x (pos_c - pos_j)            geometric_computing.py:53-75.
// The gradient flows through the minimising candidate only (torch.min / scatter_min backward).  The planes are
// recomputed with the forward's ATen rounding so that the same candidate wins.
constexpr int TGEO_WARPS = 8;
constexpr int TGEO_MAXDEG = 64;

__global__ void __launch_bounds__(TGEO_WARPS * 32)
triplet_torsion_bwd_kernel(const float* __restrict__ pos, const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                           const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ trip_ptr,
                           const float* __restrict__ dtorsion, int n_edges, float* __restrict__ dpos) {
  __shared__ float planes[TGEO_WARPS][TGEO_MAXDEG][3];
  __shared__ int32_t ks[TGEO_WARPS][TGEO_MAXDEG];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int e = blockIdx.x * TGEO_WARPS + w;
  if (e >= n_edges) return;
  const int j = src[e], i = dst[e];
  const int base = row_ptr[j], d = min(row_ptr[j + 1] - base, TGEO_MAXDEG);
  const f3 pj = load3(pos, j);
  const f3 u = sub3(load3(pos, i), pj);
  const float n = norm3_aten(u);
  for (int s = lane; s < d; s += 32) {
    const int k = src[base + s];
    ks[w][s] = k;
    const f3 pl = cross_aten(u, sub3(load3(pos, k), pj));
    planes[w][s][0] = pl.x; planes[w][s][1] = pl.y; planes[w][s][2] = pl.z;
  }
  __syncwarp();
  int p_i = d;
  for (int s = 0; s < d; ++s) if (ks[w][s] == i) p_i = s;
  const int t0 = trip_ptr[e];
  f3 gi = {0.f, 0.f, 0.f}, gj = {0.f, 0.f, 0.f};
  for (int s = lane; s < d; s += 32) {
    if (s == p_i) continue;
    const float g = dtorsion[t0 + s - (s > p_i ? 1 : 0)];
    const f3 p1 = {planes[w][s][0], planes[w][s][1], planes[w][s][2]};
    float best = __int_as_float(0x7f800000), bta = 1.f, btb = 0.f;
    int bc = -1;
    for (int c = 0; c < d; ++c) {
      if (c == p_i) continue;
      const f3 p2 = {planes[w][c][0], planes[w][c][1], planes[w][c][2]};
      const float ta = sum3_aten(mul3(p1, p2));
      const float tb = __fdiv_rn(sum3_aten(mul3(cross_aten(p1, p2), u)), n);
      float tor = atan2f(tb, ta);
      if (tor <= 0.0f) tor = __fadd_rn(tor, 6.2831855f);
      if (tor < best) { best = tor; bc = c; bta = ta; btb = tb; }
    }
    const float den = bta * bta + btb * btb;
    if (bc < 0 || den == 0.f || g == 0.f) continue;
    const float g_ta = -btb / den * g, g_tb = bta / den * g;
    const f3 p2 = {planes[w][bc][0], planes[w][bc][1], planes[w][bc][2]};
    const f3 q = cross3(p1, p2);
    const float sq = q.x * u.x + q.y * u.y + q.z * u.z;
    const float g_s = g_tb / n, g_n = -g_tb * sq / (n * n);
    f3 g_p1 = scale3(p2, g_ta), g_p2 = scale3(p1, g_ta);
    const f3 g_q = scale3(u, g_s);
    f3 g_u = add3(scale3(q, g_s), scale3(u, g_n / n));
    g_p1 = add3(g_p1, cross3(p2, g_q));
    g_p2 = add3(g_p2, cross3(g_q, p1));
    const int k = ks[w][s], c = ks[w][bc];
    const f3 vk = sub3(load3(pos, k), pj), vc = sub3(load3(pos, c), pj);
    g_u = add3(g_u, add3(cross3(vk, g_p1), cross3(vc, g_p2)));
    const f3 g_vk = cross3(g_p1, u), g_vc = cross3(g_p2, u);
    atomic_add3(dpos, k, g_vk);
    atomic_add3(dpos, c, g_vc);
    gi = add3(gi, g_u);
    gj = add3(gj, add3(g_u, add3(g_vk, g_vc)));
  }
  gi = warp_sum3(gi);
  gj = warp_sum3(gj);
  if (lane == 0) {
    atomic_add3(dpos, i, gi);
    atomic_add3(dpos, j, scale3(gj, -1.f));
  }
}

// ddist[e] = sum_g dgauss[e,g] * gauss[e,g] * 2 coeff (d - mu_g)  +  dcut[e] * (-0.5 sin(d pi / c) pi / c)
__global__ void schnet_edge_features_bwd_kernel(const float* __restrict__ dist, int64_t n_edges,
                                                const float* __restrict__ offset, int n_gauss, float coeff,
                                                float inv_cutoff, const float* __restrict__ dgauss,
                                                const float* __restrict__ dcut, float* __restrict__ ddist) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const float d = dist[e];
  float acc = 0.f;
  if (dgauss)
    for (int g = 0; g < n_gauss; ++g) {
      const float t = d - __ldg(offset + g);
      acc = fmaf(dgauss[e * n_gauss + g], expf(coeff * t * t) * 2.0f * coeff * t, acc);
    }
  if (dcut) {
    const float w = 3.14159274101257324f * inv_cutoff;
    acc = fmaf(dcut[e], -0.5f * sinf(d * w) * w, acc);
  }
  ddist[e] = acc;
}


// ---- second order (force TRAINING: loss.backward() through forces taken with create_graph=True, run.py:110-123) ----
// Backward of edge_dist_bwd, i.e. of  dpos = sum_e ddist_e (+u_e at i, -u_e at j),  u_e = (pos_i - pos_j) / d_e,
// given G = d(loss)/d(dpos) [N,3]:   with w_e = G_i - G_j
//   d(ddist)_e = u_e . w_e ;   d(pos_i) += ddist_e (w_e - (u_e . w_e) u_e) / d_e ,  d(pos_j) -= the same.
__global__ void edge_dist_bwd2_kernel(const float* __restrict__ pos, const int32_t* __restrict__ src,
                                      const int32_t* __restrict__ dst, const float* __restrict__ dist,
                                      const float* __restrict__ ddist, const float* __restrict__ G, int n_edges,
                                      float* __restrict__ d_ddist, float* __restrict__ d_pos) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const float d = dist[e];
  if (d == 0.f) { d_ddist[e] = 0.f; return; }
  const int j = src[e], i = dst[e];
  const f3 u = scale3(sub3(load3(pos, i), load3(pos, j)), 1.0f / d);
  const f3 w = sub3(load3(G, i), load3(G, j));
  const float uw = u.x * w.x + u.y * w.y + u.z * w.z;
  d_ddist[e] = uw;
  const f3 h = scale3(add3(w, scale3(u, -uw)), ddist[e] / d);
  atomic_add3(d_pos, i, h);
  atomic_add3(d_pos, j, scale3(h, -1.f));
}

// Backward of schnet_edge_features_bwd (ddist = sum_g dgauss gauss' + dcut cut') given g = d(loss)/d(ddist) [E]:
//   d(dgauss)[e,k] = g_e gauss_k'(d_e),  d(dcut)[e] = g_e cut'(d_e),  d(dist)[e] = g_e (sum_k dgauss gauss_k'' + dcut cut'')
//   gauss = exp(c t^2), t = d - mu:  gauss' = 2 c t gauss,  gauss'' = (2c + 4 c^2 t^2) gauss;   cut = 0.5 (cos(d w) + 1), w = pi / cutoff
__global__ void schnet_edge_features_bwd2_kernel(const float* __restrict__ dist, int64_t n_edges,
                                                 const float* __restrict__ offset, int n_gauss, float coeff,
                                                 float inv_cutoff, const float* __restrict__ dgauss,
                                                 const float* __restrict__ dcut, const float* __restrict__ g,
                                                 float* __restrict__ d_dgauss, float* __restrict__ d_dcut,
                                                 float* __restrict__ d_dist) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const float d = dist[e], ge = g[e];
  float acc = 0.f;
  for (int k = 0; k < n_gauss; ++k) {
    const float t = d - __ldg(offset + k);
    const float ga = expf(coeff * t * t);
    const float g1 = 2.0f * coeff * t * ga;
    if (d_dgauss) d_dgauss[e * n_gauss + k] = ge * g1;
    if (dgauss) acc = fmaf(dgauss[e * n_gauss + k], (2.0f * coeff + 4.0f * coeff * coeff * t * t) * ga, acc);
  }
  const float w = 3.14159274101257324f * inv_cutoff;
  if (d_dcut) d_dcut[e] = ge * (-0.5f * w * sinf(d * w));
  if (dcut) acc = fmaf(dcut[e], -0.5f * w * w * cosf(d * w), acc);
  d_dist[e] = ge * acc;
}

// out[r] = sum_c a[r, c] * b[r, c]   (one warp per row)
__global__ void rowdot_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t rows, int width,
                              float* __restrict__ out) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  float acc = 0.f;
  for (int c = lane; c < width; c += 32) acc = fmaf(a[r * width + c], b[r * width + c], acc);
#pragma unroll
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) out[r] = acc;
}

// ---------------------------------------------------------------------------------- forward-mode geometry (force training)
// Training ON forces (reference run.py:110-123) needs d/d(theta) of  c . dE/dpos  for a fixed per-atom vector c; that is
// the parameter gradient of the DIRECTIONAL derivative of E along c (dig_b200/autograd_jvp.py).  The geometry side of
// that derivative is first order: the tangents of dist / angle / torsion along c,
//   dist_dot[e] = u_hat . (c_i - c_j),   angle_dot[t] = g_u . (c_i - c_j) + g_v . (c_k - c_j),   torsion_dot[t] likewise
// with exactly the per-triplet gradients g_u, g_v, ... the backward kernels above scatter (so J c and J^T w agree to
// rounding; tests check <J c, w> = <c, J^T w>).  One thread per edge / one warp per (j -> i) edge, same enumeration.
__global__ void edge_dist_jvp_kernel(const float* __restrict__ pos, const float* __restrict__ cvec,
                                     const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                     const float* __restrict__ dist, int n_edges, float* __restrict__ dist_dot) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const float d = dist[e];
  if (d == 0.f) { dist_dot[e] = 0.f; return; }
  const int j = src[e], i = dst[e];
  const f3 u = sub3(load3(pos, i), load3(pos, j)), dc = sub3(load3(cvec, i), load3(cvec, j));
  dist_dot[e] = (u.x * dc.x + u.y * dc.y + u.z * dc.z) / d;
}

__device__ __forceinline__ float dot3(const f3 a, const f3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

__global__ void __launch_bounds__(256)
triplet_angle_jvp_kernel(const float* __restrict__ pos, const float* __restrict__ cvec, const int32_t* __restrict__ src,
                         const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                         const int32_t* __restrict__ trip_ptr, int n_edges, float* __restrict__ angle_dot) {
  const int lane = threadIdx.x & 31;
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (e >= n_edges) return;
  const int j = src[e], i = dst[e];
  const int base = row_ptr[j], d = row_ptr[j + 1] - base;
  int p_i = d;
  for (int s0 = 0; s0 < d; s0 += 32) {
    const int sl = s0 + lane;
    const unsigned hit = __ballot_sync(0xffffffffu, sl < d && src[base + sl] == i);
    if (hit) p_i = s0 + __ffs(hit) - 1;
  }
  const f3 pj = load3(pos, j), cj = load3(cvec, j);
  const f3 u = sub3(load3(pos, i), pj), cu = sub3(load3(cvec, i), cj);
  const int t0 = trip_ptr[e];
  for (int s = lane; s < d; s += 32) {
    if (s == p_i) continue;
    const int k = src[base + s];
    const f3 v = sub3(load3(pos, k), pj), cv = sub3(load3(cvec, k), cj);
    const float a = dot3(u, v);
    const f3 w = cross3(u, v);
    const float b = sqrtf(dot3(w, w));
    const float den = a * a + b * b;
    float out = 0.f;
    if (den != 0.f) {
      const float ga = -b / den, gb = a / den;
      f3 gu = scale3(v, ga), gv = scale3(u, ga);
      if (b > 0.f) {
        const f3 wh = scale3(w, 1.0f / b);
        gu = add3(gu, scale3(cross3(v, wh), gb));
        gv = add3(gv, scale3(cross3(wh, u), gb));
      }
      out = dot3(gu, cu) + dot3(gv, cv);
    }
    angle_dot[t0 + s - (s > p_i ? 1 : 0)] = out;
  }
}

__global__ void __launch_bounds__(TGEO_WARPS * 32)
triplet_torsion_jvp_kernel(const float* __restrict__ pos, const float* __restrict__ cvec, const int32_t* __restrict__ src,
                           const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                           const int32_t* __restrict__ trip_ptr, int n_edges, float* __restrict__ torsion_dot) {
  __shared__ float planes[TGEO_WARPS][TGEO_MAXDEG][3];
  __shared__ int32_t ks[TGEO_WARPS][TGEO_MAXDEG];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int e = blockIdx.x * TGEO_WARPS + w;
  if (e >= n_edges) return;
  const int j = src[e], i = dst[e];
  const int base = row_ptr[j], d = min(row_ptr[j + 1] - base, TGEO_MAXDEG);
  const f3 pj = load3(pos, j), cj = load3(cvec, j);
  const f3 u = sub3(load3(pos, i), pj), cu = sub3(load3(cvec, i), cj);
  const float n = norm3_aten(u);
  for (int s = lane; s < d; s += 32) {
    const int k = src[base + s];
    ks[w][s] = k;
    const f3 pl = cross_aten(u, sub3(load3(pos, k), pj));
    planes[w][s][0] = pl.x; planes[w][s][1] = pl.y; planes[w][s][2] = pl.z;
  }
  __syncwarp();
  int p_i = d;
  for (int s = 0; s < d; ++s) if (ks[w][s] == i) p_i = s;
  const int t0 = trip_ptr[e];
  for (int s = lane; s < d; s += 32) {
    if (s == p_i) continue;
    const f3 p1 = {planes[w][s][0], planes[w][s][1], planes[w][s][2]};
    float best = __int_as_float(0x7f800000), bta = 1.f, btb = 0.f;
    int bc = -1;
    for (int c = 0; c < d; ++c) {              // same candidate search (and rounding) as the forward / backward kernels
      if (c == p_i) continue;
      const f3 p2 = {planes[w][c][0], planes[w][c][1], planes[w][c][2]};
      const float ta = sum3_aten(mul3(p1, p2));
      const float tb = __fdiv_rn(sum3_aten(mul3(cross_aten(p1, p2), u)), n);
      float tor = atan2f(tb, ta);
      if (tor <= 0.0f) tor = __fadd_rn(tor, 6.2831855f);
      if (tor < best) { best = tor; bc = c; bta = ta; btb = tb; }
    }
    const float den = bta * bta + btb * btb;
    float out = 0.f;
    if (bc >= 0 && den != 0.f) {
      const float g_ta = -btb / den, g_tb = bta / den;
      const f3 p2 = {planes[w][bc][0], planes[w][bc][1], planes[w][bc][2]};
      const f3 q = cross3(p1, p2);
      const float sq = dot3(q, u);
      const float g_s = g_tb / n, g_n = -g_tb * sq / (n * n);
      f3 g_p1 = scale3(p2, g_ta), g_p2 = scale3(p1, g_ta);
      const f3 g_q = scale3(u, g_s);
      f3 g_u = add3(scale3(q, g_s), scale3(u, g_n / n));
      g_p1 = add3(g_p1, cross3(p2, g_q));
      g_p2 = add3(g_p2, cross3(g_q, p1));
      const int k = ks[w][s], c = ks[w][bc];
      const f3 vk = sub3(load3(pos, k), pj), vc = sub3(load3(pos, c), pj);
      g_u = add3(g_u, add3(cross3(vk, g_p1), cross3(vc, g_p2)));
      const f3 g_vk = cross3(g_p1, u), g_vc = cross3(g_p2, u);
      out = dot3(g_u, cu) + dot3(g_vk, sub3(load3(cvec, k), cj)) + dot3(g_vc, sub3(load3(cvec, c), cj));
    }
    torsion_dot[t0 + s - (s > p_i ? 1 : 0)] = out;
  }
}

// ------------------------------------------------------------------------------ xyz_to_dat's derivatives, any in-degree
// The triplets of xyz_to_dat(..., use_torsion=True) with `tors_arg` (dig3d_triplet_geometry_any_degree_arg): the torsion
// of triplet t = (k -> j -> i) is the candidate in slot tors_arg[t] of j's in-edges, c = src[row_ptr[j] + tors_arg[t]],
// so no kernel below searches for it again.
//
// The per-triplet gradients are written once, templated on the scalar: float gives the gradient, `dual` (value and
// tangent) evaluated with the tangent seeded by G gives, in the same pass, the gradient's value (<grad, G> is the JVP)
// and its directional derivative along G (the Hessian-vector product H G).  Conventions (DESIGN.md §6): a collinear
// angle (|ji x jk| = 0) keeps only the atan2 term in a = ji . jk, whose coefficient -b / (a^2 + b^2) is then 0, and the
// tangent of |w| at w = 0 is taken as 0; a^2 + b^2 = 0 and |ji| = 0 pass nothing; the self candidate c = k is the
// constant 2 pi or its rounding residue (plane1 x plane1) and passes nothing.  The derivative kernels of the models
// (triplet_angle_bwd_kernel above, shared and unchanged) form cross products with ATen's fused rounding instead.
// `dual` and its arithmetic: dual.cuh.
template <typename T>
struct v3 {
  T x, y, z;
};
template <typename T>
__device__ __forceinline__ v3<T> operator+(const v3<T> a, const v3<T> b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <typename T>
__device__ __forceinline__ v3<T> operator*(const v3<T> a, const T s) { return {a.x * s, a.y * s, a.z * s}; }
template <typename T>
__device__ __forceinline__ T dot(const v3<T> a, const v3<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
// The cross product's value from separately rounded products (no FMA contraction): exactly parallel copies of a vector
// (an atom at the same position as another) then give exactly 0, so the conventions for a zero cross product apply.
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ dual mul_rn(dual a, dual b) { return {__fmul_rn(a.v, b.v), a.d * b.v + a.v * b.d}; }
template <typename T>
__device__ __forceinline__ v3<T> cross(const v3<T> a, const v3<T> b) {
  return {mul_rn(a.y, b.z) - mul_rn(a.z, b.y), mul_rn(a.z, b.x) - mul_rn(a.x, b.z), mul_rn(a.x, b.y) - mul_rn(a.y, b.x)};
}

// theta = atan2(b, a), a = u . v, w = u x v, b = |w|  ->  (d theta / du, d theta / dv); false: passes nothing.
template <typename T>
__device__ __forceinline__ bool angle_grad(const v3<T> u, const v3<T> v, v3<T>& g_u, v3<T>& g_v) {
  const T a = dot(u, v);
  const v3<T> w = cross(u, v);
  const T b = sqrt_t(dot(w, w));
  const T den = a * a + b * b;
  if (val(den) == 0.f) return false;
  const T ga = -b / den, gb = a / den;
  g_u = v * ga;
  g_v = u * ga;
  if (val(b) > 0.f) {
    const v3<T> wh = w * (T{1.f} / b);
    g_u = g_u + cross(v, wh) * gb;
    g_v = g_v + cross(wh, u) * gb;
  }
  return true;
}

// tau = atan2(tb, ta), p1 = u x vk, p2 = u x vc, ta = p1 . p2, tb = ((p1 x p2) . u) / |u|
//   -> (d tau / du, d tau / dvk, d tau / dvc); false: passes nothing.
template <typename T>
__device__ __forceinline__ bool torsion_grad(const v3<T> u, const v3<T> vk, const v3<T> vc, v3<T>& g_u, v3<T>& g_vk,
                                             v3<T>& g_vc) {
  const T n = sqrt_t(dot(u, u));
  if (val(n) == 0.f) return false;
  const v3<T> p1 = cross(u, vk), p2 = cross(u, vc);
  const T ta = dot(p1, p2);
  const v3<T> q = cross(p1, p2);
  const T tb = dot(q, u) / n;
  const T den = ta * ta + tb * tb;
  if (val(den) == 0.f) return false;
  const T g_ta = -tb / den, g_tb = ta / den;
  const T g_s = g_tb / n;                           // d tau / d (q . u)
  const T g_n = -(g_tb * tb) / n;                   // d tau / d |u| (tb = (q . u) / |u|)
  const v3<T> g_q = u * g_s;                        // (p1 x p2) . g_q = p1 . (p2 x g_q) = p2 . (g_q x p1)
  const v3<T> g_p1 = p2 * g_ta + cross(p2, g_q);
  const v3<T> g_p2 = p1 * g_ta + cross(g_q, p1);
  g_u = q * g_s + u * (g_n / n) + cross(vk, g_p1) + cross(vc, g_p2);
  g_vk = cross(g_p1, u);
  g_vc = cross(g_p2, u);
  return true;
}

__device__ __forceinline__ v3<float> to_v3(const f3 a) { return {a.x, a.y, a.z}; }
__device__ __forceinline__ f3 to_f3(const v3<float> a) { return {a.x, a.y, a.z}; }
__device__ __forceinline__ v3<dual> to_dual(const f3 a, const f3 da) {
  return {{a.x, da.x}, {a.y, da.y}, {a.z, da.z}};
}
__device__ __forceinline__ f3 value3(const v3<dual> a) { return {a.x.v, a.y.v, a.z.v}; }
__device__ __forceinline__ f3 tangent3(const v3<dual> a) { return {a.x.d, a.y.d, a.z.d}; }

// Slot of i among j's in-edges (d if absent), one ballot per 32 slots: triplet tt of edge (j -> i) is slot
// s = tt + (tt >= p_i) of j's in-edges.
__device__ __forceinline__ int slot_of(const int32_t* __restrict__ src, int base, int d, int i, int lane) {
  int p_i = d;
  for (int s0 = 0; s0 < d; s0 += 32) {
    const int sl = s0 + lane;
    const unsigned hit = __ballot_sync(0xffffffffu, sl < d && src[base + sl] == i);
    if (hit) { p_i = s0 + __ffs(hit) - 1; break; }
  }
  return p_i;
}

// dpos of sum_t dtorsion[t] torsion[t], any in-degree: one warp per edge e = (j -> i), lanes over its triplets.  The i
// and j parts are summed over the warp (one atomic triple each per edge); k and c get atomics.
__global__ void __launch_bounds__(256)
triplet_torsion_bwd_arg_kernel(const float* __restrict__ pos, const int32_t* __restrict__ src,
                               const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                               const int32_t* __restrict__ trip_ptr, const int32_t* __restrict__ tors_arg,
                               const float* __restrict__ dtorsion, int n_edges, float* __restrict__ dpos) {
  const int lane = threadIdx.x & 31;
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (e >= n_edges) return;
  const int j = src[e], i = dst[e];
  const int base = row_ptr[j], d = row_ptr[j + 1] - base;
  const int t0 = trip_ptr[e], nt = trip_ptr[e + 1] - t0;
  if (nt == 0) return;
  const int p_i = slot_of(src, base, d, i, lane);
  const f3 pj = load3(pos, j);
  const v3<float> u = to_v3(sub3(load3(pos, i), pj));
  f3 gi = {0.f, 0.f, 0.f}, gj = {0.f, 0.f, 0.f};
  for (int tt = lane; tt < nt; tt += 32) {
    const int s = tt + (tt >= p_i ? 1 : 0), a = tors_arg[t0 + tt];
    const float g = dtorsion[t0 + tt];
    if (a < 0 || a == s || g == 0.f) continue;
    const int k = src[base + s], c = src[base + a];
    v3<float> g_u, g_vk, g_vc;
    if (!torsion_grad(u, to_v3(sub3(load3(pos, k), pj)), to_v3(sub3(load3(pos, c), pj)), g_u, g_vk, g_vc)) continue;
    const f3 hk = to_f3(g_vk * g), hc = to_f3(g_vc * g), hu = to_f3(g_u * g);
    atomic_add3(dpos, k, hk);
    atomic_add3(dpos, c, hc);
    gi = add3(gi, hu);
    gj = add3(gj, add3(hu, add3(hk, hc)));
  }
  gi = warp_sum3(gi);
  gj = warp_sum3(gj);
  if (lane == 0) {
    atomic_add3(dpos, i, gi);
    atomic_add3(dpos, j, scale3(gj, -1.f));
  }
}

// Backward of (triplet_angle_bwd + triplet_torsion_bwd_arg), i.e. of dpos = sum_t dangle_t grad angle_t + dtorsion_t
// grad torsion_t, given G = d(loss) / d(dpos) [N, 3]:
//   d_dangle[t] = <grad angle_t, G>,  d_dtorsion[t] = <grad torsion_t, G>,
//   d_pos += dangle_t H_angle_t G + dtorsion_t H_torsion_t G.
// dangle / dtorsion null: that term is absent (its Hessian term is zero; d_dangle / d_dtorsion are still written when
// given).  Same warp-per-edge layout as triplet_torsion_bwd_arg_kernel; d_dangle / d_dtorsion are written for every
// triplet (0 where the conventions pass nothing).
__global__ void __launch_bounds__(256)
triplet_geometry_bwd2_kernel(const float* __restrict__ pos, const int32_t* __restrict__ src,
                             const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                             const int32_t* __restrict__ trip_ptr, const int32_t* __restrict__ tors_arg,
                             const float* __restrict__ dangle, const float* __restrict__ dtorsion,
                             const float* __restrict__ G, int n_edges, float* __restrict__ d_dangle,
                             float* __restrict__ d_dtorsion, float* __restrict__ d_pos) {
  const int lane = threadIdx.x & 31;
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (e >= n_edges) return;
  const int j = src[e], i = dst[e];
  const int base = row_ptr[j], d = row_ptr[j + 1] - base;
  const int t0 = trip_ptr[e], nt = trip_ptr[e + 1] - t0;
  if (nt == 0) return;
  const int p_i = slot_of(src, base, d, i, lane);
  const f3 pj = load3(pos, j), Gj = load3(G, j);
  const f3 Gu = sub3(load3(G, i), Gj);
  const v3<dual> u = to_dual(sub3(load3(pos, i), pj), Gu);
  const bool want_angle = dangle || d_dangle, want_torsion = dtorsion || d_dtorsion;
  f3 hi = {0.f, 0.f, 0.f}, hj = {0.f, 0.f, 0.f};
  for (int tt = lane; tt < nt; tt += 32) {
    const int t = t0 + tt, s = tt + (tt >= p_i ? 1 : 0);
    const int k = src[base + s];
    const f3 Gk = sub3(load3(G, k), Gj);
    const v3<dual> vk = to_dual(sub3(load3(pos, k), pj), Gk);
    if (want_angle) {
      v3<dual> g_u, g_v;
      float jvp = 0.f;
      if (angle_grad(u, vk, g_u, g_v)) {
        jvp = dot(to_v3(value3(g_u)), to_v3(Gu)) + dot(to_v3(value3(g_v)), to_v3(Gk));
        const float w = dangle ? dangle[t] : 0.f;
        if (w != 0.f) {
          const f3 hu = scale3(tangent3(g_u), w), hk = scale3(tangent3(g_v), w);
          atomic_add3(d_pos, k, hk);
          hi = add3(hi, hu);
          hj = add3(hj, add3(hu, hk));
        }
      }
      if (d_dangle) d_dangle[t] = jvp;
    }
    if (want_torsion) {
      const int a = tors_arg[t];
      float jvp = 0.f;
      if (a >= 0 && a != s) {
        const int c = src[base + a];
        const f3 Gc = sub3(load3(G, c), Gj);
        v3<dual> g_u, g_vk, g_vc;
        if (torsion_grad(u, vk, to_dual(sub3(load3(pos, c), pj), Gc), g_u, g_vk, g_vc)) {
          jvp = dot(to_v3(value3(g_u)), to_v3(Gu)) + dot(to_v3(value3(g_vk)), to_v3(Gk)) +
                dot(to_v3(value3(g_vc)), to_v3(Gc));
          const float w = dtorsion ? dtorsion[t] : 0.f;
          if (w != 0.f) {
            const f3 hu = scale3(tangent3(g_u), w), hk = scale3(tangent3(g_vk), w), hc = scale3(tangent3(g_vc), w);
            atomic_add3(d_pos, k, hk);
            atomic_add3(d_pos, c, hc);
            hi = add3(hi, hu);
            hj = add3(hj, add3(hu, add3(hk, hc)));
          }
        }
      }
      if (d_dtorsion) d_dtorsion[t] = jvp;
    }
  }
  hi = warp_sum3(hi);
  hj = warp_sum3(hj);
  if (lane == 0) {
    atomic_add3(d_pos, i, hi);
    atomic_add3(d_pos, j, scale3(hj, -1.f));
  }
}

}  // namespace dig3d

using namespace dig3d;

extern "C" {

int dig3d_triplet_torsion_bwd_arg(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                                  const int32_t* trip_ptr, const int32_t* tors_arg, const float* dtorsion,
                                  int64_t n_edges, float* dpos, void* stream) {
  DIG3D_REQUIRE(pos && src && dst && row_ptr && trip_ptr && tors_arg && dtorsion && dpos,
                "triplet_torsion_bwd_arg: null pointer");
  DIG3D_REQUIRE(n_edges >= 0 && n_edges < (1ll << 26), "triplet_torsion_bwd_arg: %lld edges", (long long)n_edges);
  if (n_edges == 0) return DIG3D_OK;
  triplet_torsion_bwd_arg_kernel<<<ceil_div(n_edges * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      pos, src, dst, row_ptr, trip_ptr, tors_arg, dtorsion, (int)n_edges, dpos);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_geometry_bwd2(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                                const int32_t* trip_ptr, const int32_t* tors_arg, const float* dangle,
                                const float* dtorsion, const float* g_dpos, int64_t n_edges, float* d_dangle,
                                float* d_dtorsion, float* d_pos, void* stream) {
  DIG3D_REQUIRE(pos && src && dst && row_ptr && trip_ptr && g_dpos && d_pos, "triplet_geometry_bwd2: null pointer");
  DIG3D_REQUIRE(!(dtorsion || d_dtorsion) || tors_arg, "triplet_geometry_bwd2: the torsion terms need tors_arg");
  DIG3D_REQUIRE(n_edges >= 0 && n_edges < (1ll << 26), "triplet_geometry_bwd2: %lld edges", (long long)n_edges);
  if (n_edges == 0) return DIG3D_OK;
  triplet_geometry_bwd2_kernel<<<ceil_div(n_edges * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      pos, src, dst, row_ptr, trip_ptr, tors_arg, dangle, dtorsion, g_dpos, (int)n_edges, d_dangle, d_dtorsion,
      d_pos);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_edge_dist_bwd(const float* pos, const int32_t* src, const int32_t* dst, const float* dist, const float* ddist,
                        int64_t n_edges, float* dpos, void* stream) {
  DIG3D_REQUIRE(pos && src && dst && dist && ddist && dpos, "edge_dist_bwd: null pointer");
  if (n_edges == 0) return DIG3D_OK;
  edge_dist_bwd_kernel<<<ceil_div(n_edges, 256), 256, 0, (cudaStream_t)stream>>>(pos, src, dst, dist, ddist,
                                                                                (int)n_edges, dpos);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_angle_bwd(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                            const int32_t* trip_ptr, const float* dangle, int64_t n_edges, float* dpos, void* stream) {
  DIG3D_REQUIRE(pos && src && dst && row_ptr && trip_ptr && dangle && dpos, "triplet_angle_bwd: null pointer");
  if (n_edges == 0) return DIG3D_OK;
  triplet_angle_bwd_kernel<<<ceil_div(n_edges * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      pos, src, dst, row_ptr, trip_ptr, dangle, (int)n_edges, dpos);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_torsion_bwd(const float* pos, const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                              const int32_t* trip_ptr, const float* dtorsion, int64_t n_edges, float* dpos, void* stream) {
  DIG3D_REQUIRE(pos && src && dst && row_ptr && trip_ptr && dtorsion && dpos, "triplet_torsion_bwd: null pointer");
  if (n_edges == 0) return DIG3D_OK;
  triplet_torsion_bwd_kernel<<<ceil_div(n_edges, TGEO_WARPS), TGEO_WARPS * 32, 0, (cudaStream_t)stream>>>(
      pos, src, dst, row_ptr, trip_ptr, dtorsion, (int)n_edges, dpos);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_geometry_jvp(const float* pos, const float* cvec, const int32_t* src, const int32_t* dst,
                       const int32_t* row_ptr, const int32_t* trip_ptr, const float* dist, int64_t n_edges,
                       float* dist_dot, float* angle_dot, float* torsion_dot, void* stream) {
  DIG3D_REQUIRE(pos && cvec && src && dst && dist && dist_dot, "geometry_jvp: null pointer");
  DIG3D_REQUIRE((!angle_dot && !torsion_dot) || (row_ptr && trip_ptr), "geometry_jvp: triplet tangents need row_ptr / trip_ptr");
  if (n_edges == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  edge_dist_jvp_kernel<<<ceil_div(n_edges, 256), 256, 0, st>>>(pos, cvec, src, dst, dist, (int)n_edges, dist_dot);
  DIG3D_LAUNCH_CHECK();
  if (angle_dot) {
    triplet_angle_jvp_kernel<<<ceil_div(n_edges * 32, 256), 256, 0, st>>>(pos, cvec, src, dst, row_ptr, trip_ptr,
                                                                          (int)n_edges, angle_dot);
    DIG3D_LAUNCH_CHECK();
  }
  if (torsion_dot) {
    triplet_torsion_jvp_kernel<<<ceil_div(n_edges, TGEO_WARPS), TGEO_WARPS * 32, 0, st>>>(
        pos, cvec, src, dst, row_ptr, trip_ptr, (int)n_edges, torsion_dot);
    DIG3D_LAUNCH_CHECK();
  }
  return DIG3D_OK;
}

int dig3d_schnet_edge_features_bwd(const float* dist, int64_t n_edges, const float* offset, int32_t n_gauss,
                                   double coeff, double cutoff, const float* dgauss, const float* dcut, float* ddist,
                                   void* stream) {
  DIG3D_REQUIRE(dist && offset && ddist && n_gauss > 0 && (dgauss || dcut), "schnet_edge_features_bwd: bad arguments");
  if (n_edges == 0) return DIG3D_OK;
  schnet_edge_features_bwd_kernel<<<ceil_div(n_edges, 256), 256, 0, (cudaStream_t)stream>>>(
      dist, n_edges, offset, n_gauss, (float)coeff, (float)(1.0 / cutoff), dgauss, dcut, ddist);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_rowdot(const float* a, const float* b, int64_t rows, int32_t width, float* out, void* stream) {
  DIG3D_REQUIRE(a && b && out && width > 0, "rowdot: bad arguments");
  if (rows == 0) return DIG3D_OK;
  rowdot_kernel<<<ceil_div(rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(a, b, rows, width, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_edge_dist_bwd2(const float* pos, const int32_t* src, const int32_t* dst, const float* dist, const float* ddist,
                         const float* g_dpos, int64_t n_edges, float* d_ddist, float* d_pos, void* stream) {
  DIG3D_REQUIRE(pos && src && dst && dist && ddist && g_dpos && d_ddist && d_pos, "edge_dist_bwd2: null pointer");
  if (n_edges == 0) return DIG3D_OK;
  edge_dist_bwd2_kernel<<<ceil_div(n_edges, 256), 256, 0, (cudaStream_t)stream>>>(pos, src, dst, dist, ddist, g_dpos,
                                                                                 (int)n_edges, d_ddist, d_pos);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_schnet_edge_features_bwd2(const float* dist, int64_t n_edges, const float* offset, int32_t n_gauss,
                                    double coeff, double cutoff, const float* dgauss, const float* dcut, const float* g,
                                    float* d_dgauss, float* d_dcut, float* d_dist, void* stream) {
  DIG3D_REQUIRE(dist && offset && g && d_dist && n_gauss > 0, "schnet_edge_features_bwd2: bad arguments");
  if (n_edges == 0) return DIG3D_OK;
  schnet_edge_features_bwd2_kernel<<<ceil_div(n_edges, 256), 256, 0, (cudaStream_t)stream>>>(
      dist, n_edges, offset, n_gauss, (float)coeff, (float)(1.0 / cutoff), dgauss, dcut, g, d_dgauss, d_dcut, d_dist);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
