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
#include "dual.cuh"
#include "generated/basis_gemnet_2_3.cuh"
#include "generated/basis_gemnet_2_3_d2.cuh"

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

// The edges whose vectors the angles of edge e = (j -> i) read (comenet.py:331-354): e itself, i's nearest and
// second-nearest in-edges, and the reference edges of i and of j.
struct ComenetEdgeRefs {
  int e0i, e1i, iref, jref;
};
__device__ __forceinline__ ComenetEdgeRefs comenet_edge_refs(const int32_t* __restrict__ src,
                                                             const int32_t* __restrict__ dst,
                                                             const int32_t* __restrict__ a0_in,
                                                             const int32_t* __restrict__ a1_in,
                                                             const int32_t* __restrict__ a0_out,
                                                             const int32_t* __restrict__ a1_out, int e) {
  const int j = src[e], i = dst[e];
  const int e0i = a0_in[i], e1i = a1_in[i], e0j = a0_out[j], e1j = a1_out[j];
  const int n0 = src[e0i], n0_j = dst[e0j];
  return {e0i, e1i, (n0 == j) ? e1i : e0i,                               // comenet.py:344-348
          (n0_j == i) ? e1j : e0j};                                      // comenet.py:350-354
}

// theta / phi / tau of one edge with the intermediates their derivatives need.  The forward kernel and the two force
// kernels below evaluate the angles with this one function, so the derivatives are taken at the bit-equal angles.
struct ComenetEdgeGeom {
  f3 pji, in0, in1, iref, jref;      // the five edge vectors
  f3 pl1, pl2, c2, q1, q2, c3;       // planes; c2 = pl1 x pl2, c3 = q1 x q2
  float a1, b1;                      // theta = fold(atan2(b1, a1))
  float d;                           // |pji|
  float a2, s2;                      // phi = fold(atan2(s2 / d, a2))
  float a3, s3;                      // tau = fold(atan2(s3 / d, a3))
  float theta, phi, tau;
};
template <bool FROM_VEC>
__device__ __forceinline__ ComenetEdgeGeom comenet_edge_geom(const float* __restrict__ pos,
                                                             const int32_t* __restrict__ src,
                                                             const int32_t* __restrict__ dst, int e,
                                                             const ComenetEdgeRefs r) {
  ComenetEdgeGeom G;
  G.pji = edge_vec<FROM_VEC>(pos, src, dst, e);
  G.in0 = edge_vec<FROM_VEC>(pos, src, dst, r.e0i);
  G.in1 = edge_vec<FROM_VEC>(pos, src, dst, r.e1i);
  G.iref = edge_vec<FROM_VEC>(pos, src, dst, r.iref);
  G.jref = edge_vec<FROM_VEC>(pos, src, dst, r.jref);
  const f3 mji = neg3(G.pji);
  // theta                                                                comenet.py:365-368
  G.pl1 = cross_aten(mji, G.in0);
  G.b1 = norm3_aten(G.pl1);
  G.a1 = sum3_aten(mul3(mji, G.in0));
  G.theta = fold_pi(atan2f(G.b1, G.a1));
  // phi                                                                  comenet.py:371-377
  G.d = norm3_aten(G.pji);
  G.pl2 = cross_aten(mji, G.in1);
  G.c2 = cross_aten(G.pl1, G.pl2);
  G.s2 = sum3_aten(mul3(G.c2, G.pji));
  G.a2 = sum3_aten(mul3(G.pl1, G.pl2));
  G.phi = fold_pi(atan2f(__fdiv_rn(G.s2, G.d), G.a2));
  // tau                                                                  comenet.py:380-385
  G.q1 = cross_aten(G.pji, G.jref);
  G.q2 = cross_aten(G.pji, G.iref);
  G.c3 = cross_aten(G.q1, G.q2);
  G.s3 = sum3_aten(mul3(G.c3, G.pji));
  G.a3 = sum3_aten(mul3(G.q1, G.q2));
  G.tau = fold_pi(atan2f(__fdiv_rn(G.s3, G.d), G.a3));
  return G;
}

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
  const ComenetEdgeGeom G = comenet_edge_geom<FROM_VEC>(
      pos, src, dst, e, comenet_edge_refs(src, dst, a0_in, a1_in, a0_out, a1_out, e));
  const float theta = G.theta, phi = G.phi, tau = G.tau;
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

// ------------------------------------------------------------------ forces: derivatives of feature1 / feature2 in pos
// Reverse mode (dig3d_comenet_features_bwd) and forward mode (dig3d_comenet_features_tangent) of the kernel above for
// the reference's op sequence (comenet.py:297-385, features.py:289-348) with ATen's derivative conventions where a
// value is singular: the norm of a zero vector and atan2(0, 0) pass no gradient (norm_backward / atan2_backward mask
// them).  The reference-atom argmins are piecewise constant: no derivative.
// Aliased cross products.  When two of the vectors a cross product reads are the same edge -- routine: j is i's nearest
// in-neighbour on one in-edge of every node (pos_in0 == pos_ji), a node with a single in-edge has e0i == e1i, a node
// with a single out-edge is its own jref -- the product is a x a, identically zero as a function of the positions, and
// its derivative is exactly zero.  ATen's value is the FMA rounding residue of a x a (SURVEY.md 5.9b), and autograd
// differentiates the bilinear form instead: two opposite terms of size |g| / |residue| (~1e7 |g| for phi) that only
// cancel to the last bits of their own size, so torch's forces on such graphs carry O(|g|) noise that changes with
// the order of its sums (run to run on the CPU with several threads, and with every atomic order on the GPU).  These
// kernels take the exact derivative: the terms of an aliased product are zero.  Both kernels use the same partial
// derivatives and the same rule, so one is exactly the transpose of the other.
__device__ __forceinline__ f3 add3(const f3 a, const f3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ f3 scale3(const f3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ f3 axpy3(float s, const f3 a, const f3 b) {
  return {fmaf(s, a.x, b.x), fmaf(s, a.y, b.y), fmaf(s, a.z, b.z)};
}
__device__ __forceinline__ float dot3(const f3 a, const f3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }
__device__ __forceinline__ f3 cross3(const f3 a, const f3 b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
// d atan2(y, x) / dy and / dx; both 0 at (0, 0) as in ATen's atan2_backward
__device__ __forceinline__ void atan2_partials(float y, float x, float& py, float& px) {
  const float den = fmaf(x, x, y * y);
  py = den == 0.f ? 0.f : x / den;
  px = den == 0.f ? 0.f : -y / den;
}

// d(theta, phi, tau)/d(its inputs) at one edge: the scalar partials shared by both modes
struct ComenetEdgePartials {
  float th_b1, th_a1;                // theta
  float ph_b2, ph_a2;                // phi (b2 = s2 / d)
  float ta_b3, ta_a3;                // tau (b3 = s3 / d)
  float inv_b1;                      // 1 / |pl1|, 0 for pl1 == 0 (norm_backward)
  float inv_d;                       // 1 / d (the features' vecs.norm(): 0 for d == 0)
  // cross products whose two operands are the same edge vector (derivative exactly zero, see above)
  bool pl1_0, pl2_0, c2_0, q1_0, q2_0, c3_0;
};
// Whether the edge vectors v1 (edge e1) and v2 (edge e2) lie on one line as functions of the inputs, so that their cross
// product is identically zero: the same edge, or -- FROM_VEC, periodic images -- two self-image edges of one atom
// (row == col: vec = offset . cell) whose vectors are exactly parallel (offsets o and -o, or o and 2o, which is routine
// in a cell smaller than twice the nearest-neighbour distance).  Exactness: the products of fp32 values are exact in
// fp64.
__device__ __forceinline__ bool exactly_parallel(const f3 a, const f3 b) {
  const double ax = a.x, ay = a.y, az = a.z, bx = b.x, by = b.y, bz = b.z;
  return ay * bz == az * by && az * bx == ax * bz && ax * by == ay * bx;
}
template <bool FROM_VEC>
__device__ __forceinline__ bool on_one_line(int e1, int e2, const f3 v1, const f3 v2, const int32_t* __restrict__ src,
                                            const int32_t* __restrict__ dst) {
  if (e1 == e2) return true;
  if (!FROM_VEC) return false;
  return src[e1] == dst[e1] && src[e2] == dst[e2] && dst[e1] == dst[e2] && exactly_parallel(v1, v2);
}

template <bool FROM_VEC>
__device__ __forceinline__ ComenetEdgePartials comenet_edge_partials(const ComenetEdgeGeom& G,
                                                                     const ComenetEdgeRefs r, int e,
                                                                     const int32_t* __restrict__ src,
                                                                     const int32_t* __restrict__ dst) {
  ComenetEdgePartials P;
  P.pl1_0 = on_one_line<FROM_VEC>(r.e0i, e, G.in0, G.pji, src, dst);        // pl1 = (-pji) x in0
  P.pl2_0 = on_one_line<FROM_VEC>(r.e1i, e, G.in1, G.pji, src, dst);        // pl2 = (-pji) x in1
  P.c2_0 = on_one_line<FROM_VEC>(r.e0i, r.e1i, G.in0, G.in1, src, dst);     // pl1 x pl2 with pl1 || pl2
  P.q1_0 = on_one_line<FROM_VEC>(r.jref, e, G.jref, G.pji, src, dst);       // q1 = pji x jref
  P.q2_0 = on_one_line<FROM_VEC>(r.iref, e, G.iref, G.pji, src, dst);       // q2 = pji x iref
  P.c3_0 = on_one_line<FROM_VEC>(r.iref, r.jref, G.iref, G.jref, src, dst); // q1 x q2 with q1 || q2
  atan2_partials(G.b1, G.a1, P.th_b1, P.th_a1);
  atan2_partials(__fdiv_rn(G.s2, G.d), G.a2, P.ph_b2, P.ph_a2);
  atan2_partials(__fdiv_rn(G.s3, G.d), G.a3, P.ta_b3, P.ta_a3);
  P.inv_b1 = G.b1 == 0.f ? 0.f : 1.0f / G.b1;
  P.inv_d = G.d == 0.f ? 0.f : 1.0f / G.d;
  return P;
}

// the basis at x = dist / cutoff and its derivatives (the generated closed forms of basis_gemnet_2_3)
struct ComenetEdgeBasis {
  float rb[6], rbd[6], y0[2], y0d[2], ylm[4], ylmt[4], ylmp[4];
};
__device__ __forceinline__ void comenet_edge_basis(float x, const ComenetEdgeGeom& G, ComenetEdgeBasis& B) {
  basis_gemnet_2_3::bessel(x, B.rb);
  basis_gemnet_2_3::bessel_dx(x, B.rbd);
  basis_gemnet_2_3::yl0(G.tau, B.y0);
  basis_gemnet_2_3::yl0_dtheta(G.tau, B.y0d);
  basis_gemnet_2_3::ylm(G.theta, G.phi, B.ylm);
  basis_gemnet_2_3::ylm_dtheta(G.theta, G.phi, B.ylmt);
  basis_gemnet_2_3::ylm_dphi(G.theta, G.phi, B.ylmp);
}

// Pass 1: per edge e, d(loss)/d(edge vector) of the five vectors its angles read, written to work[e][role][3] with
// roles 0 = pji (e itself), 1 = in0 (e0i), 2 = in1 (e1i), 3 = iref, 4 = jref.  FROM_VEC: the OCP variant, the edge
// vectors read from `pos` = vec [E, 3] (see edge_vec).
template <bool FROM_VEC>
__global__ void comenet_features_bwd_edge_kernel(const float* __restrict__ pos, const float* __restrict__ dist,
                                                 const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                                 const int32_t* __restrict__ a0_in, const int32_t* __restrict__ a1_in,
                                                 const int32_t* __restrict__ a0_out, const int32_t* __restrict__ a1_out,
                                                 int n_edges, float inv_cutoff, const float* __restrict__ df1,
                                                 const float* __restrict__ df2, float* __restrict__ work) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const ComenetEdgeRefs rf = comenet_edge_refs(src, dst, a0_in, a1_in, a0_out, a1_out, e);
  const ComenetEdgeGeom G = comenet_edge_geom<FROM_VEC>(pos, src, dst, e, rf);
  const ComenetEdgePartials P = comenet_edge_partials<FROM_VEC>(G, rf, e, src, dst);
  ComenetEdgeBasis B;
  comenet_edge_basis(__fmul_rn(dist[e], inv_cutoff), G, B);
  // features -> d(rbf), d theta, d phi, d tau                            features.py:289-295,340-348
  float grb[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float gth = 0.f, gph = 0.f, gta = 0.f;
#pragma unroll
  for (int l = 0; l < 2; ++l)
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float g = __ldg(df2 + (size_t)e * NF2 + l * 3 + r);
      grb[l * 3 + r] = fmaf(g, B.y0[l], grb[l * 3 + r]);
      gta = fmaf(g * B.rb[l * 3 + r], B.y0d[l], gta);
    }
#pragma unroll
  for (int h = 0; h < 4; ++h)
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int k = (h == 0 ? 0 : 1) * 3 + r;
      const float g = __ldg(df1 + (size_t)e * NF1 + h * 3 + r);
      grb[k] = fmaf(g, B.ylm[h], grb[k]);
      gth = fmaf(g * B.rb[k], B.ylmt[h], gth);
      gph = fmaf(g * B.rb[k], B.ylmp[h], gph);
    }
  float gx = 0.f;
#pragma unroll
  for (int k = 0; k < 6; ++k) gx = fmaf(grb[k], B.rbd[k], gx);
  const float gdist = gx * inv_cutoff;
  // angles -> vectors
  const f3 M = neg3(G.pji);
  f3 gP = scale3(G.pji, gdist * P.inv_d), gM = {0.f, 0.f, 0.f}, gA = {0.f, 0.f, 0.f};
  // theta = atan2(|pl1|, M . in0)
  const float g_a1 = gth * P.th_a1;
  f3 gpl1 = scale3(G.pl1, gth * P.th_b1 * P.inv_b1);
  gM = axpy3(g_a1, G.in0, gM);
  gA = axpy3(g_a1, M, gA);
  // phi = atan2(s2 / d, pl1 . pl2), s2 = (pl1 x pl2) . pji
  const float g_b2 = gph * P.ph_b2, g_a2 = gph * P.ph_a2;
  const float g_s2 = g_b2 / G.d;
  float g_d = -g_b2 * G.s2 / (G.d * G.d);
  const f3 gc2 = P.c2_0 ? f3{0.f, 0.f, 0.f} : scale3(G.pji, g_s2);
  gP = axpy3(g_s2, G.c2, gP);
  gpl1 = add3(gpl1, axpy3(g_a2, G.pl2, cross3(G.pl2, gc2)));
  f3 gpl2 = axpy3(g_a2, G.pl1, cross3(gc2, G.pl1));
  if (P.pl1_0) gpl1 = {0.f, 0.f, 0.f};
  if (P.pl2_0) gpl2 = {0.f, 0.f, 0.f};
  // tau = atan2(s3 / d, q1 . q2), s3 = (q1 x q2) . pji, q1 = pji x jref, q2 = pji x iref
  const float g_b3 = gta * P.ta_b3, g_a3 = gta * P.ta_a3;
  const float g_s3 = g_b3 / G.d;
  g_d -= g_b3 * G.s3 / (G.d * G.d);
  const f3 gc3 = P.c3_0 ? f3{0.f, 0.f, 0.f} : scale3(G.pji, g_s3);
  gP = axpy3(g_s3, G.c3, gP);
  f3 gq1 = axpy3(g_a3, G.q2, cross3(G.q2, gc3));
  f3 gq2 = axpy3(g_a3, G.q1, cross3(gc3, G.q1));
  if (P.q1_0) gq1 = {0.f, 0.f, 0.f};
  if (P.q2_0) gq2 = {0.f, 0.f, 0.f};
  gP = add3(gP, add3(cross3(G.jref, gq1), cross3(G.iref, gq2)));
  const f3 gS = cross3(gq1, G.pji), gR = cross3(gq2, G.pji);
  // d = sqrt(sum(pji^2)) of phi / tau
  gP = axpy3(g_d / G.d, G.pji, gP);
  // pl1 = M x in0, pl2 = M x in1
  gM = add3(gM, add3(cross3(G.in0, gpl1), cross3(G.in1, gpl2)));
  gA = add3(gA, cross3(gpl1, M));
  const f3 gB = cross3(gpl2, M);
  gP = sub3(gP, gM);
  float* w = work + (size_t)e * 15;
  const f3 out[5] = {gP, gA, gB, gR, gS};
#pragma unroll
  for (int k = 0; k < 5; ++k) { w[3 * k] = out[k].x; w[3 * k + 1] = out[k].y; w[3 * k + 2] = out[k].z; }
}

// Pass 2: dvec[e'] = the sum, in edge order, of every pass-1 contribution to edge e'.  An edge e reads e' as in0 / in1 /
// iref only if both end in the same node (dst[e] == dst[e']): the in-edges of dst[e']; as jref only if both start in the
// same node: the out-edges of src[e'].  No atomics: the result is the same bits run to run.
__global__ void comenet_features_bwd_gather_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                                   const int32_t* __restrict__ row_ptr,
                                                   const int32_t* __restrict__ out_ptr,
                                                   const int32_t* __restrict__ out_list,
                                                   const int32_t* __restrict__ a0_in, const int32_t* __restrict__ a1_in,
                                                   const int32_t* __restrict__ a0_out,
                                                   const int32_t* __restrict__ a1_out, int n_edges,
                                                   const float* __restrict__ work, float* __restrict__ dvec) {
  const int ep = blockIdx.x * blockDim.x + threadIdx.x;
  if (ep >= n_edges) return;
  const int j = src[ep], i = dst[ep];
  const float* w = work + (size_t)ep * 15;
  float ax = w[0], ay = w[1], az = w[2];
  {
    const int e0i = a0_in[i], e1i = a1_in[i], n0 = src[e0i];
    for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e) {
      const int iref = (n0 == src[e]) ? e1i : e0i;
      const float* c = work + (size_t)e * 15;
      if (e0i == ep) { ax += c[3]; ay += c[4]; az += c[5]; }
      if (e1i == ep) { ax += c[6]; ay += c[7]; az += c[8]; }
      if (iref == ep) { ax += c[9]; ay += c[10]; az += c[11]; }
    }
  }
  {
    const int e0j = a0_out[j], e1j = a1_out[j], n0_j = dst[e0j];
    for (int k = out_ptr[j]; k < out_ptr[j + 1]; ++k) {
      const int e = out_list[k];
      const int jref = (n0_j == dst[e]) ? e1j : e0j;
      if (jref == ep) {
        const float* c = work + (size_t)e * 15;
        ax += c[12]; ay += c[13]; az += c[14];
      }
    }
  }
  dvec[3 * (size_t)ep] = ax; dvec[3 * (size_t)ep + 1] = ay; dvec[3 * (size_t)ep + 2] = az;
}

// Pass 3: vec[e] = pos[src[e]] - pos[dst[e]]  ->  dpos[n] = sum of dvec over n's out-edges - sum over its in-edges
__global__ void comenet_features_bwd_node_kernel(const int32_t* __restrict__ row_ptr,
                                                 const int32_t* __restrict__ out_ptr,
                                                 const int32_t* __restrict__ out_list, int n_nodes,
                                                 const float* __restrict__ dvec, float* __restrict__ dpos) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_nodes) return;
  float ax = 0.f, ay = 0.f, az = 0.f;
  for (int k = out_ptr[n]; k < out_ptr[n + 1]; ++k) {
    const int e = out_list[k];
    ax += dvec[3 * (size_t)e]; ay += dvec[3 * (size_t)e + 1]; az += dvec[3 * (size_t)e + 2];
  }
  for (int e = row_ptr[n]; e < row_ptr[n + 1]; ++e) {
    ax -= dvec[3 * (size_t)e]; ay -= dvec[3 * (size_t)e + 1]; az -= dvec[3 * (size_t)e + 2];
  }
  dpos[3 * (size_t)n] = ax; dpos[3 * (size_t)n + 1] = ay; dpos[3 * (size_t)n + 2] = az;
}

// Forward mode: f1_dot / f2_dot of every edge along the per-atom displacement cvec [N, 3].  FROM_VEC: the edge vectors
// are read from `pos` = vec [E, 3]; their tangent is still cvec[src] - cvec[dst] (the cell is held fixed).
template <bool FROM_VEC>
__global__ void comenet_features_tangent_kernel(const float* __restrict__ pos, const float* __restrict__ dist,
                                                const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                                const int32_t* __restrict__ a0_in, const int32_t* __restrict__ a1_in,
                                                const int32_t* __restrict__ a0_out, const int32_t* __restrict__ a1_out,
                                                int n_edges, float inv_cutoff, const float* __restrict__ cvec,
                                                float* __restrict__ f1_dot, float* __restrict__ f2_dot) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const ComenetEdgeRefs r = comenet_edge_refs(src, dst, a0_in, a1_in, a0_out, a1_out, e);
  const ComenetEdgeGeom G = comenet_edge_geom<FROM_VEC>(pos, src, dst, e, r);
  const ComenetEdgePartials P = comenet_edge_partials<FROM_VEC>(G, r, e, src, dst);
  ComenetEdgeBasis B;
  comenet_edge_basis(__fmul_rn(dist[e], inv_cutoff), G, B);
  const f3 zero = {0.f, 0.f, 0.f};
  const f3 dP = edge_vec<false>(cvec, src, dst, e), dA = edge_vec<false>(cvec, src, dst, r.e0i);
  const f3 dB = edge_vec<false>(cvec, src, dst, r.e1i), dR = edge_vec<false>(cvec, src, dst, r.iref);
  const f3 dS = edge_vec<false>(cvec, src, dst, r.jref);
  const f3 M = neg3(G.pji), dM = neg3(dP);
  const float ddist = dot3(G.pji, dP) * P.inv_d;
  // theta
  const f3 dpl1 = P.pl1_0 ? zero : add3(cross3(dM, G.in0), cross3(M, dA));
  const float da1 = dot3(dM, G.in0) + dot3(M, dA);
  const float db1 = dot3(G.pl1, dpl1) * P.inv_b1;
  const float dth = fmaf(P.th_b1, db1, P.th_a1 * da1);
  // phi
  const float dd = dot3(G.pji, dP) / G.d;
  const f3 dpl2 = P.pl2_0 ? zero : add3(cross3(dM, G.in1), cross3(M, dB));
  const float da2 = dot3(dpl1, G.pl2) + dot3(G.pl1, dpl2);
  const f3 dc2 = P.c2_0 ? zero : add3(cross3(dpl1, G.pl2), cross3(G.pl1, dpl2));
  const float ds2 = dot3(dc2, G.pji) + dot3(G.c2, dP);
  const float db2 = ds2 / G.d - G.s2 * dd / (G.d * G.d);
  const float dph = fmaf(P.ph_b2, db2, P.ph_a2 * da2);
  // tau
  const f3 dq1 = P.q1_0 ? zero : add3(cross3(dP, G.jref), cross3(G.pji, dS));
  const f3 dq2 = P.q2_0 ? zero : add3(cross3(dP, G.iref), cross3(G.pji, dR));
  const float da3 = dot3(dq1, G.q2) + dot3(G.q1, dq2);
  const f3 dc3 = P.c3_0 ? zero : add3(cross3(dq1, G.q2), cross3(G.q1, dq2));
  const float ds3 = dot3(dc3, G.pji) + dot3(G.c3, dP);
  const float db3 = ds3 / G.d - G.s3 * dd / (G.d * G.d);
  const float dta = fmaf(P.ta_b3, db3, P.ta_a3 * da3);
  // features
  const float dx = ddist * inv_cutoff;
#pragma unroll
  for (int l = 0; l < 2; ++l)
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const int k = l * 3 + q;
      f2_dot[(size_t)e * NF2 + k] = fmaf(B.rbd[k] * dx, B.y0[l], B.rb[k] * B.y0d[l] * dta);
    }
#pragma unroll
  for (int h = 0; h < 4; ++h)
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const int k = (h == 0 ? 0 : 1) * 3 + q;
      f1_dot[(size_t)e * NF1 + h * 3 + q] =
          fmaf(B.rbd[k] * dx, B.ylm[h], B.rb[k] * fmaf(B.ylmt[h], dth, B.ylmp[h] * dph));
    }
}

// ------------------------------------------------------------------ Hessian-vector products: reverse of the tangent
// dpos = sum_e sum_k g_k (d2 f_k / dpos2) cvec with g1 / g2 = d loss / d f1_dot / f2_dot: the reverse of the tangent
// kernel above in the positions (its reverse in cvec is features_bwd itself).  It is d/de of J(pos + e cvec)^T g, so
// this is pass 1 of the backward evaluated on dual numbers (value, tangent along cvec) seeded with df1 = g1,
// df2 = g2; the tangent part of the five edge-vector gradients then goes through the backward's gather and node passes,
// which are linear and do not depend on pos.  The values, partials and aliasing flags are those of the first-order
// kernels and the intermediate tangents those of the tangent kernel, so the conventions carry over: the reference atoms
// are constant, an aliased cross product is a constant (its value the residue, its tangent 0, its gradient terms 0),
// and a zero norm or atan2(0, 0) passes nothing in either part.
struct df3 {
  dual x, y, z;
};
__device__ __forceinline__ df3 make_df3(const f3 v, const f3 t) { return {{v.x, t.x}, {v.y, t.y}, {v.z, t.z}}; }
__device__ __forceinline__ f3 tangent3(const df3 a) { return {a.x.d, a.y.d, a.z.d}; }
__device__ __forceinline__ dual scale(const dual a, float s) { return {a.v * s, a.d * s}; }
__device__ __forceinline__ dual fmad(const dual a, const dual b, const dual c) {
  return {fmaf(a.v, b.v, c.v), fmaf(a.d, b.v, fmaf(a.v, b.d, c.d))};
}
__device__ __forceinline__ df3 neg3(const df3 a) { return {-a.x, -a.y, -a.z}; }
__device__ __forceinline__ df3 add3(const df3 a, const df3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ df3 sub3(const df3 a, const df3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ df3 scale3(const df3 a, const dual s) { return {a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ df3 axpy3(const dual s, const df3 a, const df3 b) {
  return {fmad(s, a.x, b.x), fmad(s, a.y, b.y), fmad(s, a.z, b.z)};
}
__device__ __forceinline__ df3 cross3(const df3 a, const df3 b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
// atan2_partials with their tangents; py / px are atan2_partials' values at (y.v, x.v)
__device__ __forceinline__ void atan2_partials_dual(const dual y, const dual x, float py, float px, dual& Py, dual& Px) {
  const float den = fmaf(x.v, x.v, y.v * y.v);
  if (den == 0.f) { Py = {0.f, 0.f}; Px = {0.f, 0.f}; return; }
  const float dden = 2.f * fmaf(x.v, x.d, y.v * y.d);
  Py = {py, (x.d - py * dden) / den};
  Px = {px, (-y.d - px * dden) / den};
}

// Pass 1 on duals: work[e][role][3] = the tangent of pass 1's five edge-vector gradients (same roles)
template <bool FROM_VEC>
__global__ void comenet_features_tangent_bwd_edge_kernel(const float* __restrict__ pos, const float* __restrict__ dist,
                                                         const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                                         const int32_t* __restrict__ a0_in,
                                                         const int32_t* __restrict__ a1_in,
                                                         const int32_t* __restrict__ a0_out,
                                                         const int32_t* __restrict__ a1_out, int n_edges,
                                                         float inv_cutoff, const float* __restrict__ cvec,
                                                         const float* __restrict__ g1, const float* __restrict__ g2,
                                                         float* __restrict__ work) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const ComenetEdgeRefs r = comenet_edge_refs(src, dst, a0_in, a1_in, a0_out, a1_out, e);
  const ComenetEdgeGeom G = comenet_edge_geom<FROM_VEC>(pos, src, dst, e, r);
  const ComenetEdgePartials P = comenet_edge_partials<FROM_VEC>(G, r, e, src, dst);
  ComenetEdgeBasis B;
  const float x = __fmul_rn(dist[e], inv_cutoff);
  comenet_edge_basis(x, G, B);
  // the tangents along cvec, as comenet_features_tangent_kernel computes them
  const f3 zero = {0.f, 0.f, 0.f};
  const f3 dP = edge_vec<false>(cvec, src, dst, e), dA = edge_vec<false>(cvec, src, dst, r.e0i);
  const f3 dB = edge_vec<false>(cvec, src, dst, r.e1i), dR = edge_vec<false>(cvec, src, dst, r.iref);
  const f3 dS = edge_vec<false>(cvec, src, dst, r.jref);
  const f3 Mv = neg3(G.pji), dM = neg3(dP);
  const float ddist = dot3(G.pji, dP) * P.inv_d;
  const f3 dpl1 = P.pl1_0 ? zero : add3(cross3(dM, G.in0), cross3(Mv, dA));
  const float da1 = dot3(dM, G.in0) + dot3(Mv, dA);
  const float db1 = dot3(G.pl1, dpl1) * P.inv_b1;
  const float dth = fmaf(P.th_b1, db1, P.th_a1 * da1);
  const float dd = dot3(G.pji, dP) / G.d;
  const f3 dpl2 = P.pl2_0 ? zero : add3(cross3(dM, G.in1), cross3(Mv, dB));
  const float da2 = dot3(dpl1, G.pl2) + dot3(G.pl1, dpl2);
  const f3 dc2 = P.c2_0 ? zero : add3(cross3(dpl1, G.pl2), cross3(G.pl1, dpl2));
  const float ds2 = dot3(dc2, G.pji) + dot3(G.c2, dP);
  const float db2 = ds2 / G.d - G.s2 * dd / (G.d * G.d);
  const float dph = fmaf(P.ph_b2, db2, P.ph_a2 * da2);
  const f3 dq1 = P.q1_0 ? zero : add3(cross3(dP, G.jref), cross3(G.pji, dS));
  const f3 dq2 = P.q2_0 ? zero : add3(cross3(dP, G.iref), cross3(G.pji, dR));
  const float da3 = dot3(dq1, G.q2) + dot3(G.q1, dq2);
  const f3 dc3 = P.c3_0 ? zero : add3(cross3(dq1, G.q2), cross3(G.q1, dq2));
  const float ds3 = dot3(dc3, G.pji) + dot3(G.c3, dP);
  const float db3 = ds3 / G.d - G.s3 * dd / (G.d * G.d);
  const float dta = fmaf(P.ta_b3, db3, P.ta_a3 * da3);
  // the basis and its first derivatives as duals (tangents from the generated second derivatives)
  float rbdd[6], y0dd[2], ytt[4], ytp[4], ypp[4];
  basis_gemnet_2_3::bessel_dxx(x, rbdd);
  basis_gemnet_2_3::yl0_dtheta2(G.tau, y0dd);
  basis_gemnet_2_3::ylm_dtheta2(G.theta, G.phi, ytt);
  basis_gemnet_2_3::ylm_dtheta_dphi(G.theta, G.phi, ytp);
  basis_gemnet_2_3::ylm_dphi2(G.theta, G.phi, ypp);
  const float dx = ddist * inv_cutoff;
  dual rb[6], rbd[6], y0[2], y0d[2], ylm[4], ylmt[4], ylmp[4];
#pragma unroll
  for (int k = 0; k < 6; ++k) { rb[k] = {B.rb[k], B.rbd[k] * dx}; rbd[k] = {B.rbd[k], rbdd[k] * dx}; }
#pragma unroll
  for (int l = 0; l < 2; ++l) { y0[l] = {B.y0[l], B.y0d[l] * dta}; y0d[l] = {B.y0d[l], y0dd[l] * dta}; }
#pragma unroll
  for (int h = 0; h < 4; ++h) {
    ylm[h] = {B.ylm[h], fmaf(B.ylmt[h], dth, B.ylmp[h] * dph)};
    ylmt[h] = {B.ylmt[h], fmaf(ytt[h], dth, ytp[h] * dph)};
    ylmp[h] = {B.ylmp[h], fmaf(ytp[h], dth, ypp[h] * dph)};
  }
  // features -> d(rbf), d theta, d phi, d tau (pass 1, on duals)
  const dual dz = {0.f, 0.f};
  dual grb[6] = {dz, dz, dz, dz, dz, dz};
  dual gth = dz, gph = dz, gta = dz;
#pragma unroll
  for (int l = 0; l < 2; ++l)
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const float g = __ldg(g2 + (size_t)e * NF2 + l * 3 + q);
      grb[l * 3 + q] = fmad(dual{g, 0.f}, y0[l], grb[l * 3 + q]);
      gta = fmad(scale(rb[l * 3 + q], g), y0d[l], gta);
    }
#pragma unroll
  for (int h = 0; h < 4; ++h)
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const int k = (h == 0 ? 0 : 1) * 3 + q;
      const float g = __ldg(g1 + (size_t)e * NF1 + h * 3 + q);
      grb[k] = fmad(dual{g, 0.f}, ylm[h], grb[k]);
      gth = fmad(scale(rb[k], g), ylmt[h], gth);
      gph = fmad(scale(rb[k], g), ylmp[h], gph);
    }
  dual gx = dz;
#pragma unroll
  for (int k = 0; k < 6; ++k) gx = fmad(grb[k], rbd[k], gx);
  const dual gdist = scale(gx, inv_cutoff);
  // angles -> vectors
  const df3 pji = make_df3(G.pji, dP), M = make_df3(Mv, dM), in0 = make_df3(G.in0, dA), in1 = make_df3(G.in1, dB);
  const df3 iref = make_df3(G.iref, dR), jref = make_df3(G.jref, dS);
  const df3 pl1 = make_df3(G.pl1, dpl1), pl2 = make_df3(G.pl2, dpl2), c2 = make_df3(G.c2, dc2);
  const df3 q1 = make_df3(G.q1, dq1), q2 = make_df3(G.q2, dq2), c3 = make_df3(G.c3, dc3);
  const df3 zd = {dz, dz, dz};
  const dual d = {G.d, dd}, s2 = {G.s2, ds2}, s3 = {G.s3, ds3};
  const dual inv_d = {P.inv_d, -P.inv_d * P.inv_d * dd}, inv_b1 = {P.inv_b1, -P.inv_b1 * P.inv_b1 * db1};
  dual th_b1, th_a1, ph_b2, ph_a2, ta_b3, ta_a3;
  atan2_partials_dual({G.b1, db1}, {G.a1, da1}, P.th_b1, P.th_a1, th_b1, th_a1);
  atan2_partials_dual({__fdiv_rn(G.s2, G.d), db2}, {G.a2, da2}, P.ph_b2, P.ph_a2, ph_b2, ph_a2);
  atan2_partials_dual({__fdiv_rn(G.s3, G.d), db3}, {G.a3, da3}, P.ta_b3, P.ta_a3, ta_b3, ta_a3);
  df3 gP = scale3(pji, gdist * inv_d), gM = zd, gA = zd;
  // theta = atan2(|pl1|, M . in0)
  const dual g_a1 = gth * th_a1;
  df3 gpl1 = scale3(pl1, gth * th_b1 * inv_b1);
  gM = axpy3(g_a1, in0, gM);
  gA = axpy3(g_a1, M, gA);
  // phi = atan2(s2 / d, pl1 . pl2), s2 = (pl1 x pl2) . pji
  const dual g_b2 = gph * ph_b2, g_a2 = gph * ph_a2;
  const dual g_s2 = g_b2 / d;
  dual g_d = -g_b2 * s2 / (d * d);
  const df3 gc2 = P.c2_0 ? zd : scale3(pji, g_s2);
  gP = axpy3(g_s2, c2, gP);
  gpl1 = add3(gpl1, axpy3(g_a2, pl2, cross3(pl2, gc2)));
  df3 gpl2 = axpy3(g_a2, pl1, cross3(gc2, pl1));
  if (P.pl1_0) gpl1 = zd;
  if (P.pl2_0) gpl2 = zd;
  // tau = atan2(s3 / d, q1 . q2), s3 = (q1 x q2) . pji, q1 = pji x jref, q2 = pji x iref
  const dual g_b3 = gta * ta_b3, g_a3 = gta * ta_a3;
  const dual g_s3 = g_b3 / d;
  g_d = g_d - g_b3 * s3 / (d * d);
  const df3 gc3 = P.c3_0 ? zd : scale3(pji, g_s3);
  gP = axpy3(g_s3, c3, gP);
  df3 gq1 = axpy3(g_a3, q2, cross3(q2, gc3));
  df3 gq2 = axpy3(g_a3, q1, cross3(gc3, q1));
  if (P.q1_0) gq1 = zd;
  if (P.q2_0) gq2 = zd;
  gP = add3(gP, add3(cross3(jref, gq1), cross3(iref, gq2)));
  const df3 gS = cross3(gq1, pji), gR = cross3(gq2, pji);
  // d = sqrt(sum(pji^2)) of phi / tau
  gP = axpy3(g_d / d, pji, gP);
  // pl1 = M x in0, pl2 = M x in1
  gM = add3(gM, add3(cross3(in0, gpl1), cross3(in1, gpl2)));
  gA = add3(gA, cross3(gpl1, M));
  const df3 gB = cross3(gpl2, M);
  gP = sub3(gP, gM);
  float* w = work + (size_t)e * 15;
  const f3 out[5] = {tangent3(gP), tangent3(gA), tangent3(gB), tangent3(gR), tangent3(gS)};
#pragma unroll
  for (int k = 0; k < 5; ++k) { w[3 * k] = out[k].x; w[3 * k + 1] = out[k].y; w[3 * k + 2] = out[k].z; }
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

// The cell term of the kernel above: dcell[g][a][b] = sum over graph g's edges of cell_offsets[e][a] * dvec[e][b].  One
// CTA per graph over its contiguous edge range (target-sorted order); each thread sums a fixed stride of edges, then a
// fixed shared-memory tree: no float atomics, the same bits run to run.
constexpr int CELL_BWD_THREADS = 256;
__global__ void __launch_bounds__(CELL_BWD_THREADS)
pbc_cell_bwd_kernel(const float* __restrict__ dvec, const float* __restrict__ cell_offsets,
                    const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ graph_ptr,
                    float* __restrict__ dcell) {
  __shared__ float red[9][CELL_BWD_THREADS];
  const int g = blockIdx.x, t = threadIdx.x;
  const int lo = row_ptr[graph_ptr[g]], hi = row_ptr[graph_ptr[g + 1]];
  float acc[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) acc[k] = 0.f;
  for (int e = lo + t; e < hi; e += CELL_BWD_THREADS) {
    const f3 o = load3(cell_offsets, e), d = load3(dvec, e);
    const float oa[3] = {o.x, o.y, o.z}, db[3] = {d.x, d.y, d.z};
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) acc[3 * a + b] = fmaf(oa[a], db[b], acc[3 * a + b]);
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) red[k][t] = acc[k];
  __syncthreads();
  for (int s = CELL_BWD_THREADS / 2; s > 0; s >>= 1) {
    if (t < s)
#pragma unroll
      for (int k = 0; k < 9; ++k) red[k][t] += red[k][t + s];
    __syncthreads();
  }
  if (t < 9) dcell[(size_t)g * 9 + t] = red[t][0];
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

}  // extern "C"

// Passes 2 and 3 of the features backward: work[0, 15E) (the five edge-vector gradients of every edge) -> dvec =
// work[15E, 18E) -> dpos
static int comenet_vec_grads_to_dpos(const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                                     const int32_t* out_ptr, const int32_t* out_list, const int32_t* refs,
                                     int64_t n_nodes, int64_t n_edges, float* work, float* dpos, cudaStream_t st) {
  float* dvec = work + 15 * n_edges;
  if (n_edges) {
    comenet_features_bwd_gather_kernel<<<ceil_div(n_edges, 128), 128, 0, st>>>(
        src, dst, row_ptr, out_ptr, out_list, refs, refs + n_nodes, refs + 2 * n_nodes, refs + 3 * n_nodes,
        (int)n_edges, work, dvec);
    DIG3D_LAUNCH_CHECK();
  }
  comenet_features_bwd_node_kernel<<<ceil_div(n_nodes, 128), 128, 0, st>>>(row_ptr, out_ptr, out_list, (int)n_nodes,
                                                                           dvec, dpos);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

// The three passes of the features backward (pos [N,3], or FROM_VEC: vec [E,3]) and the tangent kernel's launch
template <bool FROM_VEC>
static int comenet_features_bwd_launch(const float* pos, const float* dist, const int32_t* src, const int32_t* dst,
                                       const int32_t* row_ptr, const int32_t* out_ptr, const int32_t* out_list,
                                       const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                                       const float* dfeature1, const float* dfeature2, float* work, float* dpos,
                                       void* stream) {
  if (n_nodes == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int32_t* a0i = refs; const int32_t* a1i = refs + n_nodes;
  const int32_t* a0o = refs + 2 * n_nodes; const int32_t* a1o = refs + 3 * n_nodes;
  if (n_edges) {
    comenet_features_bwd_edge_kernel<FROM_VEC><<<ceil_div(n_edges, 128), 128, 0, st>>>(
        pos, dist, src, dst, a0i, a1i, a0o, a1o, (int)n_edges, 1.0f / (float)cutoff, dfeature1, dfeature2, work);
    DIG3D_LAUNCH_CHECK();
  }
  return comenet_vec_grads_to_dpos(src, dst, row_ptr, out_ptr, out_list, refs, n_nodes, n_edges, work, dpos, st);
}

template <bool FROM_VEC>
static int comenet_features_tangent_launch(const float* pos, const float* dist, const int32_t* src, const int32_t* dst,
                                           const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                                           const float* cvec, float* feature1_dot, float* feature2_dot, void* stream) {
  if (n_nodes == 0 || n_edges == 0) return DIG3D_OK;
  comenet_features_tangent_kernel<FROM_VEC><<<ceil_div(n_edges, 128), 128, 0, (cudaStream_t)stream>>>(
      pos, dist, src, dst, refs, refs + n_nodes, refs + 2 * n_nodes, refs + 3 * n_nodes, (int)n_edges,
      1.0f / (float)cutoff, cvec, feature1_dot, feature2_dot);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

// The reverse of the tangent in the positions: pass 1 on duals, then passes 2 and 3 of the backward
template <bool FROM_VEC>
static int comenet_features_tangent_bwd_launch(const float* pos, const float* dist, const int32_t* src,
                                               const int32_t* dst, const int32_t* row_ptr, const int32_t* out_ptr,
                                               const int32_t* out_list, const int32_t* refs, int64_t n_nodes,
                                               int64_t n_edges, double cutoff, const float* cvec, const float* g1,
                                               const float* g2, float* work, float* dpos, void* stream) {
  if (n_nodes == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (n_edges) {
    comenet_features_tangent_bwd_edge_kernel<FROM_VEC><<<ceil_div(n_edges, 128), 128, 0, st>>>(
        pos, dist, src, dst, refs, refs + n_nodes, refs + 2 * n_nodes, refs + 3 * n_nodes, (int)n_edges,
        1.0f / (float)cutoff, cvec, g1, g2, work);
    DIG3D_LAUNCH_CHECK();
  }
  return comenet_vec_grads_to_dpos(src, dst, row_ptr, out_ptr, out_list, refs, n_nodes, n_edges, work, dpos, st);
}

extern "C" {

int dig3d_comenet_features_bwd(const float* pos, const float* dist, const int32_t* src, const int32_t* dst,
                               const int32_t* row_ptr, const int32_t* out_ptr, const int32_t* out_list,
                               const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                               const float* dfeature1, const float* dfeature2, float* work, float* dpos,
                               void* stream) {
  DIG3D_REQUIRE(pos && dist && src && dst && row_ptr && out_ptr && out_list && refs && dfeature1 && dfeature2 &&
                    work && dpos, "comenet_features_bwd: null pointer");
  return comenet_features_bwd_launch<false>(pos, dist, src, dst, row_ptr, out_ptr, out_list, refs, n_nodes, n_edges,
                                            cutoff, dfeature1, dfeature2, work, dpos, stream);
}

int dig3d_comenet_features_tangent(const float* pos, const float* dist, const int32_t* src, const int32_t* dst,
                                   const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                                   const float* cvec, float* feature1_dot, float* feature2_dot, void* stream) {
  DIG3D_REQUIRE(pos && dist && src && dst && refs && cvec && feature1_dot && feature2_dot,
                "comenet_features_tangent: null pointer");
  return comenet_features_tangent_launch<false>(pos, dist, src, dst, refs, n_nodes, n_edges, cutoff, cvec,
                                                feature1_dot, feature2_dot, stream);
}

int dig3d_comenet_features_bwd_vec(const float* vec, const float* dist, const int32_t* src, const int32_t* dst,
                                   const int32_t* row_ptr, const int32_t* out_ptr, const int32_t* out_list,
                                   const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                                   const float* dfeature1, const float* dfeature2, float* work, float* dpos,
                                   void* stream) {
  DIG3D_REQUIRE(vec && dist && src && dst && row_ptr && out_ptr && out_list && refs && dfeature1 && dfeature2 &&
                    work && dpos, "comenet_features_bwd_vec: null pointer");
  return comenet_features_bwd_launch<true>(vec, dist, src, dst, row_ptr, out_ptr, out_list, refs, n_nodes, n_edges,
                                           cutoff, dfeature1, dfeature2, work, dpos, stream);
}

int dig3d_comenet_features_tangent_vec(const float* vec, const float* dist, const int32_t* src, const int32_t* dst,
                                       const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                                       const float* cvec, float* feature1_dot, float* feature2_dot, void* stream) {
  DIG3D_REQUIRE(vec && dist && src && dst && refs && cvec && feature1_dot && feature2_dot,
                "comenet_features_tangent_vec: null pointer");
  return comenet_features_tangent_launch<true>(vec, dist, src, dst, refs, n_nodes, n_edges, cutoff, cvec,
                                               feature1_dot, feature2_dot, stream);
}

int dig3d_comenet_features_tangent_bwd(const float* pos, const float* dist, const int32_t* src, const int32_t* dst,
                                       const int32_t* row_ptr, const int32_t* out_ptr, const int32_t* out_list,
                                       const int32_t* refs, int64_t n_nodes, int64_t n_edges, double cutoff,
                                       const float* cvec, const float* g1, const float* g2, float* work, float* dpos,
                                       void* stream) {
  DIG3D_REQUIRE(pos && dist && src && dst && row_ptr && out_ptr && out_list && refs && cvec && g1 && g2 && work &&
                    dpos, "comenet_features_tangent_bwd: null pointer");
  return comenet_features_tangent_bwd_launch<false>(pos, dist, src, dst, row_ptr, out_ptr, out_list, refs, n_nodes,
                                                    n_edges, cutoff, cvec, g1, g2, work, dpos, stream);
}

int dig3d_comenet_features_tangent_bwd_vec(const float* vec, const float* dist, const int32_t* src,
                                           const int32_t* dst, const int32_t* row_ptr, const int32_t* out_ptr,
                                           const int32_t* out_list, const int32_t* refs, int64_t n_nodes,
                                           int64_t n_edges, double cutoff, const float* cvec, const float* g1,
                                           const float* g2, float* work, float* dpos, void* stream) {
  DIG3D_REQUIRE(vec && dist && src && dst && row_ptr && out_ptr && out_list && refs && cvec && g1 && g2 && work &&
                    dpos, "comenet_features_tangent_bwd_vec: null pointer");
  return comenet_features_tangent_bwd_launch<true>(vec, dist, src, dst, row_ptr, out_ptr, out_list, refs, n_nodes,
                                                   n_edges, cutoff, cvec, g1, g2, work, dpos, stream);
}

int dig3d_pbc_cell_bwd(const float* dvec, const float* cell_offsets, const int32_t* row_ptr, const int32_t* graph_ptr,
                       int64_t n_graphs, float* dcell, void* stream) {
  DIG3D_REQUIRE(dvec && cell_offsets && row_ptr && graph_ptr && dcell, "pbc_cell_bwd: null pointer");
  if (n_graphs == 0) return DIG3D_OK;
  pbc_cell_bwd_kernel<<<(int)n_graphs, CELL_BWD_THREADS, 0, (cudaStream_t)stream>>>(dvec, cell_offsets, row_ptr,
                                                                                     graph_ptr, dcell);
  DIG3D_LAUNCH_CHECK();
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
