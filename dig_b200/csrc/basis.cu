// Radial / angular basis evaluation (sm_90a).
//
//   dist_emb    spherenet/features.py:167-182   env(d/c) * sin(freq * d/c)
//   angle_emb   spherenet/features.py:185-222   j~_ln(d_kj/c) * Y_l0(angle)          -> sbf [T, ns*nr]
//               dimenetpp/features.py:183-220   same with env(d_kj/c) folded in
//   torsion_emb spherenet/features.py:225-263   j~_bn(d_kj/c) * Y_f(angle, torsion)  -> tbf [T, ns*ns*nr]
//
// The closed forms are the generated headers (dig_b200/codegen.py): one correctly rounded fp32
// op per node of the reference's lambdified expression.  The fused model path never materialises
// sbf / tbf: dig3d_triplet_basis_project_lists contracts them with lin_sbf1 / lin_t1 of ALL layers at
// once, grouped by the (k->j) edge so the radial half of the contraction is done once per edge.
#include "common.cuh"
#include "harmonics.cuh"
#include "generated/basis_dimenet_7_6.cuh"
#include "generated/basis_dimenet_3_6.cuh"
#include "generated/basis_gemnet_2_3.cuh"
#include "generated/basis_dimenet_7_6_d2.cuh"
#include "generated/basis_dimenet_3_6_d2.cuh"

namespace dig3d {

struct B76 {
  static constexpr int NS = basis_dimenet_7_6::NS, NR = basis_dimenet_7_6::NR;
  static constexpr int NB = NS * NR, NY = NS * NS;
  __device__ static void bessel(float x, float (&o)[NB]) { basis_dimenet_7_6::bessel(x, o); }
  __device__ static void bessel_order(int l, float x, float (&o)[NR]) { basis_dimenet_7_6::bessel_order(l, x, o); }
  __device__ static void yl0(float t, float (&o)[NS]) { basis_dimenet_7_6::yl0(t, o); }
  __device__ static void ylm(float t, float p, float (&o)[NY]) { basis_dimenet_7_6::ylm(t, p, o); }
  __device__ static void bessel_dx(float x, float (&o)[NB]) { basis_dimenet_7_6::bessel_dx(x, o); }
  __device__ static void yl0_dtheta(float t, float (&o)[NS]) { basis_dimenet_7_6::yl0_dtheta(t, o); }
  __device__ static void ylm_dtheta(float t, float p, float (&o)[NY]) { basis_dimenet_7_6::ylm_dtheta(t, p, o); }
  __device__ static void ylm_dphi(float t, float p, float (&o)[NY]) { basis_dimenet_7_6::ylm_dphi(t, p, o); }
  __device__ static void bessel_dxx(float x, float (&o)[NB]) { basis_dimenet_7_6::bessel_dxx(x, o); }
  __device__ static void yl0_dtheta2(float t, float (&o)[NS]) { basis_dimenet_7_6::yl0_dtheta2(t, o); }
  __device__ static void ylm_dtheta2(float t, float p, float (&o)[NY]) { basis_dimenet_7_6::ylm_dtheta2(t, p, o); }
  __device__ static void ylm_dtheta_dphi(float t, float p, float (&o)[NY]) { basis_dimenet_7_6::ylm_dtheta_dphi(t, p, o); }
  __device__ static void ylm_dphi2(float t, float p, float (&o)[NY]) { basis_dimenet_7_6::ylm_dphi2(t, p, o); }
};
struct B36 {
  static constexpr int NS = basis_dimenet_3_6::NS, NR = basis_dimenet_3_6::NR;
  static constexpr int NB = NS * NR, NY = NS * NS;
  __device__ static void bessel(float x, float (&o)[NB]) { basis_dimenet_3_6::bessel(x, o); }
  __device__ static void bessel_order(int l, float x, float (&o)[NR]) { basis_dimenet_3_6::bessel_order(l, x, o); }
  __device__ static void yl0(float t, float (&o)[NS]) { basis_dimenet_3_6::yl0(t, o); }
  __device__ static void ylm(float t, float p, float (&o)[NY]) { basis_dimenet_3_6::ylm(t, p, o); }
  __device__ static void bessel_dx(float x, float (&o)[NB]) { basis_dimenet_3_6::bessel_dx(x, o); }
  __device__ static void yl0_dtheta(float t, float (&o)[NS]) { basis_dimenet_3_6::yl0_dtheta(t, o); }
  __device__ static void ylm_dtheta(float t, float p, float (&o)[NY]) { basis_dimenet_3_6::ylm_dtheta(t, p, o); }
  __device__ static void ylm_dphi(float t, float p, float (&o)[NY]) { basis_dimenet_3_6::ylm_dphi(t, p, o); }
  __device__ static void bessel_dxx(float x, float (&o)[NB]) { basis_dimenet_3_6::bessel_dxx(x, o); }
  __device__ static void yl0_dtheta2(float t, float (&o)[NS]) { basis_dimenet_3_6::yl0_dtheta2(t, o); }
  __device__ static void ylm_dtheta2(float t, float p, float (&o)[NY]) { basis_dimenet_3_6::ylm_dtheta2(t, p, o); }
  __device__ static void ylm_dtheta_dphi(float t, float p, float (&o)[NY]) { basis_dimenet_3_6::ylm_dtheta_dphi(t, p, o); }
  __device__ static void ylm_dphi2(float t, float p, float (&o)[NY]) { basis_dimenet_3_6::ylm_dphi2(t, p, o); }
};
struct G23 {
  static constexpr int NS = basis_gemnet_2_3::NS, NR = basis_gemnet_2_3::NR;
  static constexpr int NB = NS * NR, NY = NS * NS;
  __device__ static void bessel(float x, float (&o)[NB]) { basis_gemnet_2_3::bessel(x, o); }
  __device__ static void bessel_order(int l, float x, float (&o)[NR]) { basis_gemnet_2_3::bessel_order(l, x, o); }
  __device__ static void yl0(float t, float (&o)[NS]) { basis_gemnet_2_3::yl0(t, o); }
  __device__ static void ylm(float t, float p, float (&o)[NY]) { basis_gemnet_2_3::ylm(t, p, o); }
  __device__ static void bessel_dx(float x, float (&o)[NB]) { basis_gemnet_2_3::bessel_dx(x, o); }
  __device__ static void yl0_dtheta(float t, float (&o)[NS]) { basis_gemnet_2_3::yl0_dtheta(t, o); }
  __device__ static void ylm_dtheta(float t, float p, float (&o)[NY]) { basis_gemnet_2_3::ylm_dtheta(t, p, o); }
  __device__ static void ylm_dphi(float t, float p, float (&o)[NY]) { basis_gemnet_2_3::ylm_dphi(t, p, o); }
};

// Envelope.forward (features.py:159-164), ATen-CUDA op order:
//   1./x -> reciprocal;  x.pow(p-1) -> powf (x*x / x*x*x for exponents 2 / 3)
__device__ __forceinline__ float envelope(float x, int p, float a, float b, float c) {
  const float rcp = __fdiv_rn(1.0f, x);
  float p0;
  const int q = p - 1;
  if (q == 2) p0 = __fmul_rn(x, x);
  else if (q == 3) p0 = __fmul_rn(__fmul_rn(x, x), x);
  else if (q == 1) p0 = x;
  else p0 = powf(x, (float)q);
  const float p1 = __fmul_rn(p0, x);
  const float p2 = __fmul_rn(p1, x);
  float r = __fadd_rn(rcp, __fmul_rn(a, p0));
  r = __fadd_rn(r, __fmul_rn(b, p1));
  r = __fadd_rn(r, __fmul_rn(c, p2));
  return r;
}

// rbf0 [E, NR] and the Bessel values [E, NB] of every edge, one edge's work spread over NS + 1 threads: blockIdx.y =
// Bessel order l (its NR entries, the same expression trees and roundings as bessel(): codegen.emit_bessel_orders) or NS
// for the six rbf0 sines.  One thread per edge would walk ~80 sinf / cosf calls back to back on ~7 resident warps per SM
// (latency bound: 50 us for 34 k edges); split by order the launch has 8x the warps and the critical path is the longest
// single order.  dist / cutoff is dist * (1.0f / cutoff), as ATen CUDA divides by a scalar.
template <class BS>
__global__ void __launch_bounds__(128)
edge_basis_split_kernel(const float* __restrict__ dist, int n_edges, float inv_cutoff, int p, float ea, float eb, float ec,
                        const float* __restrict__ freq, int env_on_bessel, float* __restrict__ rbf0,
                        float* __restrict__ bess) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int part = blockIdx.y;
  if (e >= n_edges) return;
  const float x = __fmul_rn(dist[e], inv_cutoff);
  if (part == BS::NS) {
    if (!rbf0) return;
    const float env = envelope(x, p, ea, eb, ec);
#pragma unroll
    for (int n = 0; n < BS::NR; ++n)
      rbf0[(size_t)e * BS::NR + n] = __fmul_rn(env, sinf(__fmul_rn(__ldg(freq + n), x)));
    return;
  }
  if (!bess) return;
  float b[BS::NR];
  BS::bessel_order(part, x, b);
  const float env = env_on_bessel ? envelope(x, p, ea, eb, ec) : 1.0f;
#pragma unroll
  for (int n = 0; n < BS::NR; ++n)
    bess[(size_t)e * BS::NB + part * BS::NR + n] = env_on_bessel ? __fmul_rn(env, b[n]) : b[n];
}


// d(loss)/d(freq[n]) = sum_e drbf0[e][n] * env(x_e) * cos(freq[n] * x_e) * x_e     (training path; rbf0 = env * sin(freq x),
// reference spherenet/features.py:180-182 -- freq is the only trainable tensor of the basis layers)
__global__ void rbf_freq_grad_kernel(const float* __restrict__ dist, int64_t n_edges, float inv_cutoff, int p, float ea,
                                     float eb, float ec, const float* __restrict__ freq, int nr,
                                     const float* __restrict__ drbf0, float* __restrict__ dfreq) {
  float part[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_edges; e += (int64_t)gridDim.x * blockDim.x) {
    const float x = __fmul_rn(dist[e], inv_cutoff);
    const float ex = envelope(x, p, ea, eb, ec) * x;
    for (int n = 0; n < nr; ++n) part[n] = fmaf(drbf0[e * nr + n], ex * cosf(__ldg(freq + n) * x), part[n]);
  }
  for (int n = 0; n < nr; ++n) {
    float v = part[n];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(dfreq + n, v);
  }
}

template <class BS>
__global__ void triplet_basis_kernel(const float* __restrict__ bess, const float* __restrict__ angle,
                                     const float* __restrict__ torsion, const int32_t* __restrict__ idx_kj,
                                     int n_triplets, float* __restrict__ sbf, float* __restrict__ tbf) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_triplets) return;
  const float* rb = bess + (size_t)idx_kj[t] * BS::NB;
  const float th = angle[t];
  if (sbf) {
    float y0[BS::NS];
    BS::yl0(th, y0);
#pragma unroll
    for (int l = 0; l < BS::NS; ++l)
#pragma unroll
      for (int n = 0; n < BS::NR; ++n)
        sbf[(size_t)t * BS::NB + l * BS::NR + n] = __fmul_rn(__ldg(rb + l * BS::NR + n), y0[l]);
  }
  if (tbf) {
    float y[BS::NY];
    BS::ylm(th, torsion[t], y);
    // (rbf[idx_kj].view(-1,1,n,k) * cbf.view(-1,n,n,1)): out[(a*n+b)*k+r] = rbf[b*k+r]*cbf[a*n+b]
#pragma unroll
    for (int ab = 0; ab < BS::NY; ++ab)
#pragma unroll
      for (int r = 0; r < BS::NR; ++r)
        tbf[(size_t)t * (BS::NY * BS::NR) + ab * BS::NR + r] =
            __fmul_rn(__ldg(rb + (ab % BS::NS) * BS::NR + r), y[ab]);
  }
}

// ------------------------------------------------------------------ fused basis + projection
// One warp per (k->j) edge.  Lane q = (layer l, basis row m), q = l*B + m, L*B == 32.
//   R[ab]  = sum_r bess[kj][b*nr+r] * w_t1[l][m][(ab)*nr+r]        (ab = a*ns+b)   -- per edge
//   Rs[l'] = sum_r bess[kj][l'*nr+r] * w_sbf1[l][m][l'*nr+r]                        -- per edge
// then for every triplet (k->j->i) that uses this edge:
//   t_p[t][q]   = sum_ab Y_ab(angle_t, torsion_t) * R[ab]
//   sbf_p[t][q] = sum_l' Y_l'0(angle_t) * Rs[l']
// The harmonics of up to 32 triplets are evaluated with lane == triplet, parked in shared
// memory, then consumed with lane == (l, m).
// The library launches it without the torsion factor (DimeNet++); the torsion models run
// triplet_basis_project_packed_kernel below.
constexpr int PRJ_WARPS = 8;
constexpr int PRJ_LD = 33;  // lane stride of the transposed weight tables (conflict-free both ways)

template <class BS, bool TORSION>
struct PrjSmem {
  static constexpr int NYT = TORSION ? BS::NY : 1;
  float wt[TORSION ? BS::NY * BS::NR * PRJ_LD : 1];   // [c][lane]: w_t1[lane][c]
  float ws[BS::NB * PRJ_LD];                          // [c][lane]: w_sbf1[lane][c]
  float bess[PRJ_WARPS][BS::NB];
  static constexpr int YLD = ((NYT + BS::NS + 3) / 4) * 4;   // harmonics row, padded for float4 broadcasts
  alignas(16) float y[PRJ_WARPS][32][YLD];
  int32_t trip[PRJ_WARPS][32];
};

// Persistent CTAs (grid ~ 2 per SM): the first-projection weights of all layers are staged ONCE per
// CTA into shared memory, transposed so that lane q reads row q without bank conflicts.
template <class BS, bool TORSION>
__global__ void __launch_bounds__(PRJ_WARPS * 32)
triplet_basis_project_kernel(const float* __restrict__ bess, const float* __restrict__ angle,
                             const float* __restrict__ torsion, const int32_t* __restrict__ src,
                             const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                             const int32_t* __restrict__ trip_ptr, const int32_t* __restrict__ graph_ptr,
                             const int64_t* __restrict__ batch, int n_edges, int n_triplets,
                             const float* __restrict__ w_sbf1, const float* __restrict__ w_t1,
                             float* __restrict__ sbf_p, float* __restrict__ t_p) {
  constexpr int NS = BS::NS, NR = BS::NR, NB = BS::NB, NY = BS::NY;
  constexpr int NYT = TORSION ? NY : 1;
  extern __shared__ __align__(16) unsigned char prj_smem_raw[];
  PrjSmem<BS, TORSION>& sm = *reinterpret_cast<PrjSmem<BS, TORSION>*>(prj_smem_raw);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (TORSION)
    for (int id = threadIdx.x; id < 32 * NY * NR; id += PRJ_WARPS * 32)
      sm.wt[(id % (NY * NR)) * PRJ_LD + id / (NY * NR)] = __ldg(w_t1 + id);
  for (int id = threadIdx.x; id < 32 * NB; id += PRJ_WARPS * 32)
    sm.ws[(id % NB) * PRJ_LD + id / NB] = __ldg(w_sbf1 + id);
  __syncthreads();
  for (int kj = blockIdx.x * PRJ_WARPS + w; kj < n_edges; kj += gridDim.x * PRJ_WARPS) {
    const int k = src[kj], j = dst[kj];
    __syncwarp();
    for (int c = lane; c < NB; c += 32) sm.bess[w][c] = __ldg(bess + (size_t)kj * NB + c);
    __syncwarp();
    // per-edge radial contraction
    float R[NYT], Rs[NS];
#pragma unroll
    for (int b = 0; b < NS; ++b) {     // radial order b outermost: its NR Bessel values are read once
      float rb[NR];
#pragma unroll
      for (int r = 0; r < NR; ++r) rb[r] = sm.bess[w][b * NR + r];
      float acc = 0.f;
#pragma unroll
      for (int r = 0; r < NR; ++r) acc = fmaf(rb[r], sm.ws[(b * NR + r) * PRJ_LD + lane], acc);
      Rs[b] = acc;
      if (TORSION) {
#pragma unroll
        for (int a = 0; a < NS; ++a) {
          const int ab = a * NS + b;
          float acc_t = 0.f;
#pragma unroll
          for (int r = 0; r < NR; ++r) acc_t = fmaf(rb[r], sm.wt[(ab * NR + r) * PRJ_LD + lane], acc_t);
          R[ab] = acc_t;
        }
      }
    }
    // enumerate the out-edges e = (j -> i), i != k, of j: candidates are the nodes of j's graph
    const int jbase = row_ptr[j], dj = row_ptr[j + 1] - jbase;
    const int rank_k = kj - jbase;  // position of k among j's in-neighbours
    const int g = (int)batch[j];
    const int lo = graph_ptr[g], hi = graph_ptr[g + 1];
    for (int c0 = lo; c0 < hi; c0 += 32) {
      const int i = c0 + lane;
      int t = -1;
      if (i < hi && i != k && i != j) {
        const int ib = row_ptr[i], di = row_ptr[i + 1] - ib;
        int a = 0, b = di;  // binary search j among i's in-neighbour sources (ascending)
        while (a < b) { int mid = (a + b) >> 1; if (src[ib + mid] < j) a = mid + 1; else b = mid; }
        if (a < di && src[ib + a] == j) {
          const int e = ib + a;
          // slot of k in e's triplet list: rank_k minus one if i precedes k in j's in-list
          int a2 = 0, b2 = dj;
          while (a2 < b2) { int mid = (a2 + b2) >> 1; if (src[jbase + mid] < i) a2 = mid + 1; else b2 = mid; }
          const bool i_in = (a2 < dj && src[jbase + a2] == i);
          t = trip_ptr[e] + rank_k - ((i_in && a2 < rank_k) ? 1 : 0);
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, t >= 0);
      if (t >= 0) {
        const int slot = __popc(m & ((1u << lane) - 1));
        sm.trip[w][slot] = t;
        const float th = angle[t];
        float y0[NS];
        BS::yl0(th, y0);
#pragma unroll
        for (int l = 0; l < NS; ++l) sm.y[w][slot][NYT + l] = y0[l];
        if (TORSION) {
          float y[NY];
          BS::ylm(th, torsion[t], y);
#pragma unroll
          for (int ab = 0; ab < NY; ++ab) sm.y[w][slot][ab] = y[ab];
        }
      }
      __syncwarp();
      const int cnt = __popc(m);
      for (int s = 0; s < cnt; ++s) {
        const int tt = sm.trip[w][s];
        // harmonics of triplet s: float4 broadcasts (row stride padded to a multiple of 4 floats)
        float yv[PrjSmem<BS, TORSION>::YLD];
#pragma unroll
        for (int i = 0; i < PrjSmem<BS, TORSION>::YLD; i += 4) {
          const float4 q = *reinterpret_cast<const float4*>(&sm.y[w][s][i]);
          yv[i] = q.x; yv[i + 1] = q.y; yv[i + 2] = q.z; yv[i + 3] = q.w;
        }
        float acc_s = 0.f;
#pragma unroll
        for (int l = 0; l < NS; ++l) acc_s = fmaf(yv[NYT + l], Rs[l], acc_s);
        // layer-major output [4][T][8]: each layer later streams its own contiguous 32 B per triplet
        const size_t o = ((size_t)(lane >> 3) * n_triplets + tt) * 8 + (lane & 7);
        sbf_p[o] = acc_s;
        if (TORSION) {
          float acc_t = 0.f;
#pragma unroll
          for (int ab = 0; ab < NY; ++ab) acc_t = fmaf(yv[ab], R[ab], acc_t);
          t_p[o] = acc_t;
        }
      }
      __syncwarp();
    }
  }
}

// ------------------------------------------------------------------ fused projection, packed (torsion models)
// Same traversal and outputs as triplet_basis_project_kernel with the torsion factor, rebuilt around the FP32 issue
// rate (that organisation is bound by its FP32 instruction count):
//   * per-edge radial contraction: for a Bessel order b the NS + 1 outputs Rs[b], R[a*NS + b] share their NR Bessel
//     values, so they run as (NS + 1) / 2 paired FFMA chains on pairs of OUTPUTS -- the weights of a pair sit side by side in
//     shared memory (one LDS.64 per pair of FFMAs), the Bessel values are staged duplicated;
//     every half is the r-ascending chain of the scalar kernel;
//   * the harmonics of a triplet are stored in that pair order ({Y_b0, Y[0*NS+b]}, {Y[1*NS+b], Y[2*NS+b]}, ...; row
//     stride 60 floats: the 16-byte stores of eight lanes fall into eight different bank groups), so the per-triplet
//     contraction is NS * (NS+1) / 2 paired FFMAs on natural register pairs; sbf_p keeps the scalar kernel's summation order,
//     t_p is summed as (NS+1)/2 interleaved partial sums;
//   * the harmonics come from the recurrences of harmonics.cuh (two sincosf + ~250 multiply-adds) instead of the
//     node-by-node closed forms (~1200 instructions); the radial contraction runs AFTER the harmonics so that its 56
//     result registers are not live while they are evaluated.
template <class BS>
struct PrjPackSmem {
  static constexpr int NP = (BS::NS + 1) / 2;                       // output pairs per Bessel order
  static constexpr int ROW = BS::NS * NP * 2;                       // harmonics per triplet in pair order
  static constexpr int YLD = (ROW / 4) % 2 ? ROW : ROW + 4;         // odd number of 16-byte chunks per row
  float2 wp[BS::NS * NP * BS::NR * 32];                             // [(b, p, r)][lane]
  float2 bess2[PRJ_WARPS][BS::NB];                                  // {v, v}
  alignas(16) float y[PRJ_WARPS][32][YLD];
  int32_t trip[PRJ_WARPS][32];
};

template <class BS>
__global__ void __launch_bounds__(PRJ_WARPS * 32, 2)
triplet_basis_project_packed_kernel(const float* __restrict__ bess, const float* __restrict__ angle,
                                    const float* __restrict__ torsion, const int32_t* __restrict__ src,
                                    const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                                    const int32_t* __restrict__ trip_ptr, const int32_t* __restrict__ graph_ptr,
                                    const int64_t* __restrict__ batch, int n_edges, int n_triplets,
                                    const float* __restrict__ w_sbf1, const float* __restrict__ w_t1,
                                    float* __restrict__ sbf_p, float* __restrict__ t_p,
                                    const int32_t* __restrict__ out_ptr, const int32_t* __restrict__ out_list,
                                    const int32_t* __restrict__ pos_in) {
  constexpr int NS = BS::NS, NR = BS::NR, NB = BS::NB, NY = BS::NY;
  using SM = PrjPackSmem<BS>;
  constexpr int NP = SM::NP, ROW = SM::ROW;
  static_assert((NS + 1) % 2 == 0 && ROW % 4 == 0, "packed projection: NS must be odd");
  extern __shared__ __align__(16) unsigned char prj_smem_raw[];
  SM& sm = *reinterpret_cast<SM*>(prj_smem_raw);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  // output o of order b: o = 0 -> Rs[b] (lin_sbf1 column b*NR + r), o >= 1 -> R[(o-1)*NS + b] (lin_t1 column ...)
  for (int id = threadIdx.x; id < NS * NP * NR * 32; id += PRJ_WARPS * 32) {
    const int q = id & 31, r = (id >> 5) % NR, p = ((id >> 5) / NR) % NP, b = (id >> 5) / (NR * NP);
    float v[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int o = 2 * p + h;
      v[h] = o == 0 ? __ldg(w_sbf1 + q * NB + b * NR + r) : __ldg(w_t1 + q * (NY * NR) + ((o - 1) * NS + b) * NR + r);
    }
    sm.wp[id] = make_float2(v[0], v[1]);
  }
  __syncthreads();
  for (int kj = blockIdx.x * PRJ_WARPS + w; kj < n_edges; kj += gridDim.x * PRJ_WARPS) {
    const int k = src[kj], j = dst[kj];
    __syncwarp();
    for (int c = lane; c < NB; c += 32) {
      const float v = __ldg(bess + (size_t)kj * NB + c);
      sm.bess2[w][c] = make_float2(v, v);
    }
    const int jbase = row_ptr[j], dj = row_ptr[j + 1] - jbase;
    const int rank_k = kj - jbase;  // position of k among j's in-neighbours
    const bool lists = out_ptr != nullptr;
    int lo, hi;
    if (lists) { lo = out_ptr[j]; hi = out_ptr[j + 1]; }
    else { const int g = (int)batch[j]; lo = graph_ptr[g]; hi = graph_ptr[g + 1]; }
    for (int c0 = lo; c0 < hi; c0 += 32) {
      // out-edges e = (j -> i), i != k: from the list of the graph build (entry c0 + lane; the position of i among j's
      // in-neighbours comes with it, i == k <=> that position is rank_k), or searched among the nodes of j's graph
      const int i = c0 + lane;
      int t = -1;
      if (lists) {
        if (i < hi) {
          const int e = out_list[i], p = pos_in[e];
          if (p != rank_k) t = trip_ptr[e] + rank_k - (p < rank_k ? 1 : 0);
        }
      } else if (i < hi && i != k && i != j) {
        const int ib = row_ptr[i], di = row_ptr[i + 1] - ib;
        int a = 0, b = di;
        while (a < b) { int mid = (a + b) >> 1; if (src[ib + mid] < j) a = mid + 1; else b = mid; }
        if (a < di && src[ib + a] == j) {
          const int e = ib + a;
          int a2 = 0, b2 = dj;
          while (a2 < b2) { int mid = (a2 + b2) >> 1; if (src[jbase + mid] < i) a2 = mid + 1; else b2 = mid; }
          const bool i_in = (a2 < dj && src[jbase + a2] == i);
          t = trip_ptr[e] + rank_k - ((i_in && a2 < rank_k) ? 1 : 0);
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, t >= 0);
      const int cnt = __popc(m);
      if (cnt == 0) continue;
      if (t >= 0) {
        const int slot = __popc(m & ((1u << lane) - 1));
        sm.trip[w][slot] = t;
        float y[NY], y0[NS];
        ylm_recurrence<NS>(angle[t], torsion[t], y, y0);
        float yp[ROW];
#pragma unroll
        for (int b = 0; b < NS; ++b)
#pragma unroll
          for (int o = 0; o <= NS; ++o) yp[(b * NP + (o >> 1)) * 2 + (o & 1)] = o == 0 ? y0[b] : y[(o - 1) * NS + b];
        float4* row = reinterpret_cast<float4*>(&sm.y[w][slot][0]);
#pragma unroll
        for (int c = 0; c < ROW / 4; ++c) row[c] = make_float4(yp[4 * c], yp[4 * c + 1], yp[4 * c + 2], yp[4 * c + 3]);
      }
      __syncwarp();
      // per-edge radial contraction, lane = output column q (4 layers x 8)
      float2 R[NS][NP];
#pragma unroll
      for (int b = 0; b < NS; ++b) {
        float2 rb[NR];
#pragma unroll
        for (int r = 0; r < NR; ++r) rb[r] = sm.bess2[w][b * NR + r];
#pragma unroll
        for (int p = 0; p < NP; ++p) {
          float2 acc = make_float2(0.f, 0.f);
#pragma unroll
          for (int r = 0; r < NR; ++r) acc = ffma2(rb[r], sm.wp[((b * NP + p) * NR + r) * 32 + lane], acc);
          R[b][p] = acc;
        }
      }
      for (int s = 0; s < cnt; ++s) {
        const int tt = sm.trip[w][s];
        const float4* row = reinterpret_cast<const float4*>(&sm.y[w][s][0]);
        float2 acc[NP];
#pragma unroll
        for (int p = 0; p < NP; ++p) acc[p] = make_float2(0.f, 0.f);
#pragma unroll
        for (int c = 0; c < ROW / 4; ++c) {
          const float4 v = row[c];                     // pairs 2c, 2c + 1 of the row = (b, p) in b-major order
          const int i0 = 2 * c, i1 = 2 * c + 1;
          acc[i0 % NP] = ffma2(make_float2(v.x, v.y), R[i0 / NP][i0 % NP], acc[i0 % NP]);
          acc[i1 % NP] = ffma2(make_float2(v.z, v.w), R[i1 / NP][i1 % NP], acc[i1 % NP]);
        }
        // acc[0].x = sum_b Y_b0 Rs[b] (b ascending, as the scalar kernel); everything else belongs to t_p
        float2 rest = make_float2(0.f, 0.f);
#pragma unroll
        for (int p = 1; p < NP; ++p) rest = fadd2(rest, acc[p]);
        const size_t o = ((size_t)(lane >> 3) * n_triplets + tt) * 8 + (lane & 7);
        sbf_p[o] = acc[0].x;
        t_p[o] = (acc[0].y + rest.x) + rest.y;
      }
      __syncwarp();
    }
  }
}

// ------------------------------------------------------------------ backward of the fused projection (training path)
// d(loss)/d(lin_sbf1.weight), d(loss)/d(lin_t1.weight) of up to four layers from d sbf_p[l][T, 8] / d t_p[l][T, 8]:
//   dW_t1[q][(a*ns+b)*nr + r] = sum_kj ( sum_{t uses kj} d t_p[q][t] * Y_ab(t) ) * bess[kj][b*nr + r]      (q = layer*8 + row)
// Same traversal as the forward kernel (one warp per (k->j) edge, lane = q, the harmonics of its triplets parked in
// shared memory); the inner sum G[ab] stays in registers, the outer product with the edge's Bessel values goes into a
// per-CTA shared-memory accumulator (shared atomics, lane-distinct banks) that is flushed once per CTA.  The [T, 294]
// basis is never materialised.
struct PrjGradPtrs { const float* ds[4]; const float* dt[4]; };   // passed by value as a kernel argument

template <class BS, bool TORSION>
struct PrjBwdSmem {
  static constexpr int NYT = TORSION ? BS::NY : 1;
  float dwt[TORSION ? BS::NY * BS::NR * PRJ_LD : 1];
  float dws[BS::NB * PRJ_LD];
  float bess[PRJ_WARPS][BS::NB];
  static constexpr int YLD = ((NYT + BS::NS + 3) / 4) * 4;
  alignas(16) float y[PRJ_WARPS][32][YLD];
  int32_t trip[PRJ_WARPS][32];
};

template <class BS, bool TORSION>
__global__ void __launch_bounds__(PRJ_WARPS * 32)
triplet_basis_project_bwd_kernel(const float* __restrict__ bess, const float* __restrict__ angle,
                                 const float* __restrict__ torsion, const int32_t* __restrict__ src,
                                 const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                                 const int32_t* __restrict__ trip_ptr, const int32_t* __restrict__ graph_ptr,
                                 const int64_t* __restrict__ batch, int n_edges, PrjGradPtrs gp,
                                 float* __restrict__ dw_sbf1 /*[32, NB]*/, float* __restrict__ dw_t1 /*[32, NY*NR]*/) {
  constexpr int NS = BS::NS, NR = BS::NR, NB = BS::NB, NY = BS::NY;
  constexpr int NYT = TORSION ? NY : 1;
  using SM = PrjBwdSmem<BS, TORSION>;
  extern __shared__ __align__(16) unsigned char prj_smem_raw[];
  SM& sm = *reinterpret_cast<SM*>(prj_smem_raw);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (TORSION)
    for (int id = threadIdx.x; id < NY * NR * PRJ_LD; id += PRJ_WARPS * 32) sm.dwt[id] = 0.f;
  for (int id = threadIdx.x; id < NB * PRJ_LD; id += PRJ_WARPS * 32) sm.dws[id] = 0.f;
  __syncthreads();
  const float* my_ds = gp.ds[lane >> 3];
  const float* my_dt = TORSION ? gp.dt[lane >> 3] : nullptr;
  const int mrow = lane & 7;
  for (int kj = blockIdx.x * PRJ_WARPS + w; kj < n_edges; kj += gridDim.x * PRJ_WARPS) {
    const int k = src[kj], j = dst[kj];
    __syncwarp();
    for (int c = lane; c < NB; c += 32) sm.bess[w][c] = __ldg(bess + (size_t)kj * NB + c);
    float G[NYT], Gs[NS];
#pragma unroll
    for (int i = 0; i < NYT; ++i) G[i] = 0.f;
#pragma unroll
    for (int i = 0; i < NS; ++i) Gs[i] = 0.f;
    const int jbase = row_ptr[j], dj = row_ptr[j + 1] - jbase;
    const int rank_k = kj - jbase;
    const int g = (int)batch[j];
    const int lo = graph_ptr[g], hi = graph_ptr[g + 1];
    for (int c0 = lo; c0 < hi; c0 += 32) {
      const int i = c0 + lane;
      int t = -1;
      if (i < hi && i != k && i != j) {
        const int ib = row_ptr[i], di = row_ptr[i + 1] - ib;
        int a = 0, b = di;
        while (a < b) { int mid = (a + b) >> 1; if (src[ib + mid] < j) a = mid + 1; else b = mid; }
        if (a < di && src[ib + a] == j) {
          const int e = ib + a;
          int a2 = 0, b2 = dj;
          while (a2 < b2) { int mid = (a2 + b2) >> 1; if (src[jbase + mid] < i) a2 = mid + 1; else b2 = mid; }
          const bool i_in = (a2 < dj && src[jbase + a2] == i);
          t = trip_ptr[e] + rank_k - ((i_in && a2 < rank_k) ? 1 : 0);
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, t >= 0);
      if (t >= 0) {
        const int slot = __popc(m & ((1u << lane) - 1));
        sm.trip[w][slot] = t;
        const float th = angle[t];
        float y0[NS];
        BS::yl0(th, y0);
#pragma unroll
        for (int l = 0; l < NS; ++l) sm.y[w][slot][NYT + l] = y0[l];
        if (TORSION) {
          float y[NY];
          BS::ylm(th, torsion[t], y);
#pragma unroll
          for (int ab = 0; ab < NY; ++ab) sm.y[w][slot][ab] = y[ab];
        }
      }
      __syncwarp();
      const int cnt = __popc(m);
      for (int s = 0; s < cnt; ++s) {
        const int tt = sm.trip[w][s];
        float yv[SM::YLD];
#pragma unroll
        for (int i = 0; i < SM::YLD; i += 4) {
          const float4 q = *reinterpret_cast<const float4*>(&sm.y[w][s][i]);
          yv[i] = q.x; yv[i + 1] = q.y; yv[i + 2] = q.z; yv[i + 3] = q.w;
        }
        const float d_s = my_ds ? __ldg(my_ds + (size_t)tt * 8 + mrow) : 0.f;
#pragma unroll
        for (int l = 0; l < NS; ++l) Gs[l] = fmaf(d_s, yv[NYT + l], Gs[l]);
        if (TORSION) {
          const float d_t = my_dt ? __ldg(my_dt + (size_t)tt * 8 + mrow) : 0.f;
#pragma unroll
          for (int ab = 0; ab < NY; ++ab) G[ab] = fmaf(d_t, yv[ab], G[ab]);
        }
      }
      __syncwarp();
    }
    // outer product with the edge's Bessel values into the CTA accumulators
#pragma unroll
    for (int b = 0; b < NS; ++b) {
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        const float rb = sm.bess[w][b * NR + r];
        atomicAdd(&sm.dws[(b * NR + r) * PRJ_LD + lane], Gs[b] * rb);
        if (TORSION) {
#pragma unroll
          for (int a = 0; a < NS; ++a)
            atomicAdd(&sm.dwt[((a * NS + b) * NR + r) * PRJ_LD + lane], G[a * NS + b] * rb);
        }
      }
    }
  }
  __syncthreads();
  for (int id = threadIdx.x; id < 32 * NB; id += PRJ_WARPS * 32) {
    const int q = id / NB, c = id % NB;
    atomicAdd(dw_sbf1 + id, sm.dws[c * PRJ_LD + q]);
  }
  if (TORSION)
    for (int id = threadIdx.x; id < 32 * NY * NR; id += PRJ_WARPS * 32) {
      const int q = id / (NY * NR), c = id % (NY * NR);
      atomicAdd(dw_t1 + id, sm.dwt[c * PRJ_LD + q]);
    }
}

// ------------------------------------------------------------------ force path: d(basis)/d(dist), d(basis)/d(angle)
// env'(x) = -1/x^2 + a (p-1) x^(p-2) + b p x^(p-1) + c (p+1) x^p
__device__ __forceinline__ float envelope_dx(float x, int p, float a, float b, float c) {
  const float xp2 = powf(x, (float)(p - 2));
  const float xp1 = xp2 * x, xp0 = xp1 * x;
  return -1.0f / (x * x) + a * (float)(p - 1) * xp2 + b * (float)p * xp1 + c * (float)(p + 1) * xp0;
}

// Per edge: ddist[e] = sum_n drbf0[e][n] * d(env(x) sin(freq_n x))/dx / cutoff   (x = dist / cutoff), and the
// x-derivative of the edge's (enveloped) Bessel basis, kept for triplet_basis_project_bwd_geom.
template <class BS>
__global__ void edge_basis_bwd_kernel(const float* __restrict__ dist, int n_edges, float inv_cutoff, int p, float ea,
                                      float eb, float ec, const float* __restrict__ freq, int env_on_bessel,
                                      const float* __restrict__ drbf0, float* __restrict__ ddist,
                                      float* __restrict__ bess_dx) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const float x = __fmul_rn(dist[e], inv_cutoff);
  const float env = envelope(x, p, ea, eb, ec), envd = envelope_dx(x, p, ea, eb, ec);
  if (ddist) {
    float acc = 0.f;
    if (drbf0) {
#pragma unroll
      for (int n = 0; n < BS::NR; ++n) {
        const float f = __ldg(freq + n);
        acc = fmaf(drbf0[(size_t)e * BS::NR + n], envd * sinf(f * x) + env * f * cosf(f * x), acc);
      }
    }
    ddist[e] = acc * inv_cutoff;
  }
  if (bess_dx) {
    float b[BS::NB], bd[BS::NB];
    BS::bessel(x, b);
    BS::bessel_dx(x, bd);
#pragma unroll
    for (int c = 0; c < BS::NB; ++c)
      bess_dx[(size_t)e * BS::NB + c] = env_on_bessel ? fmaf(envd, b[c], env * bd[c]) : bd[c];
  }
}

// ------------------------------------------------------------------ forward-mode basis (force training, autograd_jvp.py)
// Tangents of the edge bases along a displacement with dist_dot[e] = d(dist_e)/d(eps):
//   rbf0_dot[e][n] = d(env(x) sin(f_n x))/dx * dist_dot / cutoff,   bess_dot[e][c] = d(bess[e][c])/dx * dist_dot / cutoff.
template <class BS>
__global__ void edge_basis_tangent_kernel(const float* __restrict__ dist, const float* __restrict__ dist_dot, int n_edges,
                                          float inv_cutoff, int p, float ea, float eb, float ec,
                                          const float* __restrict__ freq, int env_on_bessel,
                                          float* __restrict__ rbf0_dot, float* __restrict__ bess_dot) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const float x = __fmul_rn(dist[e], inv_cutoff);
  const float xd = dist_dot[e] * inv_cutoff;
  const float env = envelope(x, p, ea, eb, ec), envd = envelope_dx(x, p, ea, eb, ec);
  if (rbf0_dot) {
#pragma unroll
    for (int n = 0; n < BS::NR; ++n) {
      const float f = __ldg(freq + n);
      rbf0_dot[(size_t)e * BS::NR + n] = (envd * sinf(f * x) + env * f * cosf(f * x)) * xd;
    }
  }
  if (bess_dot) {
    float b[BS::NB], bd[BS::NB];
    BS::bessel(x, b);
    BS::bessel_dx(x, bd);
#pragma unroll
    for (int c = 0; c < BS::NB; ++c)
      bess_dot[(size_t)e * BS::NB + c] = (env_on_bessel ? fmaf(envd, b[c], env * bd[c]) : bd[c]) * xd;
  }
}

// d(loss)/d(freq[n]) through rbf0_dot:  sum_e G[e][n] * xd_e * d/df ( env' sin(f x) + env f cos(f x) )
//                                     = sum_e G[e][n] * xd_e * ( env' x cos(f x) + env (cos(f x) - f x sin(f x)) )
__global__ void rbf_freq_grad_tangent_kernel(const float* __restrict__ dist, const float* __restrict__ dist_dot,
                                             int64_t n_edges, float inv_cutoff, int p, float ea, float eb, float ec,
                                             const float* __restrict__ freq, int nr, const float* __restrict__ g_dot,
                                             float* __restrict__ dfreq) {
  float part[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_edges; e += (int64_t)gridDim.x * blockDim.x) {
    const float x = __fmul_rn(dist[e], inv_cutoff);
    const float xd = dist_dot[e] * inv_cutoff;
    const float env = envelope(x, p, ea, eb, ec), envd = envelope_dx(x, p, ea, eb, ec);
    for (int n = 0; n < nr; ++n) {
      const float f = __ldg(freq + n);
      float sn, cs;
      sincosf(f * x, &sn, &cs);
      part[n] = fmaf(g_dot[e * nr + n] * xd, envd * x * cs + env * (cs - f * x * sn), part[n]);
    }
  }
  for (int n = 0; n < nr; ++n) {
    float v = part[n];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(dfreq + n, v);
  }
}

// Tangents of the materialised triplet bases (layouts of triplet_basis_kernel):
//   sbf_dot[t][l,n]  = Y_l0'(th) th_dot bess[kj][l,n] + Y_l0(th) bess_dot[kj][l,n]
//   tbf_dot[t][ab,r] = (dY_ab/dth th_dot + dY_ab/dph ph_dot) bess[kj][b,r] + Y_ab bess_dot[kj][b,r]
template <class BS>
__global__ void triplet_basis_tangent_kernel(const float* __restrict__ bess, const float* __restrict__ bess_dot,
                                             const float* __restrict__ angle, const float* __restrict__ angle_dot,
                                             const float* __restrict__ torsion, const float* __restrict__ torsion_dot,
                                             const int32_t* __restrict__ idx_kj, int n_triplets,
                                             float* __restrict__ sbf_dot, float* __restrict__ tbf_dot) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_triplets) return;
  const float* rb = bess + (size_t)idx_kj[t] * BS::NB;
  const float* rd = bess_dot + (size_t)idx_kj[t] * BS::NB;
  const float th = angle[t], thd = angle_dot[t];
  if (sbf_dot) {
    float y0[BS::NS], y0d[BS::NS];
    BS::yl0(th, y0);
    BS::yl0_dtheta(th, y0d);
#pragma unroll
    for (int l = 0; l < BS::NS; ++l)
#pragma unroll
      for (int n = 0; n < BS::NR; ++n)
        sbf_dot[(size_t)t * BS::NB + l * BS::NR + n] =
            fmaf(y0d[l] * thd, __ldg(rb + l * BS::NR + n), y0[l] * __ldg(rd + l * BS::NR + n));
  }
  if (tbf_dot) {
    const float ph = torsion[t], phd = torsion_dot[t];
    float y[BS::NY], yd[BS::NY];
    BS::ylm_dtheta(th, ph, yd);
    BS::ylm_dphi(th, ph, y);
#pragma unroll
    for (int ab = 0; ab < BS::NY; ++ab) yd[ab] = fmaf(yd[ab], thd, y[ab] * phd);
    BS::ylm(th, ph, y);
#pragma unroll
    for (int ab = 0; ab < BS::NY; ++ab)
#pragma unroll
      for (int r = 0; r < BS::NR; ++r)
        tbf_dot[(size_t)t * (BS::NY * BS::NR) + ab * BS::NR + r] =
            fmaf(yd[ab], __ldg(rb + (ab % BS::NS) * BS::NR + r), y[ab] * __ldg(rd + (ab % BS::NS) * BS::NR + r));
  }
}

// Reverse mode of triplet_basis_kernel (the transpose of triplet_basis_tangent_kernel), for the generic triplet branch
// (materialised bases, any int_emb_size / basis_emb_size) on the force path:
//   dangle[t]   = sum_{l,n}  d_sbf[t][l,n]  Y_l0'(th) bess[kj][l,n] + sum_{ab,r} d_tbf[t][ab,r] dY_ab/dth bess[kj][b,r]
//   dtorsion[t] = sum_{ab,r} d_tbf[t][ab,r] dY_ab/dph bess[kj][b,r]
//   ddist[kj]   = (1/cutoff) sum_{t: idx_kj[t] = kj} ( sum_{l,n} d_sbf[t][l,n] Y_l0 bess_dx[kj][l,n]
//                                                     + sum_{ab,r} d_tbf[t][ab,r] Y_ab bess_dx[kj][b,r] )
// with bess_dx = d(bess)/dx, x = dist / cutoff (edge_basis_bwd_kernel).  The harmonics and their derivatives are the
// generated closed forms the forward and tangent kernels call, so the three cannot drift apart.
// One warp per (k->j) edge; lane = one triplet that uses the edge as its k->j edge, found through the out-edge lists of
// j (edges j->i, 32 per pass): the triplet of (k->j, j->i) sits at trip_ptr[ji] + rank(k) - (rank(i) < rank(k)), the
// order triplet_geometry writes (rank = position among j's in-edges; pos_in[ji] = rank(i), deg(j) when i is none).
// Every triplet is the k->j triplet of exactly one edge, so dangle / dtorsion are written once each, and ddist[kj] is a
// sum the warp owns: per-lane partials in pass order, then a fixed butterfly.  No float atomics and no kj-sorted copy
// of the triplets: the result is the same bit for bit from run to run.  Edges that are no triplet's k->j edge get 0.
constexpr int TBB_WARPS = 4;

template <class BS>
__global__ void __launch_bounds__(TBB_WARPS * 32)
triplet_basis_bwd_kernel(const float* __restrict__ bess, const float* __restrict__ bess_dx,
                         const float* __restrict__ angle, const float* __restrict__ torsion,
                         const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                         const int32_t* __restrict__ trip_ptr, const int32_t* __restrict__ out_ptr,
                         const int32_t* __restrict__ out_list, const int32_t* __restrict__ pos_in, int n_edges,
                         const float* __restrict__ d_sbf, const float* __restrict__ d_tbf, float inv_cutoff,
                         float* __restrict__ ddist, float* __restrict__ dangle, float* __restrict__ dtorsion) {
  constexpr int NS = BS::NS, NR = BS::NR, NB = BS::NB, NY = BS::NY;
  __shared__ float sb[TBB_WARPS][NB], sbd[TBB_WARPS][NB];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kj = blockIdx.x * TBB_WARPS + w;
  if (kj >= n_edges) return;                                   // uniform per warp
  for (int c = lane; c < NB; c += 32) {
    sb[w][c] = bess[(size_t)kj * NB + c];
    sbd[w][c] = bess_dx[(size_t)kj * NB + c];
  }
  __syncwarp();
  const int j = dst[kj], rank_k = kj - row_ptr[j];
  const int o_lo = out_ptr[j], o_hi = out_ptr[j + 1];
  float acc_x = 0.f;
  for (int o0 = o_lo; o0 < o_hi; o0 += 32) {
    const int o = o0 + lane;
    if (o >= o_hi) continue;
    const int ji = out_list[o], rank_i = pos_in[ji];
    if (rank_i == rank_k) continue;                            // i == k: no triplet
    const int t = trip_ptr[ji] + rank_k - (rank_i < rank_k ? 1 : 0);
    const float th = angle[t];
    float dth = 0.f, dph = 0.f, dx = 0.f;
    if (d_sbf) {
      const float* ds = d_sbf + (size_t)t * NB;
      float y0[NS], y0d[NS];
      BS::yl0(th, y0);
      BS::yl0_dtheta(th, y0d);
#pragma unroll
      for (int l = 0; l < NS; ++l) {
        float h = 0.f, hd = 0.f;
#pragma unroll
        for (int n = 0; n < NR; ++n) {
          const float gr = ds[l * NR + n];
          h = fmaf(gr, sb[w][l * NR + n], h);
          hd = fmaf(gr, sbd[w][l * NR + n], hd);
        }
        dth = fmaf(y0d[l], h, dth);
        dx = fmaf(y0[l], hd, dx);
      }
    }
    if (d_tbf) {
      const float ph = torsion[t];
      const float* dt = d_tbf + (size_t)t * (NY * NR);
      float H[NY], Hd[NY];
#pragma unroll
      for (int ab = 0; ab < NY; ++ab) {
        const int b = ab % NS;
        float h = 0.f, hd = 0.f;
#pragma unroll
        for (int r = 0; r < NR; ++r) {
          const float gr = dt[ab * NR + r];
          h = fmaf(gr, sb[w][b * NR + r], h);
          hd = fmaf(gr, sbd[w][b * NR + r], hd);
        }
        H[ab] = h;
        Hd[ab] = hd;
      }
      {
        float y[NY];
        BS::ylm(th, ph, y);
#pragma unroll
        for (int ab = 0; ab < NY; ++ab) dx = fmaf(y[ab], Hd[ab], dx);
      }
      {
        float y[NY];
        BS::ylm_dtheta(th, ph, y);
#pragma unroll
        for (int ab = 0; ab < NY; ++ab) dth = fmaf(y[ab], H[ab], dth);
      }
      {
        float y[NY];
        BS::ylm_dphi(th, ph, y);
#pragma unroll
        for (int ab = 0; ab < NY; ++ab) dph = fmaf(y[ab], H[ab], dph);
      }
    }
    dangle[t] = dth;
    if (dtorsion) dtorsion[t] = dph;
    acc_x += dx;
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) acc_x += __shfl_xor_sync(0xffffffffu, acc_x, off);
  if (lane == 0) ddist[kj] = acc_x * inv_cutoff;
}

// ------------------------------------------------------------------ reverse mode of the tangent kernels (Hessians)
// The tangents above are first derivatives of the bases times the geometry tangents.  Their reverse mode in the VALUE
// inputs (dist, angle, torsion) needs the second derivatives: the closed forms of generated/basis_<tag>_d2.cuh and
//   env''(x) = 2/x^3 + a (p-1)(p-2) x^(p-3) + b p (p-1) x^(p-2) + c (p+1) p x^(p-1).
// Their reverse mode in the tangent inputs is a first-order backward.  d(H v) = one reverse pass over the tangent
// network along v (autograd_jvp.py), so these kernels are what reaches the positions from a force's gradient.
__device__ __forceinline__ float envelope_dxx(float x, int p, float a, float b, float c) {
  const float xp3 = powf(x, (float)(p - 3));
  const float xp2 = xp3 * x, xp1 = xp2 * x;
  return 2.0f / (x * x * x) + a * (float)((p - 1) * (p - 2)) * xp3 + b * (float)(p * (p - 1)) * xp2 +
         c * (float)((p + 1) * p) * xp1;
}

// Reverse of rbf0_dot[e][n] = f_n'(x) xd  (f_n = env(x) sin(freq_n x), x = dist / cutoff, xd = dist_dot / cutoff)
// given G = d(loss)/d(rbf0_dot):
//   d_dist[e]     = sum_n G[e][n] f_n''(x) xd / cutoff,   d_dist_dot[e] = sum_n G[e][n] f_n'(x) / cutoff
// and, when bess_dxx is given, d2(bess)/dx2 of the edge (enveloped as the forward's bess when env_on_bessel), which
// triplet_basis_tangent_bwd reads.  One thread per edge, each output written once.
template <class BS>
__global__ void edge_basis_tangent_bwd_kernel(const float* __restrict__ dist, const float* __restrict__ dist_dot,
                                              int n_edges, float inv_cutoff, int p, float ea, float eb, float ec,
                                              const float* __restrict__ freq, int env_on_bessel,
                                              const float* __restrict__ g_rbf0_dot, float* __restrict__ d_dist,
                                              float* __restrict__ d_dist_dot, float* __restrict__ bess_dxx) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const float x = __fmul_rn(dist[e], inv_cutoff);
  const float env = envelope(x, p, ea, eb, ec), envd = envelope_dx(x, p, ea, eb, ec);
  const float envdd = envelope_dxx(x, p, ea, eb, ec);
  if (g_rbf0_dot) {
    const float xd = dist_dot[e] * inv_cutoff;
    float a1 = 0.f, a2 = 0.f;
#pragma unroll
    for (int n = 0; n < BS::NR; ++n) {
      const float f = __ldg(freq + n);
      float sn, cs;
      sincosf(f * x, &sn, &cs);
      const float gn = g_rbf0_dot[(size_t)e * BS::NR + n];
      a1 = fmaf(gn, envd * sn + env * f * cs, a1);
      a2 = fmaf(gn, envdd * sn + 2.0f * envd * f * cs - env * f * f * sn, a2);
    }
    d_dist[e] = a2 * xd * inv_cutoff;
    d_dist_dot[e] = a1 * inv_cutoff;
  }
  if (bess_dxx) {
    float b2[BS::NB];
    BS::bessel_dxx(x, b2);
    if (env_on_bessel) {
      float b[BS::NB], b1[BS::NB];
      BS::bessel(x, b);
      BS::bessel_dx(x, b1);
#pragma unroll
      for (int c = 0; c < BS::NB; ++c) b2[c] = envdd * b[c] + 2.0f * envd * b1[c] + env * b2[c];
    }
#pragma unroll
    for (int c = 0; c < BS::NB; ++c) bess_dxx[(size_t)e * BS::NB + c] = b2[c];
  }
}

// Reverse of triplet_basis_tangent_kernel (with bess_dot = B'(x) xd folded in) in all of its inputs, given
// Gs = d(loss)/d(sbf_dot) and Gt = d(loss)/d(tbf_dot).  Per triplet, with H_k[l] = sum_n Gs[l,n] B^(k)[kj][l,n]
// (B, B', B'' the edge's Bessel values and x-derivatives) and Y = Y_l0(th):
//   d_angle      = sum_l Y'' thd H0 + Y' xd H1         d_angle_dot = sum_l Y' H0
//   d_x (kj)     = sum_l Y' thd H1 + Y xd H2           d_xd (kj)   = sum_l Y H1
// and for the torsion branch, with Y = Y_ab(th, ph), Yd = Y_th thd + Y_ph phd and H_k[ab] = sum_r Gt[ab,r] B^(k)[b,r]:
//   d_angle     += sum_ab (Y_thth thd + Y_thph phd) H0 + Y_th xd H1     d_angle_dot   += sum_ab Y_th H0
//   d_torsion    = sum_ab (Y_thph thd + Y_phph phd) H0 + Y_ph xd H1     d_torsion_dot  = sum_ab Y_ph H0
//   d_x         += sum_ab Yd H1 + Y xd H2                                d_xd          += sum_ab Y H1
// (x-derivatives of the Bessel part: H1 / H2 with B', B'').
// d_dist[kj] = sum d_x / cutoff and d_dist_dot[kj] = sum d_xd / cutoff over the triplets whose k->j edge is kj.  The
// triplets of an edge are found as in triplet_basis_bwd_kernel (one warp per k->j edge, the out-edge lists of j), so
// the edge sums are owned by one warp: no float atomics, the same bits on every run.
template <class BS>
__global__ void __launch_bounds__(TBB_WARPS * 32)
triplet_basis_tangent_bwd_kernel(const float* __restrict__ bess, const float* __restrict__ bess_dx,
                                 const float* __restrict__ bess_dxx, const float* __restrict__ dist_dot,
                                 const float* __restrict__ angle, const float* __restrict__ angle_dot,
                                 const float* __restrict__ torsion, const float* __restrict__ torsion_dot,
                                 const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                                 const int32_t* __restrict__ trip_ptr, const int32_t* __restrict__ out_ptr,
                                 const int32_t* __restrict__ out_list, const int32_t* __restrict__ pos_in, int n_edges,
                                 const float* __restrict__ g_sbf, const float* __restrict__ g_tbf, float inv_cutoff,
                                 float* __restrict__ d_dist, float* __restrict__ d_dist_dot,
                                 float* __restrict__ d_angle, float* __restrict__ d_angle_dot,
                                 float* __restrict__ d_torsion, float* __restrict__ d_torsion_dot) {
  constexpr int NS = BS::NS, NR = BS::NR, NB = BS::NB, NY = BS::NY;
  __shared__ float sb[TBB_WARPS][3][NB];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kj = blockIdx.x * TBB_WARPS + w;
  if (kj >= n_edges) return;                                   // uniform per warp
  for (int c = lane; c < NB; c += 32) {
    sb[w][0][c] = bess[(size_t)kj * NB + c];
    sb[w][1][c] = bess_dx[(size_t)kj * NB + c];
    sb[w][2][c] = bess_dxx[(size_t)kj * NB + c];
  }
  __syncwarp();
  const float xd = dist_dot[kj] * inv_cutoff;
  const int j = dst[kj], rank_k = kj - row_ptr[j];
  const int o_lo = out_ptr[j], o_hi = out_ptr[j + 1];
  float acc_x = 0.f, acc_xd = 0.f;
  for (int o0 = o_lo; o0 < o_hi; o0 += 32) {
    const int o = o0 + lane;
    if (o >= o_hi) continue;
    const int ji = out_list[o], rank_i = pos_in[ji];
    if (rank_i == rank_k) continue;                            // i == k: no triplet
    const int t = trip_ptr[ji] + rank_k - (rank_i < rank_k ? 1 : 0);
    const float th = angle[t], thd = angle_dot[t];
    float dth = 0.f, dthd = 0.f, dph = 0.f, dphd = 0.f, dx = 0.f, dxd = 0.f;
    if (g_sbf) {
      const float* gs = g_sbf + (size_t)t * NB;
      float y0[NS], y1[NS], y2[NS];
      BS::yl0(th, y0);
      BS::yl0_dtheta(th, y1);
      BS::yl0_dtheta2(th, y2);
#pragma unroll
      for (int l = 0; l < NS; ++l) {
        float h0 = 0.f, h1 = 0.f, h2 = 0.f;
#pragma unroll
        for (int n = 0; n < NR; ++n) {
          const float gr = gs[l * NR + n];
          h0 = fmaf(gr, sb[w][0][l * NR + n], h0);
          h1 = fmaf(gr, sb[w][1][l * NR + n], h1);
          h2 = fmaf(gr, sb[w][2][l * NR + n], h2);
        }
        dth = fmaf(y2[l] * thd, h0, fmaf(y1[l] * xd, h1, dth));
        dthd = fmaf(y1[l], h0, dthd);
        dx = fmaf(y1[l] * thd, h1, fmaf(y0[l] * xd, h2, dx));
        dxd = fmaf(y0[l], h1, dxd);
      }
    }
    if (g_tbf) {
      const float ph = torsion[t], phd = torsion_dot[t];
      const float* gt = g_tbf + (size_t)t * (NY * NR);
      // H0 is kept per (a, b); H1 / H2 are recomputed where they are read (registers: the harmonics take NY each)
      auto hk = [&](int ab, int k) {
        const int b = ab % NS;
        float h = 0.f;
#pragma unroll
        for (int r = 0; r < NR; ++r) h = fmaf(gt[ab * NR + r], sb[w][k][b * NR + r], h);
        return h;
      };
      float H0[NY];
#pragma unroll
      for (int ab = 0; ab < NY; ++ab) H0[ab] = hk(ab, 0);
      {
        float y[NY];
        BS::ylm(th, ph, y);
#pragma unroll
        for (int ab = 0; ab < NY; ++ab) {
          dx = fmaf(y[ab] * xd, hk(ab, 2), dx);
          dxd = fmaf(y[ab], hk(ab, 1), dxd);
        }
      }
      {
        float y[NY];
        BS::ylm_dtheta(th, ph, y);
#pragma unroll
        for (int ab = 0; ab < NY; ++ab) {
          const float h1 = hk(ab, 1);
          dth = fmaf(y[ab] * xd, h1, dth);
          dthd = fmaf(y[ab], H0[ab], dthd);
          dx = fmaf(y[ab] * thd, h1, dx);
        }
      }
      {
        float y[NY];
        BS::ylm_dphi(th, ph, y);
#pragma unroll
        for (int ab = 0; ab < NY; ++ab) {
          const float h1 = hk(ab, 1);
          dph = fmaf(y[ab] * xd, h1, dph);
          dphd = fmaf(y[ab], H0[ab], dphd);
          dx = fmaf(y[ab] * phd, h1, dx);
        }
      }
      {
        float y[NY];
        BS::ylm_dtheta2(th, ph, y);
#pragma unroll
        for (int ab = 0; ab < NY; ++ab) dth = fmaf(y[ab] * thd, H0[ab], dth);
      }
      {
        float y[NY];
        BS::ylm_dtheta_dphi(th, ph, y);
#pragma unroll
        for (int ab = 0; ab < NY; ++ab) {
          dth = fmaf(y[ab] * phd, H0[ab], dth);
          dph = fmaf(y[ab] * thd, H0[ab], dph);
        }
      }
      {
        float y[NY];
        BS::ylm_dphi2(th, ph, y);
#pragma unroll
        for (int ab = 0; ab < NY; ++ab) dph = fmaf(y[ab] * phd, H0[ab], dph);
      }
    }
    d_angle[t] = dth;
    d_angle_dot[t] = dthd;
    if (d_torsion) d_torsion[t] = dph;
    if (d_torsion_dot) d_torsion_dot[t] = dphd;
    acc_x += dx;
    acc_xd += dxd;
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) {
    acc_x += __shfl_xor_sync(0xffffffffu, acc_x, off);
    acc_xd += __shfl_xor_sync(0xffffffffu, acc_xd, off);
  }
  if (lane == 0) {
    d_dist[kj] = acc_x * inv_cutoff;
    d_dist_dot[kj] = acc_xd * inv_cutoff;
  }
}

// Backward of the fused projection w.r.t. the geometry (forces):
//   sbf_p[q][t] = sum_l  Y_l0(angle_t)            Rs[q][l],   Rs[q][l]  = sum_r bess[kj][l,r]  w_sbf1[q][l,r]
//   t_p[q][t]   = sum_ab Y_ab(angle_t, torsion_t) R[q][ab],   R[q][ab]  = sum_r bess[kj][b,r]  w_t1[q][ab,r]
// => dangle[t]   = sum_l Y_l0' Hs[l] + sum_ab dY_ab/dtheta H[ab],   Hs[l] = sum_q d sbf_p[q][t] Rs[q][l],  H[ab] = sum_q d t_p[q][t] R[q][ab]
//    dtorsion[t] = sum_ab dY_ab/dphi H[ab]
//    ddist[kj]   = (1/cutoff) sum_{t uses kj} ( sum_l Y_l0 Hsd[l] + sum_ab Y_ab Hd[ab] ),  Hsd / Hd from d(bess)/dx.
// One warp per (k->j) edge: first lane = q builds the four per-edge matrices in shared memory, then lane = TRIPLET
// (the candidate enumeration of the forward kernel already yields one triplet per lane) contracts them with its 32
// upstream gradients; the harmonics and their derivatives are evaluated in registers, nothing per-triplet is staged.
constexpr int PRJG_WARPS = 4;

template <class BS, bool TORSION>
struct PrjGeomSmem {
  static constexpr int NYT = TORSION ? BS::NY : 1;
  float wt[TORSION ? BS::NY * BS::NR * PRJ_LD : 1];
  float ws[BS::NB * PRJ_LD];
  float bess[PRJG_WARPS][BS::NB];
  float bessd[PRJG_WARPS][BS::NB];
  alignas(16) float R[PRJG_WARPS][NYT][32];
  alignas(16) float Rd[PRJG_WARPS][NYT][32];
  alignas(16) float Rs[PRJG_WARPS][BS::NS][32];
  alignas(16) float Rsd[PRJG_WARPS][BS::NS][32];
};

__device__ __forceinline__ void dot32(const float (&d)[32], const float* __restrict__ row, const float* __restrict__ rowd,
                                      float& h, float& hd) {
  float a0 = 0.f, a1 = 0.f;
#pragma unroll
  for (int q = 0; q < 32; q += 4) {
    const float4 r = *reinterpret_cast<const float4*>(row + q);
    const float4 rd = *reinterpret_cast<const float4*>(rowd + q);
    a0 = fmaf(d[q], r.x, a0); a0 = fmaf(d[q + 1], r.y, a0); a0 = fmaf(d[q + 2], r.z, a0); a0 = fmaf(d[q + 3], r.w, a0);
    a1 = fmaf(d[q], rd.x, a1); a1 = fmaf(d[q + 1], rd.y, a1); a1 = fmaf(d[q + 2], rd.z, a1); a1 = fmaf(d[q + 3], rd.w, a1);
  }
  h = a0;
  hd = a1;
}

__device__ __forceinline__ void load_grad32(const float* const (&ptr)[4], int t, float (&d)[32]) {
#pragma unroll
  for (int l = 0; l < 4; ++l) {
    if (ptr[l]) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(ptr[l] + (size_t)t * 8));
      const float4 b = __ldg(reinterpret_cast<const float4*>(ptr[l] + (size_t)t * 8 + 4));
      d[l * 8] = a.x; d[l * 8 + 1] = a.y; d[l * 8 + 2] = a.z; d[l * 8 + 3] = a.w;
      d[l * 8 + 4] = b.x; d[l * 8 + 5] = b.y; d[l * 8 + 6] = b.z; d[l * 8 + 7] = b.w;
    } else {
#pragma unroll
      for (int m = 0; m < 8; ++m) d[l * 8 + m] = 0.f;
    }
  }
}

template <class BS, bool TORSION>
__global__ void __launch_bounds__(PRJG_WARPS * 32)
triplet_basis_project_bwd_geom_kernel(const float* __restrict__ bess, const float* __restrict__ bess_dx,
                                      const float* __restrict__ angle, const float* __restrict__ torsion,
                                      const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                      const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ trip_ptr,
                                      const int32_t* __restrict__ graph_ptr, const int64_t* __restrict__ batch,
                                      int n_edges, PrjGradPtrs gp, const float* __restrict__ w_sbf1,
                                      const float* __restrict__ w_t1, float inv_cutoff, float* __restrict__ ddist,
                                      float* __restrict__ dangle, float* __restrict__ dtorsion) {
  constexpr int NS = BS::NS, NR = BS::NR, NB = BS::NB, NY = BS::NY;
  using SM = PrjGeomSmem<BS, TORSION>;
  extern __shared__ __align__(16) unsigned char prj_smem_raw[];
  SM& sm = *reinterpret_cast<SM*>(prj_smem_raw);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (TORSION)
    for (int id = threadIdx.x; id < 32 * NY * NR; id += PRJG_WARPS * 32)
      sm.wt[(id % (NY * NR)) * PRJ_LD + id / (NY * NR)] = __ldg(w_t1 + id);
  for (int id = threadIdx.x; id < 32 * NB; id += PRJG_WARPS * 32) sm.ws[(id % NB) * PRJ_LD + id / NB] = __ldg(w_sbf1 + id);
  __syncthreads();
  for (int kj = blockIdx.x * PRJG_WARPS + w; kj < n_edges; kj += gridDim.x * PRJG_WARPS) {
    const int k = src[kj], j = dst[kj];
    __syncwarp();
    for (int c = lane; c < NB; c += 32) {
      sm.bess[w][c] = __ldg(bess + (size_t)kj * NB + c);
      sm.bessd[w][c] = __ldg(bess_dx + (size_t)kj * NB + c);
    }
    __syncwarp();
    // lane = q: per-edge radial contractions (values and x-derivatives)
#pragma unroll
    for (int b = 0; b < NS; ++b) {
      float rb[NR], rbd[NR];
#pragma unroll
      for (int r = 0; r < NR; ++r) { rb[r] = sm.bess[w][b * NR + r]; rbd[r] = sm.bessd[w][b * NR + r]; }
      float a0 = 0.f, a1 = 0.f;
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        const float wv = sm.ws[(b * NR + r) * PRJ_LD + lane];
        a0 = fmaf(rb[r], wv, a0);
        a1 = fmaf(rbd[r], wv, a1);
      }
      sm.Rs[w][b][lane] = a0;
      sm.Rsd[w][b][lane] = a1;
      if (TORSION) {
#pragma unroll
        for (int a = 0; a < NS; ++a) {
          const int ab = a * NS + b;
          float c0 = 0.f, c1 = 0.f;
#pragma unroll
          for (int r = 0; r < NR; ++r) {
            const float wv = sm.wt[(ab * NR + r) * PRJ_LD + lane];
            c0 = fmaf(rb[r], wv, c0);
            c1 = fmaf(rbd[r], wv, c1);
          }
          sm.R[w][ab][lane] = c0;
          sm.Rd[w][ab][lane] = c1;
        }
      }
    }
    __syncwarp();
    float acc_x = 0.f;
    const int jbase = row_ptr[j], dj = row_ptr[j + 1] - jbase;
    const int rank_k = kj - jbase;
    const int g = (int)batch[j];
    const int lo = graph_ptr[g], hi = graph_ptr[g + 1];
    for (int c0 = lo; c0 < hi; c0 += 32) {
      const int i = c0 + lane;
      int t = -1;
      if (i < hi && i != k && i != j) {
        const int ib = row_ptr[i], di = row_ptr[i + 1] - ib;
        int a = 0, b = di;
        while (a < b) { int mid = (a + b) >> 1; if (src[ib + mid] < j) a = mid + 1; else b = mid; }
        if (a < di && src[ib + a] == j) {
          const int e = ib + a;
          int a2 = 0, b2 = dj;
          while (a2 < b2) { int mid = (a2 + b2) >> 1; if (src[jbase + mid] < i) a2 = mid + 1; else b2 = mid; }
          const bool i_in = (a2 < dj && src[jbase + a2] == i);
          t = trip_ptr[e] + rank_k - ((i_in && a2 < rank_k) ? 1 : 0);
        }
      }
      if (t < 0) continue;                                  // lanes are independent from here on
      const float th = angle[t];
      float d[32];
      float dth = 0.f, dph = 0.f, dx = 0.f;
      {
        load_grad32(gp.ds, t, d);
        float y0[NS], y0d[NS];
        BS::yl0(th, y0);
        BS::yl0_dtheta(th, y0d);
#pragma unroll
        for (int l = 0; l < NS; ++l) {
          float h, hd;
          dot32(d, sm.Rs[w][l], sm.Rsd[w][l], h, hd);
          dth = fmaf(y0d[l], h, dth);
          dx = fmaf(y0[l], hd, dx);
        }
      }
      if (TORSION) {
        const float ph = torsion[t];
        load_grad32(gp.dt, t, d);
        float H[NY], Hd[NY];
#pragma unroll
        for (int ab = 0; ab < NY; ++ab) dot32(d, sm.R[w][ab], sm.Rd[w][ab], H[ab], Hd[ab]);
        {
          float y[NY];
          BS::ylm(th, ph, y);
#pragma unroll
          for (int ab = 0; ab < NY; ++ab) dx = fmaf(y[ab], Hd[ab], dx);
        }
        {
          float y[NY];
          BS::ylm_dtheta(th, ph, y);
#pragma unroll
          for (int ab = 0; ab < NY; ++ab) dth = fmaf(y[ab], H[ab], dth);
        }
        {
          float y[NY];
          BS::ylm_dphi(th, ph, y);
#pragma unroll
          for (int ab = 0; ab < NY; ++ab) dph = fmaf(y[ab], H[ab], dph);
        }
        dtorsion[t] = dph;
      }
      dangle[t] = dth;
      acc_x += dx;
    }
    __syncwarp();
#pragma unroll
    for (int o = 16; o; o >>= 1) acc_x += __shfl_xor_sync(0xffffffffu, acc_x, o);
    if (lane == 0) ddist[kj] = acc_x * inv_cutoff;
  }
}

template <class BS>
static int launch_edge_basis(const float* dist, int64_t n_edges, double cutoff, int exponent,
                             const float* freq, int env_on_bessel, float* rbf0, float* bess,
                             cudaStream_t st) {
  const int p = exponent + 1;
  const float a = (float)(-(p + 1) * (p + 2) / 2.0), b = (float)(p * (p + 2)), c = (float)(-p * (p + 1) / 2.0);
  const float inv = 1.0f / (float)cutoff;
  edge_basis_split_kernel<BS><<<dim3(ceil_div(n_edges, 128), BS::NS + 1), 128, 0, st>>>(
      dist, (int)n_edges, inv, p, a, b, c, freq, env_on_bessel, rbf0, bess);
  return 0;
}

}  // namespace dig3d

using namespace dig3d;

extern "C" {

int dig3d_edge_basis(const float* dist, int64_t n_edges, double cutoff, int32_t envelope_exponent,
                     const float* freq, int32_t basis_id, int32_t envelope_on_bessel, float* rbf0,
                     float* bess, void* stream) {
  DIG3D_REQUIRE(dist && (rbf0 || bess), "edge_basis: null pointer");
  DIG3D_REQUIRE(!rbf0 || freq, "edge_basis: rbf0 requested without freq");
  if (n_edges == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  switch (basis_id) {
    case 0: launch_edge_basis<B76>(dist, n_edges, cutoff, envelope_exponent, freq, envelope_on_bessel, rbf0, bess, st); break;
    case 1: launch_edge_basis<B36>(dist, n_edges, cutoff, envelope_exponent, freq, envelope_on_bessel, rbf0, bess, st); break;
    case 2: launch_edge_basis<G23>(dist, n_edges, cutoff, envelope_exponent, freq, envelope_on_bessel, rbf0, bess, st); break;
    default: set_error("edge_basis: unknown basis_id %d", basis_id); return DIG3D_EUNSUPPORTED;
  }
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_rbf_freq_grad(const float* dist, int64_t n_edges, double cutoff, int32_t envelope_exponent,
                        const float* freq, int32_t num_radial, const float* drbf0, float* dfreq, void* stream) {
  DIG3D_REQUIRE(dist && freq && drbf0 && dfreq && num_radial > 0 && num_radial <= 8, "rbf_freq_grad: bad arguments");
  if (n_edges == 0) return DIG3D_OK;
  const int p = envelope_exponent + 1;
  const float a = (float)(-(p + 1) * (p + 2) / 2.0), b = (float)(p * (p + 2)), c = (float)(-p * (p + 1) / 2.0);
  int grid = ceil_div(n_edges, 256);
  if (grid > 592) grid = 592;
  rbf_freq_grad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(dist, n_edges, 1.0f / (float)cutoff, p, a, b, c, freq,
                                                               num_radial, drbf0, dfreq);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_basis(const float* bess, const float* angle, const float* torsion, const int32_t* idx_kj,
                        int64_t n_triplets, int32_t basis_id, float* sbf, float* tbf, void* stream) {
  DIG3D_REQUIRE(bess && angle && idx_kj && (sbf || tbf), "triplet_basis: null pointer");
  DIG3D_REQUIRE(!tbf || torsion, "triplet_basis: tbf requested without torsion");
  if (n_triplets == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ceil_div(n_triplets, 128);
  switch (basis_id) {
    case 0: triplet_basis_kernel<B76><<<grid, 128, 0, st>>>(bess, angle, torsion, idx_kj, (int)n_triplets, sbf, tbf); break;
    case 1: triplet_basis_kernel<B36><<<grid, 128, 0, st>>>(bess, angle, torsion, idx_kj, (int)n_triplets, sbf, tbf); break;
    default: set_error("triplet_basis: unsupported basis_id %d", basis_id); return DIG3D_EUNSUPPORTED;
  }
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_edge_basis_tangent(const float* dist, const float* dist_dot, int64_t n_edges, double cutoff,
                             int32_t envelope_exponent, const float* freq, int32_t basis_id, int32_t envelope_on_bessel,
                             float* rbf0_dot, float* bess_dot, void* stream) {
  DIG3D_REQUIRE(dist && dist_dot && (rbf0_dot || bess_dot), "edge_basis_tangent: null pointer");
  DIG3D_REQUIRE(!rbf0_dot || freq, "edge_basis_tangent: rbf0_dot needs freq");
  if (n_edges == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int p = envelope_exponent + 1;
  const float a = -(float)((p + 1) * (p + 2)) / 2.f, b = (float)(p * (p + 2)), c = -(float)(p * (p + 1)) / 2.f;
  const float inv = 1.0f / (float)cutoff;
  const int grid = ceil_div(n_edges, 128);
  switch (basis_id) {
    case 0: edge_basis_tangent_kernel<B76><<<grid, 128, 0, st>>>(dist, dist_dot, (int)n_edges, inv, p, a, b, c, freq, envelope_on_bessel, rbf0_dot, bess_dot); break;
    case 1: edge_basis_tangent_kernel<B36><<<grid, 128, 0, st>>>(dist, dist_dot, (int)n_edges, inv, p, a, b, c, freq, envelope_on_bessel, rbf0_dot, bess_dot); break;
    default: set_error("edge_basis_tangent: unsupported basis_id %d", basis_id); return DIG3D_EUNSUPPORTED;
  }
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_rbf_freq_grad_tangent(const float* dist, const float* dist_dot, int64_t n_edges, double cutoff,
                                int32_t envelope_exponent, const float* freq, int32_t nr, const float* g_dot,
                                float* dfreq, void* stream) {
  DIG3D_REQUIRE(dist && dist_dot && freq && g_dot && dfreq, "rbf_freq_grad_tangent: null pointer");
  DIG3D_REQUIRE(nr >= 1 && nr <= 8, "rbf_freq_grad_tangent: num_radial=%d outside [1,8]", nr);
  if (n_edges == 0) return DIG3D_OK;
  const int p = envelope_exponent + 1;
  const float a = -(float)((p + 1) * (p + 2)) / 2.f, b = (float)(p * (p + 2)), c = -(float)(p * (p + 1)) / 2.f;
  const int grid = (int)(ceil_div(n_edges, 256) < 296 ? ceil_div(n_edges, 256) : 296);
  rbf_freq_grad_tangent_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(dist, dist_dot, n_edges, 1.0f / (float)cutoff, p,
                                                                      a, b, c, freq, nr, g_dot, dfreq);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_basis_tangent(const float* bess, const float* bess_dot, const float* angle, const float* angle_dot,
                                const float* torsion, const float* torsion_dot, const int32_t* idx_kj,
                                int64_t n_triplets, int32_t basis_id, float* sbf_dot, float* tbf_dot, void* stream) {
  DIG3D_REQUIRE(bess && bess_dot && angle && angle_dot && idx_kj && (sbf_dot || tbf_dot), "triplet_basis_tangent: null pointer");
  DIG3D_REQUIRE(!tbf_dot || (torsion && torsion_dot), "triplet_basis_tangent: tbf_dot requested without torsion / torsion_dot");
  if (n_triplets == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ceil_div(n_triplets, 128);
  switch (basis_id) {
    case 0: triplet_basis_tangent_kernel<B76><<<grid, 128, 0, st>>>(bess, bess_dot, angle, angle_dot, torsion, torsion_dot, idx_kj, (int)n_triplets, sbf_dot, tbf_dot); break;
    case 1: triplet_basis_tangent_kernel<B36><<<grid, 128, 0, st>>>(bess, bess_dot, angle, angle_dot, torsion, torsion_dot, idx_kj, (int)n_triplets, sbf_dot, tbf_dot); break;
    default: set_error("triplet_basis_tangent: unsupported basis_id %d", basis_id); return DIG3D_EUNSUPPORTED;
  }
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_basis_bwd(const float* bess, const float* bess_dx, const float* angle, const float* torsion,
                            const int32_t* dst, const int32_t* row_ptr, const int32_t* trip_ptr, const int32_t* out_ptr,
                            const int32_t* out_list, const int32_t* pos_in, int64_t n_edges, int64_t n_triplets,
                            int32_t basis_id, const float* d_sbf, const float* d_tbf, double cutoff, float* ddist,
                            float* dangle, float* dtorsion, void* stream) {
  DIG3D_REQUIRE(cutoff > 0.0, "triplet_basis_bwd: cutoff must be positive");
  if (n_edges == 0) return DIG3D_OK;
  // without triplets every per-triplet buffer is empty (possibly NULL): only ddist (all zeros) is written
  DIG3D_REQUIRE(bess && bess_dx && dst && row_ptr && trip_ptr && out_ptr && out_list && pos_in && ddist &&
                    (n_triplets == 0 || (angle && dangle)), "triplet_basis_bwd: null pointer");
  DIG3D_REQUIRE(n_triplets == 0 || !(d_tbf || dtorsion) || torsion, "triplet_basis_bwd: d_tbf / dtorsion need torsion");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ceil_div(n_edges, TBB_WARPS);
  const float inv = 1.0f / (float)cutoff;
  if (n_triplets == 0) { d_sbf = nullptr; d_tbf = nullptr; dtorsion = nullptr; }
  switch (basis_id) {
    case 0: triplet_basis_bwd_kernel<B76><<<grid, TBB_WARPS * 32, 0, st>>>(bess, bess_dx, angle, torsion, dst, row_ptr, trip_ptr, out_ptr, out_list, pos_in, (int)n_edges, d_sbf, d_tbf, inv, ddist, dangle, dtorsion); break;
    case 1: triplet_basis_bwd_kernel<B36><<<grid, TBB_WARPS * 32, 0, st>>>(bess, bess_dx, angle, torsion, dst, row_ptr, trip_ptr, out_ptr, out_list, pos_in, (int)n_edges, d_sbf, d_tbf, inv, ddist, dangle, dtorsion); break;
    default: set_error("triplet_basis_bwd: unsupported basis_id %d", basis_id); return DIG3D_EUNSUPPORTED;
  }
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_edge_basis_tangent_bwd(const float* dist, const float* dist_dot, int64_t n_edges, double cutoff,
                                 int32_t envelope_exponent, const float* freq, int32_t basis_id,
                                 int32_t envelope_on_bessel, const float* g_rbf0_dot, float* d_dist, float* d_dist_dot,
                                 float* bess_dxx, void* stream) {
  DIG3D_REQUIRE(dist && (g_rbf0_dot || bess_dxx), "edge_basis_tangent_bwd: null pointer");
  DIG3D_REQUIRE(!g_rbf0_dot || (dist_dot && freq && d_dist && d_dist_dot),
                "edge_basis_tangent_bwd: g_rbf0_dot needs dist_dot, freq, d_dist and d_dist_dot");
  DIG3D_REQUIRE(cutoff > 0.0, "edge_basis_tangent_bwd: cutoff must be positive");
  if (n_edges == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int p = envelope_exponent + 1;
  const float a = -(float)((p + 1) * (p + 2)) / 2.f, b = (float)(p * (p + 2)), c = -(float)(p * (p + 1)) / 2.f;
  const float inv = 1.0f / (float)cutoff;
  const int grid = ceil_div(n_edges, 128);
  switch (basis_id) {
    case 0: edge_basis_tangent_bwd_kernel<B76><<<grid, 128, 0, st>>>(dist, dist_dot, (int)n_edges, inv, p, a, b, c, freq, envelope_on_bessel, g_rbf0_dot, d_dist, d_dist_dot, bess_dxx); break;
    case 1: edge_basis_tangent_bwd_kernel<B36><<<grid, 128, 0, st>>>(dist, dist_dot, (int)n_edges, inv, p, a, b, c, freq, envelope_on_bessel, g_rbf0_dot, d_dist, d_dist_dot, bess_dxx); break;
    default: set_error("edge_basis_tangent_bwd: unsupported basis_id %d", basis_id); return DIG3D_EUNSUPPORTED;
  }
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_basis_tangent_bwd(const float* bess, const float* bess_dx, const float* bess_dxx,
                                    const float* dist_dot, const float* angle, const float* angle_dot,
                                    const float* torsion, const float* torsion_dot, const int32_t* dst,
                                    const int32_t* row_ptr, const int32_t* trip_ptr, const int32_t* out_ptr,
                                    const int32_t* out_list, const int32_t* pos_in, int64_t n_edges,
                                    int64_t n_triplets, int32_t basis_id, const float* g_sbf, const float* g_tbf,
                                    double cutoff, float* d_dist, float* d_dist_dot, float* d_angle,
                                    float* d_angle_dot, float* d_torsion, float* d_torsion_dot, void* stream) {
  DIG3D_REQUIRE(cutoff > 0.0, "triplet_basis_tangent_bwd: cutoff must be positive");
  if (n_edges == 0) return DIG3D_OK;
  // without triplets every per-triplet buffer is empty (possibly NULL): only the edge outputs (zeros) are written
  DIG3D_REQUIRE(bess && bess_dx && bess_dxx && dist_dot && dst && row_ptr && trip_ptr && out_ptr && out_list &&
                    pos_in && d_dist && d_dist_dot && (n_triplets == 0 || (angle && angle_dot && d_angle && d_angle_dot)),
                "triplet_basis_tangent_bwd: null pointer");
  DIG3D_REQUIRE(n_triplets == 0 || !(g_tbf || d_torsion || d_torsion_dot) || (torsion && torsion_dot),
                "triplet_basis_tangent_bwd: the torsion branch needs torsion and torsion_dot");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ceil_div(n_edges, TBB_WARPS);
  const float inv = 1.0f / (float)cutoff;
  if (n_triplets == 0) { g_sbf = nullptr; g_tbf = nullptr; d_torsion = nullptr; d_torsion_dot = nullptr; }
  switch (basis_id) {
    case 0: triplet_basis_tangent_bwd_kernel<B76><<<grid, TBB_WARPS * 32, 0, st>>>(bess, bess_dx, bess_dxx, dist_dot, angle, angle_dot, torsion, torsion_dot, dst, row_ptr, trip_ptr, out_ptr, out_list, pos_in, (int)n_edges, g_sbf, g_tbf, inv, d_dist, d_dist_dot, d_angle, d_angle_dot, d_torsion, d_torsion_dot); break;
    case 1: triplet_basis_tangent_bwd_kernel<B36><<<grid, TBB_WARPS * 32, 0, st>>>(bess, bess_dx, bess_dxx, dist_dot, angle, angle_dot, torsion, torsion_dot, dst, row_ptr, trip_ptr, out_ptr, out_list, pos_in, (int)n_edges, g_sbf, g_tbf, inv, d_dist, d_dist_dot, d_angle, d_angle_dot, d_torsion, d_torsion_dot); break;
    default: set_error("triplet_basis_tangent_bwd: unsupported basis_id %d", basis_id); return DIG3D_EUNSUPPORTED;
  }
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_basis_project_lists(const float* bess, const float* angle, const float* torsion,
                                      const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                                      const int32_t* trip_ptr, const int32_t* graph_ptr, const int64_t* batch,
                                      int64_t n_edges, int64_t n_triplets, int32_t basis_id, int32_t n_layers,
                                      int32_t basis_emb, const float* w_sbf1, const float* w_t1, float* sbf_p,
                                      float* t_p, const int32_t* out_ptr, const int32_t* out_list,
                                      const int32_t* pos_in, void* stream) {
  DIG3D_REQUIRE(bess && angle && src && dst && row_ptr && trip_ptr && graph_ptr && batch && w_sbf1 && sbf_p,
                "triplet_basis_project: null pointer");
  DIG3D_REQUIRE((out_ptr != nullptr) == (out_list != nullptr) && (out_ptr != nullptr) == (pos_in != nullptr),
                "triplet_basis_project: out_ptr, out_list and pos_in come together");
  DIG3D_REQUIRE(n_layers * basis_emb == 32, "triplet_basis_project: n_layers*basis_emb must be 32, got %d*%d",
                n_layers, basis_emb);
  const bool tors = (t_p != nullptr);
  DIG3D_REQUIRE(!tors || (torsion && w_t1), "triplet_basis_project: torsion path needs torsion and w_t1");
  if (n_edges == 0 || n_triplets == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int dev = 0, n_sm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  const int grid = (int)((n_edges + PRJ_WARPS - 1) / PRJ_WARPS < 2 * n_sm ? (n_edges + PRJ_WARPS - 1) / PRJ_WARPS
                                                                          : 2 * n_sm);
#define DIG3D_PRJ_ONE(BS)                                                                                   \
  {                                                                                                         \
    auto kfn = triplet_basis_project_kernel<BS, false>;                                                     \
    const size_t smem = sizeof(PrjSmem<BS, false>);                                                         \
    if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { \
      set_error("triplet_basis_project: cannot reserve %zu bytes of shared memory", smem);                  \
      return DIG3D_ECUDA;                                                                                   \
    }                                                                                                       \
    kfn<<<grid, PRJ_WARPS * 32, smem, st>>>(bess, angle, torsion, src, dst, row_ptr, trip_ptr, graph_ptr,   \
                                            batch, (int)n_edges, (int)n_triplets, w_sbf1, w_t1, sbf_p, t_p);\
  }
#define DIG3D_PRJP_ONE(BS)                                                                                  \
  {                                                                                                         \
    auto kfn = triplet_basis_project_packed_kernel<BS>;                                                     \
    const size_t smem = sizeof(PrjPackSmem<BS>);                                                            \
    if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { \
      set_error("triplet_basis_project: cannot reserve %zu bytes of shared memory", smem);                  \
      return DIG3D_ECUDA;                                                                                   \
    }                                                                                                       \
    kfn<<<grid, PRJ_WARPS * 32, smem, st>>>(bess, angle, torsion, src, dst, row_ptr, trip_ptr, graph_ptr,   \
                                            batch, (int)n_edges, (int)n_triplets, w_sbf1, w_t1, sbf_p, t_p, \
                                            out_ptr, out_list, pos_in);                                     \
  }
#define DIG3D_PRJ(BS) \
  if (tors) DIG3D_PRJP_ONE(BS) else DIG3D_PRJ_ONE(BS)
  switch (basis_id) {
    case 0: DIG3D_PRJ(B76); break;
    case 1: DIG3D_PRJ(B36); break;
    default: set_error("triplet_basis_project: unsupported basis_id %d", basis_id); return DIG3D_EUNSUPPORTED;
  }
#undef DIG3D_PRJ_ONE
#undef DIG3D_PRJP_ONE
#undef DIG3D_PRJ
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_basis_project_bwd(const float* bess, const float* angle, const float* torsion, const int32_t* src,
                                    const int32_t* dst, const int32_t* row_ptr, const int32_t* trip_ptr,
                                    const int32_t* graph_ptr, const int64_t* batch, int64_t n_edges, int64_t n_triplets,
                                    int32_t basis_id, const float* const* d_sbf_p, const float* const* d_t_p,
                                    float* dw_sbf1, float* dw_t1, void* stream) {
  DIG3D_REQUIRE(bess && angle && src && dst && row_ptr && trip_ptr && graph_ptr && batch && d_sbf_p && dw_sbf1,
                "triplet_basis_project_bwd: null pointer");
  const bool tors = (dw_t1 != nullptr);
  DIG3D_REQUIRE(!tors || (torsion && d_t_p), "triplet_basis_project_bwd: torsion path needs torsion and d_t_p");
  if (n_edges == 0 || n_triplets == 0) return DIG3D_OK;
  PrjGradPtrs gp;
  for (int l = 0; l < 4; ++l) { gp.ds[l] = d_sbf_p[l]; gp.dt[l] = tors ? d_t_p[l] : nullptr; }
  cudaStream_t st = (cudaStream_t)stream;
  int dev = 0, n_sm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  const int64_t want = (n_edges + PRJ_WARPS - 1) / PRJ_WARPS;
  const int grid = (int)(want < 2 * n_sm ? want : 2 * n_sm);
#define DIG3D_PRJB_ONE(BS, TORS)                                                                            \
  {                                                                                                         \
    auto kfn = triplet_basis_project_bwd_kernel<BS, TORS>;                                                  \
    const size_t smem = sizeof(PrjBwdSmem<BS, TORS>);                                                       \
    if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { \
      set_error("triplet_basis_project_bwd: cannot reserve %zu bytes of shared memory", smem);              \
      return DIG3D_ECUDA;                                                                                   \
    }                                                                                                       \
    kfn<<<grid, PRJ_WARPS * 32, smem, st>>>(bess, angle, torsion, src, dst, row_ptr, trip_ptr, graph_ptr,   \
                                            batch, (int)n_edges, gp, dw_sbf1, dw_t1);                       \
  }
#define DIG3D_PRJB(BS) \
  if (tors) DIG3D_PRJB_ONE(BS, true) else DIG3D_PRJB_ONE(BS, false)
  switch (basis_id) {
    case 0: DIG3D_PRJB(B76); break;
    case 1: DIG3D_PRJB(B36); break;
    default: set_error("triplet_basis_project_bwd: unsupported basis_id %d", basis_id); return DIG3D_EUNSUPPORTED;
  }
#undef DIG3D_PRJB_ONE
#undef DIG3D_PRJB
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_edge_basis_bwd(const float* dist, int64_t n_edges, double cutoff, int32_t envelope_exponent, const float* freq,
                         int32_t basis_id, int32_t envelope_on_bessel, const float* drbf0, float* ddist, float* bess_dx,
                         void* stream) {
  DIG3D_REQUIRE(dist && (ddist || bess_dx), "edge_basis_bwd: null pointer");
  DIG3D_REQUIRE(!drbf0 || (freq && ddist), "edge_basis_bwd: drbf0 needs freq and ddist");
  if (n_edges == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int p = envelope_exponent + 1;
  const float a = (float)(-(p + 1) * (p + 2) / 2.0), b = (float)(p * (p + 2)), c = (float)(-p * (p + 1) / 2.0);
  const float inv = 1.0f / (float)cutoff;
  const int grid = ceil_div(n_edges, 128);
  switch (basis_id) {
    case 0: edge_basis_bwd_kernel<B76><<<grid, 128, 0, st>>>(dist, (int)n_edges, inv, p, a, b, c, freq, envelope_on_bessel, drbf0, ddist, bess_dx); break;
    case 1: edge_basis_bwd_kernel<B36><<<grid, 128, 0, st>>>(dist, (int)n_edges, inv, p, a, b, c, freq, envelope_on_bessel, drbf0, ddist, bess_dx); break;
    default: set_error("edge_basis_bwd: unsupported basis_id %d", basis_id); return DIG3D_EUNSUPPORTED;
  }
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_triplet_basis_project_bwd_geom(const float* bess, const float* bess_dx, const float* angle,
                                         const float* torsion, const int32_t* src, const int32_t* dst,
                                         const int32_t* row_ptr, const int32_t* trip_ptr, const int32_t* graph_ptr,
                                         const int64_t* batch, int64_t n_edges, int64_t n_triplets, int32_t basis_id,
                                         const float* const* d_sbf_p, const float* const* d_t_p, const float* w_sbf1,
                                         const float* w_t1, double cutoff, float* ddist, float* dangle, float* dtorsion,
                                         void* stream) {
  DIG3D_REQUIRE(bess && bess_dx && angle && src && dst && row_ptr && trip_ptr && graph_ptr && batch && d_sbf_p &&
                    w_sbf1 && ddist && dangle, "triplet_basis_project_bwd_geom: null pointer");
  const bool tors = (dtorsion != nullptr);
  DIG3D_REQUIRE(!tors || (torsion && d_t_p && w_t1), "triplet_basis_project_bwd_geom: torsion path needs torsion, d_t_p, w_t1");
  if (n_edges == 0) return DIG3D_OK;
  PrjGradPtrs gp;
  for (int l = 0; l < 4; ++l) { gp.ds[l] = d_sbf_p[l]; gp.dt[l] = tors ? d_t_p[l] : nullptr; }
  cudaStream_t st = (cudaStream_t)stream;
  int dev = 0, n_sm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  const int64_t want = (n_edges + PRJG_WARPS - 1) / PRJG_WARPS;
  const int grid = (int)(want < 4 * n_sm ? want : 4 * n_sm);
  const float inv = 1.0f / (float)cutoff;
#define DIG3D_PRJG_ONE(BS, TORS)                                                                            \
  {                                                                                                         \
    auto kfn = triplet_basis_project_bwd_geom_kernel<BS, TORS>;                                             \
    const size_t smem = sizeof(PrjGeomSmem<BS, TORS>);                                                      \
    if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { \
      set_error("triplet_basis_project_bwd_geom: cannot reserve %zu bytes of shared memory", smem);         \
      return DIG3D_ECUDA;                                                                                   \
    }                                                                                                       \
    kfn<<<grid, PRJG_WARPS * 32, smem, st>>>(bess, bess_dx, angle, torsion, src, dst, row_ptr, trip_ptr,    \
                                             graph_ptr, batch, (int)n_edges, gp, w_sbf1, w_t1, inv, ddist,  \
                                             dangle, dtorsion);                                             \
  }
#define DIG3D_PRJG(BS) \
  if (tors) DIG3D_PRJG_ONE(BS, true) else DIG3D_PRJG_ONE(BS, false)
  switch (basis_id) {
    case 0: DIG3D_PRJG(B76); break;
    case 1: DIG3D_PRJG(B36); break;
    default: set_error("triplet_basis_project_bwd_geom: unsupported basis_id %d", basis_id); return DIG3D_EUNSUPPORTED;
  }
#undef DIG3D_PRJG_ONE
#undef DIG3D_PRJG
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
