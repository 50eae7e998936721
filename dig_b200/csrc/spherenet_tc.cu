// SphereNet / DimeNet++ update_e on the Hopper tensor cores (wgmma, sm_90a), 3xTF32.
//
// The dense edge-MLP chain of update_e (spherenet.py:154-180: lin_ji, lin_kj, lin_down, lin_up, three
// residual layers, lin) is ~96 % of the block's FLOPs.  Here each CTA owns 128 consecutive edges and runs
// the whole chain with the activations resident on chip:
//
//   * MMA: wgmma.m64n64k8.f32.tf32, the 128-edge tile as two m64 halves x N = 128/64 channels in n64 blocks.
//     fp32 parity (1e-5) rules out plain TF32, so every product is the 3xTF32 split
//     D = A_lo*W_hi + A_hi*W_lo + A_hi*W_hi with hi = rna_tf32(x), lo = rna_tf32(x - hi).
//   * A operand: the epilogue warps write the next layer's activations (already split into hi / lo planes)
//     straight into the canonical no-swizzle K-major layout in shared memory; the fp32 residual / skip value of
//     the row stays in the registers of the epilogue thread that owns it, so one A buffer (2 x 66 KB) suffices.
//   * The tensor core accumulates with truncation, a systematic shrink that adds up coherently over the chain and
//     over the nodes of a molecule.  So a wgmma chain only ever accumulates ONE K-chunk (32 = four k-steps, opened
//     by that chunk's two small correction terms); the chunk goes to one of two accumulators of the CTA's
//     accumulator-store slot (wgmma.cuh), and the epilogue warps add each finished chunk into fp32 registers with
//     round-to-nearest while the warpgroup works on the next chunk (streaming accumulation).
//   * B operand: weights are pre-split and pre-arranged (dig3d_tc_pack) as [K/32][hi|lo][8][N][4] so that a
//     K-chunk is ONE contiguous 32 KB block, streamed by cp.async.bulk (TMA engine) through a 2-stage
//     mbarrier ring.
//   * Roles (640 threads): warpgroup 0 = weight ring + wgmma, warps 4..19 = epilogue (accumulator store ->
//     registers -> bias / swish / residual -> split -> shared memory); four warps share a 32-row quarter and take
//     32 columns each.
//
// The latency-bound triplet gather (spherenet.py:163-171) runs in its own high-occupancy SIMT kernel
// (sphere_triplet_gather_kernel) and hands m[E,64] to the chain.
#include "common.cuh"
#define TC90_TM_COLS 256   // accumulator store columns per CTA slot
#include "wgmma.cuh"

namespace dig3d {
using namespace tc90;

constexpr int TC_M = 128;
constexpr int TC_EPI_WARPS = 16;
constexpr int TC_EPI_THREADS = TC_EPI_WARPS * 32;
constexpr int TC_CTRL = 128;                       // warpgroup 0: weight ring + wgmma
constexpr int TC_THREADS = TC_CTRL + TC_EPI_THREADS;   // + 16 epilogue warps
constexpr int TC_STAGES = 2;
constexpr int TC_STAGE_FLOATS = 2 * 8 * 128 * 4;   // hi + lo planes of a K=32 chunk with N = 128

// k-unit stride of the A planes, in 16-byte units: one unit of padding (LBO = 129 * 16 B) makes both the
// "lane = row" epilogue stores and the "lane = k-unit" coalesced tile loads bank-conflict free.
constexpr int TC_AKU = TC_M + 1;

struct TcSmem {
  float a_hi[32 * TC_AKU * 4];
  float a_lo[32 * TC_AKU * 4];
  float w[TC_STAGES][TC_STAGE_FLOATS];
  float bias[8][128];
  float wr[128 * 8];      // lin_rbf (kernel B) or lin_rbf2 (kernel A) rows, padded to 8
  float wr1[8 * 8];       // lin_rbf1 rows (kernel A), padded to 8
  int dst[TC_M];
  int aux[2][TC_M];       // init_e: atomic numbers of the target / source node of each row
  uint64_t full[TC_STAGES], empty[TC_STAGES], a_ready, d_ready[2], d_free[2];
  uint32_t tmem_base;
};

static_assert(sizeof(TcSmem) > TM_ONE_CTA_PER_SM_SMEM, "one CTA per SM sizes the accumulator-store slot pool");

struct TcGemm {
  const float* w;     // packed [K/32][2][8][N][4]
  const float* bias;  // [N] or null
  int K, N;
};

// x * sigmoid(x).  Default: MUFU ex2/rcp approximations (a much shorter epilogue; the energy stays within the 1e-5
// parity bound, tests/test_gpu_parity.py); libdevice expf + IEEE division selectable for experiments.
static int h_fast_swish = 1;   // host-side switch, selects the kernel instantiation
// optional timeline probe: CTA 0 of the tensor kernels records clock64() at protocol points (tools/gpu_tc_timeline.py)
__device__ long long g_tc_trace[64];
__device__ int g_tc_trace_on = 0;
#define TC_TRACE(slot) do { if (g_tc_trace_on && blockIdx.x == 0) g_tc_trace[(slot)] = clock64(); } while (0)
template <bool FAST>
__device__ __forceinline__ float swish_t(float x) {
  return FAST ? __fdividef(x, 1.0f + __expf(-x)) : __fdiv_rn(x, 1.0f + expf(-x));
}
#define swish_sel(x, fast) swish_t<FAST>(x)

// ---- control warpgroup: streams every K-chunk of every GEMM of the chain through the ring and issues its wgmma; one
// K-chunk per accumulator (columns 0 / 128 of the accumulator store), accumulators ping-pong (it & 1).  The ring's only
// consumer is this warpgroup, so a stage is refilled (chunk it + TC_STAGES) as soon as the wgmma reading it are done.
// Register split as in spherenet_h16.cu: 128 x 64 + 512 x 104 = 640 x 96.
__device__ __forceinline__ void tc_regs_ctrl() { asm volatile("setmaxnreg.dec.sync.aligned.u32 64;"); }
__device__ __forceinline__ void tc_regs_epi() { asm volatile("setmaxnreg.inc.sync.aligned.u32 104;"); }
template <int NG>
__device__ __forceinline__ void tc_produce(TcSmem& s, const TcGemm (&g)[NG], int& pq, int& pc, int& pit) {
  if (pq >= NG) return;
  const uint32_t bytes = 2u * 8u * (uint32_t)g[pq].N * 16u;
  if (threadIdx.x == 0) {
    const int st = pit % TC_STAGES;
    if (pit < 12) TC_TRACE(40 + pit);
    mbar_arrive_expect_tx(&s.full[st], bytes);
    bulk_g2s(s.w[st], g[pq].w + (size_t)pc * (bytes / 4), bytes, &s.full[st]);
  }
  ++pit;
  if (++pc == g[pq].K / 32) { pc = 0; ++pq; }
}
template <int NG>
__device__ __forceinline__ void tc_mma(TcSmem& s, const TcGemm (&g)[NG], uint32_t tmem_d) {
  const int wt = threadIdx.x;                          // 0..127
  int pq = 0, pc = 0, pit = 0;
  for (int i = 0; i < TC_STAGES; ++i) tc_produce(s, g, pq, pc, pit);
  int it = 0;
  const uint32_t a_hi = smem_u32(s.a_hi), a_lo = smem_u32(s.a_lo);
  for (int q = 0; q < NG; ++q) {
    const int chunks = g[q].K / 32, n = g[q].N;
    mbar_wait(&s.a_ready, q & 1);
    tc_fence_after();
    if (q < 4 && wt == 0) TC_TRACE(8 + 4 * q);            // A ready
    for (int c = 0; c < chunks; ++c, ++it) {
      const int st = it % TC_STAGES, ab = it & 1;
      mbar_wait(&s.full[st], (it / TC_STAGES) & 1);
      if (it >= 2) mbar_wait(&s.d_free[ab], ((it >> 1) & 1) ^ 1);   // the epilogue has drained this accumulator
      tc_fence_after();
      if (q < 4 && c == 0 && wt == 0) TC_TRACE(9 + 4 * q);   // first weight chunk landed
      for (int mh = 0; mh < 2; ++mh)
        for (int nh = 0; nh < n / 64; ++nh) {
          const uint32_t w_hi = smem_u32(s.w[st]) + (uint32_t)(nh * 64 * 16), w_lo = w_hi + 8u * n * 16u;
          const uint32_t a_m = (uint32_t)(mh * 64 * 16);
          float d[32];
          wg_fence();
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            const uint32_t a_off = a_m + (uint32_t)((c * 4 + ks) * 2 * TC_AKU * 16);
            const uint32_t b_off = (uint32_t)(ks * 2 * n * 16);
            // the chunk's corrections (magnitude 2^-11 of the main term) open the accumulator ...
            mma_tf32(d, smem_desc(a_lo + a_off, TC_AKU * 16, 128), smem_desc(w_hi + b_off, n * 16, 128), ks != 0);
            mma_tf32(d, smem_desc(a_hi + a_off, TC_AKU * 16, 128), smem_desc(w_lo + b_off, n * 16, 128), 1);
          }
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            const uint32_t a_off = a_m + (uint32_t)((c * 4 + ks) * 2 * TC_AKU * 16);
            const uint32_t b_off = (uint32_t)(ks * 2 * n * 16);
            mma_tf32(d, smem_desc(a_hi + a_off, TC_AKU * 16, 128), smem_desc(w_hi + b_off, n * 16, 128), 1);
          }                                         // ... then its four hi*hi steps are added on top
          wg_commit();
          wg_wait0();
          tm_store_frag(d, wt, tmem_d + ((uint32_t)(64 * mh) << 16) + 128u * ab + 64u * nh);
        }
      tc_fence_before();
      wg_bar();
      tc_produce(s, g, pq, pc, pit);
      if (wt == 0) mbar_arrive(&s.d_ready[ab]);
    }
    if (q < 4 && wt == 0) TC_TRACE(10 + 4 * q);           // all MMAs of the GEMM issued
  }
}

// ---- epilogue helpers (thread = one row, 64 or 32 columns in 16-column pieces)
struct EpiCtx {
  int row, part, lane_base;   // row in tile, column part (0..3), base row of the warp's quarter
  uint32_t tm;                // accumulator-store address of the CTA's slot
};
__device__ __forceinline__ EpiCtx epi_ctx(const TcSmem& s) {
  const int et = threadIdx.x - TC_CTRL, we = et >> 5, lane = et & 31;
  const int q = we & 3;         // row quarter of the warp
  return {32 * q + lane, we >> 2, 32 * q, s.tmem_base};
}
__device__ __forceinline__ void store_a(TcSmem& s, int row, int col, const float (&v)[16]) {
#pragma unroll
  for (int i = 0; i < 16; i += 4) {
    float4 h, l;
    split_tf32(v[i], h.x, l.x); split_tf32(v[i + 1], h.y, l.y); split_tf32(v[i + 2], h.z, l.z); split_tf32(v[i + 3], h.w, l.w);
    const int o = (((col + i) >> 2) * TC_AKU + row) * 4;
    *reinterpret_cast<float4*>(s.a_hi + o) = h;
    *reinterpret_cast<float4*>(s.a_lo + o) = l;
  }
}
// Streaming accumulation of one GEMM: every finished K-chunk is added (round-to-nearest) into this thread's
// fp32 registers, NP 16-column pieces starting at column col0; `it` is the global chunk counter shared
// (by construction) with the MMA issuer.
template <int NP, bool ZERO = true>
__device__ __forceinline__ void epi_accumulate(TcSmem& s, uint32_t tl, int col0, int chunks, int& it,
                                               float (&acc)[NP * 16]) {
  if (ZERO) {
#pragma unroll
    for (int i = 0; i < NP * 16; ++i) acc[i] = 0.f;
  }
  for (int c = 0; c < chunks; ++c, ++it) {
    const int ab = it & 1;
    mbar_wait(&s.d_ready[ab], (it >> 1) & 1);
    tc_fence_after();
    uint32_t r[NP][16];
#pragma unroll
    for (int p = 0; p < NP; ++p) tmem_ld16(tl + 128u * ab + col0 + 16 * p, r[p]);
    tmem_ld_wait();
    tc_fence_before();
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&s.d_free[ab]);   // one arrival per warp (512 serialised arrivals are slow)
#pragma unroll
    for (int p = 0; p < NP; ++p)
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[p * 16 + i] = __fadd_rn(acc[p * 16 + i], __uint_as_float(r[p][i]));
  }
}
// Cooperative (all epilogue threads) load of a row-major [128 x K4*4] fp32 tile from global memory into the A
// planes: a warp reads one 512-byte (K4 = 32) row segment per instruction (coalesced) and scatters its
// float4s over the k-units (conflict free thanks to the padded k-unit stride).
template <int K4>
__device__ __forceinline__ void load_a_tile(TcSmem& s, const float* __restrict__ g, int rows) {
  const int et = threadIdx.x - TC_CTRL;
#pragma unroll
  for (int k = 0; k < TC_M * K4 / TC_EPI_THREADS; ++k) {
    const int f = et + k * TC_EPI_THREADS;
    const int row = f / K4, c4 = f % K4;
    const float4 x = row < rows ? __ldg(reinterpret_cast<const float4*>(g + (size_t)row * (K4 * 4)) + c4)
                                : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 h, l;
    split_tf32(x.x, h.x, l.x); split_tf32(x.y, h.y, l.y); split_tf32(x.z, h.z, l.z); split_tf32(x.w, h.w, l.w);
    const int o = (c4 * TC_AKU + row) * 4;
    *reinterpret_cast<float4*>(s.a_hi + o) = h;
    *reinterpret_cast<float4*>(s.a_lo + o) = l;
  }
}
__device__ __forceinline__ void epi_done(TcSmem& s) {
  fence_async_smem();
  tc_fence_before();
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(&s.a_ready);
}
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, %0;" ::"n"(TC_EPI_THREADS) : "memory"); }

// ---------------------------------------------------------------------------------- triplet gather (SIMT)
// m[e] = sum_{t in trip(e)} x_down[kj(t)] * lin_sbf2(sbf_p[t]) * lin_t2(t_p[t])      spherenet.py:163-171
// ---- packed inner loop shared by the edge-centred and the warp-per-node gather ------------------------------------
// A lane owns channels `lane` and `lane + 32`.  Per triplet and channel the work is two 8-term expansions
// (lin_sbf2, lin_t2) and three products; the expansions run as paired FFMA chains (common.cuh):
//   TORSION   : the halves of a pair are the sbf and the t expansion of the SAME triplet and channel -- weights
//               {w_sbf2[c][q], w_t2[c][q]} and staged values {sbf_p[t][q], t_p[t][q]} pair up naturally;
//   !TORSION  : the halves are the sbf expansions of two CONSECUTIVE triplets (weights duplicated, staged values
//               interleaved pairwise).
// Every half is the same k-ascending fmaf chain as before, so the results are bit-identical to the scalar loops.
template <bool TORSION>
__device__ __forceinline__ void tg_load_weights(float2 (&w)[2][8], const float* __restrict__ w_sbf2,
                                                const float* __restrict__ w_t2, int lane) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float a = __ldg(w_sbf2 + (lane + 32 * h) * 8 + q);
      w[h][q] = make_float2(a, TORSION ? __ldg(w_t2 + (lane + 32 * h) * 8 + q) : a);
    }
}

// st: the warp's 64 x float2 staging area.  Lane l holds element (triplet l / 8, q = l % 8) of the chunk's first four
// triplets in (sa, ta) and of the last four in (sb, tb).
template <bool TORSION>
__device__ __forceinline__ void tg_stage(float2* st, int lane, float sa, float sb, float ta, float tb) {
  if (TORSION) {
    st[lane] = make_float2(sa, ta);
    st[lane + 32] = make_float2(sb, tb);
  } else {
    float* f = reinterpret_cast<float*>(st);
    const int q = lane & 7, u = lane >> 3;                 // (u, q) -> pair (u >> 1), half (u & 1)
    f[((u >> 1) * 8 + q) * 2 + (u & 1)] = sa;
    f[(((u >> 1) + 2) * 8 + q) * 2 + (u & 1)] = sb;
  }
}

template <bool TORSION, class XRow>
__device__ __forceinline__ void tg_accumulate(const float2* st, int n8, const float2 (&w)[2][8], XRow xrow, float& a0,
                                              float& a1) {
  if (TORSION) {
    // two triplets per step: four independent paired FFMA chains, all eight broadcast loads in flight before the first use
    // (one triplet at a time, the chain latency and the shared-memory round trip are exposed).  The staged values of a triplet past
    // the end of the chunk are zero, its row is not read, so it adds an exact 0.
#pragma unroll
    for (int up = 0; up < 4; ++up) {
      if (2 * up < n8) {
        const int u = 2 * up;
        const bool two = u + 1 < n8;
        float4 v[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = *reinterpret_cast<const float4*>(st + u * 8 + 2 * q);
        float xa0, xb0, xa1 = 0.f, xb1 = 0.f;
        xrow(u, xa0, xb0);
        if (two) xrow(u + 1, xa1, xb1);
        float2 g0 = make_float2(0.f, 0.f), g1 = g0, k0 = g0, k1 = g0;   // {lin_sbf2, lin_t2}: channel 0 / 1 of u, u + 1
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 a0q = make_float2(v[q].x, v[q].y), a1q = make_float2(v[q].z, v[q].w);
          const float2 b0q = make_float2(v[4 + q].x, v[4 + q].y), b1q = make_float2(v[4 + q].z, v[4 + q].w);
          g0 = ffma2(w[0][2 * q], a0q, g0); g1 = ffma2(w[1][2 * q], a0q, g1);
          k0 = ffma2(w[0][2 * q], b0q, k0); k1 = ffma2(w[1][2 * q], b0q, k1);
          g0 = ffma2(w[0][2 * q + 1], a1q, g0); g1 = ffma2(w[1][2 * q + 1], a1q, g1);
          k0 = ffma2(w[0][2 * q + 1], b1q, k0); k1 = ffma2(w[1][2 * q + 1], b1q, k1);
        }
        float m0 = __fmul_rn(xa0, g0.x), m1 = __fmul_rn(xb0, g1.x);
        float n0 = __fmul_rn(xa1, k0.x), n1 = __fmul_rn(xb1, k1.x);
        m0 = __fmul_rn(m0, g0.y); m1 = __fmul_rn(m1, g1.y);
        n0 = __fmul_rn(n0, k0.y); n1 = __fmul_rn(n1, k1.y);
        a0 += m0; a1 += m1;
        a0 += n0; a1 += n1;
      }
    }
  } else {
#pragma unroll
    for (int up = 0; up < 4; ++up) {
      if (2 * up < n8) {
        float2 g0 = make_float2(0.f, 0.f), g1 = make_float2(0.f, 0.f);        // triplets 2 up, 2 up + 1
#pragma unroll
        for (int q = 0; q < 8; q += 2) {
          const float4 v = *reinterpret_cast<const float4*>(st + up * 8 + q);
          const float2 v0 = make_float2(v.x, v.y), v1 = make_float2(v.z, v.w);
          g0 = ffma2(w[0][q], v0, g0); g1 = ffma2(w[1][q], v0, g1);
          g0 = ffma2(w[0][q + 1], v1, g0); g1 = ffma2(w[1][q + 1], v1, g1);
        }
        float x0, x1;
        xrow(2 * up, x0, x1);
        a0 += __fmul_rn(x0, g0.x); a1 += __fmul_rn(x1, g1.x);
        if (2 * up + 1 < n8) {
          xrow(2 * up + 1, x0, x1);
          a0 += __fmul_rn(x0, g0.y); a1 += __fmul_rn(x1, g1.y);
        }
      }
    }
  }
}

template <bool TORSION>
__global__ void __launch_bounds__(256, 3)
sphere_triplet_gather_kernel(const float* __restrict__ x_down, const float* __restrict__ sbf_p,
                             const float* __restrict__ t_p, const int32_t* __restrict__ src,
                             const int32_t* __restrict__ dst, const int32_t* __restrict__ row_ptr,
                             const int32_t* __restrict__ trip_ptr, int n_edges, const float* __restrict__ w_sbf2,
                             const float* __restrict__ w_t2, float* __restrict__ m) {
  // per warp: the projected basis rows of 8 consecutive triplets (8 x 8 floats each for sbf and t), loaded
  // with two coalesced 256-byte reads instead of 32 broadcast loads, then re-read as warp broadcasts
  __shared__ __align__(16) float2 stage[8][64];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (e >= n_edges) return;
  float2 wq[2][8];
  tg_load_weights<TORSION>(wq, w_sbf2, w_t2, lane);
  const int j = src[e], i = dst[e];
  const int base = row_ptr[j], d = row_ptr[j + 1] - base;
  // position of i among j's in-neighbours (d if absent): triplet r of this edge uses slot r + (r >= p_i)
  int p_i = d;
  for (int s0 = 0; s0 < d; s0 += 32) {
    const int sl = s0 + lane;
    const unsigned hit = __ballot_sync(0xffffffffu, sl < d && src[base + sl] == i);
    if (hit) p_i = s0 + __ffs(hit) - 1;
  }
  const int t0 = trip_ptr[e], nt = d - (p_i < d ? 1 : 0);
  float a0 = 0.f, a1 = 0.f;
  for (int r0 = 0; r0 < nt; r0 += 8) {
    const int n8 = min(8, nt - r0), lim = n8 * 8;
    const float* sp = sbf_p + (size_t)(t0 + r0) * 8;
    const float sa = lane < lim ? __ldg(sp + lane) : 0.f, sb = lane + 32 < lim ? __ldg(sp + lane + 32) : 0.f;
    float ta = 0.f, tb = 0.f;
    if (TORSION) {
      const float* tp = t_p + (size_t)(t0 + r0) * 8;
      ta = lane < lim ? __ldg(tp + lane) : 0.f; tb = lane + 32 < lim ? __ldg(tp + lane + 32) : 0.f;
    }
    float x0[8], x1[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int r = min(r0 + u, nt - 1);
      const int kj = base + r + (r >= p_i ? 1 : 0);
      x0[u] = __ldg(x_down + (size_t)kj * 64 + lane);
      x1[u] = __ldg(x_down + (size_t)kj * 64 + lane + 32);
    }
    __syncwarp();
    tg_stage<TORSION>(stage[w], lane, sa, sb, ta, tb);
    __syncwarp();
    tg_accumulate<TORSION>(stage[w], n8, wq, [&](int u, float& xa, float& xb) { xa = x0[u]; xb = x1[u]; }, a0, a1);
  }
  m[(size_t)e * 64 + lane] = a0;
  m[(size_t)e * 64 + lane + 32] = a1;
}

// ---------------------------------------------------------------------------------- triplet gather, one WARP per node
// Same result as sphere_triplet_gather_kernel, bit for bit, organised around the SOURCE node j of the edges: every
// out-edge (j -> i) sums over the same in-edges (k -> j) of j, whose x_down rows are CONTIGUOUS in the target-sorted
// edge list, so the per-triplet 256-byte L2 gathers of the edge-centred kernel become one coalesced staging of those
// rows.  Every warp is independent: it owns (node j, share `sub` of `split`), stages the rows of j's in-edges in its
// OWN shared-memory buffer with one bulk copy (cp.async.bulk, own mbarrier), finds the out-edges with lane = candidate
// atom, keeps the in-neighbour list in two registers per lane (position look-ups are ballots) and walks its out-edges,
// fetching the projected-basis values one chunk ahead.  No __syncthreads after the set-up.  split > 1 spreads a heavy
// node over several warps (each stages its own copy of the rows; out-edge r of the node goes to share r % split).
constexpr int TGW_WARPS = 4;
constexpr int TGW_MAXIN = 64;     // in-degree supported (cap + 1 <= 64, same bound as GEO_MAXDEG in graph.cu)

template <bool TORSION>
__global__ void __launch_bounds__(TGW_WARPS * 32)
sphere_triplet_gather_warp_kernel(const float* __restrict__ x_down, const float* __restrict__ sbf_p,
                                  const float* __restrict__ t_p, const int32_t* __restrict__ src,
                                  const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ trip_ptr,
                                  const int32_t* __restrict__ graph_ptr, const int64_t* __restrict__ batch,
                                  int n_nodes, int split, int cap, const float* __restrict__ w_sbf2,
                                  const float* __restrict__ w_t2, float* __restrict__ m,
                                  const int32_t* __restrict__ out_ptr, const int32_t* __restrict__ out_list,
                                  const int32_t* __restrict__ pos_in) {
  extern __shared__ __align__(128) unsigned char tgw_smem[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const size_t per_warp = (size_t)cap * 256 + 512 + 128;
  unsigned char* mine = tgw_smem + (size_t)w * per_warp;
  float (*rows)[64] = reinterpret_cast<float (*)[64]>(mine);
  float2* stage = reinterpret_cast<float2*>(mine + (size_t)cap * 256);
  uint64_t* bar = reinterpret_cast<uint64_t*>(mine + (size_t)cap * 256 + 512);
  const int task = blockIdx.x * TGW_WARPS + w;
  if (task >= n_nodes * split) return;
  const int j = task / split, sub = task - j * split;
  const int base = row_ptr[j], d = row_ptr[j + 1] - base;
  // out-edges of j: the list the graph build left (out_ptr / out_list / pos_in), or -- for graphs that came without it
  // (caller-supplied edge_index) -- a search over the nodes of j's graph
  const bool lists = out_ptr != nullptr;
  int lo, hi;
  if (lists) { lo = out_ptr[j]; hi = out_ptr[j + 1]; }
  else { const int g = (int)batch[j]; lo = graph_ptr[g]; hi = graph_ptr[g + 1]; }
  if (lane == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
    if (d > 0) {
      mbar_arrive_expect_tx(bar, (uint32_t)d * 256u);
      bulk_g2s(&rows[0][0], x_down + (size_t)base * 64, (uint32_t)d * 256u, bar);
    }
  }
  const int in_a = !lists && lane < d ? src[base + lane] : -1, in_b = !lists && lane + 32 < d ? src[base + lane + 32] : -1;
  float2 wq[2][8];
  tg_load_weights<TORSION>(wq, w_sbf2, w_t2, lane);
  __syncwarp();
  auto fetch = [&](int t_first, int left, float& sa, float& sb, float& ta, float& tb) {
    const int lim = min(8, left) * 8;
    const float* sp = sbf_p + (size_t)t_first * 8;
    sa = lane < lim ? __ldg(sp + lane) : 0.f; sb = lane + 32 < lim ? __ldg(sp + lane + 32) : 0.f;
    ta = 0.f; tb = 0.f;
    if (TORSION) {
      const float* tp = t_p + (size_t)t_first * 8;
      ta = lane < lim ? __ldg(tp + lane) : 0.f; tb = lane + 32 < lim ? __ldg(tp + lane + 32) : 0.f;
    }
  };
  // position of node i among j's in-neighbours (d if absent)
  auto position = [&](int i) {
    const unsigned ha = __ballot_sync(0xffffffffu, in_a == i), hb = __ballot_sync(0xffffffffu, in_b == i);
    return ha ? __ffs(ha) - 1 : (hb ? 32 + __ffs(hb) - 1 : d);
  };
  bool staged = false;
  int seen = 0;                      // out-edges of j met so far (all shares)
  for (int c0 = lo; c0 < hi; c0 += 32) {
    const int i = c0 + lane;
    int e_l = -1, p_l = d;
    if (lists) {
      if (i < hi) { e_l = out_list[i]; p_l = pos_in[e_l]; }
    } else if (i < hi && i != j) {
      const int ib = row_ptr[i], di = row_ptr[i + 1] - ib;
      int a = 0, b = di;
      while (a < b) { const int mid = (a + b) >> 1; if (src[ib + mid] < j) a = mid + 1; else b = mid; }
      if (a < di && src[ib + a] == j) e_l = ib + a;
    }
    const unsigned found = __ballot_sync(0xffffffffu, e_l >= 0);
    const int rank = seen + __popc(found & ((1u << lane) - 1));
    unsigned sel = __ballot_sync(0xffffffffu, e_l >= 0 && rank % split == sub);
    seen += __popc(found);
    if (!sel) continue;
    if (!staged && d > 0) { mbar_wait(bar, 0); staged = true; }
    // walk the selected out-edges; the projected-basis values of a chunk are fetched one chunk ahead (next chunk of the
    // edge, or the first chunk of the next selected edge)
    int bit = __ffs(sel) - 1;
    sel &= sel - 1;
    int e = __shfl_sync(0xffffffffu, e_l, bit), p_i = lists ? __shfl_sync(0xffffffffu, p_l, bit) : position(c0 + bit);
    int t0 = trip_ptr[e], nt = d - (p_i < d ? 1 : 0);
    float sa = 0.f, sb = 0.f, ta = 0.f, tb = 0.f;
    bool fetched = false;
    for (;;) {
      int e_n = -1, p_n = 0, t0_n = 0, nt_n = 0;
      if (sel) {
        const int bn = __ffs(sel) - 1;
        sel &= sel - 1;
        e_n = __shfl_sync(0xffffffffu, e_l, bn);
        p_n = lists ? __shfl_sync(0xffffffffu, p_l, bn) : position(c0 + bn);
        t0_n = trip_ptr[e_n]; nt_n = d - (p_n < d ? 1 : 0);
      }
      if (!fetched && nt > 0) fetch(t0, nt, sa, sb, ta, tb);
      fetched = false;
      float a0 = 0.f, a1 = 0.f;
      for (int r0 = 0; r0 < nt; r0 += 8) {
        const int n8 = min(8, nt - r0);
        __syncwarp();
        tg_stage<TORSION>(stage, lane, sa, sb, ta, tb);
        __syncwarp();
        if (r0 + 8 < nt) fetch(t0 + r0 + 8, nt - r0 - 8, sa, sb, ta, tb);
        else if (e_n >= 0 && nt_n > 0) { fetch(t0_n, nt_n, sa, sb, ta, tb); fetched = true; }
        tg_accumulate<TORSION>(stage, n8, wq, [=](int u, float& xa, float& xb) {
          const int r = r0 + u, row = r + (r >= p_i ? 1 : 0);
          xa = rows[row][lane]; xb = rows[row][lane + 32];
        }, a0, a1);
      }
      m[(size_t)e * 64 + lane] = a0;
      m[(size_t)e * 64 + lane + 32] = a1;
      if (e_n < 0) break;
      e = e_n; p_i = p_n; t0 = t0_n; nt = nt_n;
    }
  }
}

// ---------------------------------------------------------------------------------- weight packing
// W [N, K] (nn.Linear layout) -> [K/32][hi|lo][8][N][4], hi/lo = TF32 split.  One launch packs up to 16 matrices.
struct PackJob { const float* w; float* out; int N, K, trans; };   // trans: the source is stored [K, N] (W^T)
struct PackJobs { PackJob job[16]; int n; };
__global__ void tc_pack_kernel(PackJobs jobs) {
  const PackJob jb = jobs.job[blockIdx.y];
  const int total = jb.N * jb.K;
  for (int id = blockIdx.x * blockDim.x + threadIdx.x; id < total; id += gridDim.x * blockDim.x) {
    const int n = id / jb.K, k = id % jb.K;
    float h, l;
    split_tf32(__ldg(jb.w + (jb.trans ? (size_t)k * jb.N + n : (size_t)id)), h, l);
    const int c = k >> 5, ku = (k & 31) >> 2, kk = k & 3;
    const size_t blk = (size_t)c * (2 * 8 * jb.N * 4);
    jb.out[blk + ((size_t)ku * jb.N + n) * 4 + kk] = h;
    jb.out[blk + (size_t)8 * jb.N * 4 + ((size_t)ku * jb.N + n) * 4 + kk] = l;
  }
}

// ---------------------------------------------------------------------------------- update_e part A (tensor)
struct TcAParams {
  TcGemm g[3];                 // lin_ji, lin_kj, lin_down
  const float *w_rbf1, *w_rbf2;
};

template <bool FAST>
__global__ void __launch_bounds__(TC_THREADS, 1)
sphere_update_e_a_tc_kernel(const float* __restrict__ e1, const float* __restrict__ rbf0, int n_edges, TcAParams P,
                            float* __restrict__ x_ji, float* __restrict__ x_down) {
  extern __shared__ __align__(1024) unsigned char tc_raw[];
  TcSmem& s = *reinterpret_cast<TcSmem*>(tc_raw);
  const int tid = threadIdx.x, warp = tid >> 5;
  const int e0 = blockIdx.x * TC_M, rows = min(TC_M, n_edges - e0);
  if (tid == 0) {
    for (int i = 0; i < TC_STAGES; ++i) { mbar_init(&s.full[i], 1); mbar_init(&s.empty[i], 1); }
    mbar_init(&s.a_ready, TC_EPI_WARPS);
    for (int i = 0; i < 2; ++i) { mbar_init(&s.d_ready[i], 1); mbar_init(&s.d_free[i], TC_EPI_WARPS); }
    mbar_fence_init();
  }
  if (warp == 0) tmem_alloc(&s.tmem_base, 256);
  for (int i = tid; i < 2 * 128; i += TC_THREADS) s.bias[i / 128][i % 128] = __ldg(P.g[i / 128].bias + i % 128);
  for (int i = tid; i < 128 * 8; i += TC_THREADS) s.wr[i] = __ldg(P.w_rbf2 + i);      // [128][8]
  for (int i = tid; i < 64; i += TC_THREADS) s.wr1[i] = (i % 8 < 6) ? __ldg(P.w_rbf1 + (i / 8) * 6 + i % 8) : 0.f;
  tc_fence_before();
  if (tid == TC_CTRL) TC_TRACE(0);
  __syncthreads();
  tc_fence_after();
  if (tid == TC_CTRL) TC_TRACE(1);
  if (warp < TC_CTRL / 32) {
    tc_regs_ctrl();
    tc_mma(s, P.g, s.tmem_base);
  } else {
    tc_regs_epi();
    const EpiCtx c = epi_ctx(s);
    const bool valid = c.row < rows;
    const size_t ge = (size_t)(e0 + c.row);
    const uint32_t tl = c.tm + ((uint32_t)c.lane_base << 16);
    // A0 = e1 tile
    load_a_tile<32>(s, e1 + (size_t)e0 * 128, rows);
    // rbf gate coefficients of this row: r8 = lin_rbf1(rbf0[row])            spherenet.py:157
    float r8[8];
    {
      float rb[6];
#pragma unroll
      for (int n = 0; n < 6; ++n) rb[n] = valid ? __ldg(rbf0 + ge * 6 + n) : 0.f;
#pragma unroll
      for (int m = 0; m < 8; ++m) {
        float a = 0.f;
#pragma unroll
        for (int n = 0; n < 6; ++n) a = fmaf(s.wr1[m * 8 + n], rb[n], a);
        r8[m] = a;
      }
    }
    if (tid == TC_CTRL) TC_TRACE(2);
    epi_done(s);
    int it = 0;
    const int col0 = c.part * 32;
    float acc[32];
    // G0: x_ji = act(lin_ji(e1))                                                spherenet.py:154
    epi_accumulate<2>(s, tl, col0, 4, it, acc);
    if (tid == TC_CTRL) TC_TRACE(3);
    epi_done(s);   // A (= e1) is reused unchanged by lin_kj: let its MMAs run under this activation + store
    if (valid) {
#pragma unroll
      for (int i = 0; i < 32; i += 4) {
        float4 o;
        o.x = swish_sel(acc[i] + s.bias[0][col0 + i], fast);
        o.y = swish_sel(acc[i + 1] + s.bias[0][col0 + i + 1], fast);
        o.z = swish_sel(acc[i + 2] + s.bias[0][col0 + i + 2], fast);
        o.w = swish_sel(acc[i + 3] + s.bias[0][col0 + i + 3], fast);
        *reinterpret_cast<float4*>(x_ji + ge * 128 + col0 + i) = o;
      }
    }
    if (tid == TC_CTRL) TC_TRACE(4);
    // G1: x_kj = act(lin_kj(e1)) * lin_rbf2(r8)                                 spherenet.py:155-159
    epi_accumulate<2>(s, tl, col0, 4, it, acc);
    if (tid == TC_CTRL) TC_TRACE(5);
#pragma unroll
    for (int cc = 0; cc < 2; ++cc) {
      float v[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int col = col0 + cc * 16 + i;
        const float4 w0 = *reinterpret_cast<const float4*>(s.wr + col * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(s.wr + col * 8 + 4);
        const float gate = fmaf(w1.w, r8[7], fmaf(w1.z, r8[6], fmaf(w1.y, r8[5], fmaf(w1.x, r8[4],
                           fmaf(w0.w, r8[3], fmaf(w0.z, r8[2], fmaf(w0.y, r8[1], w0.x * r8[0])))))));
        v[i] = swish_sel(acc[cc * 16 + i] + s.bias[1][col], fast) * gate;
      }
      store_a(s, c.row, col0 + cc * 16, v);
    }
    if (tid == TC_CTRL) TC_TRACE(6);
    epi_done(s);
    // G2: x_down = act(lin_down(x_kj)), N = 64                                  spherenet.py:161
    {
      const int col = c.part * 16;
      float a16[16];
      epi_accumulate<1>(s, tl, col, 4, it, a16);
      if (tid == TC_CTRL) TC_TRACE(7);
      if (valid) {
#pragma unroll
        for (int i = 0; i < 16; i += 4) {
          float4 o;
          o.x = swish_sel(a16[i], fast); o.y = swish_sel(a16[i + 1], fast);
          o.z = swish_sel(a16[i + 2], fast); o.w = swish_sel(a16[i + 3], fast);
          *reinterpret_cast<float4*>(x_down + ge * 64 + col + i) = o;
        }
      }
    }
    tc_fence_before();
  }
  __syncthreads();
  if (warp == 0) tmem_dealloc(s.tmem_base, 256);
}

// ---------------------------------------------------------------------------------- update_e part B (tensor)
struct TcBParams {
  TcGemm g[8];                 // lin_up, res0.lin1, res0.lin2, lin, res1.lin1, res1.lin2, res2.lin1, res2.lin2
  const float* w_rbf;          // [128, 6]
};

template <bool FAST>
__global__ void __launch_bounds__(TC_THREADS, 1)
sphere_update_e_b_tc_kernel(const float* __restrict__ m, const float* __restrict__ x_ji,
                            const float* __restrict__ e1_in, const float* __restrict__ rbf0,
                            const int32_t* __restrict__ dst, int n_edges, TcBParams P, float* __restrict__ e1_out,
                            float* __restrict__ v_in) {
  extern __shared__ __align__(1024) unsigned char tc_raw[];
  TcSmem& s = *reinterpret_cast<TcSmem*>(tc_raw);
  const int tid = threadIdx.x, warp = tid >> 5;
  const int e0 = blockIdx.x * TC_M, rows = min(TC_M, n_edges - e0);
  if (tid == 0) {
    for (int i = 0; i < TC_STAGES; ++i) { mbar_init(&s.full[i], 1); mbar_init(&s.empty[i], 1); }
    mbar_init(&s.a_ready, TC_EPI_WARPS);
    for (int i = 0; i < 2; ++i) { mbar_init(&s.d_ready[i], 1); mbar_init(&s.d_free[i], TC_EPI_WARPS); }
    mbar_fence_init();
  }
  if (warp == 0) tmem_alloc(&s.tmem_base, 256);
  for (int i = tid; i < 8 * 128; i += TC_THREADS) {
    const float* b = P.g[i / 128].bias;
    s.bias[i / 128][i % 128] = b ? __ldg(b + i % 128) : 0.f;
  }
  for (int i = tid; i < 128 * 8; i += TC_THREADS) s.wr[i] = (i % 8 < 6) ? __ldg(P.w_rbf + (i / 8) * 6 + i % 8) : 0.f;
  for (int i = tid; i < TC_M; i += TC_THREADS) s.dst[i] = (i < rows) ? dst[e0 + i] : -1;
  tc_fence_before();
  __syncthreads();
  tc_fence_after();
  if (warp < TC_CTRL / 32) {
    tc_regs_ctrl();
    tc_mma(s, P.g, s.tmem_base);
  } else {
    tc_regs_epi();
    const EpiCtx c = epi_ctx(s);
    const bool valid = c.row < rows;
    const size_t ge = (size_t)(e0 + c.row);
    const uint32_t tl = c.tm + ((uint32_t)c.lane_base << 16);
    // A0 = m tile (K = 64)
    load_a_tile<16>(s, m + (size_t)e0 * 64, rows);
    epi_done(s);
    // The eight epilogues of the chain (spherenet.py:172-179):
    //   q=0: h = x_ji + act(lin_up(m))                       -> A, stash
    //   q=1,4,6: t = act(lin1(h))                            -> A
    //   q=2,5: h = stash + act(lin2(t))                      -> A, stash      (q=2: stash not needed afterwards)
    //   q=3: h = act(lin(h)) + e1_in                         -> A, stash
    //   q=7: h = stash + act(lin2(t))                        -> e1_out, e2 tile
    float stash[32];     // fp32 residual of this thread's (row, 32 columns), lives in registers
    int it = 0;
    const int col0 = c.part * 32;
#pragma unroll 1
    for (int q = 0; q < 8; ++q) {
      float acc[32];
      epi_accumulate<2>(s, tl, col0, q == 0 ? 2 : 4, it, acc);
      const bool add_stash = (q == 2 || q == 5 || q == 7);
      const bool to_stash = (q == 0 || q == 3 || q == 5);
#pragma unroll
      for (int cc = 0; cc < 2; ++cc) {
        const int col = col0 + cc * 16;
        float v[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = swish_sel(acc[cc * 16 + i] + s.bias[q][col + i], fast);
        if (add_stash) {
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] += stash[cc * 16 + i];
        }
        if (q == 0 || q == 3) {
          const float* gsrc = (q == 0 ? x_ji : e1_in) + ge * 128 + col;
#pragma unroll
          for (int i = 0; i < 16; i += 4) {
            const float4 x = valid ? __ldg(reinterpret_cast<const float4*>(gsrc + i)) : make_float4(0, 0, 0, 0);
            v[i] += x.x; v[i + 1] += x.y; v[i + 2] += x.z; v[i + 3] += x.w;
          }
        }
        if (q < 7) {
          store_a(s, c.row, col, v);
          if (to_stash) {
#pragma unroll
            for (int i = 0; i < 16; ++i) stash[cc * 16 + i] = v[i];
          }
        } else {
          // e1_out and e2 = lin_rbf(rbf0) * e1 (tile staged over the A planes)   spherenet.py:180
          float rb[6];
#pragma unroll
          for (int n = 0; n < 6; ++n) rb[n] = valid ? __ldg(rbf0 + ge * 6 + n) : 0.f;
          float* e2t = s.a_hi;   // [128][132] floats overlay (a_hi + a_lo are contiguous, all MMAs are done)
#pragma unroll
          for (int i = 0; i < 16; i += 4) {
            if (valid) *reinterpret_cast<float4*>(e1_out + ge * 128 + col + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              float gsum = 0.f;
#pragma unroll
              for (int n = 0; n < 6; ++n) gsum = fmaf(s.wr[(col + i + u) * 8 + n], rb[n], gsum);
              e2t[c.row * 132 + col + i + u] = gsum * v[i + u];
            }
          }
        }
      }
      if (q < 7) epi_done(s);
    }
    tc_fence_before();
    epi_bar();
    // segmented edge -> node sums of the e2 tile (target-sorted rows)             spherenet.py:211
    const int col = tid - TC_CTRL;
    if (col < 128 && rows > 0) {
      const float* e2t = s.a_hi;
      float run = 0.f;
      int cur = s.dst[0];
      bool first = true;
      for (int r = 0; r < rows; ++r) {
        const int d = s.dst[r];
        if (d != cur) {
          if (first) atomicAdd(v_in + (size_t)cur * 128 + col, run);
          else v_in[(size_t)cur * 128 + col] = run;
          first = false; run = 0.f; cur = d;
        }
        run += e2t[r * 132 + col];
      }
      atomicAdd(v_in + (size_t)cur * 128 + col, run);
    }
  }
  __syncthreads();
  if (warp == 0) tmem_dealloc(s.tmem_base, 256);
}

// ---------------------------------------------------------------------------------- init_e (tensor)
// e1 = act(lin(cat[x_i, x_j, act(lin_rbf_0(rbf))])), e2 = lin_rbf_1(rbf) * e1        spherenet.py:79-91
// The K = 384 contraction runs as three K = 128 panels whose A operand is rebuilt between panels (embedding rows
// of the target nodes, of the source nodes, then the radial term); the per-chunk partial products keep
// accumulating in the epilogue registers across the panels.
struct TcInitParams {
  TcGemm g[3];                 // the three K-panels of init_e.lin (bias applied at the end)
  const float *emb, *w_rbf0, *b_rbf0, *b_lin, *w_rbf1;
};

template <bool FAST>
__global__ void __launch_bounds__(TC_THREADS, 1)
sphere_init_e_tc_kernel(const int64_t* __restrict__ z, const int32_t* __restrict__ src,
                        const int32_t* __restrict__ dst, const float* __restrict__ rbf0, int n_edges, TcInitParams P,
                        float* __restrict__ e1, float* __restrict__ v_in) {
  extern __shared__ __align__(1024) unsigned char tc_raw[];
  TcSmem& s = *reinterpret_cast<TcSmem*>(tc_raw);
  const int tid = threadIdx.x, warp = tid >> 5;
  const int e0 = blockIdx.x * TC_M, rows = min(TC_M, n_edges - e0);
  float* w0 = &s.bias[2][0];   // lin_rbf_0.weight [128][6] parked in the unused bias rows
  if (tid == 0) {
    for (int i = 0; i < TC_STAGES; ++i) { mbar_init(&s.full[i], 1); mbar_init(&s.empty[i], 1); }
    mbar_init(&s.a_ready, TC_EPI_WARPS);
    for (int i = 0; i < 2; ++i) { mbar_init(&s.d_ready[i], 1); mbar_init(&s.d_free[i], TC_EPI_WARPS); }
    mbar_fence_init();
  }
  if (warp == 0) tmem_alloc(&s.tmem_base, 256);
  for (int i = tid; i < 128; i += TC_THREADS) { s.bias[0][i] = __ldg(P.b_lin + i); s.bias[1][i] = __ldg(P.b_rbf0 + i); }
  for (int i = tid; i < 128 * 6; i += TC_THREADS) w0[i] = __ldg(P.w_rbf0 + i);
  for (int i = tid; i < 128 * 8; i += TC_THREADS) s.wr[i] = (i % 8 < 6) ? __ldg(P.w_rbf1 + (i / 8) * 6 + i % 8) : 0.f;
  for (int i = tid; i < TC_M; i += TC_THREADS) {
    const int d = (i < rows) ? dst[e0 + i] : -1, sj = (i < rows) ? src[e0 + i] : -1;
    s.dst[i] = d;
    s.aux[0][i] = d >= 0 ? (int)z[d] : 0;
    s.aux[1][i] = sj >= 0 ? (int)z[sj] : 0;
  }
  tc_fence_before();
  __syncthreads();
  tc_fence_after();
  if (warp < TC_CTRL / 32) {
    tc_regs_ctrl();
    tc_mma(s, P.g, s.tmem_base);
  } else {
    tc_regs_epi();
    const EpiCtx c = epi_ctx(s);
    const int et = tid - TC_CTRL;
    const bool valid = c.row < rows;
    const size_t ge = (size_t)(e0 + c.row);
    const uint32_t tl = c.tm + ((uint32_t)c.lane_base << 16);
    const int col0 = c.part * 32;
    float rb[6];
#pragma unroll
    for (int n = 0; n < 6; ++n) rb[n] = valid ? __ldg(rbf0 + ge * 6 + n) : 0.f;
    auto fill_embedding = [&](const int* zrow) {   // A = emb[z[node of row]]: one coalesced 512 B row per warp step
#pragma unroll
      for (int k = 0; k < TC_M * 32 / TC_EPI_THREADS; ++k) {
        const int f = et + k * TC_EPI_THREADS, row = f >> 5, c4 = f & 31;
        const float4 x = row < rows ? __ldg(reinterpret_cast<const float4*>(P.emb + (size_t)zrow[row] * 128) + c4)
                                    : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 h, l;
        split_tf32(x.x, h.x, l.x); split_tf32(x.y, h.y, l.y); split_tf32(x.z, h.z, l.z); split_tf32(x.w, h.w, l.w);
        const int o = (c4 * TC_AKU + row) * 4;
        *reinterpret_cast<float4*>(s.a_hi + o) = h;
        *reinterpret_cast<float4*>(s.a_lo + o) = l;
      }
    };
    int it = 0;
    float acc[32];
    fill_embedding(s.aux[0]);                       // panel 0: x_i
    epi_done(s);
    epi_accumulate<2, true>(s, tl, col0, 4, it, acc);
    fill_embedding(s.aux[1]);                       // panel 1: x_j
    epi_done(s);
    epi_accumulate<2, false>(s, tl, col0, 4, it, acc);
#pragma unroll
    for (int cc = 0; cc < 2; ++cc) {                // panel 2: act(lin_rbf_0(rbf))        spherenet.py:87
      float v[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int col = col0 + cc * 16 + i;
        float a = 0.f;
#pragma unroll
        for (int n = 0; n < 6; ++n) a = fmaf(w0[col * 6 + n], rb[n], a);
        v[i] = valid ? swish_sel(a + s.bias[1][col], fast) : 0.f;
      }
      store_a(s, c.row, col0 + cc * 16, v);
    }
    epi_done(s);
    epi_accumulate<2, false>(s, tl, col0, 4, it, acc);
    // e1 = act(. + b), e2 = lin_rbf_1(rbf) * e1 (tile staged over the A planes), edge -> node sums
    float* e2t = s.a_hi;
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      float o[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int col = col0 + i + u;
        o[u] = swish_sel(acc[i + u] + s.bias[0][col], fast);
        float gsum = 0.f;
#pragma unroll
        for (int n = 0; n < 6; ++n) gsum = fmaf(s.wr[col * 8 + n], rb[n], gsum);
        e2t[c.row * 132 + col] = gsum * o[u];
      }
      if (valid) *reinterpret_cast<float4*>(e1 + ge * 128 + col0 + i) = make_float4(o[0], o[1], o[2], o[3]);
    }
    tc_fence_before();
    epi_bar();
    const int col = tid - TC_CTRL;
    if (col < 128 && rows > 0) {
      float run = 0.f;
      int cur = s.dst[0];
      bool first = true;
      for (int r = 0; r < rows; ++r) {
        const int d = s.dst[r];
        if (d != cur) {
          if (first) atomicAdd(v_in + (size_t)cur * 128 + col, run);
          else v_in[(size_t)cur * 128 + col] = run;
          first = false; run = 0.f; cur = d;
        }
        run += e2t[r * 132 + col];
      }
      atomicAdd(v_in + (size_t)cur * 128 + col, run);
    }
  }
  __syncthreads();
  if (warp == 0) tmem_dealloc(s.tmem_base, 256);
}


// ---------------------------------------------------------------------------------- generic linear (training path)
// y[rows, N] = x[rows, K] W^T + bias on wgmma (3xTF32, streaming accumulation), K = NPANEL panels of K4*4 columns,
// N in {64, 128}; optionally also act_out = swish(y) (the training forward keeps the pre-activation for the backward).
template <int NPANEL>
struct TcLinParams { TcGemm g[NPANEL]; };

template <int K4>
__device__ __forceinline__ void load_a_tile_ld(TcSmem& s, const float* __restrict__ g, size_t ld, int rows) {
  const int et = threadIdx.x - TC_CTRL;
#pragma unroll
  for (int k = 0; k < TC_M * K4 / TC_EPI_THREADS; ++k) {
    const int f = et + k * TC_EPI_THREADS;
    const int row = f / K4, c4 = f % K4;
    const float4 x = row < rows ? __ldg(reinterpret_cast<const float4*>(g + (size_t)row * ld) + c4)
                                : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 h, l;
    split_tf32(x.x, h.x, l.x); split_tf32(x.y, h.y, l.y); split_tf32(x.z, h.z, l.z); split_tf32(x.w, h.w, l.w);
    const int o = (c4 * TC_AKU + row) * 4;
    *reinterpret_cast<float4*>(s.a_hi + o) = h;
    *reinterpret_cast<float4*>(s.a_lo + o) = l;
  }
}

template <int NPANEL, int N, int K4>
__global__ void __launch_bounds__(TC_THREADS, 1)
linear_tc_kernel(const float* __restrict__ x, int n_rows, TcLinParams<NPANEL> P, const float* __restrict__ bias,
                 float* __restrict__ y, float* __restrict__ act_out) {
  extern __shared__ __align__(1024) unsigned char tc_raw[];
  TcSmem& s = *reinterpret_cast<TcSmem*>(tc_raw);
  constexpr int K = NPANEL * K4 * 4;
  constexpr int PW = N / 4;                          // columns per epilogue column-part (32 or 16)
  const int tid = threadIdx.x, warp = tid >> 5;
  const int r0 = blockIdx.x * TC_M, rows = min(TC_M, n_rows - r0);
  if (tid == 0) {
    for (int i = 0; i < TC_STAGES; ++i) { mbar_init(&s.full[i], 1); mbar_init(&s.empty[i], 1); }
    mbar_init(&s.a_ready, TC_EPI_WARPS);
    for (int i = 0; i < 2; ++i) { mbar_init(&s.d_ready[i], 1); mbar_init(&s.d_free[i], TC_EPI_WARPS); }
    mbar_fence_init();
  }
  if (warp == 0) tmem_alloc(&s.tmem_base, 256);
  for (int i = tid; i < N; i += TC_THREADS) s.bias[0][i] = bias ? __ldg(bias + i) : 0.f;
  tc_fence_before();
  __syncthreads();
  tc_fence_after();
  if (warp < TC_CTRL / 32) {
    tc_regs_ctrl();
    tc_mma(s, P.g, s.tmem_base);
  } else {
    tc_regs_epi();
    const EpiCtx c = epi_ctx(s);
    const bool valid = c.row < rows;
    const uint32_t tl = c.tm + ((uint32_t)c.lane_base << 16);
    const int col0 = c.part * PW;
    int it = 0;
    float acc[PW];
#pragma unroll
    for (int p = 0; p < NPANEL; ++p) {
      load_a_tile_ld<K4>(s, x + (size_t)r0 * K + p * (K4 * 4), K, rows);
      epi_done(s);
      if (p == 0) epi_accumulate<PW / 16, true>(s, tl, col0, K4 / 8, it, acc);
      else epi_accumulate<PW / 16, false>(s, tl, col0, K4 / 8, it, acc);
    }
    if (valid) {
      float* yr = y + (size_t)(r0 + c.row) * N + col0;
      float* ar = act_out ? act_out + (size_t)(r0 + c.row) * N + col0 : nullptr;
#pragma unroll
      for (int i = 0; i < PW; i += 4) {
        float4 o;
        o.x = acc[i] + s.bias[0][col0 + i];
        o.y = acc[i + 1] + s.bias[0][col0 + i + 1];
        o.z = acc[i + 2] + s.bias[0][col0 + i + 2];
        o.w = acc[i + 3] + s.bias[0][col0 + i + 3];
        *reinterpret_cast<float4*>(yr + i) = o;
        if (ar) {
          float4 a;
          a.x = swish_t<false>(o.x); a.y = swish_t<false>(o.y); a.z = swish_t<false>(o.z); a.w = swish_t<false>(o.w);
          *reinterpret_cast<float4*>(ar + i) = a;
        }
      }
    }
  }
  __syncthreads();
  if (warp == 0) tmem_dealloc(s.tmem_base, 256);
}

static int tc_smem_attr(const void* fn, size_t bytes) {
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(%zu): %s", bytes, cudaGetErrorString(e));
    return DIG3D_ECUDA;
  }
  return DIG3D_OK;
}

template <int NPANEL, int N, int K4>
static int launch_linear_tc(const float* x, int64_t rows, const float* packed, const float* bias, float* y, float* act_out,
                            cudaStream_t st) {
  TcLinParams<NPANEL> P;
  const size_t panel = (size_t)(K4 / 8) * 2 * 8 * N * 4;      // K4/8 chunks of [hi|lo][8][N][4] floats
  for (int p = 0; p < NPANEL; ++p) P.g[p] = {packed + p * panel, nullptr, K4 * 4, N};
  auto kfn = linear_tc_kernel<NPANEL, N, K4>;
  int rc = tc_smem_attr((const void*)kfn, sizeof(TcSmem));
  if (rc) return rc;
  kfn<<<ceil_div(rows, TC_M), TC_THREADS, sizeof(TcSmem), st>>>(x, (int)rows, P, bias, y, act_out);
  return DIG3D_OK;
}


}  // namespace dig3d

using namespace dig3d;

extern "C" {

int dig3d_tc_pack(const float* const* weights, const int32_t* n, const int32_t* k, float* const* outs, int32_t count,
                  void* stream) {
  DIG3D_REQUIRE(weights && n && k && outs && count >= 1 && count <= 16, "tc_pack: bad arguments");
  PackJobs jobs;
  jobs.n = count;
  int max_total = 0;
  for (int i = 0; i < count; ++i) {
    DIG3D_REQUIRE(weights[i] && outs[i] && k[i] % 32 == 0 && n[i] % 8 == 0, "tc_pack: matrix %d has N=%d K=%d", i, n[i], k[i]);
    jobs.job[i] = {weights[i], outs[i], n[i], k[i], 0};
    max_total = max_total > n[i] * k[i] ? max_total : n[i] * k[i];
  }
  dim3 grid(ceil_div(max_total, 256), count);
  tc_pack_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(jobs);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_tc_pack_t(const float* const* weights, const int32_t* n, const int32_t* k, const int32_t* trans,
                    float* const* outs, int32_t count, void* stream) {
  DIG3D_REQUIRE(weights && n && k && trans && outs && count >= 1 && count <= 16, "tc_pack_t: bad arguments");
  PackJobs jobs;
  jobs.n = count;
  int max_total = 0;
  for (int i = 0; i < count; ++i) {
    DIG3D_REQUIRE(weights[i] && outs[i] && k[i] % 32 == 0 && n[i] % 8 == 0, "tc_pack_t: matrix %d has N=%d K=%d", i, n[i], k[i]);
    jobs.job[i] = {weights[i], outs[i], n[i], k[i], trans[i] ? 1 : 0};
    max_total = max_total > n[i] * k[i] ? max_total : n[i] * k[i];
  }
  dim3 grid(ceil_div(max_total, 256), count);
  tc_pack_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(jobs);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_linear_tc_supported(int32_t k, int32_t nout) {
  return ((nout == 128 && (k == 64 || k == 128 || k == 256 || k == 384)) || (nout == 64 && k == 128)) ? 1 : 0;
}

int dig3d_linear_tc(const float* x, int64_t rows, int32_t k, int32_t nout, const float* packed, const float* bias,
                    float* y, float* act_out, void* stream) {
  DIG3D_REQUIRE(x && packed && y, "linear_tc: null pointer");
  DIG3D_REQUIRE(dig3d_linear_tc_supported(k, nout), "linear_tc: shape %d -> %d is not compiled", k, nout);
  if (rows == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (nout == 64) rc = launch_linear_tc<1, 64, 32>(x, rows, packed, bias, y, act_out, st);
  else if (k == 64) rc = launch_linear_tc<1, 128, 16>(x, rows, packed, bias, y, act_out, st);
  else if (k == 128) rc = launch_linear_tc<1, 128, 32>(x, rows, packed, bias, y, act_out, st);
  else if (k == 256) rc = launch_linear_tc<2, 128, 32>(x, rows, packed, bias, y, act_out, st);
  else rc = launch_linear_tc<3, 128, 32>(x, rows, packed, bias, y, act_out, st);
  if (rc) return rc;
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_tc_set_fast_swish(int32_t on) {
  h_fast_swish = on ? 1 : 0;
  return DIG3D_OK;
}

int dig3d_tc_trace(int32_t on, long long* out64 /* host, 64 entries, nullable */) {
  if (out64) cudaMemcpyFromSymbol(out64, g_tc_trace, sizeof(long long) * 64);
  int v = on ? 1 : 0;
  cudaMemcpyToSymbol(g_tc_trace_on, &v, sizeof(v));
  return DIG3D_OK;
}

int dig3d_tc_timeouts(void) {
  unsigned int v = 0;
  cudaMemcpyFromSymbol(&v, tc90::g_mbar_timeout, sizeof(v));
  return (int)v;
}

int dig3d_sphere_init_e_tc(const int64_t* z, const int32_t* src, const int32_t* dst, const float* rbf0,
                           int64_t n_edges, const dig3d_init_e_weights* w, const float* packed_lin, float* e1,
                           float* v_in, void* stream) {
  DIG3D_REQUIRE(z && src && dst && rbf0 && w && packed_lin && e1 && v_in, "sphere_init_e_tc: null pointer");
  DIG3D_REQUIRE(w->emb && w->w_rbf0 && w->b_rbf0 && w->b_lin && w->w_rbf1, "sphere_init_e_tc: null weight");
  if (n_edges == 0) return DIG3D_OK;
  TcInitParams P;
  const size_t panel = (size_t)4 * 2 * 8 * 128 * 4;   // four K=32 chunks of [hi|lo][8][128][4] floats
  for (int p = 0; p < 3; ++p) P.g[p] = {packed_lin + p * panel, nullptr, 128, 128};
  P.emb = w->emb; P.w_rbf0 = w->w_rbf0; P.b_rbf0 = w->b_rbf0; P.b_lin = w->b_lin; P.w_rbf1 = w->w_rbf1;
  auto kfn = h_fast_swish ? sphere_init_e_tc_kernel<true> : sphere_init_e_tc_kernel<false>;
  int rc = tc_smem_attr((const void*)kfn, sizeof(TcSmem));
  if (rc) return rc;
  kfn<<<ceil_div(n_edges, TC_M), TC_THREADS, sizeof(TcSmem), (cudaStream_t)stream>>>(z, src, dst, rbf0, (int)n_edges, P,
                                                                                    e1, v_in);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_sphere_update_e_a_tc(const float* e1, const float* rbf0, int64_t n_edges, const dig3d_tc_update_e* w,
                               float* x_ji, float* x_down, void* stream) {
  DIG3D_REQUIRE(e1 && rbf0 && w && x_ji && x_down, "sphere_update_e_a_tc: null pointer");
  if (n_edges == 0) return DIG3D_OK;
  TcAParams P;
  P.g[0] = {w->p_ji, w->b_ji, 128, 128};
  P.g[1] = {w->p_kj, w->b_kj, 128, 128};
  P.g[2] = {w->p_down, nullptr, 128, 64};
  P.w_rbf1 = w->w_rbf1; P.w_rbf2 = w->w_rbf2;
  auto kfn = h_fast_swish ? sphere_update_e_a_tc_kernel<true> : sphere_update_e_a_tc_kernel<false>;
  int rc = tc_smem_attr((const void*)kfn, sizeof(TcSmem));
  if (rc) return rc;
  kfn<<<ceil_div(n_edges, TC_M), TC_THREADS, sizeof(TcSmem), (cudaStream_t)stream>>>(e1, rbf0, (int)n_edges, P, x_ji,
                                                                                    x_down);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_sphere_triplet_gather(const float* x_down, const float* sbf_p, const float* t_p, int32_t ld_p,
                                const int32_t* src, const int32_t* dst, const int32_t* row_ptr,
                                const int32_t* trip_ptr, int64_t n_edges, const float* w_sbf2, const float* w_t2,
                                float* m, void* stream) {
  DIG3D_REQUIRE(x_down && sbf_p && src && dst && row_ptr && trip_ptr && w_sbf2 && m, "sphere_triplet_gather: null pointer");
  DIG3D_REQUIRE((t_p != nullptr) == (w_t2 != nullptr), "sphere_triplet_gather: t_p and w_t2 must agree");
  DIG3D_REQUIRE(ld_p == 8, "sphere_triplet_gather: expects the layer-major [T, 8] slices (ld_p == 8), got %d", ld_p);
  if (n_edges == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int gblocks = ceil_div(n_edges * 32, 256);
  if (t_p)
    sphere_triplet_gather_kernel<true><<<gblocks, 256, 0, st>>>(x_down, sbf_p, t_p, src, dst, row_ptr, trip_ptr,
                                                               (int)n_edges, w_sbf2, w_t2, m);
  else
    sphere_triplet_gather_kernel<false><<<gblocks, 256, 0, st>>>(x_down, sbf_p, t_p, src, dst, row_ptr, trip_ptr,
                                                                (int)n_edges, w_sbf2, w_t2, m);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_sphere_triplet_gather_warp(const float* x_down, const float* sbf_p, const float* t_p, int32_t ld_p,
                                     const int32_t* src, const int32_t* row_ptr, const int32_t* trip_ptr,
                                     const int32_t* graph_ptr, const int64_t* batch, int64_t n_nodes, int32_t cap,
                                     int32_t split, const float* w_sbf2, const float* w_t2, float* m,
                                     const int32_t* out_ptr, const int32_t* out_list, const int32_t* pos_in,
                                     void* stream) {
  DIG3D_REQUIRE(x_down && sbf_p && src && row_ptr && trip_ptr && graph_ptr && batch && w_sbf2 && m,
                "sphere_triplet_gather_warp: null pointer");
  DIG3D_REQUIRE((out_ptr != nullptr) == (out_list != nullptr) && (out_ptr != nullptr) == (pos_in != nullptr),
                "sphere_triplet_gather_warp: out_ptr, out_list and pos_in come together");
  DIG3D_REQUIRE((t_p != nullptr) == (w_t2 != nullptr), "sphere_triplet_gather_warp: t_p and w_t2 must agree");
  DIG3D_REQUIRE(ld_p == 8, "sphere_triplet_gather_warp: expects the layer-major [T, 8] slices (ld_p == 8), got %d", ld_p);
  DIG3D_REQUIRE(cap >= 1 && cap <= TGW_MAXIN, "sphere_triplet_gather_warp: cap=%d outside [1,%d]", cap, TGW_MAXIN);
  DIG3D_REQUIRE(split >= 1 && split <= 32, "sphere_triplet_gather_warp: split=%d outside [1,32]", split);
  DIG3D_REQUIRE(((uintptr_t)x_down & 15) == 0, "sphere_triplet_gather_warp: x_down must be 16-byte aligned");
  if (n_nodes == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = (size_t)TGW_WARPS * ((size_t)cap * 256 + 512 + 128);
  const int grid = ceil_div(n_nodes * split, TGW_WARPS);
  auto kfn = t_p ? sphere_triplet_gather_warp_kernel<true> : sphere_triplet_gather_warp_kernel<false>;
  if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
    set_error("sphere_triplet_gather_warp: cannot reserve %zu bytes of shared memory", smem);
    return DIG3D_ECUDA;
  }
  kfn<<<grid, TGW_WARPS * 32, smem, st>>>(x_down, sbf_p, t_p, src, row_ptr, trip_ptr, graph_ptr, batch, (int)n_nodes,
                                          (int)split, (int)cap, w_sbf2, w_t2, m, out_ptr, out_list, pos_in);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_sphere_update_e_b_tc(const float* m, const float* e1_in, const float* x_ji, const float* rbf0,
                               const int32_t* dst, int64_t n_edges, const dig3d_tc_update_e* w, float* e1_out,
                               float* v_in, void* stream) {
  DIG3D_REQUIRE(m && e1_in && x_ji && rbf0 && dst && w && e1_out && v_in, "sphere_update_e_b_tc: null pointer");
  if (n_edges == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  TcBParams P;
  P.g[0] = {w->p_up, nullptr, 64, 128};
  for (int i = 0; i < 2; ++i) P.g[1 + i] = {w->p_res[i], w->b_res[i], 128, 128};
  P.g[3] = {w->p_lin, w->b_lin, 128, 128};
  for (int i = 2; i < 6; ++i) P.g[2 + i] = {w->p_res[i], w->b_res[i], 128, 128};
  P.w_rbf = w->w_rbf;
  auto kfn = h_fast_swish ? sphere_update_e_b_tc_kernel<true> : sphere_update_e_b_tc_kernel<false>;
  int rc = tc_smem_attr((const void*)kfn, sizeof(TcSmem));
  if (rc) return rc;
  kfn<<<ceil_div(n_edges, TC_M), TC_THREADS, sizeof(TcSmem), st>>>(m, x_ji, e1_in, rbf0, dst, (int)n_edges, P, e1_out,
                                                                   v_in);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
