// SphereNet / DimeNet++ dense chains on 3xFP16 wgmma.  Two engines:
//   * init_e, update_e (parts A and B of an interaction block) and update_v run on the register-accumulator engine
//     (section "update_e: register-accumulator engine" below): activations stay in wgmma register fragments (update_v:
//     in per-consumer operand planes) from layer to layer.
//   * the generic linear runs on the second-generation two-tile store engine: TWO 128-edge tiles in
//     flight per CTA (one CTA per SM), accumulators handed to row-per-thread epilogues through the accumulator store.
//
// The two-tile store engine:
// The first-generation chain (spherenet_tc.cu, 3xTF32) has fp32-sized operand planes (2 x 66 KB) and room for one
// tile per CTA, so the tensor core waits during every epilogue.  Here:
//
//   * operands are split into TWO FP16 planes after a power-of-two pre-scale, x*8 = hi + lo (+ 2^-22 x),
//     w*64 = hi + lo: fp16 carries the same 11 significant bits as TF32, so the three-product form
//     D = A_lo*W_hi + A_hi*W_lo + A_hi*W_hi keeps fp32-level accuracy (tools/emulate_split.py: energy error
//     2.2e-7 vs 3.6e-7 for 3xTF32), while f16 wgmma moves K = 16 per instruction (twice TF32) and the planes are
//     half the size: two tiles' A operands (132 KB) + a 5-stage weight ring (80 KB) fit in shared memory.  The
//     pre-scales keep `lo` in fp16's normal range for |x| > 0.03 (below that the ABSOLUTE error floor is 4e-9);
//     activations must stay below 8190 in magnitude - a larger value overflows to inf/NaN in the energies and
//     raises the flag read by dig3d_h16_overflow() (the 3xTF32 chain has fp32 range).
//   * the control warpgroup alternates between the two tiles layer by layer: while tile X's eight epilogue warps
//     run the exposed activation phase of layer q, the tensor core runs layer q of tile Y, and vice versa.  Each
//     K = 64 chunk goes to one of two accumulators of the CTA's accumulator-store slot (wgmma.cuh; see the
//     truncation note in spherenet_tc.cu), shared by the tiles; the fp32 residual / skip rows live in the other
//     half of the slot (2 x 128 columns) instead of registers, which lets one epilogue thread own 64 columns of a row.
//   * roles (640 threads): warpgroup 0 = weight ring (cp.async.bulk) + wgmma, warps 4..11 = epilogue of tile X,
//     warps 12..19 = epilogue of tile Y (two warps per 32-row quarter, 64 columns each).
//
// Reference ops: update_e.forward spherenet.py:150-182 (dimenetpp.py:133-161), init.forward spherenet.py:79-91,
// update_v.forward spherenet.py:212-215.
#include <cuda_fp16.h>
#include "common.cuh"
#define TC90_TM_COLS 512   // accumulator store columns per CTA slot
#include "wgmma.cuh"

namespace dig3d {
using namespace tc90;

constexpr int H_M = 128;
constexpr int H_AKU = H_M + 1;                     // k-unit stride of the A planes in 16-byte units (padded)
constexpr int H_PLANE = 16 * H_AKU * 16;           // bytes of one fp16 plane of a [128 x 128] operand tile
constexpr int H_STAGES = 5;                       // 80 KB of weight slabs in flight (the L2 -> smem latency is ~2 k cycles)
constexpr int H_SLAB_K = 32;                       // ring granularity: K = 32 slab = [hi|lo][4 k-units][N][8 halves]
constexpr int H_STAGE_BYTES = 2 * 4 * 128 * 16;    // 16 KB (N = 128)
constexpr int H_TILE_WARPS = 8;
constexpr int H_TILE_THREADS = H_TILE_WARPS * 32;
constexpr int H_CTRL_THREADS = 128;                // warpgroup 0: weight ring + wgmma
constexpr int H_THREADS = H_CTRL_THREADS + 2 * H_TILE_THREADS;
constexpr int H_CTRL_WARPS = H_CTRL_THREADS / 32;
// Register re-allocation between the warpgroups (setmaxnreg): the kernels are compiled for 96 registers (640 threads);
// the control warpgroup (ring + wgmma, one 32-register m64n64 accumulator) then drops to 64 and each epilogue warp
// grows to 104 (the CTA pool is conserved: 128 x 64 + 512 x 104 = 640 x 96), which lets an epilogue thread keep its
// 64 accumulator values plus the staging registers.
__device__ __forceinline__ void h_regs_ctrl() { asm volatile("setmaxnreg.dec.sync.aligned.u32 64;"); }
__device__ __forceinline__ void h_regs_epi() { asm volatile("setmaxnreg.inc.sync.aligned.u32 104;"); }
constexpr float H_SA = 8.0f, H_SW = 64.0f;
constexpr float H_INV = 1.0f / (H_SA * H_SW);
// |activation| limit of the chain: the split rounds x * H_SA to fp16, which overflows to inf from 65520 (the midpoint
// between 65504 and 2^16) on, so |x| must stay below 65520 / H_SA = 8190
constexpr int H_LDS = 129;                         // row stride (floats) of the fp32 staging overlay of a tile's planes

struct HSmem {
  unsigned char a[2][2][H_PLANE];                  // [tile][hi | lo]
  unsigned char w[H_STAGES][H_STAGE_BYTES];
  float bias[8][128];
  float wr[128 * 8];
  int dst[2][H_M];
  // d_ready / d_free are indexed [tile][accumulator]: each barrier has ONE waiter that sees every phase in order
  // (a parity wait may never lag or lead its barrier by two phases, which a barrier shared by the tiles allows)
  uint64_t full[H_STAGES], empty[H_STAGES], a_ready[2], d_ready[2][2], d_free[2][2];
  uint32_t tmem_base;
};
static_assert(sizeof(HSmem) <= 227 * 1024, "HSmem exceeds the shared memory of an SM");
static_assert(sizeof(HSmem) > TM_ONE_CTA_PER_SM_SMEM, "one CTA per SM sizes the accumulator-store slot pool");
static_assert(2 * H_PLANE == H_M * H_LDS * 4, "the fp32 staging overlay must cover exactly one tile's planes");

struct HGemm {
  const unsigned char* w;   // packed slabs (dig3d_h16_pack)
  const float* bias;        // [N] or null
  int K, N;
  int tile_stride;          // bytes added to `w` for the second tile's job of a layer
};

static __device__ unsigned int g_h16_overflow = 0;
static int h16_fast_swish = 1;
// optional timeline probe: CTA 0 of the update_e kernels records clock64() at protocol points (tools/gpu_h16_timeline.py)
static __device__ long long g_h16_trace[128];
static __device__ int g_h16_trace_on = 0;

// x * sigmoid(x).  FAST (default): MUFU ex2 / rcp approximations in their flush-to-zero forms (the non-ftz forms
// cost three extra instructions per element for denormal inputs that cannot occur here); the energy stays within the
// 1e-5 parity bound (tests/test_gpu_parity.py).  FAST = false: libdevice expf + IEEE division.
__device__ __forceinline__ float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_ftz(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// The FAST forms spell every rounding out (__fmul_rn / __fadd_rn cannot be contracted into an FFMA), so that how the
// epilogues are scheduled cannot change a result bit.  One exception: hswish's final product stays a plain multiply,
// which its callers either store or scale by H_SA (an exact power of two, which ptxas folds into the same FMUL as .M8).
template <bool FAST>
__device__ __forceinline__ float hswish(float x) {
  return FAST ? x * rcp_ftz(__fadd_rn(1.0f, ex2_ftz(__fmul_rn(x, -1.4426950408889634f))))
              : __fdiv_rn(x, 1.0f + expf(-x));
}
// H_SA * swish(t8 / H_SA): the chain keeps its activations pre-scaled by the operand scale, so the split needs no
// multiply and the scale costs nothing (it is folded into the accumulator scale and the bias).
template <bool FAST>
__device__ __forceinline__ float hswish8(float t8) {
  return FAST ? __fmul_rn(t8, rcp_ftz(__fadd_rn(1.0f, ex2_ftz(__fmul_rn(t8, -1.4426950408889634f / H_SA)))))
              : __fdiv_rn(t8, 1.0f + expf(-t8 * (1.0f / H_SA)));
}
// hswish8(t8) + r, with the final product and the add as ONE rounding in the FAST form (t8 * rcp + r, one FFMA)
template <bool FAST>
__device__ __forceinline__ float hswish8_plus(float t8, float r) {
  return FAST ? fmaf(t8, rcp_ftz(__fadd_rn(1.0f, ex2_ftz(__fmul_rn(t8, -1.4426950408889634f / H_SA)))), r)
              : hswish8<false>(t8) + r;
}

// ---- control warpgroup: streams every K = 32 slab of every job (layer x tile) through the ring and issues the
// wgmma of each K = 64 chunk (two slabs).  Jobs alternate between the tiles; each chunk goes to one of the two
// accumulators (columns 0 / 128 of the accumulator store), shared by the tiles: before chunk `ch` overwrites
// accumulator ch & 1, the tile that used it last (chunk ch - 2, possibly the other tile) must have drained it.
// The ring has no "empty" handshake: its only consumer is this warpgroup, which refills a stage (slab it + H_STAGES)
// as soon as the wgmma reading it (slab it) have completed.
struct HRing {   // producer cursor over (job q, tile t, slab c)
  int q, t, c;
};
__device__ __forceinline__ void h_produce(HSmem& s, const HGemm* g, int ng, int ntile, HRing& r, int& it) {
  if (r.q >= ng) return;
  const uint32_t bytes = 2u * 4u * (uint32_t)g[r.q].N * 16u;
  if (threadIdx.x == 0) {
    const int st = it % H_STAGES;
    mbar_arrive_expect_tx(&s.full[st], bytes);
    bulk_g2s(s.w[st], g[r.q].w + (size_t)r.t * g[r.q].tile_stride + (size_t)r.c * bytes, bytes, &s.full[st]);
  }
  ++it;
  if (++r.c == g[r.q].K / H_SLAB_K) { r.c = 0; if (++r.t == ntile) { r.t = 0; ++r.q; } }
}
__device__ __forceinline__ void h_mma_n(HSmem& s, const HGemm* g, int ng, int ntile, uint32_t tmem) {
  const int wt = threadIdx.x;                            // 0..127
  HRing ring = {0, 0, 0};
  int pit = 0;
  for (int i = 0; i < H_STAGES; ++i) h_produce(s, g, ng, ntile, ring, pit);
  int it = 0, ch = 0;
  int uses00 = 0, uses01 = 0, uses10 = 0, uses11 = 0;   // uses[tile][accumulator] so far
  int last0 = -1, last1 = -1;                            // tile that used accumulator 0 / 1 last
  for (int q = 0; q < ng; ++q) {
    const int nslab = g[q].K / H_SLAB_K, n = g[q].N;
    for (int t = 0; t < ntile; ++t) {
      mbar_wait(&s.a_ready[t], q & 1);
      tc_fence_after();
      const uint32_t a_hi = smem_u32(s.a[t][0]), a_lo = smem_u32(s.a[t][1]);
      for (int c = 0; c < nslab; c += 2, it += 2) {
        const int ab = ch & 1;
        const int lt = ab ? last1 : last0;
        if (lt >= 0) {
          const int u = lt ? (ab ? uses11 : uses10) : (ab ? uses01 : uses00);
          mbar_wait(&s.d_free[lt][ab], (u - 1) & 1);   // that tile's epilogue has drained this accumulator
        }
        mbar_wait(&s.full[it % H_STAGES], (it / H_STAGES) & 1);
        mbar_wait(&s.full[(it + 1) % H_STAGES], ((it + 1) / H_STAGES) & 1);
        tc_fence_after();
        for (int mh = 0; mh < 2; ++mh)
          for (int nh = 0; nh < n / 64; ++nh) {
            float d[32];
            wg_fence();
#pragma unroll
            for (int sl = 0; sl < 2; ++sl) {
              const uint32_t w_hi = smem_u32(s.w[(it + sl) % H_STAGES]) + (uint32_t)(nh * 64 * 16), w_lo = w_hi + 4u * n * 16u;
              const uint32_t a_m = (uint32_t)(mh * 64 * 16);
#pragma unroll
              for (int ks = 0; ks < 2; ++ks) {   // the slab's corrections (2^-11 of the main term) first ...
                const uint32_t a_off = a_m + (uint32_t)(((c + sl) * 4 + ks * 2) * H_AKU * 16), b_off = (uint32_t)(ks * 2 * n * 16);
                mma_f16(d, smem_desc(a_lo + a_off, H_AKU * 16, 128), smem_desc(w_hi + b_off, n * 16, 128), (sl | ks) != 0);
                mma_f16(d, smem_desc(a_hi + a_off, H_AKU * 16, 128), smem_desc(w_lo + b_off, n * 16, 128), 1);
              }
#pragma unroll
              for (int ks = 0; ks < 2; ++ks) {   // ... then its two hi*hi steps
                const uint32_t a_off = a_m + (uint32_t)(((c + sl) * 4 + ks * 2) * H_AKU * 16), b_off = (uint32_t)(ks * 2 * n * 16);
                mma_f16(d, smem_desc(a_hi + a_off, H_AKU * 16, 128), smem_desc(w_hi + b_off, n * 16, 128), 1);
              }
            }
            wg_commit();
            wg_wait0();
            tm_store_frag(d, wt, tmem + ((uint32_t)(64 * mh) << 16) + 128u * ab + 64u * nh);
          }
        tc_fence_before();
        wg_bar();                                         // every wgmma of the chunk done, its rows stored
        h_produce(s, g, ng, ntile, ring, pit);
        h_produce(s, g, ng, ntile, ring, pit);
        if (wt == 0) mbar_arrive(&s.d_ready[t][ab]);
        if (t) { if (ab) ++uses11; else ++uses10; } else { if (ab) ++uses01; else ++uses00; }
        if (ab) last1 = t; else last0 = t;
        ++ch;
      }
    }
  }
}

// ---- epilogue context: thread = one row of its tile, NC = 64 (N = 128) or 32 (N = 64) columns
struct HCtx {
  int t, et, row, half;     // tile in the pair, thread index within the tile's epilogue, row, column half
  uint32_t tl;              // accumulator-store address of this warp's row quarter, column 0
  int ntile, ch;            // tiles in this CTA, global accumulator-chunk counter (same sequence as the issuer's)
  int use0, use1;           // chunks of THIS tile drained from accumulator 0 / 1 so far (barrier phases)
  bool bad;                 // a non-finite value reached an OUTPUT of the kernel (fp16 operand range exceeded upstream)
  unsigned char *ahi, *alo; // operand planes this thread writes
};
__device__ __forceinline__ HCtx h_ctx(HSmem& s, int ntile) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = (warp - H_CTRL_WARPS) / H_TILE_WARPS, we = (warp - H_CTRL_WARPS) % H_TILE_WARPS;
  const int quarter = warp & 3;   // rows [32*(warp%4), +32) of the tile
  return {t, (int)threadIdx.x - H_CTRL_THREADS - t * H_TILE_THREADS, 32 * quarter + lane, we >> 2,
          s.tmem_base + ((uint32_t)(32 * quarter) << 16), ntile, 0, 0, 0, false, s.a[t][0], s.a[t][1]};
}
__device__ __forceinline__ void h_tile_bar(int t) {
  asm volatile("bar.sync %0, %1;" ::"r"(1 + t), "n"(H_TILE_THREADS) : "memory");
}
__device__ __forceinline__ void h_epi_done(HSmem& s, int t) {
  fence_async_smem();
  tc_fence_before();
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(&s.a_ready[t]);
}
// 8 consecutive K elements of a row (one k-unit), ALREADY multiplied by H_SA: split into fp16 hi / lo, one 16-byte
// store per plane.  A value beyond the fp16 range becomes inf here and NaN in the products; the kernels flag
// non-finite OUTPUTS (HCtx::bad) instead of paying a range test per operand element.
__device__ __forceinline__ void h_store_ku(HSmem& s, const HCtx& c, int row, int ku, const float (&x)[8]) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __half2 hh = __floats2half2_rn(x[2 * i], x[2 * i + 1]);
    const float2 hf = __half22float2(hh);
    const __half2 ll = __floats2half2_rn(x[2 * i] - hf.x, x[2 * i + 1] - hf.y);
    h[i] = *reinterpret_cast<const uint32_t*>(&hh);
    l[i] = *reinterpret_cast<const uint32_t*>(&ll);
  }
  const int o = (ku * H_AKU + row) * 16;
  *reinterpret_cast<uint4*>(c.ahi + o) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(c.alo + o) = make_uint4(l[0], l[1], l[2], l[3]);
}
__device__ __forceinline__ bool h_finite(float x) { return fabsf(x) <= 3.402823466e38f; }
// Cooperative load of a row-major [rows x KU*8] fp32 tile (leading dimension ld floats) into the tile's planes:
// a warp reads 32 consecutive k-units (1 KB when ld == KU*8) per step.
template <int KU>
__device__ __forceinline__ void h_load_tile(HSmem& s, HCtx& c, const float* __restrict__ g, size_t ld, int rows) {
#pragma unroll
  for (int k = 0; k < H_M * KU / H_TILE_THREADS; ++k) {
    const int f = c.et + k * H_TILE_THREADS, row = f / KU, ku = f % KU;
    float x[8];
    if (row < rows) {
      const float4 p0 = __ldg(reinterpret_cast<const float4*>(g + (size_t)row * ld + ku * 8));
      const float4 p1 = __ldg(reinterpret_cast<const float4*>(g + (size_t)row * ld + ku * 8 + 4));
      x[0] = p0.x * H_SA; x[1] = p0.y * H_SA; x[2] = p0.z * H_SA; x[3] = p0.w * H_SA;
      x[4] = p1.x * H_SA; x[5] = p1.y * H_SA; x[6] = p1.z * H_SA; x[7] = p1.w * H_SA;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) x[i] = 0.f;
    }
    h_store_ku(s, c, row, ku, x);
  }
}
// The same load in two halves, so that the global-memory round trip of the FIRST operand tile overlaps the kernel's
// set-up (barrier init, accumulator-store slot, bias / index loads): fetch before the set-up barrier, commit after it.
// et / t are passed explicitly because the epilogue context does not exist yet.
template <int KU>
struct HTileRegs { float4 v[H_M * KU / H_TILE_THREADS][2]; };
template <int KU>
__device__ __forceinline__ void h_tile_fetch(HTileRegs<KU>& r, int et, const float* __restrict__ g, size_t ld, int rows) {
#pragma unroll
  for (int k = 0; k < H_M * KU / H_TILE_THREADS; ++k) {
    const int f = et + k * H_TILE_THREADS, row = f / KU, ku = f % KU;
    if (row < rows) {
      r.v[k][0] = __ldg(reinterpret_cast<const float4*>(g + (size_t)row * ld + ku * 8));
      r.v[k][1] = __ldg(reinterpret_cast<const float4*>(g + (size_t)row * ld + ku * 8 + 4));
    } else {
      r.v[k][0] = r.v[k][1] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}
template <int KU>
__device__ __forceinline__ void h_tile_commit(HSmem& s, const HCtx& c, const HTileRegs<KU>& r) {
#pragma unroll
  for (int k = 0; k < H_M * KU / H_TILE_THREADS; ++k) {
    const int f = c.et + k * H_TILE_THREADS, row = f / KU, ku = f % KU;
    const float4 p0 = r.v[k][0], p1 = r.v[k][1];
    const float x[8] = {p0.x * H_SA, p0.y * H_SA, p0.z * H_SA, p0.w * H_SA, p1.x * H_SA, p1.y * H_SA, p1.z * H_SA, p1.w * H_SA};
    h_store_ku(s, c, row, ku, x);
  }
}
// Streaming accumulation of this tile's job: each finished K = 64 chunk is added (round to nearest) into the
// thread's fp32 registers; NP 16-column pieces starting at column col0.  The global chunk counter advances over the
// other tile's chunks of the same layer without touching a barrier (they use that tile's own barriers).
template <int NP, bool FIRST>
__device__ __forceinline__ void h_drain(HSmem& s, HCtx& c, int col0, int chunks, float (&acc)[NP * 16]) {
  if (c.t == 1) c.ch += chunks;
  for (int k = 0; k < chunks; ++k, ++c.ch) {
    const int ab = c.ch & 1;
    const int use = ab ? c.use1 : c.use0;
    mbar_wait(&s.d_ready[c.t][ab], use & 1);
    if (ab) ++c.use1; else ++c.use0;
    tc_fence_after();
    const uint32_t ta = c.tl + 128u * ab + col0;
    if (FIRST && k == 0) {            // straight into the accumulator registers: all loads in flight, one wait
#pragma unroll
      for (int p = 0; p < NP; ++p) tmem_ld16f(ta + 16 * p, &acc[p * 16]);
      tmem_ld_wait();
    } else {
#pragma unroll
      for (int p = 0; p < NP; p += 2) {
        uint32_t r[2][16];
        tmem_ld16(ta + 16 * p, r[0]);
        if (p + 1 < NP) tmem_ld16(ta + 16 * p + 16, r[1]);
        tmem_ld_wait();
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          acc[p * 16 + i] = __fadd_rn(acc[p * 16 + i], __uint_as_float(r[0][i]));
          if (p + 1 < NP) acc[p * 16 + 16 + i] = __fadd_rn(acc[p * 16 + 16 + i], __uint_as_float(r[1][i]));
        }
      }
    }
    tc_fence_before();
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&s.d_free[c.t][ab]);   // one arrival per warp
  }
  if (c.t == 0 && c.ntile == 2) c.ch += chunks;
}
__device__ __forceinline__ void h_setup(HSmem& s, int a_ready_warps = H_TILE_WARPS, int d_free_warps = H_TILE_WARPS) {
  if (threadIdx.x == 0) {
    for (int i = 0; i < H_STAGES; ++i) { mbar_init(&s.full[i], 1); mbar_init(&s.empty[i], 1); }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&s.a_ready[i], a_ready_warps);
      for (int j = 0; j < 2; ++j) { mbar_init(&s.d_ready[i][j], 1); mbar_init(&s.d_free[i][j], d_free_warps); }
    }
    mbar_fence_init();
  }
  if ((threadIdx.x >> 5) == 0) tmem_alloc(&s.tmem_base, 512);
}
__device__ __forceinline__ void h_finish(HSmem& s, const HCtx* c) {
  if (c && c->bad) atomicOr(&g_h16_overflow, 1u);
  tc_fence_before();
  __syncthreads();
  if ((threadIdx.x >> 5) == 0) tmem_dealloc(s.tmem_base, 512);
}
// Same with an output leading dimension (the tile is a column slice of a wider row-major matrix).
// `res` (nullable, same leading dimension): added to the tile in the coalesced store phase (fused residual / skip add).
template <int W>
__device__ __forceinline__ void h_store_tile_strided(HSmem& s, const HCtx& c, int col0, const float (&v)[W / 2],
                                                     float* __restrict__ out, int ld, int rows,
                                                     const float* __restrict__ res = nullptr) {
  constexpr int LD = W + 1, RPW = 128 / W;
  float* st = reinterpret_cast<float*>(s.a[c.t][0]);
#pragma unroll
  for (int i = 0; i < W / 2; ++i) st[c.row * LD + col0 + i] = v[i];
  h_tile_bar(c.t);
  const int w = c.et >> 5, lane = c.et & 31;
  for (int r0 = w * RPW; r0 < rows; r0 += H_TILE_WARPS * RPW) {
    const int r = r0 + (RPW == 2 ? (lane >> 4) : 0), c4 = 4 * (RPW == 2 ? (lane & 15) : lane);
    if (r < rows) {
      const float* src = st + r * LD + c4;
      float4 o = make_float4(src[0], src[1], src[2], src[3]);
      if (res) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(res + (size_t)r * ld + c4));
        o.x += q.x; o.y += q.y; o.z += q.z; o.w += q.w;
      }
      *reinterpret_cast<float4*>(out + (size_t)r * ld + c4) = o;
    }
  }
}

// ---------------------------------------------------------------------------------- weight packing
// W [N, K] fp32 (nn.Linear layout) -> K/32 slabs of [hi|lo][4 k-units][N][8 halves], w*64 = hi + lo.
struct HPackJob { const float* w; unsigned char* out; int N, K, trans; };   // trans > 0: the source is stored [K, trans] (a column slice of W^T's source)
struct HPackJobs { HPackJob job[16]; };
__global__ void h16_pack_kernel(HPackJobs jobs) {
  const HPackJob jb = jobs.job[blockIdx.y];
  const int total = jb.N * jb.K;
  for (int id = blockIdx.x * blockDim.x + threadIdx.x; id < total; id += gridDim.x * blockDim.x) {
    const int n = id / jb.K, k = id % jb.K;
    const float x = __ldg(jb.w + (jb.trans ? (size_t)k * jb.trans + n : (size_t)id)) * H_SW;
    const __half h = __float2half_rn(x);
    const __half l = __float2half_rn(x - __half2float(h));
    const int c = k >> 5, ku = (k & 31) >> 3, kk = k & 7;
    const size_t slab = (size_t)c * (2 * 4 * jb.N * 16);
    const size_t o = ((size_t)ku * jb.N + n) * 16 + kk * 2;
    *reinterpret_cast<__half*>(jb.out + slab + o) = h;
    *reinterpret_cast<__half*>(jb.out + slab + (size_t)4 * jb.N * 16 + o) = l;
  }
}

// ---------------------------------------------------------------------------------- update_e: register-accumulator engine
// Part B of update_e (lin_up, the residual layers, lin; spherenet.py:172-179, edge -> node sum :211) and part A
// (lin_ji, lin_kj, lin_down; spherenet.py:154-161) keep every activation of a 64-edge unit in wgmma register fragments:
//
//   * roles (384 threads): warpgroup 0 is the producer -- one thread streams the packed weight slabs of every layer
//     through a ring of R_STAGES K = 32 slabs (cp.async.bulk, full / empty mbarriers; a stage is refilled once both
//     consumers' MMAs that read it have completed).  Warpgroups 1 and 2 are consumers, each working on one 64-row unit
//     at a time: a consumer issues its own wgmma with A FROM REGISTERS and B from the ring, then runs the layer's
//     epilogue on the accumulator fragment while the other consumer's MMAs keep the tensor pipe busy (ping-pong).
//     Consumer 1 starts after consumer 0 has issued its first layer; the stagger then persists because each consumer's
//     MMAs queue behind the other's.
//   * the m64nN accumulator fragment has the layout of the register A operand of the next layer's m64k16 steps
//     (wgmma.cuh, frag_a_src): the epilogue splits each activated pair into the fp16 hi / lo registers of the next A in
//     place -- no operand planes, no accumulator store, no handshakes inside a unit's chain.
//   * the numerics are those of the two-tile store engine this replaces: operands pre-scaled by H_SA / H_SW and split
//     hi / lo with round-to-nearest; K = 64 chunks, each started with scale-d = 0 (the tensor core truncates while it
//     accumulates), summed with __fadd_rn in chunk order; the same product order inside a chunk (per K = 32 slab
//     lo*W_hi and hi*W_lo for both k-steps, then hi*W_hi); the same epilogue arithmetic per element.
//   * the fp32 skip / residual rows and then the e2 tile live in a [64][R_LDS] fp32 tile per consumer in shared memory;
//     a thread touches only its own fragment elements there until e2 is summed by column.  Every output (e1, x_ji,
//     x_down) is stored straight from the fragment: one warp store covers 8 rows x 32 bytes, whole sectors.
//   * persistent grid of min(SMs, units / 2) CTAs: consumer w of CTA b takes units b + (2 k + w) gridDim.x, so the
//     units beyond the last full round of pairs go to different SMs instead of a whole second CTA wave.
constexpr int R_UNIT = 64;              // edges per consumer unit: the M of one wgmma
constexpr int R_STAGES = 8;             // two K = 128, N = 128 layers: one consumer may hold a layer the other has left
constexpr int R_LDS = 136;              // row stride (floats) of a consumer tile: 8-byte fragment accesses are conflict free
constexpr int R_WG = 128;
constexpr int R_EPI_J = 8;              // column pairs per group of the e2 epilogues: tile stores wait for the group's loads
constexpr int R_THREADS = 3 * R_WG;     // producer warpgroup + two consumer warpgroups
// setmaxnreg: the kernel is compiled for 168 registers (384 threads); the producer drops to 40 and the consumers grow to
// 232 (128 x 40 + 256 x 232 <= 64 K): a consumer holds the A operand (64), the chunk-0 and chunk-1 accumulators (2 x 64).
__device__ __forceinline__ void r_regs_producer() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void r_regs_consumer() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

struct RSmem {
  unsigned char w[R_STAGES][H_STAGE_BYTES];
  float tile[2][R_UNIT * R_LDS];        // per consumer: skip / residual rows (x H_SA), then e2
  float rbf[2][R_UNIT * 6];             // per consumer: rbf0 rows of its unit
  float bias[8][128];                   // part B biases (x H_SA)
  float bias_a[2][128];                 // part A: b_ji (x 1), b_kj (x H_SA)
  float wr[128 * 8];                    // part B: lin_rbf [128][6] padded to 8
  float wr1[64];                        // part A: lin_rbf1 [8][6] padded to 8
  float wr2[128 * 8];                   // part A: lin_rbf2 [128][8]
  int dst[2][R_UNIT];
  uint64_t full[R_STAGES], empty[R_STAGES];
};
static_assert(sizeof(RSmem) <= 227 * 1024, "RSmem exceeds the shared memory of an SM");

// part B; part B + part A of the next block; part A; init_e; init_e + part A of block 0
enum { RE_B = 0, RE_BA = 1, RE_A = 2, RE_I = 3, RE_IA = 4 };
struct REParams {
  HGemm g[11];                          // B: lin_up, res0.lin1, res0.lin2, lin, res1.lin1, res1.lin2, res2.lin1, res2.lin2
                                        // BA: + lin_ji, lin_kj, lin_down of the NEXT block;  A: lin_ji, lin_kj, lin_down
                                        // I: init lin (K = 128 rbf panel, or K = 384 = three panels);  IA: + part A
  const float* w_rbf;                   // B: lin_rbf [128, 6];  I: init lin_rbf_1 [128, 6]
  const float *w_rbf1, *w_rbf2;         // A: lin_rbf1 [8, 6], lin_rbf2 [128, 8] (BA: of the next block)
  float *x_ji, *x_down;                 // A: outputs (BA: of the next block)
  const int64_t* z;                     // I: atomic numbers
  const int32_t* src;                   // I: source node of each edge
  const float *emb, *w_rbf0, *b_rbf0, *b_lin;   // I: init weights (emb: three-panel form)
  const float *tab_i, *tab_j;           // I, table form: [emb rows, 128] = emb W[:, 0:128]^T and emb W[:, 128:256]^T
};

__device__ __forceinline__ void r_bar(int cw) { asm volatile("bar.sync %0, %1;" ::"r"(1 + cw), "n"(R_WG) : "memory"); }
// 4 / 8-byte asynchronous copies global -> shared; a source size of 0 writes zeros (rows past the last edge)
__device__ __forceinline__ void cp_async4(void* sm, const void* g, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(sm)), "l"(g), "r"(valid ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_async8(void* sm, const void* g, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(sm)), "l"(g), "r"(valid ? 8 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// A pair of consecutive K elements, ALREADY multiplied by H_SA -> fp16 hi / lo registers (the split of h_store_ku).
__device__ __forceinline__ void r_split(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 hh = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(hh);
  const __half2 ll = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&hh);
  lo = *reinterpret_cast<const uint32_t*>(&ll);
}
struct RA { uint32_t hi[8][4], lo[8][4]; };   // register A operand of a K <= 128 layer: [k-step][register]
// activated m64n128 fragment (x H_SA) -> A operand of the next layer
__device__ __forceinline__ void r_acc_to_a(const float (&v)[64], RA& a, float scale = 1.0f) {
#pragma unroll
  for (int s = 0; s < 8; ++s)
#pragma unroll
    for (int r = 0; r < 4; ++r) r_split(v[frag_a_src(s, r)] * scale, v[frag_a_src(s, r) + 1] * scale, a.hi[s][r], a.lo[s][r]);
}
// rows [0, rows) of a row-major fp32 [64 x 16 KS] tile (leading dimension ld) -> A operand (x H_SA); other rows zero
template <int KS>
__device__ __forceinline__ void r_load_a(RA& a, const float* __restrict__ g, int ld, int rows, int wt) {
#pragma unroll
  for (int s = 0; s < KS; ++s)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int row = frag_a_row(wt, r), col = frag_a_col(wt, s, r);
      const float2 x = row < rows ? __ldg(reinterpret_cast<const float2*>(g + (size_t)row * ld + col)) : make_float2(0.f, 0.f);
      r_split(x.x * H_SA, x.y * H_SA, a.hi[s][r], a.lo[s][r]);
    }
}
// fp32 rows of a [E, 128] tensor -> this thread's fragment elements of the consumer tile (unscaled; zeros past `rows`)
__device__ __forceinline__ void r_fetch_rows(float* tile, const float* __restrict__ src, int rows, int fr, int fc) {
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = fr + 8 * h, col = 8 * j + fc;
      cp_async8(tile + row * R_LDS + col, src + (size_t)(row < rows ? row : 0) * 128 + col, row < rows);
    }
  cp_async_commit();
}

// ---- weight ring, consumer side: `it` counts the slabs of the producer's sequence this consumer has passed
__device__ __forceinline__ void r_release(RSmem& s, int it, int n) {   // the MMAs reading slabs it .. it + n - 1 are done
  __syncwarp();
  if ((threadIdx.x & 31) == 0)
    for (int i = 0; i < n; ++i) mbar_arrive(&s.empty[(it + i) % R_STAGES]);   // one arrival per consumer warp
}
// chunk CH (K = 64: slabs it + 2 CH, + 1) of a layer with N output columns into t, the slab's corrections (2^-11 of the
// main term) first, then its two hi*hi steps; the first product starts the chunk (scale-d = 0)
template <int CH, int N>
__device__ __forceinline__ void r_chunk(RSmem& s, const RA& a, float (&t)[N / 2], int it) {
#pragma unroll
  for (int sl = 0; sl < 2; ++sl) {
    const uint32_t w_hi = smem_u32(s.w[(it + 2 * CH + sl) % R_STAGES]), w_lo = w_hi + 4u * N * 16u;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const int k = 4 * CH + 2 * sl + ks;
      const uint32_t b_off = (uint32_t)(ks * 2 * N * 16);
      mma_f16_rs(t, a.lo[k], smem_desc(w_hi + b_off, N * 16, 128), (sl | ks) != 0);
      mma_f16_rs(t, a.hi[k], smem_desc(w_lo + b_off, N * 16, 128), 1);
    }
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
      mma_f16_rs(t, a.hi[4 * CH + 2 * sl + ks], smem_desc(w_hi + (uint32_t)(ks * 2 * N * 16), N * 16, 128), 1);
  }
}
// one layer (K = 64 NCH): chunk 0 -> acc, chunk 1 -> d; r_complete waits, frees the slabs and adds d to acc
template <int NCH, int N>
__device__ __forceinline__ void r_issue(RSmem& s, const RA& a, float (&acc)[N / 2], float (&d)[N / 2], int it) {
#pragma unroll
  for (int i = 0; i < 2 * NCH; ++i) mbar_wait(&s.full[(it + i) % R_STAGES], ((it + i) / R_STAGES) & 1);
  wg_fence();
  r_chunk<0, N>(s, a, acc, it);
  if (NCH == 2) r_chunk<1, N>(s, a, d, it);
  wg_commit();
}
template <int NCH, int N>
__device__ __forceinline__ void r_complete(RSmem& s, float (&acc)[N / 2], const float (&d)[N / 2], int& it) {
  wg_wait0();
  r_release(s, it, 2 * NCH);
  it += 2 * NCH;
  if (NCH == 2) {
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = __fadd_rn(acc[i], d[i]);
  }
}
// a K = 128 panel issued into acc (chunk 0) and d (chunk 1) on top of the earlier panels' sum parked in the consumer
// tile: acc = (tile + chunk 0) + chunk 1, the chunk order of the store engine's drains
__device__ __forceinline__ void r_complete_onto(RSmem& s, float (&acc)[64], const float (&d)[64], const float* tile,
                                                int fr, int fc, int& it) {
  wg_wait0();
  r_release(s, it, 4);
  it += 4;
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = 4 * j + 2 * h;
      const float2 t = *reinterpret_cast<const float2*>(tile + (fr + 8 * h) * R_LDS + 8 * j + fc);
      acc[i] = __fadd_rn(__fadd_rn(t.x, acc[i]), d[i]);
      acc[i + 1] = __fadd_rn(__fadd_rn(t.y, acc[i + 1]), d[i + 1]);
    }
}
// the thread's fragment elements of column pairs j0 .. j0 + NJ - 1 (default: all) -> the consumer tile.  The epilogues
// write the tile only after the shared-memory reads of a whole group of elements: the compiler cannot tell a tile
// store from a later bias / gate-weight / tile load (one dynamic shared-memory base, different registers), so a store
// ahead of a load keeps the next element's loads behind it and leaves one element's latency chain (loads, two MUFU
// ops, the FP32 ops) exposed at a time.
template <int NJ = 16>
__device__ __forceinline__ void r_park(const float (&acc)[64], float* tile, int fr, int fc, int j0 = 0) {
#pragma unroll
  for (int j = j0; j < j0 + NJ; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float2*>(tile + (fr + 8 * h) * R_LDS + 8 * j + fc) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
}
// rbf0 rows fr, fr + 8 of the unit
__device__ __forceinline__ void r_rbf_rows(const float* rbf, int fr, float (&rb)[2][6]) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int n = 0; n < 6; ++n) rb[h][n] = rbf[(fr + 8 * h) * 6 + n];
}
// the e2 gate lin_rbf(rbf0[row]) at one column (w0, w1: its lin_rbf row; shared by the thread's two rows)
__device__ __forceinline__ float r_gate6(const float4& w0, const float2& w1, const float (&rb)[6]) {
  return fmaf(w1.y, rb[5], fmaf(w1.x, rb[4], fmaf(w0.w, rb[3], fmaf(w0.z, rb[2], fmaf(w0.y, rb[1], __fmul_rn(w0.x, rb[0]))))));
}
// a consumer without a unit in this round still passes every slab of it (the ring counts both consumers per stage)
__device__ __forceinline__ void r_skip(RSmem& s, int& it, int n) {
  for (int i = 0; i < n; ++i, ++it) {
    mbar_wait(&s.full[it % R_STAGES], (it / R_STAGES) & 1);
    r_release(s, it, 1);
  }
}

// e2 of a unit (staged [64][R_LDS] fp32) -> edge -> node sums; thread = column, rows in order.  Rows are target-sorted:
// a segment touching the first or last row of the unit may continue in a neighbouring unit and is added with an
// atomic, interior segments are plain stores (v_in is zeroed before the launch).  Every node's in-edge segment is split
// across at most two writers: the radius graph caps the in-degree at 32, so a segment spans at most two 64-row units,
// and two atomicAdds onto zero commute (0 + a + b == 0 + b + a) -- the sums are deterministic.
__device__ __forceinline__ void r_segment_sums(const float* tile, const int* dst, int rows, int col,
                                               float* __restrict__ v_in) {
  float run = 0.f;
  int cur = dst[0];
  bool first = true;
  for (int r = 0; r < rows; ++r) {
    const int d = dst[r];
    if (d != cur) {
      if (first) atomicAdd(v_in + (size_t)cur * 128 + col, run);
      else v_in[(size_t)cur * 128 + col] = run;
      first = false; run = 0.f; cur = d;
    }
    run += tile[r * R_LDS + col];
  }
  atomicAdd(v_in + (size_t)cur * 128 + col, run);
}

// MODE = RE_B: part B of a block; RE_BA: part B of block l, then part A of block l + 1 on the e1 fragment still in
// registers (one launch, one e1 read less per block); RE_A: part A on e1 read from memory (layer 0); RE_I: init_e
// (spherenet.py:79-91, edge -> node sum :211); RE_IA: init_e, then part A of block 0 on the e1 fragment.  Per element
// the modes compute what the store engine computed, so RE_BA == RE_B followed by RE_A and RE_IA == RE_I followed by
// RE_A bit for bit.  TABLE (RE_I / RE_IA): the embedding panels of init_e come from the tables (ops.init_e_tables).
template <bool FAST, int MODE, bool TABLE = false>
__global__ void __launch_bounds__(R_THREADS, 1)
sphere_update_e_h16_kernel(const float* __restrict__ m, const float* __restrict__ x_ji,
                           const float* __restrict__ e1_in, const float* __restrict__ rbf0,
                           const int32_t* __restrict__ dst, int n_edges, REParams P, float* __restrict__ e1_out,
                           float* __restrict__ v_in) {
  constexpr bool INIT = MODE == RE_I || MODE == RE_IA;
  constexpr int NG = MODE == RE_B ? 8 : MODE == RE_BA ? 11 : MODE == RE_I ? 1 : MODE == RE_IA ? 4 : 3;   // layers per unit
  extern __shared__ __align__(1024) unsigned char h_raw[];
  RSmem& s = *reinterpret_cast<RSmem*>(h_raw);
  const int tid = threadIdx.x, wg = tid / R_WG;
  // (values live across setmaxnreg are recomputed after it: a register carried over would be spilled)
  auto n_units = [&]() { return (n_edges + R_UNIT - 1) / R_UNIT; };
  auto rounds = [&]() {   // units of consumer 0
    return (n_units() - (int)blockIdx.x + 2 * (int)gridDim.x - 1) / (2 * (int)gridDim.x);
  };
  const bool trace = g_h16_trace_on && blockIdx.x == 0;
  if (tid == 0 && trace) { g_h16_trace[100] = clock64(); g_h16_trace[101] = (long long)global_ns(); }
  if (tid == 0) {
    for (int i = 0; i < R_STAGES; ++i) { mbar_init(&s.full[i], 1); mbar_init(&s.empty[i], 8); }
    mbar_fence_init();
  }
  if (INIT) {   // bias[0] = lin.bias, bias[1] = lin_rbf_0.bias (both unscaled), bias[2..7] = lin_rbf_0.weight [128][6]
    for (int i = tid; i < 128; i += R_THREADS) { s.bias[0][i] = __ldg(P.b_lin + i); s.bias[1][i] = __ldg(P.b_rbf0 + i); }
    for (int i = tid; i < 128 * 6; i += R_THREADS) (&s.bias[2][0])[i] = __ldg(P.w_rbf0 + i);
  } else if (MODE != RE_A) {
    for (int i = tid; i < 8 * 128; i += R_THREADS) {
      const float* b = P.g[i / 128].bias;
      s.bias[i / 128][i % 128] = b ? H_SA * __ldg(b + i % 128) : 0.f;          // the chain runs pre-scaled by H_SA
    }
  }
  if (MODE != RE_A)
    for (int i = tid; i < 128 * 8; i += R_THREADS) s.wr[i] = (i % 8 < 6) ? __ldg(P.w_rbf + (i / 8) * 6 + i % 8) : 0.f;
  if (MODE != RE_B && MODE != RE_I) {
    constexpr int GA = MODE == RE_A ? 0 : MODE == RE_IA ? 1 : 8;
    for (int i = tid; i < 2 * 128; i += R_THREADS)     // lin_ji's output leaves unscaled, lin_kj's feeds an operand (x H_SA)
      s.bias_a[i / 128][i % 128] = (i / 128 ? H_SA : 1.0f) * __ldg(P.g[GA + i / 128].bias + i % 128);
    for (int i = tid; i < 128 * 8; i += R_THREADS) s.wr2[i] = __ldg(P.w_rbf2 + i);
    for (int i = tid; i < 64; i += R_THREADS) s.wr1[i] = (i % 8 < 6) ? __ldg(P.w_rbf1 + (i / 8) * 6 + i % 8) : 0.f;
  }
  __syncthreads();
  if (tid == 0 && trace) g_h16_trace[104] = clock64();

  if (wg == 0) {
    // ---- producer: every K = 32 slab of every layer, once per round (both consumers read each slab)
    r_regs_producer();
    if (tid == 0) {
      int it = 0;
      const int nr = rounds();
      for (int k = 0; k < nr; ++k)
        for (int q = 0; q < NG; ++q) {
          const uint32_t bytes = 2u * 4u * (uint32_t)P.g[q].N * 16u;
          for (int c = 0; c < P.g[q].K / H_SLAB_K; ++c, ++it) {
            const int st = it % R_STAGES;
            if (it >= R_STAGES) mbar_wait(&s.empty[st], ((it / R_STAGES) + 1) & 1);
            mbar_arrive_expect_tx(&s.full[st], bytes);
            bulk_g2s(s.w[st], P.g[q].w + (size_t)c * bytes, bytes, &s.full[st]);
          }
        }
    }
    return;
  }

  // ---- consumers
  r_regs_consumer();
  const int cw = threadIdx.x / R_WG - 1, wt = threadIdx.x & (R_WG - 1);
  const int nu = n_units(), nr = rounds();
  const int fr = frag_row(wt), fc = frag_col(wt);   // this thread's fragment rows fr, fr + 8 and columns 8 j + fc (+1)
  float* tile = s.tile[cw];
  const float* rbf = s.rbf[cw];
  int slabs = 0;
  for (int q = 0; q < NG; ++q) slabs += P.g[q].K / H_SLAB_K;
  // timeline probe (tools/gpu_h16_timeline.py): CTA 0, first unit of each consumer, four points per layer
  const bool probe = g_h16_trace_on && blockIdx.x == 0 && wt == 0;
  int lq = 0;
  auto tp = [&](bool on, int point) { if (on) g_h16_trace[cw * 48 + lq * 4 + point] = clock64(); };
  bool staggered = cw == 1, bad = false;
  auto stagger = [&]() {
    if (!staggered) { asm volatile("bar.arrive 3, %0;" ::"n"(2 * R_WG) : "memory"); staggered = true; }
  };
  if (cw == 1) asm volatile("bar.sync 3, %0;" ::"n"(2 * R_WG) : "memory");   // after consumer 0's first layer is issued
  int it = 0;
#pragma unroll 1
  for (int k = 0; k < nr; ++k) {
    const int unit = blockIdx.x + (2 * k + cw) * gridDim.x;
    if (unit >= nu) { r_skip(s, it, slabs); continue; }
    const int e0 = unit * R_UNIT, rows = min(R_UNIT, n_edges - e0);
    const bool tr = probe && k == 0;
    lq = 0;
    r_bar(cw);   // the previous unit is done with tile / rbf / dst
    for (int i = wt; i < R_UNIT * 6; i += R_WG)
      cp_async4(&s.rbf[cw][i], rbf0 + (size_t)e0 * 6 + (i < rows * 6 ? i : 0), i < rows * 6);
    RA a;
    float acc[64], d[64];
    if (INIT) {
      // e1 = act(lin(cat[x_i, x_j, act(lin_rbf_0(rbf0))])), e2 = lin_rbf_1(rbf0) * e1          spherenet.py:79-91
      if (wt < R_UNIT) cp_async4(&s.dst[cw][wt], dst + e0 + (wt < rows ? wt : 0), wt < rows);
      cp_async_commit();
      int zi[2], zj[2];   // atomic numbers of the target / source node of rows fr, fr + 8 (0 past the last edge)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int e = e0 + fr + 8 * h;
        const bool ok = fr + 8 * h < rows;
        zi[h] = ok ? (int)__ldg(P.z + __ldg(dst + e)) : 0;
        zj[h] = ok ? (int)__ldg(P.z + __ldg(P.src + e)) : 0;
      }
      auto embedding_a = [&](const int (&zr)[2]) {   // A = H_SA * emb[z]
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int h = r & 1, row = fr + 8 * h, col = frag_a_col(wt, k, r);
            const float2 x = row < rows ? __ldg(reinterpret_cast<const float2*>(P.emb + (size_t)zr[h] * 128 + col))
                                        : make_float2(0.f, 0.f);
            r_split(x.x * H_SA, x.y * H_SA, a.hi[k][r], a.lo[k][r]);
          }
      };
      auto rbf_a = [&]() {   // A = H_SA * act(lin_rbf_0(rbf0))                                     spherenet.py:87
        const float* w0 = &s.bias[2][0];
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int h = r & 1, row = fr + 8 * h, col = frag_a_col(wt, k, r);
            float x[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              float t = 0.f;
#pragma unroll
              for (int n = 0; n < 6; ++n) t = fmaf(w0[(col + u) * 6 + n], rbf[row * 6 + n], t);
              x[u] = row < rows ? H_SA * hswish<FAST>(__fadd_rn(t, s.bias[1][col + u])) : 0.f;   // one FMUL.M8 (see hswish)
            }
            r_split(x[0], x[1], a.hi[k][r], a.lo[k][r]);
          }
      };
      if (TABLE) {
        // W_i emb[z_i] + W_j emb[z_j] of the thread's elements (L2-resident tables) -> tile, while rbf0 arrives
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = fr + 8 * h, col = 8 * j + fc;
            const float2 ti = __ldg(reinterpret_cast<const float2*>(P.tab_i + (size_t)zi[h] * 128 + col));
            const float2 tj = __ldg(reinterpret_cast<const float2*>(P.tab_j + (size_t)zj[h] * 128 + col));
            *reinterpret_cast<float2*>(tile + row * R_LDS + col) = make_float2(ti.x + tj.x, ti.y + tj.y);
          }
        cp_async_wait_all();
        r_bar(cw);                                                   // rbf / dst of the unit: visible to all
        rbf_a();
        r_issue<2, 128>(s, a, acc, d, it);
        stagger();
        r_complete<2, 128>(s, acc, d, it);
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = fr + 8 * h, col = 8 * j + fc, i = 4 * j + 2 * h;
            const float2 t = *reinterpret_cast<const float2*>(tile + row * R_LDS + col);
            acc[i] = __fmul_rn(fmaf(acc[i], H_INV, t.x), H_SA * H_SW);
            acc[i + 1] = __fmul_rn(fmaf(acc[i + 1], H_INV, t.y), H_SA * H_SW);
          }
      } else {   // K = 384 as three K = 128 panels, A rebuilt between them; six chunks summed in order
        embedding_a(zi);                                             // panel 0: x_i
        r_issue<2, 128>(s, a, acc, d, it);
        stagger();
        r_complete<2, 128>(s, acc, d, it);
        r_park(acc, tile, fr, fc);                                   // (the running sum waits in the tile)
        embedding_a(zj);                                             // panel 1: x_j
        r_issue<2, 128>(s, a, acc, d, it);
        r_complete_onto(s, acc, d, tile, fr, fc, it);
        r_park(acc, tile, fr, fc);
        cp_async_wait_all();
        r_bar(cw);
        rbf_a();                                                     // panel 2: act(lin_rbf_0(rbf0))
        r_issue<2, 128>(s, a, acc, d, it);
        r_complete_onto(s, acc, d, tile, fr, fc, it);
      }
      // e1 = act(. + b) and the e2 tile; edge -> node sums                                     spherenet.py:211
      {
        float rb[2][6], e2[64];
        r_rbf_rows(rbf, fr, rb);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int col = 8 * j + fc + u;
            const float b = s.bias[0][col];
            const float4 w0 = *reinterpret_cast<const float4*>(s.wr + col * 8);
            const float2 w1 = *reinterpret_cast<const float2*>(s.wr + col * 8 + 4);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int i = 4 * j + 2 * h + u;
              const float o = hswish<FAST>(fmaf(acc[i], H_INV, b));
              bad |= !h_finite(o);
              e2[i] = __fmul_rn(r_gate6(w0, w1, rb[h]), o);
              acc[i] = o;
            }
          }
          if (j % R_EPI_J == R_EPI_J - 1) r_park<R_EPI_J>(e2, tile, fr, fc, j + 1 - R_EPI_J);
        }
      }
      r_bar(cw);
      r_segment_sums(tile, s.dst[cw], rows, wt, v_in);
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = fr + 8 * h, i = 4 * j + 2 * h;
          if (row < rows)
            *reinterpret_cast<float2*>(e1_out + (size_t)(e0 + row) * 128 + 8 * j + fc) = make_float2(acc[i], acc[i + 1]);
        }
      if (MODE == RE_IA) r_acc_to_a(acc, a, H_SA);        // part A of block 0: operand H_SA * e1
    } else if (MODE != RE_A) {
      if (wt < R_UNIT) cp_async4(&s.dst[cw][wt], dst + e0 + (wt < rows ? wt : 0), wt < rows);
      r_fetch_rows(tile, x_ji + (size_t)e0 * 128, rows, fr, fc);     // skip rows of q = 0
      r_load_a<4>(a, m + (size_t)e0 * 64, 64, rows, wt);             // A0 = m (K = 64)
      // The eight layers of the chain (spherenet.py:172-179), tile = the fp32 skip / residual row (x H_SA):
      //   q=0: h = x_ji + act(lin_up(m))                       -> A, tile
      //   q=1,4,6: t = act(lin1(h))                            -> A
      //   q=2,5: h = tile + act(lin2(t))                       -> A, tile      (q=2: then tile <- e1_in)
      //   q=3: h = act(lin(h)) + e1_in                         -> A, tile
      //   q=7: e1 = tile + act(lin2(t))                        -> e1_out, e2 tile
#pragma unroll 1
      for (int q = 0; q < 7; ++q, ++lq) {
        tp(tr, 0);
        if (q == 0) {
          r_issue<1, 128>(s, a, acc, d, it);
          stagger();
          tp(tr, 1);
          r_complete<1, 128>(s, acc, d, it);
        } else {
          r_issue<2, 128>(s, a, acc, d, it);
          tp(tr, 1);
          r_complete<2, 128>(s, acc, d, it);
        }
        tp(tr, 2);
        const bool add_tile = q == 0 || q == 2 || q == 3 || q == 5;
        const bool to_tile = q == 0 || q == 3 || q == 5;
        const float tile_scale = (q == 0 || q == 3) ? H_SA : 1.0f;   // x_ji / e1_in arrive unscaled (x H_SA is exact)
        if (q == 0 || q == 3) cp_async_wait_all();
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 b = *reinterpret_cast<const float2*>(&s.bias[q][8 * j + fc]);   // shared by both rows
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int i = 4 * j + 2 * h;
            float v0 = hswish8<FAST>(fmaf(acc[i], H_SA * H_INV, b.x));
            float v1 = hswish8<FAST>(fmaf(acc[i + 1], H_SA * H_INV, b.y));
            if (add_tile) {
              const float2 r = *reinterpret_cast<const float2*>(tile + (fr + 8 * h) * R_LDS + 8 * j + fc);
              v0 = fmaf(r.x, tile_scale, v0);
              v1 = fmaf(r.y, tile_scale, v1);
            }
            acc[i] = v0;
            acc[i + 1] = v1;
          }
        }
        if (to_tile) r_park(acc, tile, fr, fc);
        r_acc_to_a(acc, a);
        if (q == 0) r_bar(cw);                                            // rbf / dst of the unit: visible to all
        if (q == 2) r_fetch_rows(tile, e1_in + (size_t)e0 * 128, rows, fr, fc);   // read above; q = 3 adds e1_in
        tp(tr, 3);
      }
      // q = 7: e1 = tile + act(lin2(t)); e2 = lin_rbf(rbf0) * e1 staged in the tile for the edge -> node sums
      tp(tr, 0);
      r_issue<2, 128>(s, a, acc, d, it);
      tp(tr, 1);
      r_complete<2, 128>(s, acc, d, it);
      tp(tr, 2);
      {
        float rb[2][6], e2[64];
        r_rbf_rows(rbf, fr, rb);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          float2 r[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) r[h] = *reinterpret_cast<const float2*>(tile + (fr + 8 * h) * R_LDS + 8 * j + fc);
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int col = 8 * j + fc + u;
            const float b = s.bias[7][col];
            const float4 w0 = *reinterpret_cast<const float4*>(s.wr + col * 8);
            const float2 w1 = *reinterpret_cast<const float2*>(s.wr + col * 8 + 4);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int i = 4 * j + 2 * h + u;
              const float o = __fmul_rn(hswish8_plus<FAST>(fmaf(acc[i], H_SA * H_INV, b), u ? r[h].y : r[h].x), 1.0f / H_SA);
              bad |= !h_finite(o);
              e2[i] = __fmul_rn(r_gate6(w0, w1, rb[h]), o);
              acc[i] = o;
            }
          }
          if (j % R_EPI_J == R_EPI_J - 1) r_park<R_EPI_J>(e2, tile, fr, fc, j + 1 - R_EPI_J);
        }
      }
      tp(tr, 3);
      ++lq;
      r_bar(cw);
      r_segment_sums(tile, s.dst[cw], rows, wt, v_in);   // spherenet.py:211
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = fr + 8 * h, i = 4 * j + 2 * h;
          if (row < rows)
            *reinterpret_cast<float2*>(e1_out + (size_t)(e0 + row) * 128 + 8 * j + fc) = make_float2(acc[i], acc[i + 1]);
        }
      if (tr) g_h16_trace[96 + cw] = clock64();
      if (MODE == RE_BA) r_acc_to_a(acc, a, H_SA);        // part A of the next block: operand H_SA * e1
    } else {
      cp_async_commit();
      r_load_a<8>(a, e1_in + (size_t)e0 * 128, 128, rows, wt);
    }
    if (MODE != RE_B && MODE != RE_I) {
      // G0: x_ji = act(lin_ji(e1))                                                spherenet.py:154
      tp(tr, 0);
      r_issue<2, 128>(s, a, acc, d, it);
      stagger();
      tp(tr, 1);
      r_complete<2, 128>(s, acc, d, it);
      tp(tr, 2);
      {
        float2 b[16];   // read ahead of the x_ji stores, which the compiler cannot tell from shared-memory writes
#pragma unroll
        for (int j = 0; j < 16; ++j) b[j] = *reinterpret_cast<const float2*>(&s.bias_a[0][8 * j + fc]);
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = fr + 8 * h, col = 8 * j + fc, i = 4 * j + 2 * h;
            if (row < rows) {
              const float2 o = make_float2(hswish<FAST>(fmaf(acc[i], H_INV, b[j].x)), hswish<FAST>(fmaf(acc[i + 1], H_INV, b[j].y)));
              bad |= !(h_finite(o.x) && h_finite(o.y));   // e1 (part A's split operand) out of range: the flag of RE_A
              *reinterpret_cast<float2*>(P.x_ji + (size_t)(e0 + row) * 128 + col) = o;
            }
          }
      }
      if (MODE == RE_A) { cp_async_wait_all(); r_bar(cw); }   // rbf of the unit: visible to all
      tp(tr, 3);
      ++lq;
      // G1: x_kj = act(lin_kj(e1)) * lin_rbf2(lin_rbf1(rbf0)), on the same operand    spherenet.py:155-159
      tp(tr, 0);
      r_issue<2, 128>(s, a, acc, d, it);
      tp(tr, 1);
      r_complete<2, 128>(s, acc, d, it);
      tp(tr, 2);
      {
        float r8[2][8];                                // gate coefficients of the two rows: lin_rbf1(rbf0[row])
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int mm = 0; mm < 8; ++mm) {
            float x = 0.f;
#pragma unroll
            for (int n = 0; n < 6; ++n) x = fmaf(s.wr1[mm * 8 + n], rbf[(fr + 8 * h) * 6 + n], x);
            r8[h][mm] = x;
          }
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int col = 8 * j + fc + u;   // lin_rbf2 row and bias of the column: shared by the thread's two rows
            const float4 w0 = *reinterpret_cast<const float4*>(s.wr2 + col * 8);
            const float4 w1 = *reinterpret_cast<const float4*>(s.wr2 + col * 8 + 4);
            const float b = s.bias_a[1][col];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int i = 4 * j + 2 * h + u;
              const float* g = r8[h];
              const float gate = fmaf(w1.w, g[7], fmaf(w1.z, g[6], fmaf(w1.y, g[5], fmaf(w1.x, g[4],
                                 fmaf(w0.w, g[3], fmaf(w0.z, g[2], fmaf(w0.y, g[1], __fmul_rn(w0.x, g[0]))))))));
              acc[i] = __fmul_rn(hswish8<FAST>(fmaf(acc[i], H_SA * H_INV, b)), gate);
            }
          }
      }
      r_acc_to_a(acc, a);
      tp(tr, 3);
      ++lq;
      // G2: x_down = act(lin_down(x_kj)), N = 64                                  spherenet.py:161
      {
        float a64[32], d64[32];
        tp(tr, 0);
        r_issue<2, 64>(s, a, a64, d64, it);
        tp(tr, 1);
        r_complete<2, 64>(s, a64, d64, it);
        tp(tr, 2);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = fr + 8 * h, i = 4 * j + 2 * h;
            if (row < rows) {
              const float2 o = make_float2(hswish<FAST>(a64[i] * H_INV), hswish<FAST>(a64[i + 1] * H_INV));
              bad |= !(h_finite(o.x) && h_finite(o.y));   // x_kj's split (lin_down's operand) out of range
              *reinterpret_cast<float2*>(P.x_down + (size_t)(e0 + row) * 64 + 8 * j + fc) = o;
            }
          }
        tp(tr, 3);
      }
    }
  }
  stagger();   // consumer 0 of a CTA without units still meets consumer 1 at the start barrier
  if (bad) atomicOr(&g_h16_overflow, 1u);
  if (probe && cw == 0) { g_h16_trace[102] = clock64(); g_h16_trace[103] = (long long)global_ns(); }
}

template <int MODE, bool TABLE = false>
static int launch_update_e_h16(const float* m, const float* x_ji, const float* e1_in, const float* rbf0,
                               const int32_t* dst, int64_t n_edges, const REParams& P, float* e1_out, float* v_in,
                               cudaStream_t st) {
  auto kfn = h16_fast_swish ? sphere_update_e_h16_kernel<true, MODE, TABLE> : sphere_update_e_h16_kernel<false, MODE, TABLE>;
  cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(RSmem));
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(%zu): %s", sizeof(RSmem), cudaGetErrorString(e));
    return DIG3D_ECUDA;
  }
  int dev = 0, n_sm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  const int units = (int)ceil_div(n_edges, R_UNIT);
  const int grid = min(n_sm, (units + 1) / 2);
  kfn<<<grid, R_THREADS, sizeof(RSmem), st>>>(m, x_ji, e1_in, rbf0, dst, (int)n_edges, P, e1_out, v_in);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

// ---------------------------------------------------------------------------------- update_v (node MLP)
// v = lin_up(v_in) ; v = act(lins[l](v)) ... ; out = lin(v)                              spherenet.py:212-215
// H = 128 -> O = 256 -> O ... -> out_channels on the register-accumulator engine's roles (producer warpgroup with the
// cp.async.bulk ring, two consumer warpgroups on 64-node units, setmaxnreg 40 / 232).  A K = 256 operand does not fit
// in registers next to an m64n256 accumulator pair, so each consumer keeps its operand in shared memory as fp16 hi / lo
// planes (64 rows x 256, wgmma with A from shared memory) and computes a 256-wide layer as two N = 128 halves: the first
// half's activated values stay in registers while the second half runs, then both become the next operand.  The
// per-element arithmetic is the store engine's (pre-scales, split, K = 64 chunks summed in order, bias / swish).  The
// final 256 -> out_channels dot product: each thread sums its 64 columns of a row in column order, the four threads of
// a row are added in a fixed butterfly order.  All blocks (init_v + update_vs) run in one launch: the units of a pair of
// consumers belong to the same block (both read the same weight slabs), pairs are dealt round-robin over the grid.
struct HVBlock {
  const unsigned char* p[9];     // packed lin_up [256 x 128], lins[l] [256 x 256] (rows 0..127 then 128..255)
  const float* b[9];             // biases [256]
  const float* w_out;            // [out_channels, 256]
};
struct HVParams { HVBlock blk[8]; int n_lins, out_channels; };

constexpr int V_STAGES = 6;                                  // K = 32 slabs in flight (N = 128)
constexpr int V_PLANE = 32 * R_UNIT * 16;                    // bytes of one fp16 plane of a [64 x 256] operand
struct VSmem {
  unsigned char a[2][2][V_PLANE];                            // [consumer][hi | lo]: [k-unit][row][8 halves]
  unsigned char w[V_STAGES][H_STAGE_BYTES];
  uint64_t full[V_STAGES], empty[V_STAGES];
};
static_assert(sizeof(VSmem) <= 227 * 1024, "VSmem exceeds the shared memory of an SM");

// chunk CH (K = 64) of an N = 128 layer half, A from the consumer's planes, slabs it + 2 CH, + 1; same product order as
// r_chunk (corrections first, the first product starts the chunk)
__device__ __forceinline__ void v_chunk(VSmem& s, uint32_t a_hi, uint32_t a_lo, int ch, float (&t)[64], int it) {
#pragma unroll
  for (int sl = 0; sl < 2; ++sl) {
    const uint32_t w_hi = smem_u32(s.w[(it + 2 * ch + sl) % V_STAGES]), w_lo = w_hi + 4u * 128 * 16u;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const uint32_t a_off = (uint32_t)((4 * ch + 2 * sl + ks) * 2 * R_UNIT * 16), b_off = (uint32_t)(ks * 2 * 128 * 16);
      const uint64_t bh = smem_desc(w_hi + b_off, 128 * 16, 128), bl = smem_desc(w_lo + b_off, 128 * 16, 128);
      mma_f16_ss(t, smem_desc(a_lo + a_off, R_UNIT * 16, 128), bh, (sl | ks) != 0);
      mma_f16_ss(t, smem_desc(a_hi + a_off, R_UNIT * 16, 128), bl, 1);
    }
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const uint32_t a_off = (uint32_t)((4 * ch + 2 * sl + ks) * 2 * R_UNIT * 16), b_off = (uint32_t)(ks * 2 * 128 * 16);
      mma_f16_ss(t, smem_desc(a_hi + a_off, R_UNIT * 16, 128), smem_desc(w_hi + b_off, 128 * 16, 128), 1);
    }
  }
}
__device__ __forceinline__ void v_wait_slabs(VSmem& s, int it, int n) {
  for (int i = 0; i < n; ++i) mbar_wait(&s.full[(it + i) % V_STAGES], ((it + i) / V_STAGES) & 1);
}
__device__ __forceinline__ void v_release(VSmem& s, int it, int n) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0)
    for (int i = 0; i < n; ++i) mbar_arrive(&s.empty[(it + i) % V_STAGES]);
}
// one N = 128 half of a layer with NCH K = 64 chunks: acc = c0, acc += c1, ... (fp32, round to nearest, in order)
__device__ __forceinline__ void v_half(VSmem& s, uint32_t a_hi, uint32_t a_lo, int nch, float (&acc)[64],
                                      float (&d)[64], int& it) {
  v_wait_slabs(s, it, 2);
  wg_fence();
  v_chunk(s, a_hi, a_lo, 0, acc, it);
  wg_commit();
  wg_wait0();
  v_release(s, it, 2);
#pragma unroll 1
  for (int ch = 1; ch < nch; ++ch) {
    v_wait_slabs(s, it + 2 * ch, 2);
    wg_fence();
    v_chunk(s, a_hi, a_lo, ch, d, it);
    wg_commit();
    wg_wait0();
    v_release(s, it + 2 * ch, 2);
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = __fadd_rn(acc[i], d[i]);
  }
  it += 2 * nch;
}
// this thread's fragment elements (x H_SA) of columns [col0, col0 + 128) -> fp16 hi / lo planes
__device__ __forceinline__ void v_store_a(unsigned char* hi, unsigned char* lo, const float (&v)[64], int col0, int fr,
                                         int fc) {
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int col = col0 + 8 * j + fc, i = 4 * j + 2 * h;
      uint32_t xh, xl;
      r_split(v[i], v[i + 1], xh, xl);
      const int o = ((col >> 3) * R_UNIT + fr + 8 * h) * 16 + (col & 7) * 2;
      *reinterpret_cast<uint32_t*>(hi + o) = xh;
      *reinterpret_cast<uint32_t*>(lo + o) = xl;
    }
}

template <bool FAST>
__global__ void __launch_bounds__(R_THREADS, 1)
sphere_update_v_h16_kernel(const float* __restrict__ v_in_all, int n_nodes, int n_blocks, HVParams P,
                           float* __restrict__ v_out_all) {
  extern __shared__ __align__(1024) unsigned char h_raw[];
  VSmem& s = *reinterpret_cast<VSmem*>(h_raw);
  const int tid = threadIdx.x, wg = tid / R_WG;
  // (values live across setmaxnreg are recomputed after it)
  auto upb = [&]() { return (n_nodes + R_UNIT - 1) / R_UNIT; };             // units per block
  auto ppb = [&]() { return (upb() + 1) / 2; };                              // unit pairs per block
  auto rounds = [&]() { return (n_blocks * ppb() - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x; };
  if (tid == 0) {
    for (int i = 0; i < V_STAGES; ++i) { mbar_init(&s.full[i], 1); mbar_init(&s.empty[i], 8); }
    mbar_fence_init();
  }
  __syncthreads();
  const int ng = P.n_lins + 1;

  if (wg == 0) {
    // ---- producer: per pair, every K = 32 slab of both N halves of every layer of the pair's block
    r_regs_producer();
    if (tid == 0) {
      int it = 0;
      const int nr = rounds(), np = ppb();
      const uint32_t bytes = 2u * 4u * 128u * 16u;
      for (int k = 0; k < nr; ++k) {
        const HVBlock& B = P.blk[(blockIdx.x + k * gridDim.x) / np];
        for (int q = 0; q < ng; ++q) {
          const int K = q ? 256 : 128;
          for (int t = 0; t < 2; ++t)
            for (int c = 0; c < K / H_SLAB_K; ++c, ++it) {
              const int st = it % V_STAGES;
              if (it >= V_STAGES) mbar_wait(&s.empty[st], ((it / V_STAGES) + 1) & 1);
              mbar_arrive_expect_tx(&s.full[st], bytes);
              bulk_g2s(s.w[st], B.p[q] + (size_t)t * K * 128 * 4 + (size_t)c * bytes, bytes, &s.full[st]);
            }
        }
      }
    }
    return;
  }

  // ---- consumers
  r_regs_consumer();
  const int cw = threadIdx.x / R_WG - 1, wt = threadIdx.x & (R_WG - 1);
  const int fr = frag_row(wt), fc = frag_col(wt), C = P.out_channels;
  const int nr = rounds(), np = ppb(), nu = upb();
  unsigned char *ahi = s.a[cw][0], *alo = s.a[cw][1];
  const uint32_t a_hi = smem_u32(ahi), a_lo = smem_u32(alo);
  int slabs = 2 * 128 / H_SLAB_K + 2 * (ng - 1) * 256 / H_SLAB_K;
  bool staggered = cw == 1, bad = false;
  auto stagger = [&]() {
    if (!staggered) { asm volatile("bar.arrive 3, %0;" ::"n"(2 * R_WG) : "memory"); staggered = true; }
  };
  if (cw == 1) asm volatile("bar.sync 3, %0;" ::"n"(2 * R_WG) : "memory");   // after consumer 0's first half is issued
  int it = 0;
#pragma unroll 1
  for (int k = 0; k < nr; ++k) {
    const int pair = blockIdx.x + k * gridDim.x, blk = pair / np, unit = 2 * (pair % np) + cw;
    if (unit >= nu) {   // passes every slab of the round (the ring counts both consumers per stage)
      for (int i = 0; i < slabs; ++i, ++it) {
        mbar_wait(&s.full[it % V_STAGES], (it / V_STAGES) & 1);
        v_release(s, it, 1);
      }
      continue;
    }
    const HVBlock& B = P.blk[blk];
    const int r0 = unit * R_UNIT, rows = min(R_UNIT, n_nodes - r0);
    const float* vin = v_in_all + ((size_t)blk * n_nodes + r0) * 128;
    float h0[64], acc[64], d[64];
    r_bar(cw);   // the previous unit's MMAs have read the planes
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = fr + 8 * h, i = 4 * j + 2 * h;
        const float2 x = row < rows ? __ldg(reinterpret_cast<const float2*>(vin + (size_t)row * 128 + 8 * j + fc))
                                    : make_float2(0.f, 0.f);
        acc[i] = x.x * H_SA;
        acc[i + 1] = x.y * H_SA;
      }
    v_store_a(ahi, alo, acc, 0, fr, fc);                                 // A0 = v_in (K = 128)
#pragma unroll 1
    for (int q = 0; q < ng; ++q) {
      fence_async_smem();
      r_bar(cw);                                                           // the operand is complete
      const int nch = q ? 4 : 2;
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        float* v = t ? acc : h0;
        v_half(s, a_hi, a_lo, nch, acc, d, it);
        if (t == 0) stagger();
        // v8 = H_SA * (acc / (H_SA H_SW) + b) ; layers >= 1 apply the activation
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const float b = H_SA * __ldg(B.b[q] + 128 * t + 8 * j + fc + u);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int i = 4 * j + 2 * h + u;
              const float x = fmaf(acc[i], H_SA * H_INV, b);
              v[i] = q > 0 ? hswish8<FAST>(x) : x;
            }
          }
      }
      if (q + 1 < ng) {
        r_bar(cw);                                                         // every MMA of the layer has completed
        v_store_a(ahi, alo, h0, 0, fr, fc);
        v_store_a(ahi, alo, acc, 128, fr, fc);
      }
    }
    // out[row][o] = sum_c v[row][c] * w_out[o][c]: this thread's 64 columns of each of its two rows in column order,
    // then the four threads of the row in a fixed order
    for (int o = 0; o < C; ++o) {
      float part[2] = {0.f, 0.f};
#pragma unroll
      for (int t = 0; t < 2; ++t)
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const float w = __ldg(B.w_out + o * 256 + 128 * t + 8 * j + fc + u);
#pragma unroll
            for (int h = 0; h < 2; ++h) part[h] = fmaf(t ? acc[4 * j + 2 * h + u] : h0[4 * j + 2 * h + u], w, part[h]);
          }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        part[h] += __shfl_xor_sync(0xffffffffu, part[h], 1);
        part[h] += __shfl_xor_sync(0xffffffffu, part[h], 2);
        const float y = part[h] * (1.0f / H_SA);
        bad |= !h_finite(y);
        const int row = fr + 8 * h;
        if ((wt & 3) == 0 && row < rows) v_out_all[((size_t)blk * n_nodes + r0 + row) * C + o] = y;
      }
    }
  }
  stagger();   // consumer 0 of a CTA without units still meets consumer 1 at the start barrier
  if (bad) atomicOr(&g_h16_overflow, 1u);
}

// ---------------------------------------------------------------------------------- generic linear (training path)
// y[rows, ldy-strided N columns] = x[rows, K] W^T + bias (+ act_out = swish(y)) on the two-tile engine: K as NPANEL
// panels of K4*8 columns whose operand tile is rebuilt between panels (the chunk sums keep accumulating in the
// epilogue registers), N = 128 or 64 output columns per launch (a wider layer is launched once per 128-column slice).
struct HLinParams { HGemm g[3]; };

template <int NPANEL, int KU, int N>
__global__ void __launch_bounds__(H_THREADS, 1)
linear_h16_kernel(const float* __restrict__ x, int n_rows, int ldx, HLinParams P, const float* __restrict__ bias,
                  float* __restrict__ y, float* __restrict__ act_out, const float* __restrict__ residual, int ldy,
                  int tiles_per_cta, int slice_bytes) {
  extern __shared__ __align__(1024) unsigned char h_raw[];
  HSmem& s = *reinterpret_cast<HSmem*>(h_raw);
  constexpr int NC = N / 2;                                // columns per epilogue thread
  const int tid = threadIdx.x, warp = tid >> 5;
  // blockIdx.y = 128-column slice of a wider layer (all slices of one launch are N wide): its packed weights follow the
  // previous slice's, its bias / output columns start at N * slice.  Small row counts run ONE tile per CTA so that the
  // launch spreads over more SMs (a 4.7 k-row, 256-wide layer is 74 CTAs instead of 19 in two serial launches).
  {
    const int slice = blockIdx.y;
#pragma unroll
    for (int p = 0; p < NPANEL; ++p) P.g[p].w += (size_t)slice * slice_bytes;
    if (bias) bias += slice * N;
    if (y) y += slice * N;
    if (act_out) act_out += slice * N;
    if (residual) residual += slice * N;
  }
  const int n_tiles = (n_rows + H_M - 1) / H_M, tile0 = blockIdx.x * tiles_per_cta;
  const int ntile = min(tiles_per_cta, n_tiles - tile0);
  h_setup(s);
  for (int i = tid; i < N; i += H_THREADS) s.bias[0][i] = bias ? __ldg(bias + i) : 0.f;
  tc_fence_before();
  __syncthreads();
  tc_fence_after();
  HCtx c;
  bool epi = false;
  if (warp < H_CTRL_WARPS) {
    h_regs_ctrl();
    h_mma_n(s, P.g, NPANEL, ntile, s.tmem_base);
  } else if (h_regs_epi(), (c = h_ctx(s, ntile)).t < ntile) {
    epi = true;
    const int r0 = (tile0 + c.t) * H_M, rows = min(H_M, n_rows - r0);
    const int col0 = c.half * NC;
    float acc[NC];
#pragma unroll
    for (int p = 0; p < NPANEL; ++p) {
      h_load_tile<KU>(s, c, x + (size_t)r0 * ldx + p * (KU * 8), ldx, rows);
      h_epi_done(s, c.t);
      if (p == 0) h_drain<NC / 16, true>(s, c, col0, KU / 8, acc);
      else h_drain<NC / 16, false>(s, c, col0, KU / 8, acc);
    }
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      acc[i] = fmaf(acc[i], H_INV, s.bias[0][col0 + i]);
      c.bad |= !h_finite(acc[i]);   // an element of x beyond the split's range poisons its row
    }
    // outputs: y = x W^T + b (nullable) and / or act_out = swish(y); `residual` is added to the LAST of them (the skip
    // connection of a residual layer, or the second GEMM of a sum of two linears), y stays the pre-activation
    const float* res = residual ? residual + (size_t)r0 * ldy : nullptr;
    if (y) h_store_tile_strided<N>(s, c, col0, acc, y + (size_t)r0 * ldy, ldy, rows, act_out ? nullptr : res);
    if (act_out) {
#pragma unroll
      for (int i = 0; i < NC; ++i) acc[i] = hswish<false>(acc[i]);
      if (y) h_tile_bar(c.t);
      h_store_tile_strided<N>(s, c, col0, acc, act_out + (size_t)r0 * ldy, ldy, rows, res);
    }
  }
  h_finish(s, epi ? &c : nullptr);
}

static int h_smem_attr(const void* fn);
template <int NPANEL, int KU, int N>
static int launch_linear_h16(const float* x, int64_t rows, int ldx, const unsigned char* packed, const float* bias,
                             float* y, float* act_out, const float* residual, int ldy, int slices, cudaStream_t st) {
  HLinParams P;
  const size_t panel = (size_t)(KU / 4) * 2 * 4 * N * 16;      // KU/4 slabs of [hi|lo][4][N][8 halves]
  for (int p = 0; p < NPANEL; ++p) P.g[p] = {packed + p * panel, nullptr, KU * 8, N};
  auto kfn = linear_h16_kernel<NPANEL, KU, N>;
  int rc = h_smem_attr((const void*)kfn);
  if (rc) return rc;
  int dev = 0, n_sm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  const int tiles = ceil_div(rows, H_M);
  const int tpc = (ceil_div(tiles, 2) * slices < n_sm) ? 1 : 2;        // below one wave of tile pairs: one tile per CTA
  dim3 grid(ceil_div(tiles, tpc), slices);
  kfn<<<grid, H_THREADS, sizeof(HSmem), st>>>(x, (int)rows, ldx, P, bias, y, act_out, residual, ldy, tpc,
                                              4 * N * (NPANEL * KU * 8));
  return DIG3D_OK;
}

static int h_smem_attr(const void* fn) {
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HSmem));
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(%zu): %s", sizeof(HSmem), cudaGetErrorString(e));
    return DIG3D_ECUDA;
  }
  return DIG3D_OK;
}

}  // namespace dig3d

using namespace dig3d;

extern "C" {

static int h16_pack_impl(const float* const* weights, const int32_t* n, const int32_t* k, const int32_t* trans,
                         void* const* outs, int32_t count, void* stream) {
  DIG3D_REQUIRE(weights && n && k && outs && count >= 1 && count <= 16, "h16_pack: bad arguments");
  HPackJobs jobs;
  int max_total = 0;
  for (int i = 0; i < count; ++i) {
    DIG3D_REQUIRE(weights[i] && outs[i] && k[i] % 64 == 0 && n[i] % 8 == 0 && n[i] <= 128,
                  "h16_pack: matrix %d has N=%d K=%d (need K %% 64 == 0, N %% 8 == 0, N <= 128)", i, n[i], k[i]);
    jobs.job[i] = {weights[i], (unsigned char*)outs[i], n[i], k[i], trans ? trans[i] : 0};
    max_total = max_total > n[i] * k[i] ? max_total : n[i] * k[i];
  }
  dim3 grid(ceil_div(max_total, 256), count);
  h16_pack_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(jobs);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_h16_pack(const float* const* weights, const int32_t* n, const int32_t* k, void* const* outs, int32_t count,
                   void* stream) {
  return h16_pack_impl(weights, n, k, nullptr, outs, count, stream);
}

int dig3d_h16_pack_t(const float* const* weights, const int32_t* n, const int32_t* k, const int32_t* trans,
                     void* const* outs, int32_t count, void* stream) {
  DIG3D_REQUIRE(trans, "h16_pack_t: null pointer");
  return h16_pack_impl(weights, n, k, trans, outs, count, stream);
}

int dig3d_h16_set_fast_swish(int32_t on) {
  h16_fast_swish = on ? 1 : 0;
  return DIG3D_OK;
}

int dig3d_h16_overflow(int32_t clear) {
  unsigned int v = 0;
  cudaMemcpyFromSymbol(&v, g_h16_overflow, sizeof(v));
  if (clear && v) {
    unsigned int zero = 0;
    cudaMemcpyToSymbol(g_h16_overflow, &zero, sizeof(zero));
  }
  return (int)v;
}

int dig3d_h16_trace(int32_t on, long long* out128 /* host, 128 entries, nullable */) {
  if (out128) cudaMemcpyFromSymbol(out128, g_h16_trace, sizeof(long long) * 128);
  int v = on ? 1 : 0;
  cudaMemcpyToSymbol(g_h16_trace_on, &v, sizeof(v));
  return DIG3D_OK;
}

int dig3d_h16_timeouts(void) {
  unsigned int v = 0;
  cudaMemcpyFromSymbol(&v, tc90::g_mbar_timeout, sizeof(v));
  return (int)v;
}

// init_e on the register engine: tab_i / tab_j null = the three-panel form (packed = lin.weight [128, 384]), else the
// table form (packed = its rbf panel W[:, 256:384])
static void init_e_params(REParams& P, const int64_t* z, const int32_t* src, const dig3d_init_e_weights* w,
                          const void* packed, const float* tab_i, const float* tab_j) {
  P.g[0] = {(const unsigned char*)packed, nullptr, tab_i ? 128 : 384, 128};
  P.w_rbf = w->w_rbf1;
  P.z = z; P.src = src;
  P.emb = w->emb; P.w_rbf0 = w->w_rbf0; P.b_rbf0 = w->b_rbf0; P.b_lin = w->b_lin;
  P.tab_i = tab_i; P.tab_j = tab_j;
}

int dig3d_sphere_init_e_h16(const int64_t* z, const int32_t* src, const int32_t* dst, const float* rbf0,
                            int64_t n_edges, const dig3d_init_e_weights* w, const void* packed_lin, float* e1,
                            float* v_in, void* stream) {
  DIG3D_REQUIRE(z && src && dst && rbf0 && w && packed_lin && e1 && v_in, "sphere_init_e_h16: null pointer");
  DIG3D_REQUIRE(w->emb && w->w_rbf0 && w->b_rbf0 && w->b_lin && w->w_rbf1, "sphere_init_e_h16: null weight");
  if (n_edges == 0) return DIG3D_OK;
  REParams P = {};
  init_e_params(P, z, src, w, packed_lin, nullptr, nullptr);
  return launch_update_e_h16<RE_I, false>(nullptr, nullptr, nullptr, rbf0, dst, n_edges, P, e1, v_in,
                                          (cudaStream_t)stream);
}

int dig3d_sphere_init_e_h16_tab(const int64_t* z, const int32_t* src, const int32_t* dst, const float* rbf0,
                                int64_t n_edges, const dig3d_init_e_weights* w, const void* packed_rbf_panel,
                                const float* tab_i, const float* tab_j, float* e1, float* v_in, void* stream) {
  DIG3D_REQUIRE(z && src && dst && rbf0 && w && packed_rbf_panel && tab_i && tab_j && e1 && v_in,
                "sphere_init_e_h16_tab: null pointer");
  DIG3D_REQUIRE(w->w_rbf0 && w->b_rbf0 && w->b_lin && w->w_rbf1, "sphere_init_e_h16_tab: null weight");
  DIG3D_REQUIRE((((uintptr_t)tab_i | (uintptr_t)tab_j) & 15) == 0, "sphere_init_e_h16_tab: tables must be 16-byte aligned");
  if (n_edges == 0) return DIG3D_OK;
  REParams P = {};
  init_e_params(P, z, src, w, packed_rbf_panel, tab_i, tab_j);
  return launch_update_e_h16<RE_I, true>(nullptr, nullptr, nullptr, rbf0, dst, n_edges, P, e1, v_in,
                                         (cudaStream_t)stream);
}

int dig3d_sphere_init_update_e_a_h16(const int64_t* z, const int32_t* src, const int32_t* dst, const float* rbf0,
                                     int64_t n_edges, const dig3d_init_e_weights* w_init, const void* packed_init,
                                     const float* tab_i, const float* tab_j, const dig3d_tc_update_e* w, float* e1,
                                     float* v_in, float* x_ji, float* x_down, void* stream) {
  DIG3D_REQUIRE(z && src && dst && rbf0 && w_init && packed_init && w && e1 && v_in && x_ji && x_down,
                "sphere_init_update_e_a_h16: null pointer");
  DIG3D_REQUIRE(w_init->w_rbf0 && w_init->b_rbf0 && w_init->b_lin && w_init->w_rbf1 && (tab_i || w_init->emb),
                "sphere_init_update_e_a_h16: null weight");
  DIG3D_REQUIRE(!tab_i == !tab_j, "sphere_init_update_e_a_h16: tab_i and tab_j must agree");
  DIG3D_REQUIRE((((uintptr_t)tab_i | (uintptr_t)tab_j) & 15) == 0,
                "sphere_init_update_e_a_h16: tables must be 16-byte aligned");
  if (n_edges == 0) return DIG3D_OK;
  REParams P = {};
  init_e_params(P, z, src, w_init, packed_init, tab_i, tab_j);
  P.g[1] = {(const unsigned char*)w->p_ji, w->b_ji, 128, 128};
  P.g[2] = {(const unsigned char*)w->p_kj, w->b_kj, 128, 128};
  P.g[3] = {(const unsigned char*)w->p_down, nullptr, 128, 64};
  P.w_rbf1 = w->w_rbf1; P.w_rbf2 = w->w_rbf2;
  P.x_ji = x_ji; P.x_down = x_down;
  cudaStream_t st = (cudaStream_t)stream;
  return tab_i ? launch_update_e_h16<RE_IA, true>(nullptr, nullptr, nullptr, rbf0, dst, n_edges, P, e1, v_in, st)
               : launch_update_e_h16<RE_IA, false>(nullptr, nullptr, nullptr, rbf0, dst, n_edges, P, e1, v_in, st);
}

int dig3d_sphere_update_e_a_h16(const float* e1, const float* rbf0, int64_t n_edges, const dig3d_tc_update_e* w,
                                float* x_ji, float* x_down, void* stream) {
  DIG3D_REQUIRE(e1 && rbf0 && w && x_ji && x_down, "sphere_update_e_a_h16: null pointer");
  if (n_edges == 0) return DIG3D_OK;
  REParams P = {};
  P.g[0] = {(const unsigned char*)w->p_ji, w->b_ji, 128, 128};
  P.g[1] = {(const unsigned char*)w->p_kj, w->b_kj, 128, 128};
  P.g[2] = {(const unsigned char*)w->p_down, nullptr, 128, 64};
  P.w_rbf1 = w->w_rbf1; P.w_rbf2 = w->w_rbf2;
  P.x_ji = x_ji; P.x_down = x_down;
  return launch_update_e_h16<RE_A>(nullptr, nullptr, e1, rbf0, nullptr, n_edges, P, nullptr, nullptr,
                                   (cudaStream_t)stream);
}

static void update_e_b_params(REParams& P, const dig3d_tc_update_e* w) {
  P.g[0] = {(const unsigned char*)w->p_up, nullptr, 64, 128};
  for (int i = 0; i < 2; ++i) P.g[1 + i] = {(const unsigned char*)w->p_res[i], w->b_res[i], 128, 128};
  P.g[3] = {(const unsigned char*)w->p_lin, w->b_lin, 128, 128};
  for (int i = 2; i < 6; ++i) P.g[2 + i] = {(const unsigned char*)w->p_res[i], w->b_res[i], 128, 128};
  P.w_rbf = w->w_rbf;
}

int dig3d_sphere_update_e_b_h16(const float* m, const float* e1_in, const float* x_ji, const float* rbf0,
                                const int32_t* dst, int64_t n_edges, const dig3d_tc_update_e* w, float* e1_out,
                                float* v_in, void* stream) {
  DIG3D_REQUIRE(m && e1_in && x_ji && rbf0 && dst && w && e1_out && v_in, "sphere_update_e_b_h16: null pointer");
  if (n_edges == 0) return DIG3D_OK;
  REParams P = {};
  update_e_b_params(P, w);
  return launch_update_e_h16<RE_B>(m, x_ji, e1_in, rbf0, dst, n_edges, P, e1_out, v_in, (cudaStream_t)stream);
}

int dig3d_sphere_update_e_ba_h16(const float* m, const float* e1_in, const float* x_ji, const float* rbf0,
                                 const int32_t* dst, int64_t n_edges, const dig3d_tc_update_e* w,
                                 const dig3d_tc_update_e* w_next, float* e1_out, float* v_in, float* x_ji_next,
                                 float* x_down_next, void* stream) {
  DIG3D_REQUIRE(m && e1_in && x_ji && rbf0 && dst && w && w_next && e1_out && v_in && x_ji_next && x_down_next,
                "sphere_update_e_ba_h16: null pointer");
  DIG3D_REQUIRE(x_ji_next != x_ji, "sphere_update_e_ba_h16: x_ji_next must not alias x_ji (other units still read it)");
  if (n_edges == 0) return DIG3D_OK;
  REParams P = {};
  update_e_b_params(P, w);
  P.g[8] = {(const unsigned char*)w_next->p_ji, w_next->b_ji, 128, 128};
  P.g[9] = {(const unsigned char*)w_next->p_kj, w_next->b_kj, 128, 128};
  P.g[10] = {(const unsigned char*)w_next->p_down, nullptr, 128, 64};
  P.w_rbf1 = w_next->w_rbf1; P.w_rbf2 = w_next->w_rbf2;
  P.x_ji = x_ji_next; P.x_down = x_down_next;
  return launch_update_e_h16<RE_BA>(m, x_ji, e1_in, rbf0, dst, n_edges, P, e1_out, v_in, (cudaStream_t)stream);
}

int dig3d_linear_h16_supported(int32_t k, int32_t nout) {
  return ((k == 64 || k == 128 || k == 256 || k == 384) && nout >= 64 && nout % 64 == 0 && nout <= 512) ? 1 : 0;
}

/* y = x W^T + bias (+ act_out = swish(y)); packed = dig3d_h16_pack(_t) of W as consecutive [min(128, N - c), K] row
 * slices (one per 128 output columns; a trailing 64-column slice is allowed). */
int dig3d_linear_h16(const float* x, int64_t rows, int32_t k, int32_t nout, const void* packed, const float* bias,
                     float* y, float* act_out, const float* residual, void* stream) {
  DIG3D_REQUIRE(x && packed && (y || act_out), "linear_h16: null pointer");
  DIG3D_REQUIRE(dig3d_linear_h16_supported(k, nout), "linear_h16: shape %d -> %d is not compiled", k, nout);
  DIG3D_REQUIRE((((uintptr_t)x | (uintptr_t)y | (uintptr_t)act_out | (uintptr_t)residual) & 15) == 0,
                "linear_h16: 16-byte alignment");
  if (rows == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned char* pw = (const unsigned char*)packed;
  // all full 128-column slices in ONE launch (gridDim.y); a trailing 64-column slice gets its own
  for (int c0 = 0; c0 < nout;) {
    const int n = nout - c0 >= 128 ? 128 : 64;
    const int slices = n == 128 ? (nout - c0) / 128 : 1;
    const float* b = bias ? bias + c0 : nullptr;
    float* yo = y ? y + c0 : nullptr;
    float* ao = act_out ? act_out + c0 : nullptr;
    const float* ro = residual ? residual + c0 : nullptr;
    int rc;
#define DIG3D_LIN(NP, KU)                                                                                             \
    (n == 128 ? launch_linear_h16<NP, KU, 128>(x, rows, k, pw, b, yo, ao, ro, nout, slices, st)                        \
              : launch_linear_h16<NP, KU, 64>(x, rows, k, pw, b, yo, ao, ro, nout, slices, st))
    if (k == 64) rc = DIG3D_LIN(1, 8);
    else if (k == 128) rc = DIG3D_LIN(1, 16);
    else if (k == 256) rc = DIG3D_LIN(2, 16);
    else rc = DIG3D_LIN(3, 16);
#undef DIG3D_LIN
    if (rc) return rc;
    pw += (size_t)4 * n * k * slices;
    c0 += n * slices;
  }
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_sphere_update_v_h16_supported(int32_t hidden, int32_t out_emb, int32_t out_channels, int32_t n_lins) {
  return (hidden == 128 && out_emb == 256 && out_channels >= 1 && out_channels <= 4 && n_lins >= 0 && n_lins <= 8) ? 1 : 0;
}

int dig3d_sphere_update_v_h16(const float* v_in_all, int64_t n_nodes, int32_t n_blocks, int32_t out_channels,
                              int32_t n_lins, const void* const* packed /* [n_blocks][n_lins + 1] */,
                              const dig3d_update_v_weights* w, float* v_out_all, void* stream) {
  DIG3D_REQUIRE(v_in_all && packed && w && v_out_all, "sphere_update_v_h16: null pointer");
  DIG3D_REQUIRE(n_blocks >= 1 && n_blocks <= 8, "sphere_update_v_h16: n_blocks=%d outside [1,8]", n_blocks);
  DIG3D_REQUIRE(dig3d_sphere_update_v_h16_supported(128, 256, out_channels, n_lins),
                "sphere_update_v_h16: out_channels=%d / n_lins=%d not compiled", out_channels, n_lins);
  if (n_nodes == 0) return DIG3D_OK;
  HVParams P;
  P.n_lins = n_lins; P.out_channels = out_channels;
  for (int b = 0; b < n_blocks; ++b) {
    DIG3D_REQUIRE(w[b].n_lins == n_lins && w[b].w_out && w[b].b_up, "sphere_update_v_h16: block %d weights", b);
    for (int l = 0; l <= n_lins; ++l) {
      P.blk[b].p[l] = (const unsigned char*)packed[b * (n_lins + 1) + l];
      P.blk[b].b[l] = l == 0 ? w[b].b_up : w[b].b_lins[l - 1];
      DIG3D_REQUIRE(P.blk[b].p[l] && P.blk[b].b[l], "sphere_update_v_h16: block %d layer %d null", b, l);
    }
    P.blk[b].w_out = w[b].w_out;
  }
  auto kfn = h16_fast_swish ? sphere_update_v_h16_kernel<true> : sphere_update_v_h16_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(VSmem));
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(%zu): %s", sizeof(VSmem), cudaGetErrorString(e));
    return DIG3D_ECUDA;
  }
  int dev = 0, n_sm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  const int pairs = n_blocks * (int)ceil_div(ceil_div(n_nodes, R_UNIT), 2);
  kfn<<<min(n_sm, pairs), R_THREADS, sizeof(VSmem), (cudaStream_t)stream>>>(v_in_all, (int)n_nodes, n_blocks, P,
                                                                             v_out_all);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
