// Hopper (sm_90a) tensor-core layer of the dense-chain kernels: mbarrier, bulk copy (TMA engine), wgmma, and the
// accumulator store the epilogues read (no CUTLASS dependency).
//
// Conventions used by the dense-chain kernels:
//   * operands are K-major, NO swizzle, in the canonical "interleaved" layout: a [rows x K] operand tile is stored
//     as [K-units][rows][16 bytes] (a k-unit is 4 tf32 or 8 fp16 values), so the 8-row x 16-byte core matrices are
//     contiguous (128 B): SBO = 128 B (next 8 rows), LBO = the byte stride of one k-unit plane (next K elements);
//   * one warpgroup (4 warps, 128 threads) issues the wgmma.mma_async instructions of a 128-row tile as two
//     m64 halves and n64 column blocks, accumulating ONE K-chunk in registers (scale-d = 0 on its first product);
//   * in the store-engine dense chains (init_e, update_v, the generic linear, the 3xTF32 chain) the finished chunk goes
//     to the accumulator store: a slot of 128 rows x up to 512 fp32 columns in global memory (L2-resident) that the CTA
//     claims for its lifetime, addressed like tensor memory by (row << 16 | column).  The epilogue warps read whole
//     16-column row pieces of it (thread = row) while the warpgroup works on the next chunk, and the ready / free
//     handshakes are mbarriers.  Kernels whose epilogue works on the fragment layout directly (update_e's register
//     engine, triplet gather, weight gradient) keep their accumulators in registers; update_e also takes its A operand
//     from registers (mma_f16_rs).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tc90 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Bounded spin: a protocol bug must not hang the GPU.  After ~2 s without progress the wait records the event
// in g_mbar_timeout and TRAPS: the launch fails with a sticky CUDA error that the next host call reports
// (a kernel that carried on after a missed barrier would hand back garbage silently).
static __device__ unsigned int g_mbar_timeout = 0;   // one copy per translation unit
__device__ __forceinline__ uint64_t global_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ bool mbar_try(uint32_t addr, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(addr), "r"(parity)
      : "memory");
  return ok != 0;
}
static __device__ __noinline__ void mbar_timeout_trap() {
  atomicAdd(&g_mbar_timeout, 1u);
  __threadfence_system();
  __trap();
}
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  if (mbar_try(addr, parity)) return true;
  const uint64_t t0 = global_ns();
  for (;;) {
#pragma unroll 1
    for (int spin = 0; spin < 4096; ++spin)
      if (mbar_try(addr, parity)) return true;
    if (global_ns() - t0 > 2000000000ull) break;
  }
  mbar_timeout_trap();
  return false;
}

// ---- proxies / fences
// Generic-proxy shared-memory writes (operand planes) -> visible to wgmma (async proxy).
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// Ordering of the accumulator store around the mbarrier handshakes (CTA scope).
__device__ __forceinline__ void tc_fence_before() { asm volatile("fence.acq_rel.cta;" ::: "memory"); }
__device__ __forceinline__ void tc_fence_after() { asm volatile("fence.acq_rel.cta;" ::: "memory"); }

// ---- 1-D bulk copy global -> shared, completion on an mbarrier (TMA engine, no tensor map)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- named barrier of one issuing warpgroup (ids 1..2 belong to the epilogue tiles of the dense chains)
__device__ __forceinline__ void wg_bar(int id = 15) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// ---- wgmma
// K-major, no-swizzle shared-memory matrix descriptor (layout type 0).
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);            // start address, bits [0,14)
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;   // leading byte offset (next k-unit), bits [16,30)
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;   // stride byte offset (next 8 rows), bits [32,46)
  return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define TC90_D32 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15," \
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}"
#define TC90_D32_OPS(d)                                                                                          \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),   \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),    \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),   \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, fp16 operands, fp32 accumulate; accumulate = 0 overwrites D.
__device__ __forceinline__ void mma_f16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " TC90_D32 ", %32, %33, p, 1, 1, 0, 0;\n\t}"
      : TC90_D32_OPS(d)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate)
      : "memory");
}
// Same with tf32 operands (K = 8 per instruction).
__device__ __forceinline__ void mma_tf32(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " TC90_D32 ", %32, %33, p, 1, 1;\n\t}"
      : TC90_D32_OPS(d)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate)
      : "memory");
}
// Register fragment of an m64n64 accumulator: thread t of the warpgroup holds rows 16 (t/32) + (t%32)/4 (+8) and
// columns 8 j + 2 (t%4) (+1), j = 0..7: d[4j], d[4j+1] on the first row, d[4j+2], d[4j+3] on the second.  An m64n128
// accumulator continues the same pattern with j = 0..15.
__device__ __forceinline__ int frag_row(int wt) { return 16 * (wt >> 5) + ((wt & 31) >> 2); }
__device__ __forceinline__ int frag_col(int wt) { return 2 * (wt & 3); }

// ---- wgmma with A from registers
// The A operand of m64nNk16 (fp16) held in registers: thread t owns four 32-bit registers per k-step, each an fp16 pair
// of consecutive columns (lower column in the low half): a[0] = row frag_row(t), columns 2 (t%4) (+1); a[1] = row + 8,
// same columns; a[2] / a[3] = the same rows at columns + 8.  These are exactly the rows and columns of accumulator
// entries d[8 s + 2 r], d[8 s + 2 r + 1] of an m64nN fragment for k-step s (columns 16 s .. 16 s + 15): a layer's
// accumulator becomes the next layer's A operand without leaving the thread.
__device__ __forceinline__ constexpr int frag_a_src(int s, int r) { return 8 * s + 2 * r; }
// Row / column of register r of k-step s in the A operand (first column of its pair).
__device__ __forceinline__ int frag_a_row(int wt, int r) { return frag_row(wt) + 8 * (r & 1); }
__device__ __forceinline__ int frag_a_col(int wt, int s, int r) { return 16 * s + 8 * (r >> 1) + frag_col(wt); }

#define TC90_D64 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"                                          \
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"                                  \
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"                                  \
                 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}"
#define TC90_D64_OPS(d)                                                                                          \
  TC90_D32_OPS(d), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]),    \
      "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]),    \
      "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),    \
      "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]),    \
      "+f"(d[63])

// D[64 x 64] (+)= A[64 x 16] (registers) * B[64 x 16]^T (shared memory), fp16 operands, fp32 accumulate.
__device__ __forceinline__ void mma_f16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " TC90_D32 ", {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n\t}"
      : TC90_D32_OPS(d)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
      : "memory");
}
// D[64 x 128] (+)= A[64 x 16] (registers) * B[128 x 16]^T (shared memory).
__device__ __forceinline__ void mma_f16_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " TC90_D64 ", {%64,%65,%66,%67}, %68, p, 1, 1, 0;\n\t}"
      : TC90_D64_OPS(d)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
      : "memory");
}

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, both from shared memory.
__device__ __forceinline__ void mma_f16_ss(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " TC90_D64 ", %64, %65, p, 1, 1, 0, 0;\n\t}"
      : TC90_D64_OPS(d)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate)
      : "memory");
}

// ---- accumulator store (see the header comment)
// A translation unit that uses the store defines TC90_TM_COLS (columns per slot) before including this header.  The
// store is static device memory of the library (TM_SLOTS slots of 128 rows x TC90_TM_COLS fp32), so no host-side
// allocation or binding exists.  A CTA takes a free slot in tmem_alloc (atomic claim) and gives it back in
// tmem_dealloc; the slot index travels in bits [23, 32) of every address derived from the holder, so a CTA keeps its
// own slot for its whole lifetime wherever it is scheduled.  The slot count covers every SM of a Hopper part with
// one store-using CTA per SM (each such kernel asserts that two of its CTAs do not fit an SM), so a claim does not
// wait; were the pool ever exhausted, a claim waits for a resident CTA to finish.
#ifdef TC90_TM_COLS
constexpr int TM_COLS = TC90_TM_COLS;
constexpr int TM_SLOTS = 144;                 // SMs of a full GH100
constexpr int TM_SLOT_SHIFT = 23;             // address = slot << 23 | row << 16 | column
static __device__ float g_tm_store[(size_t)TM_SLOTS * 128 * TM_COLS];
static __device__ unsigned int g_tm_owner[TM_SLOTS];
// Half the shared memory of an H100 SM (228 KB) plus the 1 KB the runtime reserves per CTA: a kernel whose
// shared-memory block is larger has at most one resident CTA per SM.
constexpr size_t TM_ONE_CTA_PER_SM_SMEM = 114 * 1024;

__device__ __forceinline__ float* tm_ptr(uint32_t taddr, int lane_add) {
  const uint32_t slot = taddr >> TM_SLOT_SHIFT, row = ((taddr >> 16) & 127u) + (uint32_t)lane_add;
  return g_tm_store + ((size_t)slot * 128 + row) * TM_COLS + (taddr & 0xFFFFu);
}
// One full warp executes these (as with tensor memory); lane 0 claims / releases the slot.  tmem_dealloc follows a
// CTA-wide barrier after the last access to the slot.
__device__ __forceinline__ void tmem_alloc(uint32_t* smem_holder, uint32_t) {
  if ((threadIdx.x & 31) == 0) {
    uint32_t sm;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));   // only where the search starts: an uncontended first probe
    const uint64_t t0 = global_ns();
    for (uint32_t i = sm;; ++i) {
      const uint32_t slot = i % TM_SLOTS;
      if (atomicCAS(&g_tm_owner[slot], 0u, 1u) == 0u) {
        __threadfence();
        *smem_holder = slot << TM_SLOT_SHIFT;
        break;
      }
      if ((i & 1023) == 1023 && global_ns() - t0 > 2000000000ull) mbar_timeout_trap();
    }
  }
  __syncwarp();
}
__device__ __forceinline__ void tmem_dealloc(uint32_t taddr, uint32_t) {
  if ((threadIdx.x & 31) == 0) {
    __threadfence();
    atomicExch(&g_tm_owner[taddr >> TM_SLOT_SHIFT], 0u);
  }
  __syncwarp();
}
// Each thread of a warp reads / writes 16 consecutive columns of row ((taddr >> 16) & 127) + laneid.
__device__ __forceinline__ void tmem_ld16(uint32_t taddr, uint32_t (&r)[16]) {
  const float4* p = reinterpret_cast<const float4*>(tm_ptr(taddr, threadIdx.x & 31));
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 v = __ldcg(p + i);
    r[4 * i] = __float_as_uint(v.x); r[4 * i + 1] = __float_as_uint(v.y);
    r[4 * i + 2] = __float_as_uint(v.z); r[4 * i + 3] = __float_as_uint(v.w);
  }
}
__device__ __forceinline__ void tmem_ld16f(uint32_t taddr, float* r) {
  const float4* p = reinterpret_cast<const float4*>(tm_ptr(taddr, threadIdx.x & 31));
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 v = __ldcg(p + i);
    r[4 * i] = v.x; r[4 * i + 1] = v.y; r[4 * i + 2] = v.z; r[4 * i + 3] = v.w;
  }
}
__device__ __forceinline__ void tmem_ld_wait() {}

// Warpgroup (thread wt = 0..127) writes its m64n64 fragment to the 64 x 64 block whose top-left corner is taddr.
__device__ __forceinline__ void tm_store_frag(const float (&d)[32], int wt, uint32_t taddr) {
  float* base = tm_ptr(taddr, frag_row(wt)) + frag_col(wt);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    __stcg(reinterpret_cast<float2*>(base + 8 * j), make_float2(d[4 * j], d[4 * j + 1]));
    __stcg(reinterpret_cast<float2*>(base + 8 * TM_COLS + 8 * j), make_float2(d[4 * j + 2], d[4 * j + 3]));
  }
}
#endif  // TC90_TM_COLS

// ---- TF32 split: x = hi + lo with hi, lo both representable in TF32 (round to nearest)
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = tf32_rna(x);
  lo = tf32_rna(x - hi);
}

}  // namespace tc90
