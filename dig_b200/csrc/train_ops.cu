// Differentiable primitives for the TRAINING path (sm_90a, exact fp32).
//
// The fused inference kernels do not keep activations.  Training (reference run.py:103-135: forward,
// loss.backward(), optimizer.step()) runs the same math as a composition of the primitives below, each with a
// hand-written forward and backward kernel; torch.autograd only records the tape (dig_b200/autograd.py).
//
//   linear        y = x W^T + b                 nn.Linear at every call site of the models
//   wgrad         dW += dY^T X, db += colsum dY
//   act           swish / shifted softplus (+ derivative kernels)     spherenet.py:14, schnet.py:97-103
//   mul / add / scale
//   gather_rows   y = x[idx]                    x[i], x[j], x_kj[idx_kj] ...        (bwd: scatter_add_rows)
//   scatter_add_rows                            atomics; used for unsorted indices (sources, idx_kj)
//   (segment_sum over a sorted index lives in graph.cu)
//
// These are correctness-first kernels (first training path): tiled FFMA GEMMs for the big shapes, simple
// one-thread-per-output kernels for the skinny ones (K or N in {1, 6, 8, 42, 50, ...}).
#include "dense.cuh"

namespace dig3d {

// ------------------------------------------------------------------ linear, tiled (K % 32 == 0, NOUT in {64,128,256})
template <int NOUT, int K, int TM = 64>
struct LinSmem {
  float a[TM * (K + 4)];
  float ws[2 * NOUT * LDW];
};

// TM rows per CTA; MINB = CTAs per SM the register allocation is capped for (2 -> <= 128 registers per thread)
template <int NOUT, int K, int TM = 64, int MINB = 1>
__global__ void __launch_bounds__(DT, MINB)
linear_tiled_kernel(const float* __restrict__ x, int rows_total, const float* __restrict__ w,
                    const float* __restrict__ bias, float* __restrict__ y, float* __restrict__ act_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  LinSmem<NOUT, K, TM>& s = *reinterpret_cast<LinSmem<NOUT, K, TM>*>(smem_raw);
  {   // grouped call: blockIdx.y selects one of `groups` independent (x, w, bias, y) problems of the same shape
    const size_t gi = blockIdx.y;
    x += gi * (size_t)rows_total * K;
    w += gi * (size_t)NOUT * K;
    if (bias) bias += gi * NOUT;
    y += gi * (size_t)rows_total * NOUT;
    if (act_out) act_out += gi * (size_t)rows_total * NOUT;
  }
  constexpr int RP = TM / 16;
  const int r0 = blockIdx.x * TM, rows = min(TM, rows_total - r0);
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  tile_load<K>(s.a, K + 4, x + (size_t)r0 * K, K, rows);
  for (int id = threadIdx.x; id < (TM - rows) * K; id += DT) s.a[(rows + id / K) * (K + 4) + id % K] = 0.f;
  __syncthreads();
  float acc[RP][NOUT / 16];
  zero_acc(acc);
  gemm_tile<TM, NOUT, K>(s.a, K + 4, w, K, s.ws, acc);
#pragma unroll
  for (int p = 0; p < RP; ++p) {
    const int r = ty * RP + p;
    if (r < rows) {
#pragma unroll
      for (int q = 0; q < NOUT / 16; ++q) {
        const int c = tx + 16 * q;
        const float v = acc[p][q] + (bias ? __ldg(bias + c) : 0.f);
        y[(size_t)(r0 + r) * NOUT + c] = v;
        if (act_out) act_out[(size_t)(r0 + r) * NOUT + c] = swish(v);
      }
    }
  }
}

// ------------------------------------------------------------------ linear, naive (any shape)
__global__ void linear_naive_kernel(const float* __restrict__ x, int64_t rows, int k, int nout,
                                    const float* __restrict__ w, const float* __restrict__ bias,
                                    float* __restrict__ y, float* __restrict__ act_out) {
  int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= rows * nout) return;
  {
    const size_t gi = blockIdx.y;
    x += gi * (size_t)rows * k;
    w += gi * (size_t)nout * k;
    if (bias) bias += gi * nout;
    y += gi * (size_t)rows * nout;
    if (act_out) act_out += gi * (size_t)rows * nout;
  }
  const int64_t r = id / nout;
  const int c = (int)(id % nout);
  const float* xr = x + r * k;
  const float* wr = w + (size_t)c * k;
  float acc = 0.f;
  for (int i = 0; i < k; ++i) acc = fmaf(__ldg(xr + i), __ldg(wr + i), acc);
  const float v = acc + (bias ? __ldg(bias + c) : 0.f);
  y[id] = v;
  if (act_out) act_out[id] = swish(v);
}

// ------------------------------------------------------------------ weight gradient: dW[n][k] += sum_r dY[r][n] X[r][k]
// grid = (ceil(K/BK), ceil(NOUT/BN), row splits).  A CTA owns a BN x BK block of dW and a slice of the rows; the 256
// threads form a 16 (n) x 16 (k) grid of (BN/16) x (BK/16) register micro-tiles.  Rows are staged 32 at a time through
// shared memory with the next chunk prefetched into registers while the current one is consumed; partial blocks of the
// row splits are combined with atomicAdd (dW / db zero-initialised by the caller).
template <int BN, int BK>
__global__ void __launch_bounds__(256)
wgrad_kernel(const float* __restrict__ dy, const float* __restrict__ x, int64_t rows, int nout, int k,
             float* __restrict__ dw, float* __restrict__ db, int splits) {
  constexpr int RC = 32, MN = BN / 16, MK = BK / 16, LDN = BN + 4, LDK = BK + 4;
  const int split = blockIdx.z % splits;
  {   // grouped call: blockIdx.z = group * splits + split
    const size_t gi = blockIdx.z / splits;
    dy += gi * (size_t)rows * nout;
    x += gi * (size_t)rows * k;
    dw += gi * (size_t)nout * k;
    if (db) db += gi * nout;
  }
  constexpr int EN = RC * BN / 256, EK = RC * BK / 256;
  __shared__ __align__(16) float sdy[RC * LDN];
  __shared__ __align__(16) float sx[RC * LDK];
  const int kb = blockIdx.x * BK, nb = blockIdx.y * BN;
  const int tk = threadIdx.x & 15, tn = threadIdx.x >> 4;
  int64_t per = (rows + splits - 1) / splits;
  per = (per + RC - 1) / RC * RC;
  const int64_t r_lo = (int64_t)split * per, r_hi = min(rows, r_lo + per);
  if (r_lo >= r_hi) return;
  float pn[EN], pk[EK];
  auto fetch = [&](int64_t r0) {
#pragma unroll
    for (int i = 0; i < EN; ++i) {
      const int id = threadIdx.x + i * 256, rr = id / BN, cc = id % BN;
      const int64_t r = r0 + rr;
      pn[i] = (r < r_hi && nb + cc < nout) ? __ldg(dy + r * nout + nb + cc) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < EK; ++i) {
      const int id = threadIdx.x + i * 256, rr = id / BK, cc = id % BK;
      const int64_t r = r0 + rr;
      pk[i] = (r < r_hi && kb + cc < k) ? __ldg(x + r * k + kb + cc) : 0.f;
    }
  };
  float acc[MN][MK], bacc[MN];
#pragma unroll
  for (int i = 0; i < MN; ++i) {
    bacc[i] = 0.f;
#pragma unroll
    for (int j = 0; j < MK; ++j) acc[i][j] = 0.f;
  }
  const bool do_bias = db != nullptr && blockIdx.x == 0 && tk == 0;
  fetch(r_lo);
  for (int64_t r0 = r_lo; r0 < r_hi; r0 += RC) {
#pragma unroll
    for (int i = 0; i < EN; ++i) { const int id = threadIdx.x + i * 256; sdy[(id / BN) * LDN + id % BN] = pn[i]; }
#pragma unroll
    for (int i = 0; i < EK; ++i) { const int id = threadIdx.x + i * 256; sx[(id / BK) * LDK + id % BK] = pk[i]; }
    __syncthreads();
    if (r0 + RC < r_hi) fetch(r0 + RC);
#pragma unroll 8
    for (int rr = 0; rr < RC; ++rr) {
      float dv[MN], xv[MK];
#pragma unroll
      for (int i = 0; i < MN; ++i) dv[i] = sdy[rr * LDN + tn * MN + i];
#pragma unroll
      for (int j = 0; j < MK; ++j) xv[j] = sx[rr * LDK + tk * MK + j];
#pragma unroll
      for (int i = 0; i < MN; ++i) {
#pragma unroll
        for (int j = 0; j < MK; ++j) acc[i][j] = fmaf(dv[i], xv[j], acc[i][j]);
        if (do_bias) bacc[i] += dv[i];
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < MN; ++i) {
    const int n = nb + tn * MN + i;
    if (n >= nout) continue;
#pragma unroll
    for (int j = 0; j < MK; ++j) {
      const int kk = kb + tk * MK + j;
      if (kk < k) atomicAdd(dw + (size_t)n * k + kk, acc[i][j]);
    }
    if (do_bias) atomicAdd(db + n, bacc[i]);
  }
}

template <int BN, int BK>
static void launch_wgrad(const float* dy, const float* x, int64_t rows, int nout, int k, float* dw, float* db,
                         int groups, cudaStream_t st) {
  const int blocks = ceil_div(k, BK) * ceil_div(nout, BN) * groups;
  int64_t splits = 592 / blocks;                       // ~4 CTAs per SM in total
  const int64_t max_splits = (rows + 63) / 64;         // at least two 32-row chunks per CTA
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  dim3 grid(ceil_div(k, BK), ceil_div(nout, BN), (unsigned)(splits * groups));
  wgrad_kernel<BN, BK><<<grid, 256, 0, st>>>(dy, x, rows, nout, k, dw, db, (int)splits);
}

// ------------------------------------------------------------------ elementwise
__device__ __forceinline__ float sigmoid_f(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

// mode 0: swish (x * sigmoid(x)); mode 1: shifted softplus (softplus(x) - ln 2); mode 2: relu (pronet.py:340,464)
__global__ void act_fwd_kernel(const float* __restrict__ x, int64_t n, int mode, float* __restrict__ y) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = x[i];
  y[i] = mode == 0 ? __fmul_rn(v, sigmoid_f(v))
         : mode == 1 ? __fsub_rn(v > 20.0f ? v : log1pf(expf(v)), 0.693147182464599609375f)
                     : fmaxf(v, 0.0f);
}
// dx = dy * act'(x):  swish' = s (1 + x (1 - s)),  ssp' = sigmoid(x)
__global__ void act_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, int64_t n, int mode,
                               float* __restrict__ dx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = x[i], s = sigmoid_f(v);
  const float d = mode == 0 ? s * (1.0f + v * (1.0f - s)) : mode == 1 ? s : (v > 0.0f ? 1.0f : 0.0f);
  dx[i] = dy[i] * d;
}
// second order: d/dx of (dy * act'(x)) contracted with g:  out = g * dy * act''(x)
//   swish'' = s (1 - s) (2 + x (1 - 2 s)),  ssp'' = s (1 - s)
__global__ void act_bwd2_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ g,
                                int64_t n, int mode, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = x[i], s = sigmoid_f(v);
  const float d2 = mode == 0 ? s * (1.0f - s) * (2.0f + v * (1.0f - 2.0f * s)) : mode == 1 ? s * (1.0f - s) : 0.0f;
  out[i] = g[i] * dy[i] * d2;
}
// y = a * b (b broadcast over rows when b_rows == 1 is NOT needed here: same shape), y = a + b, y = alpha * a
__global__ void mul_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n, float* __restrict__ y) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = __fmul_rn(a[i], b[i]);
}
__global__ void add_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n, float* __restrict__ y) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = __fadd_rn(a[i], b[i]);
}
// y[r, c] = a[r, c] * s[r]   (row scale, e.g. the cosine cutoff of SchNet);  ds[r] = sum_c dy*a handled by rowdot
__global__ void rowscale_kernel(const float* __restrict__ a, const float* __restrict__ s, int64_t rows, int width,
                                float* __restrict__ y) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < rows * width) y[i] = __fmul_rn(a[i], s[i / width]);
}

// float4 forms of the streaming element-wise kernels above: the same per-element arithmetic (so the same bits), 16-byte
// accesses, four elements per thread.  A 34 k x 128 activation is 17.6 MB: the scalar kernels ran at ~40 % of the HBM rate
// (one 4-byte access per thread and instruction), these are bound by it.  Used when n % 4 == 0 and all pointers are
// 16-byte aligned; the scalar kernels remain for the rest.
__device__ __forceinline__ float act_fwd_one(float v, int mode) {
  return mode == 0 ? __fmul_rn(v, sigmoid_f(v))
         : mode == 1 ? __fsub_rn(v > 20.0f ? v : log1pf(expf(v)), 0.693147182464599609375f)
                     : fmaxf(v, 0.0f);
}
__device__ __forceinline__ float act_bwd_one(float v, float dy, int mode) {
  const float s = sigmoid_f(v);
  const float d = mode == 0 ? s * (1.0f + v * (1.0f - s)) : mode == 1 ? s : (v > 0.0f ? 1.0f : 0.0f);
  return dy * d;
}
__global__ void act_fwd4_kernel(const float4* __restrict__ x, int64_t n4, int mode, float4* __restrict__ y) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = x[i];
  y[i] = make_float4(act_fwd_one(v.x, mode), act_fwd_one(v.y, mode), act_fwd_one(v.z, mode), act_fwd_one(v.w, mode));
}
__global__ void act_bwd4_kernel(const float4* __restrict__ x, const float4* __restrict__ dy, int64_t n4, int mode,
                                float4* __restrict__ dx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = x[i], g = dy[i];
  dx[i] = make_float4(act_bwd_one(v.x, g.x, mode), act_bwd_one(v.y, g.y, mode), act_bwd_one(v.z, g.z, mode),
                      act_bwd_one(v.w, g.w, mode));
}
template <int OP>
__global__ void ewise4_kernel(const float4* __restrict__ a, const float4* __restrict__ b, int64_t n4,
                              float4* __restrict__ y) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 p = a[i], q = b[i];
  y[i] = OP == 0 ? make_float4(__fmul_rn(p.x, q.x), __fmul_rn(p.y, q.y), __fmul_rn(p.z, q.z), __fmul_rn(p.w, q.w))
                 : make_float4(__fadd_rn(p.x, q.x), __fadd_rn(p.y, q.y), __fadd_rn(p.z, q.z), __fadd_rn(p.w, q.w));
}
static inline bool vec4_ok(int64_t n, const void* a, const void* b, const void* c) {
  return n % 4 == 0 && (((uintptr_t)a | (uintptr_t)b | (uintptr_t)c) & 15) == 0;
}

// ------------------------------------------------------------------ row gather / scatter-add
template <typename IDX>
__global__ void gather_rows_kernel(const float* __restrict__ x, const IDX* __restrict__ idx, int64_t rows, int width,
                                   float* __restrict__ y) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * width) return;
  const int64_t r = i / width;
  y[i] = __ldg(x + (size_t)idx[r] * width + (i % width));
}
template <typename IDX>
__global__ void scatter_add_rows_kernel(const float* __restrict__ y, const IDX* __restrict__ idx, int64_t rows,
                                        int width, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * width) return;
  const int64_t r = i / width;
  atomicAdd(out + (size_t)idx[r] * width + (i % width), y[i]);
}


// out[c][r] = in[r][c]  (weights are tiny: <= 256 x 512)
__global__ void transpose_kernel(const float* __restrict__ in, int rows, int cols, float* __restrict__ out) {
  __shared__ float t[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    t[i][threadIdx.x] = (r < rows && c < cols) ? in[(size_t)r * cols + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < rows && c < cols) out[(size_t)c * rows + r] = t[threadIdx.x][i];
  }
}

// SchNet edge features for the training path (schnet.py:24-33, 119-127): gaussian smearing [E, G] and the cosine
// cutoff C[E]; same op order as the fused cfconv kernel (schnet.cu).
__global__ void schnet_edge_features_kernel(const float* __restrict__ dist, int64_t n_edges,
                                            const float* __restrict__ offset, int n_gauss, float coeff, float inv_cutoff,
                                            float* __restrict__ gauss, float* __restrict__ cut) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_edges * (n_gauss + 1)) return;
  const int64_t e = i / (n_gauss + 1);
  const int g = (int)(i % (n_gauss + 1));
  const float d = dist[e];
  if (g == n_gauss) {
    cut[e] = __fmul_rn(0.5f, __fadd_rn(cosf(__fmul_rn(__fmul_rn(d, 3.14159274101257324f), inv_cutoff)), 1.0f));
  } else {
    const float t = __fsub_rn(d, __ldg(offset + g));
    gauss[e * n_gauss + g] = expf(__fmul_rn(coeff, __fmul_rn(t, t)));
  }
}

// ------------------------------------------------------------------ GraphNorm (torch_geometric.nn.GraphNorm, comenet.py:160,213)
// One CTA per graph, one thread per channel.  Forward: shift = mean * mean_scale, o = h - shift, std = sqrt(mean(o^2) + eps),
// y = weight * o / std + bias (same operation order as the fused inference kernels in comenet.cu).
__global__ void graphnorm_fwd_kernel(const float* __restrict__ h, const int32_t* __restrict__ graph_ptr, int width,
                                     const float* __restrict__ weight, const float* __restrict__ bias,
                                     const float* __restrict__ mean_scale, float eps, float* __restrict__ y,
                                     float* __restrict__ shift, float* __restrict__ stdv) {
  const int g = blockIdx.x;
  const int n0 = graph_ptr[g], n1 = graph_ptr[g + 1];
  const float cnt = (float)max(n1 - n0, 1);
  for (int c = threadIdx.x; c < width; c += blockDim.x) {
    float sum = 0.f;
    for (int n = n0; n < n1; ++n) sum += h[(size_t)n * width + c];
    const float sh = __fmul_rn(__fdiv_rn(sum, cnt), __ldg(mean_scale + c));
    float sq = 0.f;
    for (int n = n0; n < n1; ++n) { const float o = __fsub_rn(h[(size_t)n * width + c], sh); sq += __fmul_rn(o, o); }
    const float sd = __fsqrt_rn(__fadd_rn(__fdiv_rn(sq, cnt), eps));
    shift[(size_t)g * width + c] = sh;
    stdv[(size_t)g * width + c] = sd;
    const float w = __ldg(weight + c), b = __ldg(bias + c);
    for (int n = n0; n < n1; ++n) {
      const float o = __fsub_rn(h[(size_t)n * width + c], sh);
      y[(size_t)n * width + c] = __fadd_rn(__fdiv_rn(__fmul_rn(w, o), sd), b);
    }
  }
}

// Backward.  With n nodes in the graph, r = 1/std, o_i = h_i - shift, A = sum dy_i o_i, B = sum dy_i, S = sum h_i:
//   d weight += A r          d bias += B
//   dv = -0.5 w A r^3        do_i = dy_i w r + 2 dv o_i / n        D = sum_i do_i = w r B + 2 dv (S - n shift) / n
//   dx_i = do_i - mean_scale D / n            d mean_scale += -(S / n) D
__global__ void graphnorm_bwd_kernel(const float* __restrict__ h, const float* __restrict__ dy,
                                     const int32_t* __restrict__ graph_ptr, int width, const float* __restrict__ weight,
                                     const float* __restrict__ mean_scale, const float* __restrict__ shift,
                                     const float* __restrict__ stdv, float* __restrict__ dx, float* __restrict__ dweight,
                                     float* __restrict__ dbias, float* __restrict__ dmean_scale) {
  const int g = blockIdx.x;
  const int n0 = graph_ptr[g], n1 = graph_ptr[g + 1];
  if (n1 <= n0) return;
  const float cnt = (float)(n1 - n0);
  for (int c = threadIdx.x; c < width; c += blockDim.x) {
    const float sh = shift[(size_t)g * width + c], r = 1.0f / stdv[(size_t)g * width + c];
    const float w = __ldg(weight + c), ms = __ldg(mean_scale + c);
    float A = 0.f, B = 0.f, S = 0.f;
    for (int n = n0; n < n1; ++n) {
      const float hv = h[(size_t)n * width + c], d = dy[(size_t)n * width + c];
      A = fmaf(d, hv - sh, A);
      B += d;
      S += hv;
    }
    const float dv = -0.5f * w * A * r * r * r;
    const float D = w * r * B + 2.0f * dv * (S - cnt * sh) / cnt;
    const float back = ms * D / cnt;
    for (int n = n0; n < n1; ++n) {
      const float o = h[(size_t)n * width + c] - sh;
      dx[(size_t)n * width + c] = dy[(size_t)n * width + c] * w * r + 2.0f * dv * o / cnt - back;
    }
    atomicAdd(dweight + c, A * r);
    atomicAdd(dbias + c, B);
    atomicAdd(dmean_scale + c, -(S / cnt) * D);
  }
}

// Forward mode of GraphNorm (force training, autograd_jvp.py) along a tangent h_dot, from the forward's shift / std.
// Per graph and channel, with n nodes, o = h - shift, std = sqrt(mean(o^2) + eps):
//   o_dot = h_dot - mean_scale * mean(h_dot)      std_dot = mean(o * o_dot) / std
//   y_dot = weight * (o_dot / std - o * std_dot / std^2)
__global__ void graphnorm_tangent_kernel(const float* __restrict__ h, const float* __restrict__ hd,
                                         const int32_t* __restrict__ graph_ptr, int width,
                                         const float* __restrict__ weight, const float* __restrict__ mean_scale,
                                         const float* __restrict__ shift, const float* __restrict__ stdv,
                                         float* __restrict__ yd) {
  const int g = blockIdx.x;
  const int n0 = graph_ptr[g], n1 = graph_ptr[g + 1];
  if (n1 <= n0) return;
  const float cnt = (float)(n1 - n0);
  for (int c = threadIdx.x; c < width; c += blockDim.x) {
    const float sh = shift[(size_t)g * width + c], sd = stdv[(size_t)g * width + c];
    const float w = __ldg(weight + c), ms = __ldg(mean_scale + c);
    float sum_d = 0.f;
    for (int n = n0; n < n1; ++n) sum_d += hd[(size_t)n * width + c];
    const float shd = ms * (sum_d / cnt);
    float A = 0.f;
    for (int n = n0; n < n1; ++n) {
      const size_t k = (size_t)n * width + c;
      A = fmaf(h[k] - sh, hd[k] - shd, A);
    }
    const float r = 1.0f / sd;
    const float sdd = A / cnt * r;
    for (int n = n0; n < n1; ++n) {
      const size_t k = (size_t)n * width + c;
      yd[k] = w * ((hd[k] - shd) * r - (h[k] - sh) * sdd * r * r);
    }
  }
}

// Reverse mode of graphnorm_tangent_kernel: gy = d loss / d y_dot -> d h, d h_dot, d weight, d mean_scale.
// With mu = mean(h), mud = mean(h_dot), r = 1/std, u = w gy, and sums over the graph's nodes:
//   d std_dot = -r^2 sum(u o)          d std = sum(u (2 o std_dot r^3 - o_dot r^2)) - d std_dot std_dot r
//   d o_k = -u_k std_dot r^2 + (d std_dot o_dot_k + d std o_k) r / n      d o_dot_k = u_k r + d std_dot o_k r / n
//   d h_k = d o_k - mean_scale sum(d o) / n            d h_dot_k = d o_dot_k - mean_scale sum(d o_dot) / n
//   d weight += sum(gy (o_dot r - o std_dot r^2))      d mean_scale += -mu sum(d o) - mud sum(d o_dot)
__global__ void graphnorm_tangent_bwd_kernel(const float* __restrict__ h, const float* __restrict__ hd,
                                             const float* __restrict__ gy, const int32_t* __restrict__ graph_ptr,
                                             int width, const float* __restrict__ weight,
                                             const float* __restrict__ mean_scale, const float* __restrict__ shift,
                                             const float* __restrict__ stdv, float* __restrict__ dh,
                                             float* __restrict__ dhd, float* __restrict__ dweight,
                                             float* __restrict__ dmean_scale) {
  const int g = blockIdx.x;
  const int n0 = graph_ptr[g], n1 = graph_ptr[g + 1];
  if (n1 <= n0) return;
  const float cnt = (float)(n1 - n0);
  for (int c = threadIdx.x; c < width; c += blockDim.x) {
    const float sh = shift[(size_t)g * width + c], sd = stdv[(size_t)g * width + c];
    const float w = __ldg(weight + c), ms = __ldg(mean_scale + c);
    float S = 0.f, Sd = 0.f;
    for (int n = n0; n < n1; ++n) { S += h[(size_t)n * width + c]; Sd += hd[(size_t)n * width + c]; }
    const float mu = S / cnt, mud = Sd / cnt, shd = ms * mud;
    float A = 0.f, G = 0.f, Go = 0.f, God = 0.f, So = 0.f, Sod = 0.f;
    for (int n = n0; n < n1; ++n) {
      const size_t k = (size_t)n * width + c;
      const float o = h[k] - sh, od = hd[k] - shd, gk = gy[k];
      A = fmaf(o, od, A);
      G += gk;
      Go = fmaf(gk, o, Go);
      God = fmaf(gk, od, God);
      So += o;
      Sod += od;
    }
    const float r = 1.0f / sd, r2 = r * r;
    const float sdd = A / cnt * r;
    const float g_sdd = -w * Go * r2;
    const float g_sd = w * (2.0f * sdd * r2 * r * Go - God * r2) - g_sdd * sdd * r;
    const float a_o = g_sdd * r / cnt, b_o = g_sd * r / cnt;          // d o_k = -w gy_k sdd r^2 + a_o od_k + b_o o_k
    const float sum_do = -w * G * sdd * r2 + a_o * Sod + b_o * So;
    const float sum_dod = w * G * r + a_o * So;
    const float back_o = ms * sum_do / cnt, back_od = ms * sum_dod / cnt;
    for (int n = n0; n < n1; ++n) {
      const size_t k = (size_t)n * width + c;
      const float o = h[k] - sh, od = hd[k] - shd, gk = gy[k];
      dh[k] = -w * gk * sdd * r2 + a_o * od + b_o * o - back_o;
      dhd[k] = w * gk * r + a_o * o - back_od;
    }
    atomicAdd(dweight + c, God * r - Go * sdd * r2);
    atomicAdd(dmean_scale + c, -mu * sum_do - mud * sum_dod);
  }
}

template <int NOUT, int K, int TM = 64, int MINB = 1>
static int launch_linear_tiled(const float* x, int64_t rows, const float* w, const float* b, float* y, float* act_out,
                               int groups, cudaStream_t st) {
  auto kfn = linear_tiled_kernel<NOUT, K, TM, MINB>;
  const size_t sm = sizeof(LinSmem<NOUT, K, TM>);
  cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
  if (e != cudaSuccess) { set_error("linear: cudaFuncSetAttribute(%zu): %s", sm, cudaGetErrorString(e)); return DIG3D_ECUDA; }
  kfn<<<dim3(ceil_div(rows, TM), groups), DT, sm, st>>>(x, (int)rows, w, b, y, act_out);
  return DIG3D_OK;
}

// tuning switch for the dominant shape (128 -> 128 on ~34 k edge rows): 0 = 64-row tiles, 1 CTA/SM by registers;
// 1 = 64-row tiles capped at 128 registers (2 CTAs/SM); 2 = 128-row tiles
static int h_lin_cfg = 1;

// ---------------------------------------------------------------------------------- fused Adam
// One pass over the flat fp32 parameter / gradient / moment buffers (torch.optim.Adam semantics, amsgrad off):
//   g += wd * p;  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2;  p -= (lr / c1) * m / (sqrt(v) / sqrt(c2) + eps)
// Replaces the ~10 multi-tensor launches of the eager optimizer; 16 B per parameter read + 12 B written.
__global__ void adam_step_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                 float* __restrict__ v, int64_t n, float lr_over_c1, float one_minus_b1, float b2,
                                 float one_minus_b2, float eps, float wd, float inv_sqrt_c2) {
  // (1 - beta) arrive as separately rounded doubles: 1.f - 0.999f is off by 1.3e-5 relative from float(1 - 0.999)
  const int64_t i4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i4 >= n) return;
  if (i4 + 4 <= n) {
    float4 pp = *reinterpret_cast<float4*>(p + i4), mm = *reinterpret_cast<float4*>(m + i4),
           vv = *reinterpret_cast<float4*>(v + i4);
    const float4 gg = *reinterpret_cast<const float4*>(g + i4);
    float* pa = &pp.x; float* ma = &mm.x; float* va = &vv.x; const float* ga = &gg.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float gk = fmaf(wd, pa[k], ga[k]);
      ma[k] = fmaf(one_minus_b1, gk - ma[k], ma[k]);             // lerp, as torch's exp_avg.lerp_(grad, 1 - beta1)
      va[k] = fmaf(va[k], b2, one_minus_b2 * gk * gk);
      pa[k] -= lr_over_c1 * __fdiv_rn(ma[k], fmaf(sqrtf(va[k]), inv_sqrt_c2, eps));
    }
    *reinterpret_cast<float4*>(p + i4) = pp; *reinterpret_cast<float4*>(m + i4) = mm; *reinterpret_cast<float4*>(v + i4) = vv;
  } else {
    for (int64_t i = i4; i < n; ++i) {
      const float gk = fmaf(wd, p[i], g[i]);
      m[i] = fmaf(one_minus_b1, gk - m[i], m[i]);
      v[i] = fmaf(v[i], b2, one_minus_b2 * gk * gk);
      p[i] -= lr_over_c1 * __fdiv_rn(m[i], fmaf(sqrtf(v[i]), inv_sqrt_c2, eps));
    }
  }
}

}  // namespace dig3d

using namespace dig3d;

extern "C" {

int dig3d_linear(const float* x, int64_t rows, int32_t k, int32_t nout, const float* w, const float* bias, float* y,
                 float* act_out, int32_t groups, void* stream) {
  DIG3D_REQUIRE(x && w && y && k > 0 && nout > 0 && groups >= 1 && groups <= 65535, "linear: bad arguments");
  if (rows == 0) return DIG3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = -100;
  if (nout == 128 && k == 128 && h_lin_cfg == 1) {
    rc = launch_linear_tiled<128, 128, 64, 2>(x, rows, w, bias, y, act_out, groups, st);
  } else if (nout == 128 && k == 128 && h_lin_cfg == 2) {
    rc = launch_linear_tiled<128, 128, 128, 1>(x, rows, w, bias, y, act_out, groups, st);
  }
#define DIG3D_LT(NO, KK) if (rc == -100 && nout == NO && k == KK) rc = launch_linear_tiled<NO, KK>(x, rows, w, bias, y, act_out, groups, st);
  DIG3D_LT(128, 128) DIG3D_LT(64, 128) DIG3D_LT(128, 64) DIG3D_LT(256, 128) DIG3D_LT(256, 256) DIG3D_LT(128, 256)
  DIG3D_LT(128, 384) DIG3D_LT(32, 32) DIG3D_LT(64, 64) DIG3D_LT(128, 32) DIG3D_LT(32, 128) DIG3D_LT(256, 64)
  DIG3D_LT(64, 256) DIG3D_LT(256, 512) DIG3D_LT(384, 128) DIG3D_LT(512, 256)
#undef DIG3D_LT
  if (rc == -100) {
    const int64_t total = rows * nout;
    linear_naive_kernel<<<dim3(ceil_div(total, 256), groups), 256, 0, st>>>(x, rows, k, nout, w, bias, y, act_out);
    rc = DIG3D_OK;
  }
  if (rc) return rc;
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_linear_set_config(int32_t cfg) {
  DIG3D_REQUIRE(cfg >= 0 && cfg <= 2, "linear_set_config: cfg must be 0, 1 or 2");
  h_lin_cfg = cfg;
  return DIG3D_OK;
}

int dig3d_wgrad(const float* dy, const float* x, int64_t rows, int32_t nout, int32_t k, float* dw, float* db,
                int32_t groups, void* stream) {
  DIG3D_REQUIRE(dy && x && dw && nout > 0 && k > 0 && groups >= 1 && groups <= 64, "wgrad: bad arguments");
  if (rows == 0) return DIG3D_OK;
  if (dig3d_wgrad_tc_supported(rows, nout, k))         // wgmma 3xTF32 (train_tc.cu) where the tile shape pays
    return dig3d_wgrad_tc(dy, x, rows, nout, k, dw, db, groups, stream);
  cudaStream_t st = (cudaStream_t)stream;
  if (nout > 16 && k > 16) launch_wgrad<64, 64>(dy, x, rows, nout, k, dw, db, groups, st);
  else if (nout > 16) launch_wgrad<64, 16>(dy, x, rows, nout, k, dw, db, groups, st);
  else if (k > 16) launch_wgrad<16, 64>(dy, x, rows, nout, k, dw, db, groups, st);
  else launch_wgrad<16, 16>(dy, x, rows, nout, k, dw, db, groups, st);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_act(const float* x, int64_t n, int32_t mode, float* y, void* stream) {
  DIG3D_REQUIRE(x && y && mode >= 0 && mode <= 2, "act: bad arguments");
  if (n == 0) return DIG3D_OK;
  if (vec4_ok(n, x, y, y))
    act_fwd4_kernel<<<ceil_div(n / 4, 256), 256, 0, (cudaStream_t)stream>>>((const float4*)x, n / 4, mode, (float4*)y);
  else
    act_fwd_kernel<<<ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(x, n, mode, y);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_act_bwd(const float* x, const float* dy, int64_t n, int32_t mode, float* dx, void* stream) {
  DIG3D_REQUIRE(x && dy && dx && mode >= 0 && mode <= 2, "act_bwd: bad arguments");
  if (n == 0) return DIG3D_OK;
  if (vec4_ok(n, x, dy, dx))
    act_bwd4_kernel<<<ceil_div(n / 4, 256), 256, 0, (cudaStream_t)stream>>>((const float4*)x, (const float4*)dy, n / 4, mode,
                                                                          (float4*)dx);
  else
    act_bwd_kernel<<<ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(x, dy, n, mode, dx);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_act_bwd2(const float* x, const float* dy, const float* g, int64_t n, int32_t mode, float* out, void* stream) {
  DIG3D_REQUIRE(x && dy && g && out && mode >= 0 && mode <= 2, "act_bwd2: bad arguments");
  if (n == 0) return DIG3D_OK;
  act_bwd2_kernel<<<ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(x, dy, g, n, mode, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, double lr,
                    double beta1, double beta2, double eps, double weight_decay, int64_t step, void* stream) {
  DIG3D_REQUIRE(param && grad && exp_avg && exp_avg_sq && step >= 1, "adam_step: bad arguments");
  DIG3D_REQUIRE((((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) == 0,
                "adam_step: the flat buffers must be 16-byte aligned");
  if (n == 0) return DIG3D_OK;
  const double c1 = 1.0 - pow(beta1, (double)step), c2 = 1.0 - pow(beta2, (double)step);
  adam_step_kernel<<<ceil_div(ceil_div(n, 4), 256), 256, 0, (cudaStream_t)stream>>>(
      param, grad, exp_avg, exp_avg_sq, n, (float)(lr / c1), (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2),
      (float)eps, (float)weight_decay, (float)(1.0 / sqrt(c2)));
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_ewise(const float* a, const float* b, int64_t n, int32_t op, float* y, void* stream) {
  DIG3D_REQUIRE(a && b && y && (op == 0 || op == 1), "ewise: bad arguments");
  if (n == 0) return DIG3D_OK;
  if (vec4_ok(n, a, b, y)) {
    if (op == 0) ewise4_kernel<0><<<ceil_div(n / 4, 256), 256, 0, (cudaStream_t)stream>>>((const float4*)a, (const float4*)b, n / 4, (float4*)y);
    else ewise4_kernel<1><<<ceil_div(n / 4, 256), 256, 0, (cudaStream_t)stream>>>((const float4*)a, (const float4*)b, n / 4, (float4*)y);
  } else if (op == 0) mul_kernel<<<ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(a, b, n, y);
  else add_kernel<<<ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(a, b, n, y);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_rowscale(const float* a, const float* s, int64_t rows, int32_t width, float* y, void* stream) {
  DIG3D_REQUIRE(a && s && y && width > 0, "rowscale: bad arguments");
  if (rows == 0) return DIG3D_OK;
  rowscale_kernel<<<ceil_div(rows * width, 256), 256, 0, (cudaStream_t)stream>>>(a, s, rows, width, y);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gather_rows(const float* x, const void* idx, int32_t idx_is_64, int64_t rows, int32_t width, float* y,
                      void* stream) {
  DIG3D_REQUIRE(x && idx && y && width > 0, "gather_rows: bad arguments");
  if (rows == 0) return DIG3D_OK;
  const int grid = ceil_div(rows * width, 256);
  if (idx_is_64) gather_rows_kernel<int64_t><<<grid, 256, 0, (cudaStream_t)stream>>>(x, (const int64_t*)idx, rows, width, y);
  else gather_rows_kernel<int32_t><<<grid, 256, 0, (cudaStream_t)stream>>>(x, (const int32_t*)idx, rows, width, y);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_scatter_add_rows(const float* y, const void* idx, int32_t idx_is_64, int64_t rows, int32_t width, float* out,
                           void* stream) {
  DIG3D_REQUIRE(y && idx && out && width > 0, "scatter_add_rows: bad arguments");
  if (rows == 0) return DIG3D_OK;
  const int grid = ceil_div(rows * width, 256);
  if (idx_is_64) scatter_add_rows_kernel<int64_t><<<grid, 256, 0, (cudaStream_t)stream>>>(y, (const int64_t*)idx, rows, width, out);
  else scatter_add_rows_kernel<int32_t><<<grid, 256, 0, (cudaStream_t)stream>>>(y, (const int32_t*)idx, rows, width, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_transpose(const float* in, int32_t rows, int32_t cols, float* out, void* stream) {
  DIG3D_REQUIRE(in && out && rows > 0 && cols > 0, "transpose: bad arguments");
  dim3 grid(ceil_div(cols, 32), ceil_div(rows, 32)), block(32, 8);
  transpose_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(in, rows, cols, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_schnet_edge_features(const float* dist, int64_t n_edges, const float* offset, int32_t n_gauss, double coeff,
                               double cutoff, float* gauss, float* cut, void* stream) {
  DIG3D_REQUIRE(dist && offset && gauss && cut && n_gauss > 0, "schnet_edge_features: bad arguments");
  if (n_edges == 0) return DIG3D_OK;
  const int64_t total = n_edges * (n_gauss + 1);
  schnet_edge_features_kernel<<<ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
      dist, n_edges, offset, n_gauss, (float)coeff, (float)(1.0 / cutoff), gauss, cut);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_graphnorm(const float* h, const int32_t* graph_ptr, int64_t n_graphs, int32_t width, const float* weight,
                    const float* bias, const float* mean_scale, double eps, float* y, float* shift, float* stdv,
                    void* stream) {
  DIG3D_REQUIRE(h && graph_ptr && weight && bias && mean_scale && y && shift && stdv && width > 0, "graphnorm: bad arguments");
  if (n_graphs == 0) return DIG3D_OK;
  graphnorm_fwd_kernel<<<(int)n_graphs, width < 256 ? width : 256, 0, (cudaStream_t)stream>>>(
      h, graph_ptr, width, weight, bias, mean_scale, (float)eps, y, shift, stdv);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_graphnorm_bwd(const float* h, const float* dy, const int32_t* graph_ptr, int64_t n_graphs, int32_t width,
                        const float* weight, const float* mean_scale, const float* shift, const float* stdv, float* dx,
                        float* dweight, float* dbias, float* dmean_scale, void* stream) {
  DIG3D_REQUIRE(h && dy && graph_ptr && weight && mean_scale && shift && stdv && dx && dweight && dbias && dmean_scale &&
                    width > 0, "graphnorm_bwd: bad arguments");
  if (n_graphs == 0) return DIG3D_OK;
  graphnorm_bwd_kernel<<<(int)n_graphs, width < 256 ? width : 256, 0, (cudaStream_t)stream>>>(
      h, dy, graph_ptr, width, weight, mean_scale, shift, stdv, dx, dweight, dbias, dmean_scale);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_graphnorm_tangent(const float* h, const float* h_dot, const int32_t* graph_ptr, int64_t n_graphs,
                            int32_t width, const float* weight, const float* mean_scale, const float* shift,
                            const float* stdv, float* y_dot, void* stream) {
  DIG3D_REQUIRE(h && h_dot && graph_ptr && weight && mean_scale && shift && stdv && y_dot && width > 0,
                "graphnorm_tangent: bad arguments");
  if (n_graphs == 0) return DIG3D_OK;
  graphnorm_tangent_kernel<<<(int)n_graphs, width < 256 ? width : 256, 0, (cudaStream_t)stream>>>(
      h, h_dot, graph_ptr, width, weight, mean_scale, shift, stdv, y_dot);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_graphnorm_tangent_bwd(const float* h, const float* h_dot, const float* dy_dot, const int32_t* graph_ptr,
                                int64_t n_graphs, int32_t width, const float* weight, const float* mean_scale,
                                const float* shift, const float* stdv, float* dh, float* dh_dot, float* dweight,
                                float* dmean_scale, void* stream) {
  DIG3D_REQUIRE(h && h_dot && dy_dot && graph_ptr && weight && mean_scale && shift && stdv && dh && dh_dot &&
                    dweight && dmean_scale && width > 0, "graphnorm_tangent_bwd: bad arguments");
  if (n_graphs == 0) return DIG3D_OK;
  graphnorm_tangent_bwd_kernel<<<(int)n_graphs, width < 256 ? width : 256, 0, (cudaStream_t)stream>>>(
      h, h_dot, dy_dot, graph_ptr, width, weight, mean_scale, shift, stdv, dh, dh_dot, dweight, dmean_scale);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
