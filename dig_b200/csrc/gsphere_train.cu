// G-SphereNet training likelihood (reference dig/ggraph3D/method/G_SphereNet/model/sphgen.py:44-79): the model-specific
// pieces of SphGen.forward and their backward.  The feature network reuses the SphereNet training primitives
// (train_ops.cu, train_sphere.cu) plus the masked re-scatters of gsphere.cu; what lives here is
//   * attention pooling over ragged step graphs (att.py:18-35), forward and backward;
//   * the six-layer affine flow in the density direction (net_utils.py:83-93) with its log-Jacobian, and its backward;
//   * tanh / sigmoid backward, and the backward of gsphere_keep_rows.
// No kernel here uses atomics: repeated runs are bit-identical.
#include <math.h>

#include "common.cuh"
#include "gsphere_att.cuh"

using namespace dig3d;

namespace {

constexpr int kThreads = 256;
constexpr int kMaxFlowLayers = 16;

int grid_for(int64_t n) {
  const int64_t b = (n + kThreads - 1) / kThreads;
  return (int)(b < 4096 ? (b > 0 ? b : 1) : 4096);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- attention pooling over ragged graphs ---------------------------------------------------------------------------
// One CTA per query, one warp per head, lane = channel of the head (d_k = 32).  The keys / values of query j are the
// rows graph_ptr[b] .. graph_ptr[b + 1] of k / v, b = qgraph[j].  Softmax as torch_geometric.utils.softmax: segment
// maximum subtracted, 1e-16 added to the sum.  stat[j, h] = (max, denominator) for the backward.
__device__ __forceinline__ float att_score(float qv, const float* __restrict__ k, int64_t row, int width, int c) {
  return __fdiv_rn(warp_sum(__fmul_rn(qv, k[row * width + c])), sqrtf(32.f));
}

__global__ void att_fwd_kernel(const float* __restrict__ q, const int64_t* __restrict__ qgraph,
                               const int32_t* __restrict__ graph_ptr, const float* __restrict__ k,
                               const float* __restrict__ v, int n_heads, float* __restrict__ out,
                               float* __restrict__ stat) {
  const int64_t j = blockIdx.x;
  const int h = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (h >= n_heads) return;
  const int width = n_heads * 32, c = h * 32 + lane;
  const int64_t b = qgraph[j];
  const int64_t r0 = graph_ptr[b], r1 = graph_ptr[b + 1];
  const float qv = q[j * width + c];
  float m = -INFINITY;
  for (int64_t r = r0; r < r1; ++r) m = fmaxf(m, att_score(qv, k, r, width, c));
  float sum = 0.f;
  for (int64_t r = r0; r < r1; ++r) sum = __fadd_rn(sum, expf(__fsub_rn(att_score(qv, k, r, width, c), m)));
  const float denom = __fadd_rn(sum, 1e-16f);
  float acc = 0.f;
  for (int64_t r = r0; r < r1; ++r) {
    const float p = __fdiv_rn(expf(__fsub_rn(att_score(qv, k, r, width, c), m)), denom);
    acc = fmaf(v[r * width + c], p, acc);
  }
  out[j * width + c] = acc;
  if (lane == 0) stat[(j * n_heads + h) * 2] = m, stat[(j * n_heads + h) * 2 + 1] = denom;
}

// Backward of the op sequence above with the maximum treated as a constant (torch_geometric detaches it):
//   dp_r = <dout, v_r>, dv_r = p_r dout, dS = -sum_r dp_r e_r / S^2, ds_r = e_r (dp_r / S + dS),
//   dq = sum_r ds_r k_r / sqrt(32), dk_r = ds_r q / sqrt(32).
// Each key row belongs to one graph and each graph has at most one query, so every dk / dv row is written by one CTA;
// rows of graphs without a query are left as the caller initialised them (zero).
__global__ void att_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ q,
                               const int64_t* __restrict__ qgraph, const int32_t* __restrict__ graph_ptr,
                               const float* __restrict__ k, const float* __restrict__ v, const float* __restrict__ stat,
                               int n_heads, float* __restrict__ dq, float* __restrict__ dk, float* __restrict__ dv) {
  const int64_t j = blockIdx.x;
  const int h = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (h >= n_heads) return;
  const int width = n_heads * 32, c = h * 32 + lane;
  const int64_t b = qgraph[j];
  const int64_t r0 = graph_ptr[b], r1 = graph_ptr[b + 1];
  const float qv = q[j * width + c], go = dout[j * width + c];
  const float m = stat[(j * n_heads + h) * 2], denom = stat[(j * n_heads + h) * 2 + 1];
  const float scale = sqrtf(32.f);
  float a = 0.f;                                             // sum_r dp_r e_r
  for (int64_t r = r0; r < r1; ++r) {
    const float e = expf(__fsub_rn(att_score(qv, k, r, width, c), m));
    a = fmaf(warp_sum(__fmul_rn(go, v[r * width + c])), e, a);
  }
  const float ds_sum = -__fdiv_rn(__fdiv_rn(a, denom), denom);
  float gq = 0.f;
  for (int64_t r = r0; r < r1; ++r) {
    const float e = expf(__fsub_rn(att_score(qv, k, r, width, c), m));
    const float dp = warp_sum(__fmul_rn(go, v[r * width + c]));
    const float dd = __fdiv_rn(__fmul_rn(e, __fadd_rn(__fdiv_rn(dp, denom), ds_sum)), scale);
    gq = fmaf(dd, k[r * width + c], gq);
    dk[r * width + c] = __fmul_rn(dd, qv);
    dv[r * width + c] = __fmul_rn(__fdiv_rn(e, denom), go);
  }
  dq[j * width + c] = gq;
}

// ---- the two kernels above at any head width d_k (lane mapping: gsphere_att.cuh) ------------------------------------
// Same op sequences; a dot product over a head sums the lane's slices in order before the segment butterfly, and the
// loops that accumulate or write per channel run once per slice.
__global__ void att_fwd_dk_kernel(const float* __restrict__ q, const int64_t* __restrict__ qgraph,
                                  const int32_t* __restrict__ graph_ptr, const float* __restrict__ k,
                                  const float* __restrict__ v, int n_heads, int d_k, int seg, float scale,
                                  float* __restrict__ out, float* __restrict__ stat) {
  const int64_t j = blockIdx.x;
  const int warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5, per_warp = 32 / seg;
  const int64_t b = qgraph[j];
  const int64_t r0 = graph_ptr[b], r1 = graph_ptr[b + 1];
  for (int h0 = warp * per_warp; h0 < n_heads; h0 += n_warps * per_warp) {      // uniform across the warp
    const HeadLanes l = head_lanes(h0, n_heads, d_k, seg);
    const int64_t hc = (int64_t)l.h * d_k;
    const float* qh = q + j * l.width + hc;
    auto score = [&](int64_t r) { return __fdiv_rn(l.dot(qh, k + r * l.width + hc), scale); };
    float m = -INFINITY;
    for (int64_t r = r0; r < r1; ++r) m = fmaxf(m, score(r));
    float sum = 0.f;
    for (int64_t r = r0; r < r1; ++r) sum = __fadd_rn(sum, expf(__fsub_rn(score(r), m)));
    const float denom = __fadd_rn(sum, 1e-16f);
    for (int i = 0; i < l.slices; ++i) {
      const bool own = l.owns(i);
      const int64_t c = l.col(i);
      float acc = 0.f;
      for (int64_t r = r0; r < r1; ++r) {
        const float p = __fdiv_rn(expf(__fsub_rn(score(r), m)), denom);
        acc = fmaf(own ? v[r * l.width + c] : 0.f, p, acc);
      }
      if (own) out[j * l.width + c] = acc;
    }
    if (l.head && l.s == 0) stat[(j * n_heads + l.h) * 2] = m, stat[(j * n_heads + l.h) * 2 + 1] = denom;
  }
}

__global__ void att_bwd_dk_kernel(const float* __restrict__ dout, const float* __restrict__ q,
                                  const int64_t* __restrict__ qgraph, const int32_t* __restrict__ graph_ptr,
                                  const float* __restrict__ k, const float* __restrict__ v,
                                  const float* __restrict__ stat, int n_heads, int d_k, int seg, float scale,
                                  float* __restrict__ dq, float* __restrict__ dk, float* __restrict__ dv) {
  const int64_t j = blockIdx.x;
  const int warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5, per_warp = 32 / seg;
  const int64_t b = qgraph[j];
  const int64_t r0 = graph_ptr[b], r1 = graph_ptr[b + 1];
  for (int h0 = warp * per_warp; h0 < n_heads; h0 += n_warps * per_warp) {      // uniform across the warp
    const HeadLanes l = head_lanes(h0, n_heads, d_k, seg);
    const int64_t hc = (int64_t)l.h * d_k;
    const float* qh = q + j * l.width + hc;
    const float* goh = dout + j * l.width + hc;
    const int64_t st = (j * n_heads + (l.head ? l.h : 0)) * 2;
    const float m = stat[st], denom = stat[st + 1];
    auto e_of = [&](int64_t r) {
      return expf(__fsub_rn(__fdiv_rn(l.dot(qh, k + r * l.width + hc), scale), m));
    };
    auto dp_of = [&](int64_t r) { return l.dot(goh, v + r * l.width + hc); };
    float a = 0.f;                                           // sum_r dp_r e_r
    for (int64_t r = r0; r < r1; ++r) {
      const float e = e_of(r);
      a = fmaf(dp_of(r), e, a);
    }
    const float ds_sum = -__fdiv_rn(__fdiv_rn(a, denom), denom);
    for (int i = 0; i < l.slices; ++i) {
      const bool own = l.owns(i);
      const int64_t c = l.col(i);
      const float qv = own ? q[j * l.width + c] : 0.f, go = own ? dout[j * l.width + c] : 0.f;
      float gq = 0.f;
      for (int64_t r = r0; r < r1; ++r) {
        const float e = e_of(r);
        const float dp = dp_of(r);
        const float dd = __fdiv_rn(__fmul_rn(e, __fadd_rn(__fdiv_rn(dp, denom), ds_sum)), scale);
        gq = fmaf(dd, own ? k[r * l.width + c] : 0.f, gq);
        if (own) {
          dk[r * l.width + c] = __fmul_rn(dd, qv);
          dv[r * l.width + c] = __fmul_rn(__fdiv_rn(e, denom), go);
        }
      }
      if (own) dq[j * l.width + c] = gq;
    }
  }
}

// ---- affine flow, density direction (net_utils.py:83-93 over :28-37) ------------------------------------------------
// st[l, r, :] = linear2 output of layer l for row r ([s | t], 2*dim wide, from one grouped GEMM).  Per layer:
// a = exp(w_l) * tanh(s), s = exp(a), x = (x + t) * s in T (float64 for the geometry latents, whose inputs are float64
// in the reference, so the sum and product promote), log_jac += log(|s| + 1e-20) in float.
__device__ __forceinline__ float ld_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double ld_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float ld_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double ld_mul(double a, double b) { return __dmul_rn(a, b); }

template <typename T>
__global__ void flow_fwd_kernel(const float* __restrict__ st, const float* __restrict__ rescale, const T* __restrict__ x0,
                                int64_t rows, int dim, int n_layers, T* __restrict__ x_out,
                                float* __restrict__ log_jac) {
  const int64_t n = rows * dim;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = k / dim;
    const int c = (int)(k - r * dim);
    T x = x0[k];
    float lj = 0.f;
    for (int l = 0; l < n_layers; ++l) {
      const float* row = st + ((int64_t)l * rows + r) * 2 * dim;
      const float s = expf(__fmul_rn(expf(rescale[l]), tanhf(row[c])));
      x = ld_mul(ld_add(x, (T)row[dim + c]), (T)s);
      const float term = logf(__fadd_rn(fabsf(s), 1e-20f));
      lj = l == 0 ? term : __fadd_rn(lj, term);
    }
    x_out[k] = x;
    log_jac[k] = lj;
  }
}

// Backward of the above for one element: the layers' inputs are recomputed forward, then, last layer first,
//   dt = g s, ds = g (x + t) (both rounded to float, as autograd casts a promoted gradient back to float) plus
//   d log_jac sign(s) / (|s| + 1e-20), da = ds s, d tanh = da exp(w), dst_s = d tanh (1 - tanh^2), g <- g s;
// part[l, k] = da tanh(s_raw) is layer l's share of d exp(w_l), reduced by flow_rescale_reduce_kernel.
template <typename T>
__global__ void flow_bwd_kernel(const float* __restrict__ st, const float* __restrict__ rescale, const T* __restrict__ x0,
                                const T* __restrict__ dx_out, const float* __restrict__ dlog_jac, int64_t rows, int dim,
                                int n_layers, float* __restrict__ dst, float* __restrict__ part) {
  const int64_t n = rows * dim;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = k / dim;
    const int c = (int)(k - r * dim);
    T xs[kMaxFlowLayers];
    T x = x0[k];
    for (int l = 0; l < n_layers; ++l) {
      const float* row = st + ((int64_t)l * rows + r) * 2 * dim;
      const float s = expf(__fmul_rn(expf(rescale[l]), tanhf(row[c])));
      xs[l] = x;
      x = ld_mul(ld_add(x, (T)row[dim + c]), (T)s);
    }
    T g = dx_out[k];
    const float gl = dlog_jac[k];
    for (int l = n_layers - 1; l >= 0; --l) {
      const int64_t base = ((int64_t)l * rows + r) * 2 * dim;
      const float ew = expf(rescale[l]);
      const float th = tanhf(st[base + c]);
      const float s = expf(__fmul_rn(ew, th));
      const float t = st[base + dim + c];
      const float dt = (float)ld_mul(g, (T)s);
      const float ds_mul = (float)ld_mul(g, ld_add(xs[l], (T)t));
      const float sg = s > 0.f ? 1.f : (s < 0.f ? -1.f : 0.f);
      const float ds_log = __fmul_rn(__fdiv_rn(gl, __fadd_rn(fabsf(s), 1e-20f)), sg);
      const float da = __fmul_rn(__fadd_rn(ds_mul, ds_log), s);
      dst[base + c] = __fmul_rn(__fmul_rn(da, ew), __fsub_rn(1.f, __fmul_rn(th, th)));
      dst[base + dim + c] = dt;
      part[(int64_t)l * n + k] = __fmul_rn(da, th);
      g = ld_mul(g, (T)s);
    }
  }
}

// drescale[l] = exp(w_l) * sum_k part[l, k]: one CTA per layer, a strided fp64 sum per thread and a fixed tree, so the
// result does not depend on scheduling.
__global__ void flow_rescale_reduce_kernel(const float* __restrict__ part, int64_t n, const float* __restrict__ rescale,
                                           float* __restrict__ drescale) {
  __shared__ double sh[kThreads];
  const int l = blockIdx.x;
  double acc = 0.0;
  for (int64_t k = threadIdx.x; k < n; k += kThreads) acc += (double)part[(int64_t)l * n + k];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int o = kThreads / 2; o; o >>= 1) {
    if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) drescale[l] = __fmul_rn((float)sh[0], expf(rescale[l]));
}

// ---- element-wise ---------------------------------------------------------------------------------------------------
// mode 0: dx = dy (1 - y^2) (tanh, y = tanh(x)); mode 1: dx = dy y (1 - y) (sigmoid, y = sigmoid(x)).
__global__ void unary_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy, int64_t n, int mode,
                                 float* __restrict__ dx) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    const float v = y[k];
    dx[k] = mode == 0 ? __fmul_rn(dy[k], __fsub_rn(1.f, __fmul_rn(v, v)))
                      : __fmul_rn(__fmul_rn(dy[k], v), __fsub_rn(1.f, v));
  }
}

// y = 1 / (1 + exp(-x)), the generation kernel's form (gsphere.cu focus_select).
__global__ void sigmoid_kernel(const float* __restrict__ x, int64_t n, float* __restrict__ y) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x)
    y[k] = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x[k])));
}

// Backward of gsphere_keep_rows: a kept row passes its gradient to x, any other row to the fallback.
__global__ void keep_rows_bwd_kernel(const int32_t* __restrict__ flag, const int32_t* __restrict__ ptr,
                                     const float* __restrict__ dy, int64_t rows, int width, float* __restrict__ dx,
                                     float* __restrict__ dfb) {
  const int64_t n = rows * width;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = k / width;
    const bool keep = flag ? flag[r] != 0 : ptr[r + 1] > ptr[r];
    const float g = dy[k];
    if (dx) dx[k] = keep ? g : 0.f;
    if (dfb) dfb[k] = keep ? 0.f : g;
  }
}

}  // namespace

extern "C" {

int dig3d_gsphere_att_fwd(const float* q, const int64_t* qgraph, const int32_t* graph_ptr, const float* k,
                          const float* v, int64_t n_queries, int32_t n_heads, float* out, float* stat, void* stream) {
  DIG3D_REQUIRE(n_heads >= 1 && n_heads <= 32 && n_queries >= 0 && n_queries < (1LL << 31),
                "gsphere_att_fwd: bad arguments (d_k is 32, at most 32 heads)");
  if (n_queries == 0) return DIG3D_OK;
  DIG3D_REQUIRE(q && qgraph && graph_ptr && k && v && out && stat, "gsphere_att_fwd: null pointer");
  att_fwd_kernel<<<(unsigned)n_queries, 32 * n_heads, 0, (cudaStream_t)stream>>>(q, qgraph, graph_ptr, k, v, n_heads,
                                                                                out, stat);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_att_bwd(const float* dout, const float* q, const int64_t* qgraph, const int32_t* graph_ptr,
                          const float* k, const float* v, const float* stat, int64_t n_queries, int32_t n_heads,
                          float* dq, float* dk, float* dv, void* stream) {
  DIG3D_REQUIRE(n_heads >= 1 && n_heads <= 32 && n_queries >= 0 && n_queries < (1LL << 31),
                "gsphere_att_bwd: bad arguments (d_k is 32, at most 32 heads)");
  if (n_queries == 0) return DIG3D_OK;
  DIG3D_REQUIRE(dout && q && qgraph && graph_ptr && k && v && stat && dq && dk && dv, "gsphere_att_bwd: null pointer");
  att_bwd_kernel<<<(unsigned)n_queries, 32 * n_heads, 0, (cudaStream_t)stream>>>(dout, q, qgraph, graph_ptr, k, v, stat,
                                                                                n_heads, dq, dk, dv);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_att_fwd_dk(const float* q, const int64_t* qgraph, const int32_t* graph_ptr, const float* k,
                             const float* v, int64_t n_queries, int32_t n_heads, int32_t d_k, float* out, float* stat,
                             void* stream) {
  DIG3D_REQUIRE(n_heads >= 1 && d_k >= 1 && n_queries >= 0 && n_queries < (1LL << 31),
                "gsphere_att_fwd_dk: bad arguments");
  if (n_queries == 0) return DIG3D_OK;
  DIG3D_REQUIRE(q && qgraph && graph_ptr && k && v && out && stat, "gsphere_att_fwd_dk: null pointer");
  const AttShape sh = att_shape(n_heads, d_k);
  att_fwd_dk_kernel<<<(unsigned)n_queries, sh.threads, 0, (cudaStream_t)stream>>>(q, qgraph, graph_ptr, k, v, n_heads,
                                                                                 d_k, sh.seg, sh.scale, out, stat);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_att_bwd_dk(const float* dout, const float* q, const int64_t* qgraph, const int32_t* graph_ptr,
                             const float* k, const float* v, const float* stat, int64_t n_queries, int32_t n_heads,
                             int32_t d_k, float* dq, float* dk, float* dv, void* stream) {
  DIG3D_REQUIRE(n_heads >= 1 && d_k >= 1 && n_queries >= 0 && n_queries < (1LL << 31),
                "gsphere_att_bwd_dk: bad arguments");
  if (n_queries == 0) return DIG3D_OK;
  DIG3D_REQUIRE(dout && q && qgraph && graph_ptr && k && v && stat && dq && dk && dv,
                "gsphere_att_bwd_dk: null pointer");
  const AttShape sh = att_shape(n_heads, d_k);
  att_bwd_dk_kernel<<<(unsigned)n_queries, sh.threads, 0, (cudaStream_t)stream>>>(
      dout, q, qgraph, graph_ptr, k, v, stat, n_heads, d_k, sh.seg, sh.scale, dq, dk, dv);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_flow_fwd(const float* st, const float* rescale, const void* x0, int32_t x_f64, int64_t rows,
                           int32_t dim, int32_t n_layers, void* x_out, float* log_jac, void* stream) {
  DIG3D_REQUIRE(dim > 0 && n_layers > 0 && n_layers <= kMaxFlowLayers && rows >= 0, "gsphere_flow_fwd: bad arguments");
  if (rows == 0) return DIG3D_OK;
  DIG3D_REQUIRE(st && rescale && x0 && x_out && log_jac, "gsphere_flow_fwd: null pointer");
  const int grid = grid_for(rows * dim);
  if (x_f64)
    flow_fwd_kernel<double><<<grid, kThreads, 0, (cudaStream_t)stream>>>(st, rescale, (const double*)x0, rows, dim,
                                                                         n_layers, (double*)x_out, log_jac);
  else
    flow_fwd_kernel<float><<<grid, kThreads, 0, (cudaStream_t)stream>>>(st, rescale, (const float*)x0, rows, dim,
                                                                        n_layers, (float*)x_out, log_jac);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_flow_bwd(const float* st, const float* rescale, const void* x0, int32_t x_f64, const void* dx_out,
                           const float* dlog_jac, int64_t rows, int32_t dim, int32_t n_layers, float* dst, float* part,
                           float* drescale, void* stream) {
  DIG3D_REQUIRE(dim > 0 && n_layers > 0 && n_layers <= kMaxFlowLayers && rows >= 0, "gsphere_flow_bwd: bad arguments");
  DIG3D_REQUIRE(drescale && (rows == 0 || (st && rescale && x0 && dx_out && dlog_jac && dst && part)),
                "gsphere_flow_bwd: null pointer");
  const int64_t n = rows * dim;
  if (n) {
    const int grid = grid_for(n);
    if (x_f64)
      flow_bwd_kernel<double><<<grid, kThreads, 0, (cudaStream_t)stream>>>(
          st, rescale, (const double*)x0, (const double*)dx_out, dlog_jac, rows, dim, n_layers, dst, part);
    else
      flow_bwd_kernel<float><<<grid, kThreads, 0, (cudaStream_t)stream>>>(
          st, rescale, (const float*)x0, (const float*)dx_out, dlog_jac, rows, dim, n_layers, dst, part);
    DIG3D_LAUNCH_CHECK();
  }
  flow_rescale_reduce_kernel<<<n_layers, kThreads, 0, (cudaStream_t)stream>>>(part, n, rescale, drescale);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_sigmoid(const float* x, int64_t n, float* y, void* stream) {
  DIG3D_REQUIRE(n >= 0 && (n == 0 || (x && y)), "gsphere_sigmoid: bad arguments");
  if (n == 0) return DIG3D_OK;
  sigmoid_kernel<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(x, n, y);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_unary_bwd(const float* y, const float* dy, int64_t n, int32_t mode, float* dx, void* stream) {
  DIG3D_REQUIRE(n >= 0 && (mode == 0 || mode == 1) && (n == 0 || (y && dy && dx)), "gsphere_unary_bwd: bad arguments");
  if (n == 0) return DIG3D_OK;
  unary_bwd_kernel<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(y, dy, n, mode, dx);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_keep_rows_bwd(const int32_t* flag, const int32_t* ptr, const float* dy, int64_t rows, int32_t width,
                                float* dx, float* dfb, void* stream) {
  DIG3D_REQUIRE((flag || ptr) && width > 0 && rows >= 0 && (dx || dfb), "gsphere_keep_rows_bwd: bad arguments");
  if (rows == 0) return DIG3D_OK;
  DIG3D_REQUIRE(dy, "gsphere_keep_rows_bwd: null pointer");
  keep_rows_bwd_kernel<<<grid_for(rows * width), kThreads, 0, (cudaStream_t)stream>>>(flag, ptr, dy, rows, width, dx,
                                                                                      dfb);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
