// Bond-length maximum mean discrepancy (reference dig/ggraph3D/utils/eval_bond_mmd_utils.py:44-97, compute_mmd): the
// bandwidth and the three Gaussian-kernel sums over one source set S and one target set T, all in fp64.
//
//   v = [source; target], n = n_s + n_t
//   bandwidth  b = fix_sigma, or sum_ij (x_i - x_j)^2 / (n^2 - n) = 2 sum_i (x_i - mean)^2 / (n - 1)     (:64-71)
//   b_k        = b / mul^(K/2) * mul^k, k < K                                                            (:73-74)
//   XX = sum_{S x S}, YY = sum_{T x T}, XY = sum_{S x T} of sum_k exp(-d^2 / b_k), diagonal included        (:76-95)
//
// Three launches on one stream: the bandwidth (one CTA, two-pass centred sum), the pair sums (persistent grid over
// 1024 x 1024 tiles, per-CTA partials into the workspace) and the fixed-order reduction of the partials.  No atomics:
// the result depends only on the inputs and the workspace length (= 3 x the grid size).
#include <math.h>

#include "common.cuh"

using namespace dig3d;

namespace {

constexpr int kThreads = 256;
constexpr int kRowsPerThread = 4;
constexpr int kTile = kThreads * kRowsPerThread;   // rows and columns of a tile
constexpr int kMaxKernels = 64;

// Fixed-order CTA sum of one value per thread (shuffle tree, then warp 0 over the eight warp sums); valid in thread 0.
__device__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; ++w) s += red[w];
  return s;
}

// b_k of the reference's bandwidth list (k < K), from b as the reference forms it.
__device__ double bandwidth_k(double b, double mul, int K, int k) {
  double p = 1.0;
  for (int i = 0; i < K / 2; ++i) p *= mul;
  double q = 1.0;
  for (int i = 0; i < k; ++i) q *= mul;
  return b / p * q;
}

// out[0] = b: fix_sigma when it is non-zero, else 2 sum (x - mean)^2 / (n - 1) -- the exact value of the reference's
// sum of squared pairwise differences over n^2 - n, without the cancellation of 2n sum x^2 - 2 (sum x)^2.
__global__ void __launch_bounds__(kThreads) bandwidth_kernel(const double* __restrict__ v, int64_t n, double fix_sigma,
                                                             double* __restrict__ out) {
  __shared__ double red[kThreads / 32];
  __shared__ double mean;
  if (fix_sigma != 0.0) {
    if (threadIdx.x == 0) out[0] = fix_sigma;
    return;
  }
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += kThreads) s += v[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) mean = s / (double)n;
  __syncthreads();
  const double m = mean;
  double q = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += kThreads) {
    const double d = v[i] - m;
    q = fma(d, d, q);
  }
  q = block_sum(q, red);
  if (threadIdx.x == 0) {
    const double dn = (double)n;
    out[0] = 2.0 * dn * q / (dn * dn - dn);
  }
}

// Tile t of a triangle -> (row tile, column tile) with row <= column.
__device__ __forceinline__ void triangle_tile(int64_t t, int64_t& r, int64_t& c) {
  // lower-triangle row a holds tiles a(a+1)/2 .. a(a+1)/2 + a; the transpose (b, a) is the upper-triangle tile
  int64_t a = (int64_t)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
  while (a * (a + 1) / 2 > t) --a;
  while ((a + 1) * (a + 2) / 2 <= t) ++a;
  const int64_t b = t - a * (a + 1) / 2;
  r = b;
  c = a;
}

// sum_k exp(x * s_k) for one pair, x = d^2.  kPow2 (mul == 2): one exp at the widest bandwidth, then squarings,
// exp(-d^2 / b_{k-1}) = exp(-d^2 / b_k)^2.  Otherwise one exp per bandwidth.  kK > 0 fixes K at compile time.
template <bool kPow2, int kK>
__device__ __forceinline__ double kernel_sum(double d2, double neg_inv_widest, const double* neg_inv, int K) {
  if (kPow2) {
    double e = exp(d2 * neg_inv_widest);
    double s = e;
    const int kk = kK > 0 ? kK : K;
#pragma unroll
    for (int k = 1; k < kk; ++k) {
      e = e * e;
      s += e;
    }
    return s;
  } else {
    double s = 0.0;
    for (int k = 0; k < K; ++k) s += exp(d2 * neg_inv[k]);
    return s;
  }
}

// Sum over one tile of sum_k exp(-(x_i - y_j)^2 / b_k), rows xr (kRowsPerThread per thread, thread-strided), columns
// col[] in shared memory.  kMasked: only rows < r_valid, columns < c_valid and, on a diagonal tile, j > i count.
template <bool kPow2, int kK, bool kMasked>
__device__ __forceinline__ double tile_sum(const double (&xr)[kRowsPerThread], const double* col, double neg_inv_widest,
                                           const double* neg_inv, int K, int r_valid, int c_valid, bool diag) {
  double acc[kRowsPerThread];
#pragma unroll
  for (int k = 0; k < kRowsPerThread; ++k) acc[k] = 0.0;
#pragma unroll 2
  for (int j = 0; j < kTile; ++j) {
    const double y = col[j];
#pragma unroll
    for (int k = 0; k < kRowsPerThread; ++k) {
      const double d = xr[k] - y;
      const double s = kernel_sum<kPow2, kK>(d * d, neg_inv_widest, neg_inv, K);
      if (kMasked) {
        const int i = threadIdx.x + k * kThreads;
        const bool keep = i < r_valid && j < c_valid && (!diag || j > i);
        acc[k] += keep ? s : 0.0;
      } else {
        acc[k] += s;
      }
    }
  }
  static_assert(kRowsPerThread == 4, "the row sums below");
  return (acc[0] + acc[1]) + (acc[2] + acc[3]);
}

// a += x with the rounding error kept in c (TwoSum): the per-thread running sum over its tiles.
__device__ __forceinline__ void two_sum_add(double& a, double& c, double x) {
  const double t = a + x;
  const double bp = t - a;
  c += (a - (t - bp)) + (x - bp);
  a = t;
}

// Persistent grid over the tiles of S x S (one triangle), T x T (one triangle) and S x T, in that order.  Off-diagonal
// pairs of the symmetric regions count twice (the tile sum is doubled), the diagonal i == j is left to the reduction.
// ws[3 * cta + region] = this CTA's sum of region (0: S x S, 1: T x T, 2: S x T).
template <bool kPow2, int kK>
__global__ void __launch_bounds__(kThreads) pairs_kernel(const double* __restrict__ v, int64_t ns, int64_t nt,
                                                         double kernel_mul, int K, const double* __restrict__ bw,
                                                         double* __restrict__ ws) {
  __shared__ double col[kTile];
  __shared__ double neg_inv[kMaxKernels];
  __shared__ double red[kThreads / 32];
  const double b = bw[0];
  if (threadIdx.x < K) neg_inv[threadIdx.x] = -1.0 / bandwidth_k(b, kernel_mul, K, threadIdx.x);
  __syncthreads();
  const double neg_inv_widest = neg_inv[K - 1];
  const int64_t ms = (ns + kTile - 1) / kTile, mt = (nt + kTile - 1) / kTile;
  const int64_t n_ss = ms * (ms + 1) / 2, n_tt = mt * (mt + 1) / 2, n_st = ms * mt;
  const int64_t n_tiles = n_ss + n_tt + n_st;
  double acc[3] = {0.0, 0.0, 0.0}, cmp[3] = {0.0, 0.0, 0.0};
  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    int region;
    int64_t r, c, row0, col0, rows, cols;
    if (t < n_ss) {
      region = 0;
      triangle_tile(t, r, c);
      row0 = 0, col0 = 0, rows = ns, cols = ns;
    } else if (t < n_ss + n_tt) {
      region = 1;
      triangle_tile(t - n_ss, r, c);
      row0 = ns, col0 = ns, rows = nt, cols = nt;
    } else {
      region = 2;
      const int64_t u = t - n_ss - n_tt;
      r = u / mt, c = u - r * mt;
      row0 = 0, col0 = ns, rows = ns, cols = nt;
    }
    const int64_t rb = r * kTile, cb = c * kTile;
    const int r_valid = (int)(rows - rb < kTile ? rows - rb : kTile);
    const int c_valid = (int)(cols - cb < kTile ? cols - cb : kTile);
    const bool diag = region < 2 && r == c;
    __syncthreads();                                   // the previous tile's columns are no longer read
    for (int j = threadIdx.x; j < kTile; j += kThreads) col[j] = j < c_valid ? v[col0 + cb + j] : 0.0;
    double xr[kRowsPerThread];
#pragma unroll
    for (int k = 0; k < kRowsPerThread; ++k) {
      const int i = threadIdx.x + k * kThreads;
      xr[k] = i < r_valid ? v[row0 + rb + i] : 0.0;
    }
    __syncthreads();
    double s;
    if (diag || r_valid < kTile || c_valid < kTile)
      s = tile_sum<kPow2, kK, true>(xr, col, neg_inv_widest, neg_inv, K, r_valid, c_valid, diag);
    else
      s = tile_sum<kPow2, kK, false>(xr, col, neg_inv_widest, neg_inv, K, r_valid, c_valid, false);
    if (region == 0) two_sum_add(acc[0], cmp[0], 2.0 * s);
    else if (region == 1) two_sum_add(acc[1], cmp[1], 2.0 * s);
    else two_sum_add(acc[2], cmp[2], s);
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const double s = block_sum(acc[q] + cmp[q], red);
    if (threadIdx.x == 0) ws[3 * blockIdx.x + q] = s;
  }
}

// out[1..3] = (XX, YY, XY) normalised, from the n_partials per-CTA partials in a fixed order; the diagonal of each
// symmetric region adds n * sum_k exp(-0 / b_k) (n * K, or NaN when the bandwidth is 0 or NaN, as in the reference).
__global__ void __launch_bounds__(kThreads) reduce_kernel(const double* __restrict__ ws, int64_t n_partials, int64_t ns,
                                                          int64_t nt, double kernel_mul, int K, double* __restrict__ out) {
  __shared__ double red[kThreads / 32];
  double diag = 0.0;
  if (threadIdx.x == 0)
    for (int k = 0; k < K; ++k) diag += exp(-(0.0 * 0.0) / bandwidth_k(out[0], kernel_mul, K, k));
  for (int q = 0; q < 3; ++q) {
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < n_partials; i += kThreads) s += ws[3 * i + q];
    s = block_sum(s, red);
    if (threadIdx.x == 0) {
      const double dns = (double)ns, dnt = (double)nt;
      if (q == 0) out[1] = (s + dns * diag) / (dns * dns);
      if (q == 1) out[2] = (s + dnt * diag) / (dnt * dnt);
      if (q == 2) out[3] = s / (dns * dnt);
    }
  }
}

}  // namespace

extern "C" {

int dig3d_mmd_terms(const double* v, int64_t n_source, int64_t n_target, double kernel_mul, int32_t kernel_num,
                    double fix_sigma, double* workspace, int64_t workspace_len, double* out, void* stream) {
  DIG3D_REQUIRE(out && workspace && (v || n_source + n_target == 0) && n_source >= 0 && n_target >= 0 &&
                    kernel_num >= 1 && kernel_num <= kMaxKernels && workspace_len >= 3 && workspace_len / 3 <= (1 << 30),
                "mmd_terms: bad arguments (1 <= kernel_num <= %d, workspace of at least 3 doubles)", kMaxKernels);
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t n = n_source + n_target;
  const int grid = (int)(workspace_len / 3);
  bandwidth_kernel<<<1, kThreads, 0, s>>>(v, n, fix_sigma, out);
  DIG3D_LAUNCH_CHECK();
  if (kernel_mul == 2.0 && kernel_num == 5)
    pairs_kernel<true, 5><<<grid, kThreads, 0, s>>>(v, n_source, n_target, kernel_mul, kernel_num, out, workspace);
  else if (kernel_mul == 2.0)
    pairs_kernel<true, 0><<<grid, kThreads, 0, s>>>(v, n_source, n_target, kernel_mul, kernel_num, out, workspace);
  else
    pairs_kernel<false, 0><<<grid, kThreads, 0, s>>>(v, n_source, n_target, kernel_mul, kernel_num, out, workspace);
  DIG3D_LAUNCH_CHECK();
  reduce_kernel<<<1, kThreads, 0, s>>>(workspace, grid, n_source, n_target, kernel_mul, kernel_num, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
