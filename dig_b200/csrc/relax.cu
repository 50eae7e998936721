// Batched FIRE relaxation (Bitzek et al., 2006; the defaults ASE's FIRE popularised), each structure on its own.
//
//  * fire_step: one CTA per active structure.  Every per-structure reduction (F.v, |F|^2, |v|^2, |dr|^2 and the max of
//    |F_i|^2) is fp64 in a fixed order: thread t adds atoms t, t + kThreads, ... in ascending order, then a shared-memory
//    tree halves the kThreads partials.  No atomics, and the order depends only on the structure's atom count, so the
//    result is bit-identical between runs and for any batch the structure sits in.  fp64 products and sums are written
//    as __dmul_rn / __dadd_rn so that no FMA contraction changes that order (tests/fire_ref.py restates it).
//  * Positions and velocities stay fp32: each new value is computed in fp64 from the fp32 inputs and rounded once.
//    Fixed atoms are never written, so their positions keep their bits (even -0.0).
//  * relax_compact: the still-running structures (status 0) in batch order, their sub-batch graph_ptr, the atom map
//    (sub-batch atom -> batch atom) and the sub-batch's `batch` vector, from one exclusive scan in one CTA.
#include "common.cuh"

using namespace dig3d;

namespace {

constexpr int kThreads = 256;
constexpr int kNMin = 5;
constexpr double kFInc = 1.1, kFDec = 0.5, kAlphaStart = 0.1, kFAlpha = 0.99;

__device__ __forceinline__ double dot3(double ax, double ay, double az, double bx, double by, double bz) {
  return __dadd_rn(__dadd_rn(__dmul_rn(ax, bx), __dmul_rn(ay, by)), __dmul_rn(az, bz));
}

// max that keeps a NaN: a structure whose forces hold a NaN never counts as converged
__device__ __forceinline__ double max_nan(double a, double b) { return (b > a || b != b) ? b : a; }

// Sum (or max) of the kThreads partials in sh[], tree by halves; the result is returned to every thread.
template <bool kMax>
__device__ __forceinline__ double block_reduce(double x, double* sh) {
  const int t = threadIdx.x;
  sh[t] = x;
  __syncthreads();
#pragma unroll
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (t < o) sh[t] = kMax ? max_nan(sh[t], sh[t + o]) : __dadd_rn(sh[t], sh[t + o]);
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

struct Atom {
  double fx, fy, fz, vx, vy, vz;
  bool free_;
};

__device__ __forceinline__ Atom load_atom(const float* __restrict__ grad, const float* __restrict__ vel,
                                          const uint8_t* __restrict__ fixed, int64_t i_batch, int64_t i_sub) {
  Atom a;
  a.free_ = !(fixed && fixed[i_batch]);
  // the force is -dE/dpos (negation is exact); a fixed atom feels none and its velocity counts in no norm
  a.fx = a.free_ ? -(double)grad[3 * i_sub] : 0.0;
  a.fy = a.free_ ? -(double)grad[3 * i_sub + 1] : 0.0;
  a.fz = a.free_ ? -(double)grad[3 * i_sub + 2] : 0.0;
  a.vx = a.free_ ? (double)vel[3 * i_batch] : 0.0;
  a.vy = a.free_ ? (double)vel[3 * i_batch + 1] : 0.0;
  a.vz = a.free_ ? (double)vel[3 * i_batch + 2] : 0.0;
  return a;
}

__global__ void __launch_bounds__(kThreads) fire_step_kernel(
    float* __restrict__ pos, float* __restrict__ vel, const float* __restrict__ grad, const float* __restrict__ energy,
    int32_t n_out, const int32_t* __restrict__ graph_ptr, const int32_t* __restrict__ active,
    const int32_t* __restrict__ sub_ptr, const uint8_t* __restrict__ fixed, double* __restrict__ dt,
    double* __restrict__ alpha, int32_t* __restrict__ n_pos, int32_t* __restrict__ steps, int32_t* __restrict__ status,
    double* __restrict__ fmax_out, float* __restrict__ energy_out, float* __restrict__ force_out, double fmax2,
    int32_t max_steps, double dt_max, double max_step) {
  __shared__ double sh[kThreads];
  __shared__ double coef[4];                 // c_v, c_f, dt, clip scale
  __shared__ int go;
  const int a = blockIdx.x;
  const int s = active[a];
  const int64_t g0 = graph_ptr[s], n = graph_ptr[s + 1] - g0, f0 = sub_ptr[a];
  const int t = threadIdx.x;

  double p = 0.0, ff = 0.0, vv = 0.0, mx = 0.0;
  for (int64_t i = t; i < n; i += kThreads) {
    const Atom at = load_atom(grad, vel, fixed, g0 + i, f0 + i);
    if (force_out) {
      force_out[3 * (g0 + i)] = (float)at.fx;
      force_out[3 * (g0 + i) + 1] = (float)at.fy;
      force_out[3 * (g0 + i) + 2] = (float)at.fz;
    }
    const double f2 = dot3(at.fx, at.fy, at.fz, at.fx, at.fy, at.fz);
    p = __dadd_rn(p, dot3(at.fx, at.fy, at.fz, at.vx, at.vy, at.vz));
    ff = __dadd_rn(ff, f2);
    vv = __dadd_rn(vv, dot3(at.vx, at.vy, at.vz, at.vx, at.vy, at.vz));
    mx = max_nan(mx, f2);
  }
  p = block_reduce<false>(p, sh);
  ff = block_reduce<false>(ff, sh);
  vv = block_reduce<false>(vv, sh);
  mx = block_reduce<true>(mx, sh);

  if (t == 0) {
    fmax_out[s] = __dsqrt_rn(mx);
    if (energy) {
      float e = 0.f;
      for (int c = 0; c < n_out; ++c) e = __fadd_rn(e, energy[(int64_t)a * n_out + c]);
      energy_out[s] = e;
    }
    int st = 0;
    if (mx < fmax2) st = 1;                                      // no free atom: mx = 0, converged
    else if (steps[s] >= max_steps) st = 2;
    status[s] = st;
    go = st == 0;
    if (go) {
      double d = dt[s], al = alpha[s], cv = 1.0, cf = 0.0;
      int np = n_pos[s];
      if (steps[s] > 0) {                                        // the first step has no power check
        if (p > 0.0) {
          cv = __dadd_rn(1.0, -al);
          cf = __ddiv_rn(__dmul_rn(al, __dsqrt_rn(vv)), __dsqrt_rn(ff));
          if (np > kNMin) {
            d = fmin(__dmul_rn(d, kFInc), dt_max);
            al = __dmul_rn(al, kFAlpha);
          }
          np += 1;
        } else {
          cv = 0.0;
          al = kAlphaStart;
          d = __dmul_rn(d, kFDec);
          np = 0;
        }
      }
      dt[s] = d;
      alpha[s] = al;
      n_pos[s] = np;
      steps[s] += 1;
      coef[0] = cv;
      coef[1] = cf;
      coef[2] = d;
    }
  }
  __syncthreads();
  if (!go) return;
  const double cv = coef[0], cf = coef[1], d = coef[2];
  // v' = (c_v v + c_f F) + dt F;  dr = dt v'
  double dr2 = 0.0;
  for (int64_t i = t; i < n; i += kThreads) {
    const Atom at = load_atom(grad, vel, fixed, g0 + i, f0 + i);
    const double wx = __dmul_rn(d, __dadd_rn(__dadd_rn(__dmul_rn(cv, at.vx), __dmul_rn(cf, at.fx)), __dmul_rn(d, at.fx)));
    const double wy = __dmul_rn(d, __dadd_rn(__dadd_rn(__dmul_rn(cv, at.vy), __dmul_rn(cf, at.fy)), __dmul_rn(d, at.fy)));
    const double wz = __dmul_rn(d, __dadd_rn(__dadd_rn(__dmul_rn(cv, at.vz), __dmul_rn(cf, at.fz)), __dmul_rn(d, at.fz)));
    dr2 = __dadd_rn(dr2, dot3(wx, wy, wz, wx, wy, wz));
  }
  dr2 = block_reduce<false>(dr2, sh);
  if (t == 0) {
    const double norm = __dsqrt_rn(dr2);
    coef[3] = norm > max_step ? __ddiv_rn(max_step, norm) : 1.0;
  }
  __syncthreads();
  const bool clip = coef[3] != 1.0;
  const double scale = coef[3];
  for (int64_t i = t; i < n; i += kThreads) {
    const Atom at = load_atom(grad, vel, fixed, g0 + i, f0 + i);
    if (!at.free_) continue;
    const double ux = __dadd_rn(__dadd_rn(__dmul_rn(cv, at.vx), __dmul_rn(cf, at.fx)), __dmul_rn(d, at.fx));
    const double uy = __dadd_rn(__dadd_rn(__dmul_rn(cv, at.vy), __dmul_rn(cf, at.fy)), __dmul_rn(d, at.fy));
    const double uz = __dadd_rn(__dadd_rn(__dmul_rn(cv, at.vz), __dmul_rn(cf, at.fz)), __dmul_rn(d, at.fz));
    double rx = __dmul_rn(d, ux), ry = __dmul_rn(d, uy), rz = __dmul_rn(d, uz);
    if (clip) {
      rx = __dmul_rn(rx, scale);
      ry = __dmul_rn(ry, scale);
      rz = __dmul_rn(rz, scale);
    }
    const int64_t j = 3 * (g0 + i);
    vel[j] = __double2float_rn(ux);
    vel[j + 1] = __double2float_rn(uy);
    vel[j + 2] = __double2float_rn(uz);
    pos[j] = __double2float_rn(__dadd_rn((double)pos[j], rx));
    pos[j + 1] = __double2float_rn(__dadd_rn((double)pos[j + 1], ry));
    pos[j + 2] = __double2float_rn(__dadd_rn((double)pos[j + 2], rz));
  }
}

constexpr int kScanThreads = 1024;

// Inclusive block scan of two int64 counters (warp shuffles, then the warp totals).
__device__ __forceinline__ void block_scan2(int64_t& x, int64_t& y, int64_t* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t ox = __shfl_up_sync(0xffffffffu, x, o), oy = __shfl_up_sync(0xffffffffu, y, o);
    if (lane >= o) x += ox, y += oy;
  }
  if (lane == 31) sh[w] = x, sh[32 + w] = y;
  __syncthreads();
  if (w == 0) {
    int64_t a = sh[lane], b = sh[32 + lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t oa = __shfl_up_sync(0xffffffffu, a, o), ob = __shfl_up_sync(0xffffffffu, b, o);
      if (lane >= o) a += oa, b += ob;
    }
    sh[lane] = a, sh[32 + lane] = b;
  }
  __syncthreads();
  if (w > 0) x += sh[w - 1], y += sh[32 + w - 1];
}

// Thread t owns structures [t * per, (t + 1) * per): count, one block scan, then write in batch order.
__global__ void __launch_bounds__(kScanThreads) compact_scan_kernel(const int32_t* __restrict__ status,
                                                                    const int32_t* __restrict__ graph_ptr,
                                                                    int64_t n_graphs, int32_t* __restrict__ active,
                                                                    int32_t* __restrict__ new_ptr,
                                                                    int32_t* __restrict__ counts) {
  __shared__ int64_t sh[64];
  const int64_t per = (n_graphs + kScanThreads - 1) / kScanThreads;
  const int64_t lo = min(n_graphs, threadIdx.x * per), hi = min(n_graphs, lo + per);
  int64_t k = 0, m = 0;
  for (int64_t s = lo; s < hi; ++s)
    if (status[s] == 0) k += 1, m += graph_ptr[s + 1] - graph_ptr[s];
  const int64_t k_own = k, m_own = m;
  block_scan2(k, m, sh);
  k -= k_own, m -= m_own;                                        // exclusive
  for (int64_t s = lo; s < hi; ++s) {
    if (status[s] != 0) continue;
    active[k] = (int32_t)s;
    new_ptr[k] = (int32_t)m;
    k += 1, m += graph_ptr[s + 1] - graph_ptr[s];
  }
  if (threadIdx.x == kScanThreads - 1) {
    new_ptr[k] = (int32_t)m;
    counts[0] = (int32_t)k;
    counts[1] = (int32_t)m;
  }
}

constexpr int kFillWarps = 8;

// One warp per active slot (slots past the active count exit): atom map and batch vector of the sub-batch.
__global__ void __launch_bounds__(32 * kFillWarps) compact_fill_kernel(const int32_t* __restrict__ graph_ptr,
                                                                       const int32_t* __restrict__ active,
                                                                       const int32_t* __restrict__ new_ptr,
                                                                       const int32_t* __restrict__ counts,
                                                                       int32_t* __restrict__ atom_map,
                                                                       int64_t* __restrict__ new_batch) {
  const int64_t a = (int64_t)blockIdx.x * kFillWarps + (threadIdx.x >> 5);
  if (a >= counts[0]) return;
  const int s = active[a];
  const int32_t g0 = graph_ptr[s], n = graph_ptr[s + 1] - g0, o = new_ptr[a];
  for (int j = threadIdx.x & 31; j < n; j += 32) {
    atom_map[o + j] = g0 + j;
    new_batch[o + j] = a;
  }
}

}  // namespace

extern "C" {

int dig3d_fire_step(float* pos, float* vel, const float* grad, const float* energy, int32_t n_out,
                    const int32_t* graph_ptr, const int32_t* active, const int32_t* sub_ptr, int64_t n_active,
                    const uint8_t* fixed, double* dt, double* alpha, int32_t* n_pos, int32_t* steps, int32_t* status,
                    double* fmax_out, float* energy_out, float* force_out, double fmax, int32_t max_steps,
                    double dt_max, double max_step, void* stream) {
  DIG3D_REQUIRE(n_active >= 0 && n_active < (1ll << 31), "fire_step: bad n_active (%lld)", (long long)n_active);
  DIG3D_REQUIRE(n_active == 0 || (pos && vel && graph_ptr && active && sub_ptr && dt && alpha && n_pos && steps &&
                                  status && fmax_out && grad),
                "fire_step: a required pointer is NULL");
  DIG3D_REQUIRE(!energy || (energy_out && n_out > 0), "fire_step: energy needs energy_out and n_out > 0");
  DIG3D_REQUIRE(fmax > 0.0 && fmax * fmax <= 1.7e308 && max_steps >= 0 && dt_max > 0.0 && max_step > 0.0,
                "fire_step: bad parameters (fmax > 0 finite, max_steps >= 0, dt_max > 0, max_step > 0)");
  if (n_active == 0) return DIG3D_OK;
  fire_step_kernel<<<(unsigned)n_active, kThreads, 0, (cudaStream_t)stream>>>(
      pos, vel, grad, energy, n_out, graph_ptr, active, sub_ptr, fixed, dt, alpha, n_pos, steps, status, fmax_out,
      energy_out, force_out, fmax * fmax, max_steps, dt_max, max_step);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_relax_compact(const int32_t* status, const int32_t* graph_ptr, int64_t n_graphs, int32_t* active,
                        int32_t* new_ptr, int32_t* atom_map, int64_t* new_batch, int32_t* counts, void* stream) {
  DIG3D_REQUIRE(n_graphs >= 0 && n_graphs < (1ll << 31), "relax_compact: bad n_graphs (%lld)", (long long)n_graphs);
  DIG3D_REQUIRE(graph_ptr && new_ptr && counts && (n_graphs == 0 || (status && active && atom_map && new_batch)),
                "relax_compact: a required pointer is NULL");
  compact_scan_kernel<<<1, kScanThreads, 0, (cudaStream_t)stream>>>(status, graph_ptr, n_graphs, active, new_ptr,
                                                                     counts);
  DIG3D_LAUNCH_CHECK();
  if (n_graphs == 0) return DIG3D_OK;
  compact_fill_kernel<<<ceil_div(n_graphs, kFillWarps), 32 * kFillWarps, 0, (cudaStream_t)stream>>>(
      graph_ptr, active, new_ptr, counts, atom_map, new_batch);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
