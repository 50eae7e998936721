// Head-to-lane mapping of G-SphereNet's attention pooling at any head width d_k (gsphere.cu attention_dk_kernel,
// gsphere_train.cu att_fwd_dk_kernel / att_bwd_dk_kernel).
//
// A head occupies a segment of `seg` lanes: d_k rounded up to a power of two below 32 (32 / seg heads share a warp),
// 32 from 32 up (one head per warp).  Lane s of a segment owns the channels s, s + seg, s + 2 seg, ... < d_k, the
// `slices` of the head; lanes past d_k add +0.  A dot product over the head is the lane's products summed in slice
// order, then the segment's xor butterfly, so at d_k = 32 it is the op sequence of the d_k = 32 kernels.  Loops that
// accumulate per channel run once per slice and recompute the scores, so every accumulator is a register at any d_k.
// One CTA per query; its warps step through the head groups.
#pragma once
#include <math.h>

namespace dig3d {

struct AttShape {
  int seg, threads;
  float scale;   // sqrt(d_k) in fp64 rounded to fp32: att.py divides an fp32 tensor by an fp64 scalar tensor
};

inline AttShape att_shape(int n_heads, int d_k) {
  int seg = 1;
  while (seg < d_k && seg < 32) seg <<= 1;
  const int per_warp = 32 / seg;
  const int64_t warps = ((int64_t)n_heads + per_warp - 1) / per_warp;
  return {seg, 32 * (int)(warps < 32 ? warps : 32), (float)sqrt((double)d_k)};
}

__device__ __forceinline__ float seg_sum(float v, int seg) {
  for (int o = seg >> 1; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct HeadLanes {
  int64_t width;   // n_heads * d_k
  int h, s, seg, slices, d_k;
  bool head;
  __device__ bool owns(int i) const { return head && s + i * seg < d_k; }
  __device__ int64_t col(int i) const { return (int64_t)h * d_k + s + i * seg; }
  // sum_c a[c] b[c] over the head's channels of rows a, b (both offset to the head's first channel)
  __device__ float dot(const float* __restrict__ a, const float* __restrict__ b) const {
    float p = __fmul_rn(owns(0) ? a[s] : 0.f, owns(0) ? b[s] : 0.f);
    for (int i = 1; i < slices; ++i)
      if (owns(i)) p = __fadd_rn(p, __fmul_rn(a[s + i * seg], b[s + i * seg]));
    return seg_sum(p, seg);
  }
};

__device__ __forceinline__ HeadLanes head_lanes(int h0, int n_heads, int d_k, int seg) {
  const int lane = threadIdx.x & 31;
  HeadLanes l;
  l.width = (int64_t)n_heads * d_k;
  l.h = h0 + lane / seg;
  l.s = lane & (seg - 1);
  l.seg = seg;
  l.slices = (d_k + seg - 1) / seg;
  l.d_k = d_k;
  l.head = l.h < n_heads;
  return l;
}

}  // namespace dig3d
