// Forward-mode dual numbers (value, tangent) for kernels that evaluate a first-order gradient, written once, along a
// direction: the tangent of the gradient is a Hessian-vector product (csrc/train_geom.cu, csrc/comenet.cu).
#pragma once

namespace dig3d {

struct dual {
  float v, d;
};
__device__ __forceinline__ float val(float a) { return a; }
__device__ __forceinline__ float val(dual a) { return a.v; }
__device__ __forceinline__ dual operator+(dual a, dual b) { return {a.v + b.v, a.d + b.d}; }
__device__ __forceinline__ dual operator-(dual a, dual b) { return {a.v - b.v, a.d - b.d}; }
__device__ __forceinline__ dual operator-(dual a) { return {-a.v, -a.d}; }
__device__ __forceinline__ dual operator*(dual a, dual b) { return {a.v * b.v, a.d * b.v + a.v * b.d}; }
__device__ __forceinline__ dual operator/(dual a, dual b) {
  const float q = a.v / b.v;
  return {q, (a.d - q * b.d) / b.v};
}
__device__ __forceinline__ float sqrt_t(float a) { return sqrtf(a); }
__device__ __forceinline__ dual sqrt_t(dual a) {
  const float r = sqrtf(a.v);
  return {r, r > 0.f ? a.d / (2.f * r) : 0.f};
}

}  // namespace dig3d
