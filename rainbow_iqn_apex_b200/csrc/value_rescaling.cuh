// Value-function rescaling (Pohlen et al. 2018, "Observe and Look Further"): the transformed Bellman operator's
//   h(x) = sign(x) (sqrt(|x| + 1) - 1) + eps x   and its inverse,
// in the cancellation-free forms below (every term non-negative), evaluated in double with explicitly rounded operations
// so that nvcc contracts nothing into an FMA: each result is the one numpy float64 computes with the same operations in
// the same order (oracle/value_rescaling.py).
//   h(x):     a = |x|;  m = a / (sqrt(a + 1) + 1);  h = copysign(m, x) + eps x
//   h^-1(y):  a = |y|;  u = (a + 1) + eps;  s = sqrt(1 + (4 eps) u);  d = ((4u) a) / (((2u - 1) + s) (s + 1));
//             h^-1 = copysign(d (d + 2), y)          (d = sqrt(x + 1) - 1 for x = h^-1(y))
#pragma once
#include <cuda_runtime.h>

namespace riqn {

__device__ __forceinline__ double vr_h(double x, double eps) {
  const double a = fabs(x);
  const double m = __ddiv_rn(a, __dadd_rn(__dsqrt_rn(__dadd_rn(a, 1.0)), 1.0));
  return __dadd_rn(copysign(m, x), __dmul_rn(eps, x));
}

__device__ __forceinline__ double vr_h_inv(double y, double eps) {
  const double a = fabs(y);
  const double u = __dadd_rn(__dadd_rn(a, 1.0), eps);
  const double s = __dsqrt_rn(__dadd_rn(1.0, __dmul_rn(__dmul_rn(4.0, eps), u)));
  const double den = __dmul_rn(__dadd_rn(__dsub_rn(__dmul_rn(2.0, u), 1.0), s), __dadd_rn(s, 1.0));
  const double d = __ddiv_rn(__dmul_rn(__dmul_rn(4.0, u), a), den);
  return copysign(__dmul_rn(d, __dadd_rn(d, 2.0)), y);
}

// eps as the entry points accept it: finite and >= 0
static inline bool vr_eps_ok(float eps) { return eps >= 0.f && isfinite(eps); }

}  // namespace riqn
