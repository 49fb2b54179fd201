// The fp64 homography arithmetic of video stabilization (stabilize.cu) and its full-frame fill (stabilize_fill.cu).  Every
// operation is rounded once, with no FMA, in the order rnc/stabilize.py's host restatements write it.
#pragma once
#include <cuda_runtime.h>

namespace rnc {

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

struct M3 {                                   // a row-major 3x3 matrix
  double m[9];
};

// pi(m p) = ((m0 x + m1 y) + m2) / ((m6 x + m7 y) + m8) and the same for y: false when the denominator is not > 0
__device__ __forceinline__ bool project(const double* m, double x, double y, double& ox, double& oy) {
  const double X = dadd(dadd(dmul(m[0], x), dmul(m[1], y)), m[2]);
  const double Y = dadd(dadd(dmul(m[3], x), dmul(m[4], y)), m[5]);
  const double w = dadd(dadd(dmul(m[6], x), dmul(m[7], y)), m[8]);
  ox = ddiv(X, w);
  oy = ddiv(Y, w);
  return w > 0.0;
}

__device__ __forceinline__ double det2(double a, double b, double c, double d) { return dsub(dmul(a, b), dmul(c, d)); }

// the adjugate of a, divided by its [2][2]
__device__ __forceinline__ M3 inv_norm(const double* a) {
  M3 C;
  C.m[0] = det2(a[4], a[8], a[5], a[7]);
  C.m[1] = det2(a[2], a[7], a[1], a[8]);
  C.m[2] = det2(a[1], a[5], a[2], a[4]);
  C.m[3] = det2(a[5], a[6], a[3], a[8]);
  C.m[4] = det2(a[0], a[8], a[2], a[6]);
  C.m[5] = det2(a[2], a[3], a[0], a[5]);
  C.m[6] = det2(a[3], a[7], a[4], a[6]);
  C.m[7] = det2(a[1], a[6], a[0], a[7]);
  C.m[8] = det2(a[0], a[4], a[1], a[3]);
  const double z = C.m[8];
#pragma unroll
  for (int k = 0; k < 9; ++k) C.m[k] = ddiv(C.m[k], z);
  return C;
}

}  // namespace rnc
