// The bilinear sample of a strided fp32 plane that frame interpolation (interp.cu) and point tracking (track.cu) share, with
// the coordinates clamped to the frame, the finiteness test both apply to flow values, and the same taps and weights on their
// own for label propagation (segment.cu).  Every operation is a __*_rn
// intrinsic, so nvcc contracts nothing into an FMA and rnc/interp.py:_sample gives the same bits on the host.
#pragma once
#include "eval_common.cuh"

namespace rnc {

// plane (b, c) of im at (px, py), bilinear with the coordinates clamped to [0, W-1] x [0, H-1]: the taps (y0, x0), (y0, x1),
// (y1, x0), (y1, x1) weighted bx*by, ax*by, bx*ay, ax*ay and added in that order
__device__ __forceinline__ float sample(const View& im, int b, int c, float px, float py, int H, int W) {
  px = fminf(fmaxf(px, 0.0f), static_cast<float>(W - 1));
  py = fminf(fmaxf(py, 0.0f), static_cast<float>(H - 1));
  const float x0 = floorf(px), y0 = floorf(py);
  const float ax = __fsub_rn(px, x0), ay = __fsub_rn(py, y0);
  const float bx = __fsub_rn(1.0f, ax), by = __fsub_rn(1.0f, ay);
  const int ix = static_cast<int>(x0), iy = static_cast<int>(y0);
  const int ix1 = min(ix + 1, W - 1), iy1 = min(iy + 1, H - 1);
  float s = __fmul_rn(im.at(b, c, iy, ix), __fmul_rn(bx, by));
  s = __fadd_rn(s, __fmul_rn(im.at(b, c, iy, ix1), __fmul_rn(ax, by)));
  s = __fadd_rn(s, __fmul_rn(im.at(b, c, iy1, ix), __fmul_rn(bx, ay)));
  return __fadd_rn(s, __fmul_rn(im.at(b, c, iy1, ix1), __fmul_rn(ax, ay)));
}

__device__ __forceinline__ bool finite(float v) { return fabsf(v) <= 3.402823466e38f; }   // false for +-inf and NaN

// sample's four taps and weights at (px, py), for a caller that combines the taps itself (segment.cu's label vote): tap i is
// (y[i >> 1], x[i & 1]) and weighs w[i], in sample's order and with its clamp and roundings
struct BilinearTaps {
  int x[2], y[2];
  float w[4];
};

__device__ __forceinline__ BilinearTaps bilinear_taps(float px, float py, int H, int W) {
  px = fminf(fmaxf(px, 0.0f), static_cast<float>(W - 1));
  py = fminf(fmaxf(py, 0.0f), static_cast<float>(H - 1));
  const float x0 = floorf(px), y0 = floorf(py);
  const float ax = __fsub_rn(px, x0), ay = __fsub_rn(py, y0);
  const float bx = __fsub_rn(1.0f, ax), by = __fsub_rn(1.0f, ay);
  const int ix = static_cast<int>(x0), iy = static_cast<int>(y0);
  return {{ix, min(ix + 1, W - 1)},
          {iy, min(iy + 1, H - 1)},
          {__fmul_rn(bx, by), __fmul_rn(ax, by), __fmul_rn(bx, ay), __fmul_rn(ax, ay)}};
}

}  // namespace rnc
