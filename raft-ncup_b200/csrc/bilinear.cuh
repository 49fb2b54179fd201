// The bilinear sample of a strided fp32 plane that the video kernels share, with the coordinates clamped to the frame, its
// taps and weights on their own for a caller that combines the taps itself, the in-frame test, the finiteness test applied
// to flow values, and the rule by which a pixel follows its flow into the other frame.  Every operation is a __*_rn
// intrinsic, so nvcc contracts nothing into an FMA and rnc/restate.py gives the same bits on the host.
#pragma once
#include "eval_common.cuh"

namespace rnc {

__device__ __forceinline__ bool finite(float v) { return fabsf(v) <= 3.402823466e38f; }   // false for +-inf and NaN

// (x, y) lies in [0, W-1] x [0, H-1]; false for NaN
__device__ __forceinline__ bool inside(float x, float y, int H, int W) {
  return x >= 0.0f && x <= static_cast<float>(W - 1) && y >= 0.0f && y <= static_cast<float>(H - 1);
}

// the bilinear taps and weights at (px, py) with the coordinates clamped to [0, W-1] x [0, H-1]: tap i is (y[i >> 1], x[i & 1])
// and weighs w(i), so the taps (y0, x0), (y0, x1), (y1, x0), (y1, x1) weigh bx*by, ax*by, bx*ay, ax*ay
struct BilinearTaps {
  int x[2], y[2];
  float ax, ay, bx, by;
  __device__ __forceinline__ float w(int i) const { return __fmul_rn(i & 1 ? ax : bx, i & 2 ? ay : by); }
};

__device__ __forceinline__ BilinearTaps bilinear_taps(float px, float py, int H, int W) {
  px = fminf(fmaxf(px, 0.0f), static_cast<float>(W - 1));
  py = fminf(fmaxf(py, 0.0f), static_cast<float>(H - 1));
  const float x0 = floorf(px), y0 = floorf(py);
  const float ax = __fsub_rn(px, x0), ay = __fsub_rn(py, y0);
  const float bx = __fsub_rn(1.0f, ax), by = __fsub_rn(1.0f, ay);
  const int ix = static_cast<int>(x0), iy = static_cast<int>(y0);
  return {{ix, min(ix + 1, W - 1)}, {iy, min(iy + 1, H - 1)}, ax, ay, bx, by};
}

// plane (b, c) of im at (px, py): the four taps weighted and added in tap order
__device__ __forceinline__ float sample(const View& im, int b, int c, float px, float py, int H, int W) {
  const BilinearTaps t = bilinear_taps(px, py, H, W);
  float s = __fmul_rn(im.at(b, c, t.y[0], t.x[0]), t.w(0));
  s = __fadd_rn(s, __fmul_rn(im.at(b, c, t.y[0], t.x[1]), t.w(1)));
  s = __fadd_rn(s, __fmul_rn(im.at(b, c, t.y[1], t.x[0]), t.w(2)));
  return __fadd_rn(s, __fmul_rn(im.at(b, c, t.y[1], t.x[1]), t.w(3)));
}

// pixel (x, y) of image b follows its flow u = flow(b, y, x) to p' = (px, py) = (x, y) + u when u is finite, occ(b, y, x) == 0
// and p' lies in the frame
__device__ __forceinline__ bool follow(const View& flow, const MaskView& occ, int b, int y, int x, int H, int W, float& px,
                                       float& py) {
  const float ux = flow.at(b, 0, y, x), uy = flow.at(b, 1, y, x);
  px = __fadd_rn(static_cast<float>(x), ux);
  py = __fadd_rn(static_cast<float>(y), uy);
  return finite(ux) && finite(uy) && occ.at(b, y, x) == 0 && inside(px, py, H, W);
}

}  // namespace rnc
