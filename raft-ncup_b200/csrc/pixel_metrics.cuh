// The float32 per-pixel arithmetic of the validation metrics, shared by rnc_flow_metrics (flow_metrics.cu) and
// rnc_region_metrics (region_metrics.cu) so that the two count every pixel the same way.
//
// Each value is what torch computes in float32 on the host: dx = flow - gt, epe = sqrt(dx*dx + dy*dy), mag the same from gt,
// outlier = epe > 3 & epe / mag > 0.05 (a Python float compared with a float32 tensor is rounded to float32).  The *_rn
// intrinsics keep nvcc from contracting any of it into an FMA, and IEEE division gives x/0 = inf and 0/0 = NaN, so a
// zero-magnitude ground truth, NaN and inf count as the torch comparisons count them.
#pragma once

namespace rnc {

struct PixelMetrics {
  float epe, mag;
  bool outlier;
};

__device__ __forceinline__ PixelMetrics pixel_metrics(float f0, float f1, float g0, float g1) {
  const float dx = __fsub_rn(f0, g0), dy = __fsub_rn(f1, g1);
  const float epe = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
  const float mag = __fsqrt_rn(__fadd_rn(__fmul_rn(g0, g0), __fmul_rn(g1, g1)));
  return {epe, mag, static_cast<bool>((epe > 3.0f) & (__fdiv_rn(epe, mag) > 0.05f))};
}

}  // namespace rnc
