// Validation metrics (evaluate.py:88-182 validate_chairs / validate_sintel / validate_kitti) for a batch of float32 flows
// against their ground truth: per image, the number of valid pixels, of EPE < 1, < 3 and < 5, of KITTI outliers, and the fp64
// sum of the valid pixels' EPE.
//
// Each pixel is what torch computes in float32 on the host (eval_common.cuh's pixel_metrics, shared with
// rnc_region_metrics), valid where valid >= 0.5.
//
// Two launches of eval_common.cuh's reductions, no host synchronisation: CTA (x, b) of the first writes the partials of its
// 2048 pixels of image b to the workspace, and the second adds each image's partials in a fixed order.  An image's sums
// depend only on that image: not on B, on its position in the batch or on which GPU ran it.
#include "eval_common.cuh"

namespace rnc {
namespace {

struct FlowPixel {
  View flow, gt;
  View valid;                  // p == nullptr: every pixel is valid
  __device__ void operator()(MetricsPart& acc, int b, int y, int x) const {
    if (valid.p && !(valid.at(b, y, x) >= 0.5f)) return;
    const PixelMetrics m = pixel_metrics(flow.at(b, 0, y, x), flow.at(b, 1, y, x), gt.at(b, 0, y, x), gt.at(b, 1, y, x));
    acc.n[0] += 1;
    acc.n[1] += m.epe < 1.0f;
    acc.n[2] += m.epe < 3.0f;
    acc.n[3] += m.epe < 5.0f;
    acc.n[4] += m.outlier;
    acc.epe_sum += static_cast<double>(m.epe);
  }
};

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

size_t rnc_flow_metrics_workspace_bytes(int B, int H, int W) {
  return eval_shape_ok(B, H, W) ? static_cast<size_t>(B) * eval_blocks(H, W) * sizeof(MetricsPart) : 0;
}

int rnc_flow_metrics(const float* flow, long long fb, long long fc, long long fy, long long fx, const float* gt, long long gb,
                     long long gc, long long gy, long long gx, const float* valid, long long vb, long long vy, long long vx,
                     int B, int H, int W, long long* counts, double* epe_sum, void* workspace, size_t workspace_bytes,
                     void* stream) {
  if (!eval_shape_ok(B, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!flow || !gt || !counts || !epe_sum || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(flow, 4) || !aligned(gt, 4) || !aligned(valid, 4) || !aligned(counts, 8) || !aligned(epe_sum, 8) ||
      !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_flow_metrics_workspace_bytes(B, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const FlowPixel px{{flow, fb, fc, fy, fx}, {gt, gb, gc, gy, gx}, {valid, vb, 0, vy, vx}};
  const int nblk = eval_blocks(H, W);
  MetricsPart* parts = static_cast<MetricsPart*>(workspace);
  cta_partials_kernel<<<dim3(nblk, B), kEvalThreads, 0, s>>>(px, H, W, parts);
  if (int st = after_launch()) return st;
  return launch_image_reduce(parts, B, nblk, 1, MetricsStore{counts, epe_sum}, s);
}

}  // extern "C"
