// Validation metrics (evaluate.py:88-182 validate_chairs / validate_sintel / validate_kitti) for a batch of float32 flows
// against their ground truth: per image, the number of valid pixels, of EPE < 1, < 3 and < 5, of KITTI outliers, and the fp64
// sum of the valid pixels' EPE.
//
// Each pixel is what torch computes in float32 on the host (pixel_metrics.cuh, shared with rnc_region_metrics), valid where
// valid >= 0.5.
//
// Two kernels, no host synchronisation: CTA (x, b) of the first writes the partials of its 2048 pixels of image b to the
// workspace, and the second adds each image's partials in a fixed order (a warp per image: lane-strided sums, then a fixed
// shuffle tree).  The grid's x extent depends only on H*W, so an image's sums depend only on that image: not on B, on its
// position in the batch or on which GPU ran it.
#include "pixel_metrics.cuh"
#include "rnc_common.cuh"

namespace rnc {
namespace {

constexpr int kMetThreads = 256;
constexpr int kMetPerThread = 8;
constexpr int kMetPerCta = kMetThreads * kMetPerThread;
constexpr int kMetCounts = 5;   // valid, epe < 1, < 3, < 5, KITTI outliers

struct MetricsPart {            // one CTA's partials; 32 bytes
  double epe_sum;
  unsigned n[kMetCounts];
  unsigned pad;
};

struct MetricsArgs {
  const float* flow;
  long long fb, fc, fy, fx;
  const float* gt;
  long long gb, gc, gy, gx;
  const float* valid;          // nullptr: every pixel is valid
  long long vb, vy, vx;
  int H, W;
};

__global__ void __launch_bounds__(kMetThreads) metrics_part_kernel(MetricsArgs a, MetricsPart* __restrict__ parts) {
  const int b = blockIdx.y;
  const int hw = a.H * a.W;
  double sum = 0.0;
  unsigned n[kMetCounts] = {0, 0, 0, 0, 0};
  for (int p = blockIdx.x * kMetPerCta + threadIdx.x, e = 0; e < kMetPerThread && p < hw; ++e, p += kMetThreads) {
    const int y = p / a.W, x = p - y * a.W;
    if (a.valid && !(a.valid[b * a.vb + y * a.vy + x * a.vx] >= 0.5f)) continue;
    const float* f = a.flow + b * a.fb + y * a.fy + x * a.fx;
    const float* g = a.gt + b * a.gb + y * a.gy + x * a.gx;
    const PixelMetrics m = pixel_metrics(f[0], f[a.fc], g[0], g[a.gc]);
    n[0] += 1;
    n[1] += m.epe < 1.0f;
    n[2] += m.epe < 3.0f;
    n[3] += m.epe < 5.0f;
    n[4] += m.outlier;
    sum += static_cast<double>(m.epe);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
#pragma unroll
  for (int c = 0; c < kMetCounts; ++c) n[c] = __reduce_add_sync(0xffffffffu, n[c]);
  __shared__ double ssum[kMetThreads / 32];
  __shared__ unsigned sn[kMetThreads / 32][kMetCounts];
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    ssum[warp] = sum;
#pragma unroll
    for (int c = 0; c < kMetCounts; ++c) sn[warp][c] = n[c];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    MetricsPart out{};
    for (int w = 0; w < kMetThreads / 32; ++w) {
      out.epe_sum += ssum[w];
#pragma unroll
      for (int c = 0; c < kMetCounts; ++c) out.n[c] += sn[w][c];
    }
    parts[static_cast<long long>(b) * gridDim.x + blockIdx.x] = out;
  }
}

// a warp per image: parts [B][nblk] -> counts [B][5], epe_sum [B]
__global__ void __launch_bounds__(kMetThreads) metrics_reduce_kernel(const MetricsPart* __restrict__ parts, int B, int nblk,
                                                                     long long* __restrict__ counts,
                                                                     double* __restrict__ epe_sum) {
  const int b = blockIdx.x * (kMetThreads / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return;
  double sum = 0.0;
  unsigned long long n[kMetCounts] = {0, 0, 0, 0, 0};
  for (int k = lane; k < nblk; k += 32) {
    const MetricsPart& q = parts[static_cast<long long>(b) * nblk + k];
    sum += q.epe_sum;
#pragma unroll
    for (int c = 0; c < kMetCounts; ++c) n[c] += q.n[c];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
#pragma unroll
    for (int c = 0; c < kMetCounts; ++c) n[c] += __shfl_xor_sync(0xffffffffu, n[c], o);
  }
  if (lane == 0) {
    epe_sum[b] = sum;
#pragma unroll
    for (int c = 0; c < kMetCounts; ++c) counts[static_cast<long long>(b) * kMetCounts + c] = static_cast<long long>(n[c]);
  }
}

bool shape_ok(int B, int H, int W) {
  return B > 0 && H > 0 && W > 0 && B <= 65535 && static_cast<long long>(H) * W < (1ll << 30);
}

int metrics_blocks(int H, int W) { return (H * W + kMetPerCta - 1) / kMetPerCta; }

bool aligned(const void* p, uintptr_t n) { return (reinterpret_cast<uintptr_t>(p) & (n - 1)) == 0; }

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

size_t rnc_flow_metrics_workspace_bytes(int B, int H, int W) {
  return shape_ok(B, H, W) ? static_cast<size_t>(B) * metrics_blocks(H, W) * sizeof(MetricsPart) : 0;
}

int rnc_flow_metrics(const float* flow, long long fb, long long fc, long long fy, long long fx, const float* gt, long long gb,
                     long long gc, long long gy, long long gx, const float* valid, long long vb, long long vy, long long vx,
                     int B, int H, int W, long long* counts, double* epe_sum, void* workspace, size_t workspace_bytes,
                     void* stream) {
  if (!shape_ok(B, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!flow || !gt || !counts || !epe_sum || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(flow, 4) || !aligned(gt, 4) || !aligned(valid, 4) || !aligned(counts, 8) || !aligned(epe_sum, 8) ||
      !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_flow_metrics_workspace_bytes(B, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const MetricsArgs a{flow, fb, fc, fy, fx, gt, gb, gc, gy, gx, valid, vb, vy, vx, H, W};
  const int nblk = metrics_blocks(H, W);
  MetricsPart* parts = static_cast<MetricsPart*>(workspace);
  metrics_part_kernel<<<dim3(nblk, B), kMetThreads, 0, s>>>(a, parts);
  if (int st = after_launch()) return st;
  const int warps = kMetThreads / 32;
  metrics_reduce_kernel<<<(B + warps - 1) / warps, kMetThreads, 0, s>>>(parts, B, nblk, counts, epe_sum);
  return after_launch();
}

}  // extern "C"
