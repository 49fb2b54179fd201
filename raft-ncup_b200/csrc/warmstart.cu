// Warm-start forward interpolation of a flow field (core/utils/utils.py:28-56, used by evaluate.py:38-40 with
// warm_start=True): every source pixel is pushed along its flow, samples landing strictly inside the image are kept, and
// each grid point takes the flow of the NEAREST kept sample (scipy.interpolate.griddata(method='nearest')).  The reference
// does this on the CPU with a k-d tree per frame; here it is an exact brute-force nearest-neighbour search on the GPU
// (H8*W8 = 7040 grid points x 7040 samples = 5e7 distance tests per frame).
#include "rnc_common.cuh"

namespace rnc {

constexpr int FI_THREADS = 256;

// flow [B][2][H][W] -> out [B][2][H][W].  Rows b >= nfwd splat along -flow and still carry +flow: the backward warm start
// (each sample moves to x - b(x) with the value b(x)), which is -forward_interpolate(-b) bit for bit.
__global__ void __launch_bounds__(FI_THREADS)
forward_interpolate_kernel(const float* __restrict__ flow, int H, int W, int nfwd, float* __restrict__ out) {
  __shared__ double sx[FI_THREADS], sy[FI_THREADS];     // sample positions in fp64, as numpy computes them (int64 + float32)
  __shared__ float sdx[FI_THREADS], sdy[FI_THREADS];
  const int b = blockIdx.y, HW = H * W;
  const bool back = b >= nfwd;
  const float* fx = flow + (size_t)b * 2 * HW;
  const float* fy = fx + HW;
  const int g = blockIdx.x * FI_THREADS + threadIdx.x;          // this thread's grid point
  const double gx = (double)(g % W), gy = (double)(g / W);
  double best = INFINITY;
  float bdx = 0.f, bdy = 0.f;                    // fill_value = 0 when no sample is valid
  for (int s0 = 0; s0 < HW; s0 += FI_THREADS) {
    const int s = s0 + threadIdx.x;
    double x1 = NAN, y1 = NAN;
    float dx = 0.f, dy = 0.f;
    if (s < HW) {
      dx = fx[s]; dy = fy[s];
      const double px = (double)(s % W) + (double)(back ? -dx : dx), py = (double)(s / W) + (double)(back ? -dy : dy);
      if (px > 0.0 && px < (double)W && py > 0.0 && py < (double)H) { x1 = px; y1 = py; }   // utils.py:44 `valid`
    }
    sx[threadIdx.x] = x1; sy[threadIdx.x] = y1; sdx[threadIdx.x] = dx; sdy[threadIdx.x] = dy;
    __syncthreads();
    const int n = min(FI_THREADS, HW - s0);
    for (int j = 0; j < n; ++j) {
      const double ex = sx[j] - gx, ey = sy[j] - gy;
      const double d2 = ex * ex + ey * ey;                           // NaN for invalid samples -> comparison false
      if (d2 < best) { best = d2; bdx = sdx[j]; bdy = sdy[j]; }
    }
    __syncthreads();
  }
  if (g < HW) {
    out[(size_t)b * 2 * HW + g] = bdx;
    out[(size_t)b * 2 * HW + HW + g] = bdy;
  }
}

}  // namespace rnc

using namespace rnc;

extern "C" int rnc_forward_interpolate_fwd(const float* flow, int B, int H, int W, float* out, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return RNC_ERR_BAD_SHAPE;
  if (!flow || !out) return RNC_ERR_BAD_POINTER;
  dim3 grid((H * W + FI_THREADS - 1) / FI_THREADS, B);
  forward_interpolate_kernel<<<grid, FI_THREADS, 0, as_stream(stream)>>>(flow, H, W, B, out);
  return after_launch();
}

extern "C" int rnc_forward_interpolate_bidir_fwd(const float* flow, int B, int H, int W, float* out, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return RNC_ERR_BAD_SHAPE;
  if (!flow || !out) return RNC_ERR_BAD_POINTER;
  dim3 grid((H * W + FI_THREADS - 1) / FI_THREADS, 2 * B);
  forward_interpolate_kernel<<<grid, FI_THREADS, 0, as_stream(stream)>>>(flow, H, W, B, out);
  return after_launch();
}
