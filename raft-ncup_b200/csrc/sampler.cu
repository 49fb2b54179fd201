// bilinear_sampler (core/utils/utils.py:59-73): F.grid_sample(img, grid, align_corners=True) with the grid given in
// pixel coordinates — bilinear, zero padding outside the image.  The standalone operator seam; inside the loop the
// lookup kernels fuse the same sampling rule (corr_lookup*.cu).
//   img    NCHW [N][C][H][W]      coords [N][h][w][2] (x, y) in pixels      out NCHW [N][C][h][w]
//   mask   optional [N][h][w][1]: 1 where 0 < x < W-1 and 0 < y < H-1 (utils.py:69-71 on the normalised grid)
#include "rnc_common.cuh"

namespace rnc {

__global__ void bilinear_sample_kernel(const float* __restrict__ img, const float* __restrict__ coords, int N, int C, int H, int W,
                                       int h, int w, float* __restrict__ out, float* __restrict__ mask) {
  const long long total = static_cast<long long>(N) * h * w;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(i / (h * w)), r = static_cast<int>(i - static_cast<long long>(n) * h * w);
    // the reference normalises to [-1, 1] and grid_sample maps back: reproduce the round trip's fp32 rounding
    float x = coords[2 * i], y = coords[2 * i + 1];
    const float xn = 2.f * x / static_cast<float>(W - 1) - 1.f, yn = 2.f * y / static_cast<float>(H - 1) - 1.f;
    x = (xn + 1.f) * 0.5f * static_cast<float>(W - 1);
    y = (yn + 1.f) * 0.5f * static_cast<float>(H - 1);
    const float fx = floorf(x), fy = floorf(y);
    const float ax = x - fx, ay = y - fy;
    const bool sane = fabsf(x) < 1.0e9f && fabsf(y) < 1.0e9f;
    const int x0 = sane ? static_cast<int>(fx) : -2, y0 = sane ? static_cast<int>(fy) : -2;
    const bool okx0 = x0 >= 0 && x0 < W, okx1 = x0 + 1 >= 0 && x0 + 1 < W;
    const bool oky0 = y0 >= 0 && y0 < H, oky1 = y0 + 1 >= 0 && y0 + 1 < H;
    const float w00 = (1.f - ax) * (1.f - ay), w10 = ax * (1.f - ay), w01 = (1.f - ax) * ay, w11 = ax * ay;
    for (int c = 0; c < C; ++c) {
      const float* p = img + (static_cast<size_t>(n) * C + c) * H * W;
      float v = 0.f;
      if (oky0 && okx0) v = fmaf(w00, p[y0 * W + x0], v);
      if (oky0 && okx1) v = fmaf(w10, p[y0 * W + x0 + 1], v);
      if (oky1 && okx0) v = fmaf(w01, p[(y0 + 1) * W + x0], v);
      if (oky1 && okx1) v = fmaf(w11, p[(y0 + 1) * W + x0 + 1], v);
      out[(static_cast<size_t>(n) * C + c) * h * w + r] = v;
    }
    if (mask) mask[i] = (xn > -1.f && yn > -1.f && xn < 1.f && yn < 1.f) ? 1.f : 0.f;
  }
}

}  // namespace rnc

using namespace rnc;

extern "C" int rnc_bilinear_sample_fwd(const float* img, const float* coords, int N, int C, int H, int W, int h, int w,
                                       float* out, float* mask, void* stream) {
  if (N <= 0 || C <= 0 || H <= 1 || W <= 1 || h <= 0 || w <= 0) return RNC_ERR_BAD_SHAPE;   // W-1 / H-1 divide (utils.py:63-64)
  if (!img || !coords || !out) return RNC_ERR_BAD_POINTER;
  long long blocks = (static_cast<long long>(N) * h * w + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  bilinear_sample_kernel<<<static_cast<int>(blocks), 256, 0, as_stream(stream)>>>(img, coords, N, C, H, W, h, w, out, mask);
  return after_launch();
}
