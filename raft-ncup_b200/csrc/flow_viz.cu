// Flow visualisation (core/utils/flow_viz.py:240-275 flow_to_image, :196-237 compute_color, :134-193 make_color_wheel) for a
// batch of float32 flows, as the reference computes it under numpy 2.x (NEP 50) promotion.
//
// Two kernels, no host synchronisation between them:
//   1. per image, the maximum radius of the flow with its unknown pixels (|u| or |v| > 1e7) zeroed.  The radius is >= +0, so
//      its float bits order as unsigned integers and an atomicMax over them is exact in any order.  A NaN radius stores
//      0xffffffff: numpy's max is then NaN and the reference's Python `max(-1, nan)` is -1;
//   2. per pixel, the colour: normalise by maxrad + eps, angle -> colour-wheel interpolation -> saturation by radius.
// Every step is rounded as numpy rounds it: the radius and its maximum in float32, then float64 from the normalisation on,
// because np.finfo(float).eps is a float64 scalar.  The *_rn intrinsics keep nvcc from contracting any of them into an FMA:
// the max-radius pixel's recomputed radius lands within an ulp or two of 1 and takes the 0.75 branch when it rounds above,
// so the roundings change colours.  The arc tangent is CUDA's float64 atan2 (within 2 ulp).
#include "rnc_common.cuh"

namespace rnc {
namespace {

constexpr int kVizThreads = 256;
constexpr int kVizPerThread = 8;                 // pass 1: pixels per thread
constexpr int kWheel = 55;                       // RY + YG + GC + CB + BM + MR
constexpr float kUnknown = 1e7f;                 // UNKNOWN_FLOW_THRESH
constexpr double kEps = 2.220446049250313e-16;   // np.finfo(float).eps
constexpr unsigned kNanBits = 0xffffffffu;

// Middlebury colour wheel, RGB: segments red-yellow 15, yellow-green 6, green-cyan 4, cyan-blue 11, blue-magenta 13,
// magenta-red 6.  In each segment one channel ramps up or down by floor(255 * j / n), which integer division gives
// exactly, one is held at 255 and one at 0.
struct WheelTable {
  unsigned char rgb[kWheel][3];
};
constexpr WheelTable make_wheel() {
  constexpr int len[6] = {15, 6, 4, 11, 13, 6};
  constexpr int ramp_ch[6] = {1, 0, 2, 1, 0, 2};   // the channel that ramps
  constexpr int rising[6] = {1, 0, 1, 0, 1, 0};    // ... up (1) or down (0)
  constexpr int full_ch[6] = {0, 1, 1, 2, 2, 0};   // the channel held at 255
  WheelTable t{};
  int k = 0;
  for (int s = 0; s < 6; ++s)
    for (int j = 0; j < len[s]; ++j, ++k) {
      const int ramp = 255 * j / len[s];
      t.rgb[k][ramp_ch[s]] = static_cast<unsigned char>(rising[s] ? ramp : 255 - ramp);
      t.rgb[k][full_ch[s]] = 255;
    }
  return t;
}
__constant__ WheelTable kWheelRGB = make_wheel();

struct VizArgs {
  const float* flow;
  long long sb, sc, sy, sx;
  int H, W;
  unsigned char* out;
  unsigned* maxbits;   // [B]
};

__device__ __forceinline__ void load_uv(const VizArgs& a, int b, int p, float& u, float& v) {
  const int y = p / a.W, x = p - y * a.W;
  const float* f = a.flow + b * a.sb + y * a.sy + x * a.sx;
  u = f[0];
  v = f[a.sc];
  if (fabsf(u) > kUnknown || fabsf(v) > kUnknown) u = v = 0.0f;   // inf is unknown; NaN is not
}

__device__ __forceinline__ float radius(float u, float v) {
  return __fsqrt_rn(__fadd_rn(__fmul_rn(u, u), __fmul_rn(v, v)));
}

__global__ void __launch_bounds__(kVizThreads) viz_maxrad_kernel(VizArgs a) {
  const int b = blockIdx.y;
  const int hw = a.H * a.W;
  unsigned m = 0;
  for (int p = blockIdx.x * kVizThreads * kVizPerThread + threadIdx.x, e = 0; e < kVizPerThread && p < hw;
       ++e, p += kVizThreads) {
    float u, v;
    load_uv(a, b, p, u, v);
    const float r = radius(u, v);
    m = max(m, isnan(r) ? kNanBits : __float_as_uint(r));
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m) atomicMax(a.maxbits + b, m);
}

__global__ void __launch_bounds__(kVizThreads) viz_color_kernel(VizArgs a) {
  const int b = blockIdx.y;
  const int hw = a.H * a.W;
  const int p = blockIdx.x * kVizThreads + threadIdx.x;
  if (p >= hw) return;
  const int y = p / a.W, x = p - y * a.W;
  const float* f = a.flow + b * a.sb + y * a.sy + x * a.sx;
  const float u0 = f[0], v0 = f[a.sc];
  unsigned char* o = a.out + (static_cast<long long>(b) * hw + p) * 3;
  if (fabsf(u0) > kUnknown || fabsf(v0) > kUnknown) {   // unknown pixels are black
    o[0] = o[1] = o[2] = 0;
    return;
  }
  const unsigned mb = a.maxbits[b];
  // maxrad + eps: np.finfo(float).eps is a float64 scalar, so this and everything after it is float64.  With a NaN in the
  // image maxrad is the Python int -1.
  const double den = __dadd_rn(mb > 0x7f800000u ? -1.0 : static_cast<double>(__uint_as_float(mb)), kEps);
  double u = __ddiv_rn(static_cast<double>(u0), den), v = __ddiv_rn(static_cast<double>(v0), den);
  const bool nan = isnan(u) || isnan(v);
  if (nan) u = v = 0.0;
  const double rad = __dsqrt_rn(__dadd_rn(__dmul_rn(u, u), __dmul_rn(v, v)));
  const double ang = __ddiv_rn(atan2(-v, -u), 3.141592653589793);
  const double fk = __dadd_rn(__dmul_rn(__ddiv_rn(__dadd_rn(ang, 1.0), 2.0), static_cast<double>(kWheel - 1)), 1.0);
  const int k0 = static_cast<int>(floor(fk));
  const int k1 = k0 + 1 == kWheel + 1 ? 1 : k0 + 1;
  const double fr = __dsub_rn(fk, static_cast<double>(k0));
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double c0 = __ddiv_rn(static_cast<double>(kWheelRGB.rgb[k0 - 1][c]), 255.0);
    const double c1 = __ddiv_rn(static_cast<double>(kWheelRGB.rgb[k1 - 1][c]), 255.0);
    double col = __dadd_rn(__dmul_rn(__dsub_rn(1.0, fr), c0), __dmul_rn(fr, c1));
    col = rad <= 1.0 ? __dsub_rn(1.0, __dmul_rn(rad, __dsub_rn(1.0, col))) : __dmul_rn(col, 0.75);
    o[c] = nan ? 0 : static_cast<unsigned char>(floor(__dmul_rn(255.0, col)));
  }
}

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

size_t rnc_flow_to_image_workspace_bytes(int B) { return B > 0 ? static_cast<size_t>(B) * sizeof(unsigned) : 0; }

int rnc_flow_to_image(const float* flow, long long sb, long long sc, long long sy, long long sx, int B, int H, int W,
                      unsigned char* out, void* workspace, size_t workspace_bytes, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || B > 65535 || static_cast<long long>(H) * W >= (1ll << 30)) return RNC_ERR_BAD_SHAPE;
  if (!flow || !out || !workspace) return RNC_ERR_BAD_POINTER;
  if ((reinterpret_cast<uintptr_t>(flow) & 3) || (reinterpret_cast<uintptr_t>(workspace) & 3)) return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_flow_to_image_workspace_bytes(B)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  VizArgs a{flow, sb, sc, sy, sx, H, W, out, static_cast<unsigned*>(workspace)};
  cudaError_t e = cudaMemsetAsync(workspace, 0, rnc_flow_to_image_workspace_bytes(B), s);
  if (e != cudaSuccess) { g_last_cuda_error = static_cast<int>(e); return RNC_ERR_CUDA; }
  const int hw = H * W;
  const int per_block = kVizThreads * kVizPerThread;
  viz_maxrad_kernel<<<dim3((hw + per_block - 1) / per_block, B), kVizThreads, 0, s>>>(a);
  int st = after_launch();
  if (st) return st;
  viz_color_kernel<<<dim3((hw + kVizThreads - 1) / kVizThreads, B), kVizThreads, 0, s>>>(a);
  return after_launch();
}

}  // extern "C"
