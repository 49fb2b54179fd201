// Forward-backward consistency of a batch of float32 flow pairs (UnFlow, Meister et al. 2018): per pixel x of image b, in
// direction F -> G (and symmetrically G -> F), the target p = x + F(x), the backward flow there G^(p), bilinear with zero
// padding on align_corners=True pixel coordinates (the semantics of utils.utils.bilinear_sampler / F.grid_sample), and
//   err = |F(x) + G^(p)|,
//   occ bit 0: |F + G^|^2 > alpha1 * (|F|^2 + |G^|^2) + alpha2, or not finite (NaN counts as inconsistent),
//   occ bit 1: p outside [0, W-1] x [0, H-1] (a NaN target is not inside).
// A pixel whose target is outside gets err = +inf and both bits; one whose sum is NaN gets err = +inf and bit 0.
//
// Every operation is a __*_rn intrinsic in the order rnc/metrics.py:host_fb_consistency writes it, so nothing is contracted
// into an FMA and the host restatement gives the same bits.  One launch for both directions of B pairs (grid z), a thread per
// pixel, no atomics and no host synchronisation; a pixel's outputs depend only on its own image.
#include "eval_common.cuh"

namespace rnc {
namespace {

constexpr int kFbThreads = 256;

struct FbArgs {
  View flow[2];                 // [0] forward, [1] backward
  unsigned char* occ[2];
  float* err[2];
  int H, W;
  float alpha1, alpha2;
};

// g's value at (x, y) of the image at base, 0 outside the frame
__device__ __forceinline__ float sample_at(const View& g, const float* base, int H, int W, int x, int y, int c) {
  return (x >= 0 && x < W && y >= 0 && y < H) ? base[c * g.c + y * g.y + x * g.x] : 0.0f;
}

__global__ void __launch_bounds__(kFbThreads) fb_consistency_kernel(FbArgs a) {
  const int dir = blockIdx.z, b = blockIdx.y;
  const int H = a.H, W = a.W;
  const long long hw = static_cast<long long>(H) * W;
  const long long p = static_cast<long long>(blockIdx.x) * kFbThreads + threadIdx.x;
  if (p >= hw) return;
  const int v = static_cast<int>(p / W), u = static_cast<int>(p - static_cast<long long>(v) * W);
  const View& f = a.flow[dir];
  const View& g = a.flow[dir ^ 1];
  const float fu = f.at(b, 0, v, u), fv = f.at(b, 1, v, u);
  const float* gb = g.pixel(b, 0, 0);
  const float px = __fadd_rn(static_cast<float>(u), fu), py = __fadd_rn(static_cast<float>(v), fv);
  const long long o = static_cast<long long>(b) * hw + p;
  if (!(px >= 0.0f && px <= static_cast<float>(W - 1) && py >= 0.0f && py <= static_cast<float>(H - 1))) {
    a.err[dir][o] = __int_as_float(0x7f800000);
    a.occ[dir][o] = 3;
    return;
  }
  const float x0 = floorf(px), y0 = floorf(py);
  const float ax = __fsub_rn(px, x0), ay = __fsub_rn(py, y0);
  const float bx = __fsub_rn(1.0f, ax), by = __fsub_rn(1.0f, ay);
  const float w00 = __fmul_rn(bx, by), w01 = __fmul_rn(ax, by), w10 = __fmul_rn(bx, ay), w11 = __fmul_rn(ax, ay);
  const int ix = static_cast<int>(x0), iy = static_cast<int>(y0);
  float gs[2];
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    float s = __fmul_rn(sample_at(g, gb, H, W, ix, iy, c), w00);
    s = __fadd_rn(s, __fmul_rn(sample_at(g, gb, H, W, ix + 1, iy, c), w01));
    s = __fadd_rn(s, __fmul_rn(sample_at(g, gb, H, W, ix, iy + 1, c), w10));
    gs[c] = __fadd_rn(s, __fmul_rn(sample_at(g, gb, H, W, ix + 1, iy + 1, c), w11));
  }
  const float su = __fadd_rn(fu, gs[0]), sv = __fadd_rn(fv, gs[1]);
  const float lhs = __fadd_rn(__fmul_rn(su, su), __fmul_rn(sv, sv));
  const float mf = __fadd_rn(__fmul_rn(fu, fu), __fmul_rn(fv, fv));
  const float mg = __fadd_rn(__fmul_rn(gs[0], gs[0]), __fmul_rn(gs[1], gs[1]));
  const float rhs = __fadd_rn(__fmul_rn(a.alpha1, __fadd_rn(mf, mg)), a.alpha2);
  const bool finite = lhs <= 3.402823466e38f;             // false for +inf and NaN
  a.err[dir][o] = finite ? __fsqrt_rn(lhs) : __int_as_float(0x7f800000);
  a.occ[dir][o] = (!finite || lhs > rhs) ? 1 : 0;
}

// its own limits, wider than eval_shape_ok's: H*W < 2^31, and H, W < 2^24 so that every pixel coordinate is exact in float32
bool shape_ok(int B, int H, int W) {
  return B > 0 && H > 0 && W > 0 && B <= 65535 && static_cast<long long>(H) * W < (1ll << 31) && H < (1 << 24) &&
         W < (1 << 24);
}

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

int rnc_fb_consistency(const float* flow_fw, long long fb, long long fc, long long fy, long long fx, const float* flow_bw,
                       long long gb, long long gc, long long gy, long long gx, int B, int H, int W, float alpha1,
                       float alpha2, unsigned char* occ_fw, unsigned char* occ_bw, float* err_fw, float* err_bw,
                       void* stream) {
  if (!shape_ok(B, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!flow_fw || !flow_bw || !occ_fw || !occ_bw || !err_fw || !err_bw) return RNC_ERR_BAD_POINTER;
  if (!aligned(flow_fw, 4) || !aligned(flow_bw, 4) || !aligned(err_fw, 4) || !aligned(err_bw, 4)) return RNC_ERR_BAD_POINTER;
  const FbArgs a{{{flow_fw, fb, fc, fy, fx}, {flow_bw, gb, gc, gy, gx}}, {occ_fw, occ_bw}, {err_fw, err_bw}, H, W, alpha1,
                 alpha2};
  const long long hw = static_cast<long long>(H) * W;
  const dim3 grid(static_cast<unsigned>((hw + kFbThreads - 1) / kFbThreads), B, 2);
  fb_consistency_kernel<<<grid, kFbThreads, 0, as_stream(stream)>>>(a);
  return after_launch();
}

}  // extern "C"
