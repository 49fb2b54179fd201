// Full-frame video stabilization (the definition: rnc/stabilize.py step 5 and DESIGN §3.22): the flows moved into the
// stabilized frames with the camera's known global motion taken out, so that only the local residual is completed across
// the uncovered border, and the global motion added back.  The kernels of stabilize.cu stay in their own file.
//
// flow_kernel<kReadd>, a thread per (video, pair, pixel u), both directions per thread:
//   transfer (kReadd false): forward, q = M_k^-1 u exactly as warp_kernel computes it (fp64, rounded once to fp32, valid when
//     w > 0 and q lies in the frame), F = bilinear.cuh's sample of F_k at q, and
//     R = pi(M_{k+1} (q + F)) - pi(M_{k+1} pi(A_k q)) in fp64, rounded once to fp32; NaN when q is not valid, F is not
//     finite or a projection has w <= 0.  Backward the same with M_{k+1}^-1, G_k, M_k and inv(A_k) for output frame k+1.
//   re-add (kReadd true), in place on the completed residuals: F~ = (pi(M_{k+1} pi(A_k q)) - u) + R~ in fp64, rounded once to
//     fp32, q = M_k^-1 u rounded to fp32 as above without the frame test; NaN when a projection has w <= 0.  Backward likewise.
// pi(P p) is ((p0 x + p1 y) + p2) / ((p6 x + p7 y) + p8) and the same for y, valid when the denominator is > 0; inv(A) is
// the adjugate divided by its [2][2], as in stabilize.cu's path.  Every operation is a __*_rn intrinsic in the order
// rnc/stabilize.py's host restatements write it, so the host gives the same bits.  No atomics, no transcendental function.
#include <cmath>

#include "bilinear.cuh"
#include "homography.cuh"

namespace rnc {
namespace {

constexpr int kFillThreads = 256;
constexpr int kMaxSide = 4096;

struct FillArgs {
  Video fw, bw;                               // [V][T-1][2][H][W], b the pair: transfer: the flows F, G; re-add: unused
  const double* motion;                       // [V][T-1][9]
  const double* maps;                         // [V][T][9], input -> output
  const double* maps_inv;                     // [V][T][9], output -> input
  float* out;                                 // [V][T-1][2][H][W] contiguous: R (transfer) or R~ -> F~ (re-add, in place)
  float* out_bw;
  int T, H, W;
};

// one direction at output pixel (x, y): src = the output -> input map of the output frame, dst = the input -> output map of
// the other frame, A = the motion from this frame's input to the other's.  Writes the two channels of the result.
template <bool kReadd>
__device__ __forceinline__ void direction(const double* src, const double* dst, const double* A, const Video& f, int v, int k,
                                          int x, int y, int H, int W, float* out, long long plane) {
  const float nan = __int_as_float(0x7fc00000);            // the host's float32 NaN, so the bits agree
  double X, Y;
  const bool wq = project(src, x, y, X, Y);
  const float qx = __double2float_rn(X), qy = __double2float_rn(Y);
  double bx, by, gx, gy;
  bool ok = wq && project(A, qx, qy, bx, by) && project(dst, bx, by, gx, gy);
  if (kReadd) {
    const float rx = out[0], ry = out[plane];
    out[0] = ok ? __double2float_rn(dadd(dsub(gx, x), static_cast<double>(rx))) : nan;
    out[plane] = ok ? __double2float_rn(dadd(dsub(gy, y), static_cast<double>(ry))) : nan;
    return;
  }
  ok = ok && inside(qx, qy, H, W);
  double ax = 0.0, ay = 0.0;
  if (ok) {
    const View im{f.video(v).pixel(k, 0, 0), 0, f.c, f.y, f.x};     // pair k's two planes
    const float ux = sample(im, 0, 0, qx, qy, H, W), uy = sample(im, 0, 1, qx, qy, H, W);
    ok = finite(ux) && finite(uy) &&
         project(dst, dadd(static_cast<double>(qx), static_cast<double>(ux)),
                 dadd(static_cast<double>(qy), static_cast<double>(uy)), ax, ay);
  }
  out[0] = ok ? __double2float_rn(dsub(ax, gx)) : nan;
  out[plane] = ok ? __double2float_rn(dsub(ay, gy)) : nan;
}

template <bool kReadd>
__global__ void __launch_bounds__(kFillThreads) flow_kernel(FillArgs a) {
  const int hw = a.H * a.W;
  const int p = blockIdx.x * kFillThreads + threadIdx.x;
  if (p >= hw) return;
  const int k = blockIdx.y, v = blockIdx.z;
  const int y = p / a.W, x = p - y * a.W;
  const long long pair = static_cast<long long>(v) * (a.T - 1) + k;
  const double* A = a.motion + pair * 9;
  const double* M = a.maps + (static_cast<long long>(v) * a.T + k) * 9;
  const double* Mi = a.maps_inv + (static_cast<long long>(v) * a.T + k) * 9;
  const long long off = pair * 2 * hw + p;
  direction<kReadd>(Mi, M + 9, A, a.fw, v, k, x, y, a.H, a.W, a.out + off, hw);
  const M3 Ai = inv_norm(A);
  direction<kReadd>(Mi + 9, M, Ai.m, a.bw, v, k, x, y, a.H, a.W, a.out_bw + off, hw);
}

bool fill_shape_ok(int V, int T, int H, int W) {
  return V > 0 && V <= 65535 && T >= 2 && T <= 65536 && H > 0 && W > 0 && H <= kMaxSide && W <= kMaxSide;
}

int launch(const FillArgs& a, int V, bool readd, void* stream) {
  const dim3 grid((a.H * a.W + kFillThreads - 1) / kFillThreads, a.T - 1, V);
  if (readd)
    flow_kernel<true><<<grid, kFillThreads, 0, as_stream(stream)>>>(a);
  else
    flow_kernel<false><<<grid, kFillThreads, 0, as_stream(stream)>>>(a);
  return after_launch();
}

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

int rnc_stabilize_flow_residual(const float* flow, long long fv, long long fk, long long fc, long long fy, long long fx,
                                const float* flow_bw, long long bv, long long bk, long long bc, long long by, long long bx,
                                const double* motion, const double* maps, const double* maps_inv, int V, int T, int H, int W,
                                float* res, float* res_bw, void* stream) {
  if (!fill_shape_ok(V, T, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!flow || !flow_bw || !motion || !maps || !maps_inv || !res || !res_bw) return RNC_ERR_BAD_POINTER;
  if (!aligned(flow, 4) || !aligned(flow_bw, 4) || !aligned(motion, 8) || !aligned(maps, 8) || !aligned(maps_inv, 8) ||
      !aligned(res, 4) || !aligned(res_bw, 4))
    return RNC_ERR_BAD_POINTER;
  const FillArgs a{{flow, fv, fk, fc, fy, fx}, {flow_bw, bv, bk, bc, by, bx}, motion, maps, maps_inv, res, res_bw, T, H, W};
  return launch(a, V, false, stream);
}

int rnc_stabilize_flow_readd(const double* motion, const double* maps, const double* maps_inv, int V, int T, int H, int W,
                             float* flow, float* flow_bw, void* stream) {
  if (!fill_shape_ok(V, T, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!motion || !maps || !maps_inv || !flow || !flow_bw) return RNC_ERR_BAD_POINTER;
  if (!aligned(motion, 8) || !aligned(maps, 8) || !aligned(maps_inv, 8) || !aligned(flow, 4) || !aligned(flow_bw, 4))
    return RNC_ERR_BAD_POINTER;
  const FillArgs a{{}, {}, motion, maps, maps_inv, flow, flow_bw, T, H, W};
  return launch(a, V, true, stream);
}

}  // extern "C"
