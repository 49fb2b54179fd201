// Blind video temporal consistency along the backward flows (the definition: rnc/temporal.py and DESIGN §3.20): one step
// k -> k+1 of the screened Poisson solve of Bonneel et al. 2015 in correction form, and the warping error's per-frame partials
// (Lai et al. 2018).
//
// rnc_temporal_step, V videos of C channels, in 5 + 2 * sweeps launches:
//   1. target_kernel, a thread per pixel p of frame k+1: p is matched (bilinear.cuh's follow) when u = G_k(p) is finite,
//      occ_bw_k(p) == 0 and p' = p + u lies in the frame.  A matched pixel samples T = O_k(p') and J = I_k(p') (bilinear.cuh's sample) and weighs
//      w = lam / (1 + alpha d2), d2 the squared colour distance of I_{k+1}(p) and J over 255; an unmatched one weighs 0.  It
//      writes D = 0, r = w (T - P) (0 where w is 0), den = n + w (n the in-frame 4-neighbours) and weak = w < lam / 4.
//   2. dist_transform.cuh's column and row passes with the non-weak pixels as sites: every pixel's exact squared distance to
//      the nearest non-weak pixel (0 in an image without one).
//   3. omega_kernel, a CTA per image: the largest of those distances, D2, by an integer maximum (exact in any order);
//      L = the least integer with L^2 >= 4 D2, s = min(pi_f32 / (L + 1), sigma) (sigma alone when D2 is 0) and
//      omega = 2 / (1 + s), each operation rounded once.
//   4. sweeps times sor_kernel<red> then sor_kernel<black>, a thread per pixel of the colour ((x + y) & 1: 0 red):
//      D += omega ((s + r) / den - D), s the in-frame 4-neighbours of D added up, left, right, down.  A colour's pixels only
//      read the other colour, so any order of its updates gives the sequential sweep's bits.
//   5. finish_kernel, a thread per pixel: O_{k+1} = P + D.
// rnc_warping_error_partials: per frame k+1 of every video, the fp64 sum over its matched pixels and channels of
// ((V_{k+1}(p) - V_k(p')) / 255)^2, V_k(p') by sample and the rest in fp64, and the count of matched pixels, through
// eval_common.cuh's two fixed-order reductions.
// Every float32 operation is a __*_rn intrinsic in the order rnc/temporal.py's host restatements write it, so the host gives
// the same bits (the warping error's fp64 sums agree to their last bits).  No atomics and no host synchronisation.
#include <cmath>

#include "bilinear.cuh"
#include "dist_transform.cuh"
#include "eval_common.cuh"

namespace rnc {
namespace {

constexpr int kStepThreads = 256;
constexpr int kMaxChannels = RNC_HARMONIC_MAX_CHANNELS;
constexpr float kPiF32 = 3.14159265358979f;

struct StepLayout {                           // the workspace
  float* D;                                   // [V][C][H][W]: the correction
  float* r;                                   // [V][C][H][W]: w (T - P)
  float* den;                                 // [V][H][W]: n + w
  int* map;                                   // [V][H][W]: the distance transform
  float* omega;                               // [V]
  unsigned char* weak;                        // [V][H][W]
};

StepLayout step_layout(Carve& ws, int V, int C, int H, int W) {
  const size_t px = static_cast<size_t>(V) * H * W;
  StepLayout l;
  l.D = ws.take<float>(px * C);
  l.r = ws.take<float>(px * C);
  l.den = ws.take<float>(px);
  l.map = ws.take<int>(px);
  l.omega = ws.take<float>(V);
  l.weak = ws.take<unsigned char>(px);
  return l;
}

struct StepArgs {
  View prev, proc, img_prev, img;             // O_k, P_{k+1} [V][C][H][W]; I_k, I_{k+1} [V][3][H][W]
  View flow;                                  // G_k [V][2][H][W]
  MaskView occ;                               // occ_bw_k [V][H][W]
  float lam, alpha;
  int C, H, W;
};

__global__ void __launch_bounds__(kStepThreads) target_kernel(StepArgs a, StepLayout l) {
  const int v = blockIdx.y, H = a.H, W = a.W, hw = H * W;
  const int p = blockIdx.x * kStepThreads + threadIdx.x;
  if (p >= hw) return;
  const int y = p / W, x = p - y * W;
  float px, py, w = 0.0f;
  const bool matched = follow(a.flow, a.occ, v, y, x, H, W, px, py);
  if (matched) {
    float d2 = -0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float e = __fdiv_rn(__fsub_rn(a.img.at(v, c, y, x), sample(a.img_prev, v, c, px, py, H, W)), 255.0f);
      d2 = __fadd_rn(d2, __fmul_rn(e, e));
    }
    w = __fdiv_rn(a.lam, __fadd_rn(1.0f, __fmul_rn(a.alpha, d2)));
  }
  const long long vp = static_cast<long long>(v) * hw + p;
  for (int c = 0; c < a.C; ++c) {
    const long long i = (static_cast<long long>(v) * a.C + c) * hw + p;
    l.D[i] = 0.0f;
    l.r[i] = w > 0.0f ? __fmul_rn(w, __fsub_rn(sample(a.prev, v, c, px, py, H, W), a.proc.at(v, c, y, x))) : 0.0f;
  }
  const int n = (y > 0) + (x > 0) + (x < W - 1) + (y < H - 1);
  l.den[vp] = __fadd_rn(static_cast<float>(n), w);
  l.weak[vp] = w < __fmul_rn(a.lam, 0.25f);
}

struct StrongSites {                          // the pixels that are not weak
  const unsigned char* weak;
  int hw, W;
  __device__ bool operator()(int v, int y, int x) const { return weak[static_cast<long long>(v) * hw + y * W + x] == 0; }
};

// a CTA per image: the largest squared distance D2, L = the least integer with L^2 >= 4 D2, and omega
__global__ void __launch_bounds__(kStepThreads) omega_kernel(int hw, float sigma, StepLayout l) {
  const int v = blockIdx.x;
  const int* m = l.map + static_cast<long long>(v) * hw;
  int d2 = 0;
  for (int p = threadIdx.x; p < hw; p += kStepThreads) d2 = max(d2, m[p]);
  d2 = __reduce_max_sync(0xffffffffu, d2);
  __shared__ int warps[kStepThreads / 32];
  if ((threadIdx.x & 31) == 0) warps[threadIdx.x >> 5] = d2;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 0; w < kStepThreads / 32; ++w) d2 = max(d2, warps[w]);
  float s = sigma;
  if (d2 > 0) {
    const long long four = 4ll * d2;
    long long L = static_cast<long long>(sqrt(static_cast<double>(four)));
    while (L * L < four) ++L;
    while (L > 0 && (L - 1) * (L - 1) >= four) --L;
    s = fminf(__fdiv_rn(kPiF32, static_cast<float>(L + 1)), sigma);
  }
  l.omega[v] = __fdiv_rn(2.0f, __fadd_rn(1.0f, s));
}

// a thread per pixel of one colour: row y's pixels of colour Colour are x = 2 e + ((y + Colour) & 1)
template <int Colour>
__global__ void __launch_bounds__(kStepThreads) sor_kernel(int C, int H, int W, StepLayout l) {
  const int v = blockIdx.y, hw = H * W, half = (W + 1) >> 1;
  const int e = blockIdx.x * kStepThreads + threadIdx.x;
  const int y = e / half;
  if (y >= H) return;
  const int x = 2 * (e - y * half) + ((y + Colour) & 1);
  if (x >= W) return;
  const long long vp = static_cast<long long>(v) * hw + y * W + x;
  const float den = l.den[vp];
  if (den == 0.0f) return;                    // an unmatched pixel of a 1x1 frame: no neighbour and no weight, D stays 0
  const float omega = l.omega[v];
  const bool up = y > 0, left = x > 0, right = x < W - 1, down = y < H - 1;
  for (int c = 0; c < C; ++c) {
    const long long i = (static_cast<long long>(v) * C + c) * hw + y * W + x;
    float* d = l.D + i;
    float s = -0.0f;                          // -0 + v == v for every v: the first neighbour starts the sum exactly
    if (up) s = __fadd_rn(s, d[-W]);
    if (left) s = __fadd_rn(s, d[-1]);
    if (right) s = __fadd_rn(s, d[1]);
    if (down) s = __fadd_rn(s, d[W]);
    const float old = *d;
    *d = __fadd_rn(old, __fmul_rn(omega, __fsub_rn(__fdiv_rn(__fadd_rn(s, l.r[i]), den), old)));
  }
}

__global__ void __launch_bounds__(kStepThreads) finish_kernel(View proc, OutView out, int C, int H, int W, StepLayout l) {
  const int v = blockIdx.y, hw = H * W;
  const int p = blockIdx.x * kStepThreads + threadIdx.x;
  if (p >= hw) return;
  const int y = p / W, x = p - y * W;
  for (int c = 0; c < C; ++c)
    out.p[v * out.b + c * out.c + y * out.y + x * out.x] =
        __fadd_rn(proc.at(v, c, y, x), l.D[(static_cast<long long>(v) * C + c) * hw + p]);
}

bool param_ok(float v) { return v >= 0.0f && v <= 3.402823466e38f; }   // finite and >= 0

bool step_shape_ok(int V, int C, int H, int W) {
  return V > 0 && V <= 65535 && C > 0 && C <= kMaxChannels && H > 0 && W > 0 && H <= kSiteMaxSide && W <= kSiteMaxSide;
}

// ------------------------------------------------------------------------------------------------ warping error

struct WarpPixel {                            // cta_partials_kernel's pixel (i, y, x): frame k+1 of video v, i = v K + k
  Video video;                                // [V][T][C][H][W], b the frame
  Video flow;                                 // [V][K][2][H][W], b the pair
  VideoMask occ;                              // [V][K][H][W], b the pair
  int K, C, H, W;
  __device__ void operator()(SumCount& acc, int i, int y, int x) const {
    const int v = i / K, k = i - v * K;
    float px, py;
    if (!follow(flow.video(v), occ.video(v), k, y, x, H, W, px, py)) return;
    const View vid = video.video(v);
    double t = 0.0;
    for (int c = 0; c < C; ++c) {
      const double e = __ddiv_rn(__dsub_rn(vid.at(k + 1, c, y, x), sample(vid, k, c, px, py, H, W)), 255.0);
      t = __dadd_rn(t, __dmul_rn(e, e));
    }
    acc.sum += t;
    acc.n += 1;
  }
};

bool warp_shape_ok(int V, int T, int C, int H, int W) {
  return V > 0 && T >= 2 && static_cast<long long>(V) * (T - 1) <= 65535 && C > 0 && eval_shape_ok(1, H, W);
}

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

size_t rnc_temporal_step_workspace_bytes(int V, int C, int H, int W) {
  if (!step_shape_ok(V, C, H, W)) return 0;
  Carve ws{nullptr};
  step_layout(ws, V, C, H, W);
  return ws.bytes;
}

int rnc_temporal_step(const float* out_prev, long long av, long long ac, long long ay, long long ax, const float* processed,
                      long long pv, long long pc, long long py, long long px, const float* frame_prev, long long iv,
                      long long ic, long long iy, long long ix, const float* frame, long long jv, long long jc, long long jy,
                      long long jx, const float* flow_bw, long long gv, long long gc, long long gy, long long gx,
                      const unsigned char* occ_bw, long long ov, long long oy, long long ox, int V, int C, int H, int W,
                      float lam, float alpha, float sigma, int sweeps, float* out, long long qv, long long qc, long long qy,
                      long long qx, void* workspace, size_t workspace_bytes, void* stream) {
  if (!step_shape_ok(V, C, H, W) || sweeps < 0 || !param_ok(lam) || !param_ok(alpha) || !param_ok(sigma))
    return RNC_ERR_BAD_SHAPE;
  if (!out_prev || !processed || !frame_prev || !frame || !flow_bw || !occ_bw || !out || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(out_prev, 4) || !aligned(processed, 4) || !aligned(frame_prev, 4) || !aligned(frame, 4) || !aligned(flow_bw, 4) ||
      !aligned(out, 4) || !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_temporal_step_workspace_bytes(V, C, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const int hw = H * W, nblk = (hw + kStepThreads - 1) / kStepThreads;
  Carve ws{static_cast<char*>(workspace)};
  const StepLayout l = step_layout(ws, V, C, H, W);
  const StepArgs a{{out_prev, av, ac, ay, ax}, {processed, pv, pc, py, px}, {frame_prev, iv, ic, iy, ix},
                   {frame, jv, jc, jy, jx},    {flow_bw, gv, gc, gy, gx},    {occ_bw, ov, 0, oy, ox},
                   lam, alpha, C, H, W};
  target_kernel<<<dim3(nblk, V), kStepThreads, 0, s>>>(a, l);
  if (int st = after_launch()) return st;
  dist2_column_kernel<<<dim3((W + kSiteColThreads - 1) / kSiteColThreads, V), kSiteColThreads, 0, s>>>(
      StrongSites{l.weak, hw, W}, H, W, l.map);
  if (int st = after_launch()) return st;
  dist2_row_kernel<<<dim3(H, V), 32, dist2_row_smem(W), s>>>(H, W, l.map, Dist2<0>{});
  if (int st = after_launch()) return st;
  omega_kernel<<<V, kStepThreads, 0, s>>>(hw, sigma, l);
  if (int st = after_launch()) return st;
  const int sor_blk = (H * ((W + 1) / 2) + kStepThreads - 1) / kStepThreads;
  for (int k = 0; k < sweeps; ++k) {
    sor_kernel<0><<<dim3(sor_blk, V), kStepThreads, 0, s>>>(C, H, W, l);
    if (int st = after_launch()) return st;
    sor_kernel<1><<<dim3(sor_blk, V), kStepThreads, 0, s>>>(C, H, W, l);
    if (int st = after_launch()) return st;
  }
  finish_kernel<<<dim3(nblk, V), kStepThreads, 0, s>>>(a.proc, {out, qv, qc, qy, qx}, C, H, W, l);
  return after_launch();
}

size_t rnc_warping_error_partials_workspace_bytes(int V, int T, int C, int H, int W) {
  return warp_shape_ok(V, T, C, H, W) ? static_cast<size_t>(V) * (T - 1) * eval_blocks(H, W) * sizeof(SumCount) : 0;
}

int rnc_warping_error_partials(const float* video, long long vv, long long vt, long long vc, long long vy, long long vx,
                               const float* flow_bw, long long gv, long long gk, long long gc, long long gy, long long gx,
                               const unsigned char* occ_bw, long long ov, long long ok, long long oy, long long ox, int V,
                               int T, int C, int H, int W, double* sum, long long* count, void* workspace,
                               size_t workspace_bytes, void* stream) {
  if (!warp_shape_ok(V, T, C, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!video || !flow_bw || !occ_bw || !sum || !count || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(video, 4) || !aligned(flow_bw, 4) || !aligned(sum, 8) || !aligned(count, 8) || !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_warping_error_partials_workspace_bytes(V, T, C, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const int K = T - 1, N = V * K, nblk = eval_blocks(H, W);
  SumCount* parts = static_cast<SumCount*>(workspace);
  cta_partials_kernel<<<dim3(nblk, N), kEvalThreads, 0, s>>>(
      WarpPixel{{video, vv, vt, vc, vy, vx}, {flow_bw, gv, gk, gc, gy, gx}, {occ_bw, ov, ok, 0, oy, ox}, K, C, H, W}, H, W,
      parts);
  if (int st = after_launch()) return st;
  return launch_image_reduce(parts, N, nblk, 1, SumCountStore{sum, count}, s);
}

}  // extern "C"
