// Frame interpolation (Baker, Scharstein, Lewis, Roth, Black and Szeliski, "A Database and Evaluation Methodology for Optical
// Flow", IJCV 2011, with fb_consistency's occlusion masks and a nearest-site hole fill; the definition: rnc/interp.py and
// DESIGN §3.15), and its interpolation error.
//
// rnc_interpolate, for B frame pairs and T times, in four launches and no host synchronisation:
//   1. interp_splat_kernel, a thread per source pixel of both frames of every image (grid z: the source frame): a source with
//      occ == 0 and a finite flow computes its photometric error e once, then for every time t proposes its motion at the
//      nearest pixel of its splat target with an integer atomicMin of the key (float bits of e) << 32 | source index.  The map
//      starts all-ones (a memset), so each pixel ends with the smallest (e, index) whatever order the threads ran in.
//   2. dist_transform.cuh's column and row passes over the B*T maps: each pixel's nearest pixel that received a proposal (a
//      feature transform; ties to the smallest column, then the smallest row), -1 in a map without one.
//   3. interp_composite_kernel, a thread per output pixel: the motion u of the winning source at that site (0 without one), the
//      two bilinear samples at x - t u and x + (1 - t) u, and the blend or the one visible sample.
// Every floating-point operation is a __*_rn intrinsic in the order rnc/interp.py:host_interpolate writes it, so nothing is
// contracted into an FMA and the host restatement gives the same bits.  No floating-point atomics: an output depends only on
// its own image and time.
//
// rnc_interp_error: per image, the fp64 sum over its pixels of sum_c (pred - gt)^2 and its pixel count, by eval_common.cuh's
// two fixed-order reductions, as rnc_flow_metrics: the order depends only on H*W, so an image's sum does not depend on N, on
// its position in the batch or on the GPU.
#include "bilinear.cuh"
#include "dist_transform.cuh"
#include "eval_common.cuh"

namespace rnc {
namespace {

constexpr int kInterpThreads = 256;
constexpr int kMaxTimes = RNC_INTERP_MAX_TIMES;
constexpr unsigned long long kNoProposal = ~0ull;

struct InterpArgs {
  View frame[2];                        // I0, I1
  View flow[2];                         // F (0 -> 1), G (1 -> 0)
  const unsigned char* occ[2];          // [B][H][W]: occ0 of F on frame 0, occ1 of G on frame 1
  unsigned long long* map;              // [B][T][H][W]
  int* site;                            // [B][T][H][W]
  float* out;                           // [B][T][3][H][W]
  int B, T, H, W;
  float t[kMaxTimes];
};

__global__ void __launch_bounds__(kInterpThreads) interp_splat_kernel(InterpArgs a) {
  const int s = blockIdx.z, b = blockIdx.y;
  const int H = a.H, W = a.W, hw = H * W;
  const int p = blockIdx.x * kInterpThreads + threadIdx.x;
  if (p >= hw) return;
  if (a.occ[s][static_cast<long long>(b) * hw + p] != 0) return;
  const int y = p / W, x = p - y * W;
  const View& f = a.flow[s];
  const float fu = f.at(b, 0, y, x), fv = f.at(b, 1, y, x);
  if (!finite(fu) || !finite(fv)) return;
  // e = sum_c |I_other(x + f) - I_own(x)|, channels in order
  const float px = __fadd_rn(static_cast<float>(x), fu), py = __fadd_rn(static_cast<float>(y), fv);
  float e = 0.0f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float d = fabsf(__fsub_rn(sample(a.frame[s ^ 1], b, c, px, py, H, W), a.frame[s].at(b, c, y, x)));
    e = c == 0 ? d : __fadd_rn(e, d);
  }
  const unsigned long long key =
      static_cast<unsigned long long>(__float_as_uint(e)) << 32 | static_cast<unsigned>(s * hw + p);
  unsigned long long* map = a.map + static_cast<long long>(b) * a.T * hw;
  for (int k = 0; k < a.T; ++k, map += hw) {
    const float tt = s == 0 ? a.t[k] : __fsub_rn(1.0f, a.t[k]);     // frame 1 travels 1 - t along G
    const float qx = rintf(__fadd_rn(static_cast<float>(x), __fmul_rn(tt, fu)));
    const float qy = rintf(__fadd_rn(static_cast<float>(y), __fmul_rn(tt, fv)));
    if (qx >= 0.0f && qx <= static_cast<float>(W - 1) && qy >= 0.0f && qy <= static_cast<float>(H - 1))
      atomicMin(map + static_cast<int>(qy) * W + static_cast<int>(qx), key);
  }
}

struct ProposalSites {                  // the pixels of a [B*T] map that received a proposal
  const unsigned long long* map;
  int H, W;
  __device__ bool operator()(int i, int y, int x) const {
    return map[(static_cast<long long>(i) * H + y) * W + x] != kNoProposal;
  }
};

struct SiteOut {                        // the row-major index of the nearest site
  static constexpr int none = -1;
  int W;
  __device__ int operator()(int, int, int q, int r, int) const { return r * W + q; }
};

__global__ void __launch_bounds__(kInterpThreads) interp_composite_kernel(InterpArgs a) {
  const int bt = blockIdx.y, b = bt / a.T, k = bt - b * a.T;
  const int H = a.H, W = a.W, hw = H * W;
  const int p = blockIdx.x * kInterpThreads + threadIdx.x;
  if (p >= hw) return;
  const int y = p / W, x = p - y * W;
  const long long img = static_cast<long long>(bt) * hw;
  const int site = a.site[img + p];
  float uu = 0.0f, uv = 0.0f;
  if (site >= 0) {
    const unsigned src = static_cast<unsigned>(a.map[img + site]);
    const int s = src >= static_cast<unsigned>(hw), q = static_cast<int>(src) - s * hw;
    const int qy = q / W, qx = q - qy * W;
    uu = a.flow[s].at(b, 0, qy, qx);
    uv = a.flow[s].at(b, 1, qy, qx);
    if (s) {                            // a frame-1 source moves by -G
      uu = -uu;
      uv = -uv;
    }
  }
  const float t = a.t[k], omt = __fsub_rn(1.0f, t);
  const float x0 = __fsub_rn(static_cast<float>(x), __fmul_rn(t, uu)), y0 = __fsub_rn(static_cast<float>(y), __fmul_rn(t, uv));
  const float x1 = __fadd_rn(static_cast<float>(x), __fmul_rn(omt, uu)), y1 = __fadd_rn(static_cast<float>(y), __fmul_rn(omt, uv));
  const float wm = static_cast<float>(W - 1), hm = static_cast<float>(H - 1);
  const long long ob = static_cast<long long>(b) * hw;
  const bool v0 = x0 >= 0.0f && x0 <= wm && y0 >= 0.0f && y0 <= hm &&
                  a.occ[0][ob + static_cast<int>(rintf(y0)) * W + static_cast<int>(rintf(x0))] == 0;
  const bool v1 = x1 >= 0.0f && x1 <= wm && y1 >= 0.0f && y1 <= hm &&
                  a.occ[1][ob + static_cast<int>(rintf(y1)) * W + static_cast<int>(rintf(x1))] == 0;
  float* out = a.out + img * 3 + p;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float s0 = sample(a.frame[0], b, c, x0, y0, H, W), s1 = sample(a.frame[1], b, c, x1, y1, H, W);
    out[static_cast<long long>(c) * hw] = v0 == v1 ? __fadd_rn(__fmul_rn(omt, s0), __fmul_rn(t, s1)) : v0 ? s0 : s1;
  }
}

struct SquaredError {                   // sum_c (pred - gt)^2 in fp64, channels in order
  View pred, gt;
  __device__ void operator()(double& acc, int n, int y, int x) const {
    double d2 = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double d = __dsub_rn(static_cast<double>(pred.at(n, c, y, x)), static_cast<double>(gt.at(n, c, y, x)));
      d2 = c == 0 ? __dmul_rn(d, d) : __dadd_rn(d2, __dmul_rn(d, d));
    }
    acc += d2;
  }
};

struct ErrorStore {                     // image n -> sq_sum [n], count [n] = H*W
  double* sq_sum;
  long long* count;
  long long hw;
  __device__ void operator()(int n, double v) const {
    sq_sum[n] = v;
    count[n] = hw;
  }
};

bool interp_shape_ok(int B, int T, int H, int W) {
  return B > 0 && T > 0 && T <= kMaxTimes && H > 0 && W > 0 && H <= kSiteMaxSide && W <= kSiteMaxSide &&
         static_cast<long long>(B) * T <= 65535;
}

size_t map_bytes(int B, int T, int H, int W) {
  return static_cast<size_t>(B) * T * H * W * sizeof(unsigned long long);
}

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

size_t rnc_interpolate_workspace_bytes(int B, int T, int H, int W) {
  return interp_shape_ok(B, T, H, W) ? map_bytes(B, T, H, W) + static_cast<size_t>(B) * T * H * W * sizeof(int) : 0;
}

int rnc_interpolate(const float* frame0, long long ab, long long ac, long long ay, long long ax, const float* frame1,
                    long long bb, long long bc, long long by, long long bx, const float* flow, long long fb, long long fc,
                    long long fy, long long fx, const float* flow_bw, long long gb, long long gc, long long gy, long long gx,
                    const unsigned char* occ0, const unsigned char* occ1, const float* times, int T, int B, int H, int W,
                    float* out, void* workspace, size_t workspace_bytes, void* stream) {
  if (!interp_shape_ok(B, T, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!frame0 || !frame1 || !flow || !flow_bw || !occ0 || !occ1 || !times || !out || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(frame0, 4) || !aligned(frame1, 4) || !aligned(flow, 4) || !aligned(flow_bw, 4) || !aligned(out, 4) ||
      !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_interpolate_workspace_bytes(B, T, H, W)) return RNC_ERR_WORKSPACE;
  InterpArgs a{{{frame0, ab, ac, ay, ax}, {frame1, bb, bc, by, bx}},
               {{flow, fb, fc, fy, fx}, {flow_bw, gb, gc, gy, gx}},
               {occ0, occ1},
               static_cast<unsigned long long*>(workspace),
               reinterpret_cast<int*>(static_cast<char*>(workspace) + map_bytes(B, T, H, W)),
               out, B, T, H, W, {}};
  for (int k = 0; k < T; ++k) {
    if (!(times[k] > 0.0f && times[k] < 1.0f)) return RNC_ERR_BAD_SHAPE;
    a.t[k] = times[k];
  }
  cudaStream_t s = as_stream(stream);
  cudaMemsetAsync(a.map, 0xff, map_bytes(B, T, H, W), s);       // every key to all-ones: no proposal yet
  if (int st = after_launch(0)) return st;
  const int hw = H * W, nblk = (hw + kInterpThreads - 1) / kInterpThreads;
  interp_splat_kernel<<<dim3(nblk, B, 2), kInterpThreads, 0, s>>>(a);
  if (int st = after_launch()) return st;
  dist2_column_kernel<<<dim3((W + kSiteColThreads - 1) / kSiteColThreads, B * T), kSiteColThreads, 0, s>>>(
      ProposalSites{a.map, H, W}, H, W, a.site);
  if (int st = after_launch()) return st;
  dist2_row_kernel<<<dim3(H, B * T), 32, dist2_row_smem(W), s>>>(H, W, a.site, SiteOut{W});
  if (int st = after_launch()) return st;
  interp_composite_kernel<<<dim3(nblk, B * T), kInterpThreads, 0, s>>>(a);
  return after_launch();
}

size_t rnc_interp_error_workspace_bytes(int N, int H, int W) {
  return eval_shape_ok(N, H, W) ? static_cast<size_t>(N) * eval_blocks(H, W) * sizeof(double) : 0;
}

int rnc_interp_error(const float* pred, long long pb, long long pc, long long py, long long px, const float* gt, long long gb,
                     long long gc, long long gy, long long gx, int N, int H, int W, double* sq_sum, long long* count,
                     void* workspace, size_t workspace_bytes, void* stream) {
  if (!eval_shape_ok(N, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!pred || !gt || !sq_sum || !count || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(pred, 4) || !aligned(gt, 4) || !aligned(sq_sum, 8) || !aligned(count, 8) || !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_interp_error_workspace_bytes(N, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const int nblk = eval_blocks(H, W);
  double* parts = static_cast<double*>(workspace);
  cta_partials_kernel<<<dim3(nblk, N), kEvalThreads, 0, s>>>(SquaredError{{pred, pb, pc, py, px}, {gt, gb, gc, gy, gx}}, H, W,
                                                              parts);
  if (int st = after_launch()) return st;
  return launch_image_reduce(parts, N, nblk, 1, ErrorStore{sq_sum, count, static_cast<long long>(H) * W}, s);
}

}  // extern "C"
