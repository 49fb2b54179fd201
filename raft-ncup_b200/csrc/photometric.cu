// The unsupervised losses of a flow F between a source image I1 and a target I2 (the definition: rnc/unsupervised.py and
// DESIGN §3.16): the census term, a soft Hamming distance between the 7x7 census transforms of g(I1) and of g(I2) warped by F,
// and the second-order edge-aware smoothness of F.  Forward and backward, no atomics: every output is a fixed-order sum, so it
// is bit-identical from run to run and a row's results do not depend on the batch around it.
//
// rnc_census_loss_fwd, five launches:
//   1. census_warp_kernel, a thread per pixel: g(I1)(p), W^(p) = g(I2) sampled bilinearly at p + F(p) (taps outside the frame
//      are 0) and its derivatives dW^/dpx, dW^/dpy, into the state (State below).
//   2. census_fwd_kernel, a 32x8 tile per CTA with a 3-pixel halo of g(I1) and W^ in shared memory (0 outside the frame): per
//      weighted pixel h = sum_d e^2 / (0.1 + e^2), l = (h + 0.01)^0.4, into a per-pixel buffer, and k = v dl/dh = v 0.4 l /
//      (h + 0.01) into the state.
//   3, 4. eval_common.cuh's cta_partials_kernel and image_reduce_kernel: per row S_r = sum v l in fp64 and M_r = sum v, in an
//      order that depends only on H*W.
//   5. row_totals_kernel, one thread: the rows' sums added in row order.
// rnc_census_loss_bwd, one launch of census_bwd_kernel (the same tiles, with k): the loss depends on W^(q) through the census
// of q and through the censuses of the 48 pixels q - d whose window holds q.  Reindexing the second set by -d (psi is odd and
// phi' odd), both are terms of q's own window:
//   dL/dW^(q) = sum_d phi'(e_d(q)) psi'(W^(q+d) - W^(q)) (k(q) + k(q+d)),
// with phi(e) = e^2 / (0.1 + e^2), psi(x) = x / sqrt(0.81 + x^2), and k = 0 outside the frame.  grad F(q) = scale dL/dW^(q)
// (dW^/dpx, dW^/dpy)(q): a gather over a fixed order of offsets.
//
// rnc_smoothness_fwd: per row, the fp64 sums of the x- and y-terms (cta_partials_kernel over a per-pixel functor, then the rows
// in row order); rnc_smoothness_bwd: per pixel, the fixed-order gather of the three x- and three y-terms that hold it.
#include "eval_common.cuh"

namespace rnc {
namespace {

constexpr int kTileX = 32, kTileY = 8, kHalo = 3;
constexpr int kTileThreads = kTileX * kTileY;
constexpr int kSx = kTileX + 2 * kHalo, kSy = kTileY + 2 * kHalo;
constexpr int kWarpThreads = 256;

// The state of N rows: fp64 planes g(I1) and W^ ([N][H][W] each), then fp32 planes dW^/dpx, dW^/dpy and k.  The intensities
// are kept in fp64 because the census compares them through differences delta: near delta = 0, where phi' has its steepest
// slope (20), a float32 rounding of g (up to 7.6e-6 at 255) would move a gradient term by up to 4e-4 of the largest one.
struct State {
  double *g1, *wh;
  float *dwx, *dwy, *k;
  __host__ __device__ State(void* base, long long n_hw)
      : g1(static_cast<double*>(base)), wh(g1 + n_hw), dwx(reinterpret_cast<float*>(wh + n_hw)), dwy(dwx + n_hw),
        k(dwy + n_hw) {}
};

__device__ __forceinline__ double gray(const View& im, int n, int y, int x) {
  const float* p = im.pixel(n, y, x);
  return 0.2989 * p[0] + 0.5870 * p[im.c] + 0.1140 * p[2 * im.c];
}

struct WarpArgs {
  View image1, image2, flow;
  State st;
  int H, W;
};

__global__ void __launch_bounds__(kWarpThreads) census_warp_kernel(WarpArgs a) {
  const int n = blockIdx.y, H = a.H, W = a.W;
  const long long hw = static_cast<long long>(H) * W;
  const int p = blockIdx.x * kWarpThreads + threadIdx.x;
  if (p >= hw) return;
  const int y = p / W, x = p - y * W;
  const float px = static_cast<float>(x) + a.flow.at(n, 0, y, x), py = static_cast<float>(y) + a.flow.at(n, 1, y, x);
  const float x0 = floorf(px), y0 = floorf(py);
  double t[4] = {0.0, 0.0, 0.0, 0.0};          // taps (x0, y0), (x0+1, y0), (x0, y0+1), (x0+1, y0+1); 0 outside the frame
  double ax = 0.0, ay = 0.0;
  // a NaN coordinate fails both range tests and samples nothing
  if (x0 >= -1.0f && x0 <= static_cast<float>(W - 1) && y0 >= -1.0f && y0 <= static_cast<float>(H - 1)) {
    ax = px - x0;
    ay = py - y0;
    const int ix = static_cast<int>(x0), iy = static_cast<int>(y0);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int tx = ix + (k & 1), ty = iy + (k >> 1);
      if (tx >= 0 && tx < W && ty >= 0 && ty < H) t[k] = gray(a.image2, n, ty, tx);
    }
  }
  const double bx = 1.0 - ax, by = 1.0 - ay;
  const long long o = static_cast<long long>(n) * hw + p;
  a.st.g1[o] = gray(a.image1, n, y, x);
  a.st.wh[o] = by * (bx * t[0] + ax * t[1]) + ay * (bx * t[2] + ax * t[3]);
  a.st.dwx[o] = static_cast<float>(by * (t[1] - t[0]) + ay * (t[3] - t[2]));
  a.st.dwy[o] = static_cast<float>(bx * (t[2] - t[0]) + ax * (t[3] - t[1]));
}

// the CTA's tile of a row's plane with its halo, 0 outside the frame
template <typename T>
__device__ __forceinline__ void load_tile(T (*dst)[kSx], const T* plane, int H, int W) {
  const int ox = blockIdx.x * kTileX - kHalo, oy = blockIdx.y * kTileY - kHalo;
  for (int i = threadIdx.x; i < kSx * kSy; i += kTileThreads) {
    const int ty = i / kSx, tx = i - ty * kSx, y = oy + ty, x = ox + tx;
    dst[ty][tx] = (x >= 0 && x < W && y >= 0 && y < H) ? plane[static_cast<long long>(y) * W + x] : T(0);
  }
}

__device__ __forceinline__ bool weighted(const unsigned char* mask, int n, int y, int x, int H, int W) {
  return x >= kHalo && x <= W - 1 - kHalo && y >= kHalo && y <= H - 1 - kHalo &&
         (mask == nullptr || mask[(static_cast<long long>(n) * H + y) * W + x] != 0);
}

struct CensusArgs {
  State st;
  const unsigned char* mask;          // [N][H][W] or NULL
  float* loss;                        // [N][H][W]: v l
  int H, W;
};

__global__ void __launch_bounds__(kTileThreads) census_fwd_kernel(CensusArgs a) {
  __shared__ double g1[kSy][kSx], wp[kSy][kSx];
  const int n = blockIdx.z, H = a.H, W = a.W;
  const long long hw = static_cast<long long>(H) * W, row = n * hw;
  load_tile(g1, a.st.g1 + row, H, W);
  load_tile(wp, a.st.wh + row, H, W);
  __syncthreads();
  const int tx = threadIdx.x % kTileX, ty = threadIdx.x / kTileX;
  const int x = blockIdx.x * kTileX + tx, y = blockIdx.y * kTileY + ty;
  if (x >= W || y >= H) return;
  float l = 0.0f, k = 0.0f;
  if (weighted(a.mask, n, y, x, H, W)) {
    const double c1 = g1[ty + kHalo][tx + kHalo], c2 = wp[ty + kHalo][tx + kHalo];
    float h = 0.0f;
#pragma unroll 7
    for (int dy = 0; dy < 2 * kHalo + 1; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2 * kHalo + 1; ++dx) {
        const float d1 = static_cast<float>(g1[ty + dy][tx + dx] - c1), d2 = static_cast<float>(wp[ty + dy][tx + dx] - c2);
        const float e = d1 * rsqrtf(0.81f + d1 * d1) - d2 * rsqrtf(0.81f + d2 * d2);
        const float e2 = e * e;
        h += e2 / (0.1f + e2);
      }
    l = powf(h + 0.01f, 0.4f);
    k = 0.4f * l / (h + 0.01f);
  }
  const long long o = row + y * static_cast<long long>(W) + x;
  a.loss[o] = l;
  a.st.k[o] = k;
}

struct CensusBwdArgs {
  State st;
  const float* scale;                 // device scalar: upstream gradient / (sum M + 1e-6)
  float* grad;                        // [N][2][H][W]
  int H, W;
};

__global__ void __launch_bounds__(kTileThreads) census_bwd_kernel(CensusBwdArgs a) {
  __shared__ double g1[kSy][kSx], wp[kSy][kSx];
  __shared__ float kk[kSy][kSx];
  const int n = blockIdx.z, H = a.H, W = a.W;
  const long long hw = static_cast<long long>(H) * W, row = n * hw;
  load_tile(g1, a.st.g1 + row, H, W);
  load_tile(wp, a.st.wh + row, H, W);
  load_tile(kk, a.st.k + row, H, W);
  __syncthreads();
  const int tx = threadIdx.x % kTileX, ty = threadIdx.x / kTileX;
  const int x = blockIdx.x * kTileX + tx, y = blockIdx.y * kTileY + ty;
  if (x >= W || y >= H) return;
  const double c1 = g1[ty + kHalo][tx + kHalo], c2 = wp[ty + kHalo][tx + kHalo];
  const float kc = kk[ty + kHalo][tx + kHalo];
  float g = 0.0f;
#pragma unroll 7
  for (int dy = 0; dy < 2 * kHalo + 1; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2 * kHalo + 1; ++dx) {
      const float kw = kc + kk[ty + dy][tx + dx];
      const float d1 = static_cast<float>(g1[ty + dy][tx + dx] - c1), d2 = static_cast<float>(wp[ty + dy][tx + dx] - c2);
      const float r2 = rsqrtf(0.81f + d2 * d2);
      const float e = d1 * rsqrtf(0.81f + d1 * d1) - d2 * r2;
      const float den = 0.1f + e * e;
      g += kw * (0.2f * e / (den * den)) * (0.81f * r2 * r2 * r2);
    }
  g *= *a.scale;
  const long long o = y * static_cast<long long>(W) + x;
  float* out = a.grad + static_cast<long long>(n) * 2 * hw + o;
  out[0] = g * a.st.dwx[row + o];
  out[hw] = g * a.st.dwy[row + o];
}

struct CensusPart {                   // a set of pixels' sum of v l and count of v; 16 bytes
  double s;
  unsigned m, pad;
  __device__ __forceinline__ CensusPart& operator+=(const CensusPart& o) {
    s += o.s;
    m += o.m;
    return *this;
  }
};

__device__ __forceinline__ CensusPart warp_sum(CensusPart v) {
  v.s = rnc::warp_sum(v.s);
  v.m = __reduce_add_sync(0xffffffffu, v.m);
  return v;
}

struct CensusPixel {
  const float* loss;
  const unsigned char* mask;
  int H, W;
  __device__ void operator()(CensusPart& acc, int n, int y, int x) const {
    acc.s += static_cast<double>(loss[(static_cast<long long>(n) * H + y) * W + x]);
    acc.m += weighted(mask, n, y, x, H, W);
  }
};

struct CensusStore {                  // row n -> S[n], M[n]
  double* s;
  long long* m;
  __device__ void operator()(int n, const CensusPart& v) const {
    s[n] = v.s;
    m[n] = v.m;
  }
};

struct SmoothPart {                   // a set of pixels' sums of x- and y-terms
  double x, y;
  __device__ __forceinline__ SmoothPart& operator+=(const SmoothPart& o) {
    x += o.x;
    y += o.y;
    return *this;
  }
};

__device__ __forceinline__ SmoothPart warp_sum(SmoothPart v) {
  v.x = rnc::warp_sum(v.x);
  v.y = rnc::warp_sum(v.y);
  return v;
}

// exp(-kappa mean_c |I(x,y) - I(x-sx, y-sy)| / 255), the edge weight of the terms centred at (x, y) along (sx, sy)
__device__ __forceinline__ float edge_weight(const View& im, int n, int y, int x, int sx, int sy, float kappa) {
  const float* p = im.pixel(n, y, x);
  const float* q = im.pixel(n, y - sy, x - sx);
  const float s = fabsf(p[0] - q[0]) + fabsf(p[im.c] - q[im.c]) + fabsf(p[2 * im.c] - q[2 * im.c]);
  return expf(-kappa * (s / 765.0f));
}

__device__ __forceinline__ float second_diff(const View& f, int n, int c, int y, int x, int sx, int sy) {
  return f.at(n, c, y + sy, x + sx) - 2.0f * f.at(n, c, y, x) + f.at(n, c, y - sy, x - sx);
}

struct SmoothPixel {
  View image, flow;
  int H, W;
  float kappa;
  __device__ void operator()(SmoothPart& acc, int n, int y, int x) const {
    if (x >= 1 && x <= W - 2) {
      const float w = edge_weight(image, n, y, x, 1, 0, kappa);
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float d = second_diff(flow, n, c, y, x, 1, 0);
        acc.x += static_cast<double>(sqrtf(d * d + 1e-6f) * w);
      }
    }
    if (y >= 1 && y <= H - 2) {
      const float w = edge_weight(image, n, y, x, 0, 1, kappa);
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float d = second_diff(flow, n, c, y, x, 0, 1);
        acc.y += static_cast<double>(sqrtf(d * d + 1e-6f) * w);
      }
    }
  }
};

struct SmoothStore {                  // row n -> sum_x[n], sum_y[n]
  double *sx, *sy;
  __device__ void operator()(int n, const SmoothPart& v) const {
    sx[n] = v.x;
    sy[n] = v.y;
  }
};

struct SmoothBwdArgs {
  View image, flow;
  const float* scale;                 // device [2]: the x- and y-terms' upstream gradient over their counts
  float* grad;                        // [N][2][H][W]
  int H, W;
  float kappa;
};

__global__ void __launch_bounds__(kWarpThreads) smoothness_bwd_kernel(SmoothBwdArgs a) {
  const int n = blockIdx.y, H = a.H, W = a.W;
  const long long hw = static_cast<long long>(H) * W;
  const int p = blockIdx.x * kWarpThreads + threadIdx.x;
  if (p >= hw) return;
  const int y = p / W, x = p - y * W;
  float g[2] = {0.0f, 0.0f};
#pragma unroll
  for (int axis = 0; axis < 2; ++axis) {
    const int sx = axis == 0, sy = axis == 1, pos = axis == 0 ? x : y, len = axis == 0 ? W : H;
    float ga[2] = {0.0f, 0.0f};
#pragma unroll
    for (int o = -1; o <= 1; ++o) {               // the terms centred at pos + o hold this pixel with weight 1, -2, 1
      const int q = pos + o;
      if (q < 1 || q > len - 2) continue;
      const int cx = x + o * sx, cy = y + o * sy;
      const float w = edge_weight(a.image, n, cy, cx, sx, sy, a.kappa);
      const float coef = o == 0 ? -2.0f : 1.0f;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float d = second_diff(a.flow, n, c, cy, cx, sx, sy);
        ga[c] += coef * (d * rsqrtf(d * d + 1e-6f)) * w;
      }
    }
    const float s = a.scale[axis];
    g[0] += s * ga[0];
    g[1] += s * ga[1];
  }
  float* out = a.grad + static_cast<long long>(n) * 2 * hw + p;
  out[0] = g[0];
  out[hw] = g[1];
}

// total[0] = a[0] + a[1] + ... in row order, total[1] = the same of b, in fp64
template <typename T>
__global__ void row_totals_kernel(const double* a, const T* b, int n, double* total) {
  double s = 0.0, t = 0.0;
  for (int r = 0; r < n; ++r) {
    s += a[r];
    t += static_cast<double>(b[r]);
  }
  total[0] = s;
  total[1] = t;
}

// N rows (a grid z extent each) of H x W >= 8 x 8 pixels, H*W < 2^30, a tile grid within 65535 rows
bool photometric_shape_ok(int N, int H, int W) {
  return eval_shape_ok(N, H, W) && H >= 8 && W >= 8 && (H + kTileY - 1) / kTileY <= 65535;
}

size_t round16(size_t n) { return (n + 15) & ~static_cast<size_t>(15); }

size_t loss_buffer_bytes(int N, int H, int W) { return round16(static_cast<size_t>(N) * H * W * sizeof(float)); }

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

size_t rnc_census_loss_workspace_bytes(int N, int H, int W) {
  return photometric_shape_ok(N, H, W)
             ? loss_buffer_bytes(N, H, W) + static_cast<size_t>(N) * eval_blocks(H, W) * sizeof(CensusPart)
             : 0;
}

int rnc_census_loss_fwd(const float* image1, long long ab, long long ac, long long ay, long long ax, const float* image2,
                        long long bb, long long bc, long long by, long long bx, const float* flow, long long fb, long long fc,
                        long long fy, long long fx, const unsigned char* mask, int N, int H, int W, double* loss_sum,
                        long long* count, double* total, void* state, void* workspace, size_t workspace_bytes,
                        void* stream) {
  if (!photometric_shape_ok(N, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!image1 || !image2 || !flow || !loss_sum || !count || !total || !state || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(image1, 4) || !aligned(image2, 4) || !aligned(flow, 4) || !aligned(loss_sum, 8) || !aligned(count, 8) ||
      !aligned(total, 8) || !aligned(state, 8) || !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_census_loss_workspace_bytes(N, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const long long hw = static_cast<long long>(H) * W;
  census_warp_kernel<<<dim3(static_cast<unsigned>((hw + kWarpThreads - 1) / kWarpThreads), N), kWarpThreads, 0, s>>>(
      WarpArgs{{image1, ab, ac, ay, ax}, {image2, bb, bc, by, bx}, {flow, fb, fc, fy, fx}, State(state, N * hw), H, W});
  if (int st = after_launch()) return st;
  float* loss = static_cast<float*>(workspace);
  census_fwd_kernel<<<dim3((W + kTileX - 1) / kTileX, (H + kTileY - 1) / kTileY, N), kTileThreads, 0, s>>>(
      CensusArgs{State(state, N * hw), mask, loss, H, W});
  if (int st = after_launch()) return st;
  const int nblk = eval_blocks(H, W);
  auto* parts = reinterpret_cast<CensusPart*>(static_cast<char*>(workspace) + loss_buffer_bytes(N, H, W));
  cta_partials_kernel<<<dim3(nblk, N), kEvalThreads, 0, s>>>(CensusPixel{loss, mask, H, W}, H, W, parts);
  if (int st = after_launch()) return st;
  if (int st = launch_image_reduce(parts, N, nblk, 1, CensusStore{loss_sum, count}, s)) return st;
  row_totals_kernel<<<1, 1, 0, s>>>(loss_sum, count, N, total);
  return after_launch();
}

int rnc_census_loss_bwd(const void* state, int N, int H, int W, const float* scale, float* grad_flow, void* stream) {
  if (!photometric_shape_ok(N, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!state || !scale || !grad_flow) return RNC_ERR_BAD_POINTER;
  if (!aligned(state, 8) || !aligned(scale, 4) || !aligned(grad_flow, 4)) return RNC_ERR_BAD_POINTER;
  const long long hw = static_cast<long long>(H) * W;
  census_bwd_kernel<<<dim3((W + kTileX - 1) / kTileX, (H + kTileY - 1) / kTileY, N), kTileThreads, 0, as_stream(stream)>>>(
      CensusBwdArgs{State(const_cast<void*>(state), N * hw), scale, grad_flow, H, W});
  return after_launch();
}

size_t rnc_smoothness_workspace_bytes(int N, int H, int W) {
  return photometric_shape_ok(N, H, W) ? static_cast<size_t>(N) * eval_blocks(H, W) * sizeof(SmoothPart) : 0;
}

int rnc_smoothness_fwd(const float* image, long long ib, long long ic, long long iy, long long ix, const float* flow,
                       long long fb, long long fc, long long fy, long long fx, int N, int H, int W, float edge_constant,
                       double* sum_x, double* sum_y, double* total, void* workspace, size_t workspace_bytes, void* stream) {
  if (!photometric_shape_ok(N, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!image || !flow || !sum_x || !sum_y || !total || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(image, 4) || !aligned(flow, 4) || !aligned(sum_x, 8) || !aligned(sum_y, 8) || !aligned(total, 8) ||
      !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_smoothness_workspace_bytes(N, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const int nblk = eval_blocks(H, W);
  auto* parts = static_cast<SmoothPart*>(workspace);
  cta_partials_kernel<<<dim3(nblk, N), kEvalThreads, 0, s>>>(
      SmoothPixel{{image, ib, ic, iy, ix}, {flow, fb, fc, fy, fx}, H, W, edge_constant}, H, W, parts);
  if (int st = after_launch()) return st;
  if (int st = launch_image_reduce(parts, N, nblk, 1, SmoothStore{sum_x, sum_y}, s)) return st;
  row_totals_kernel<<<1, 1, 0, s>>>(sum_x, sum_y, N, total);
  return after_launch();
}

int rnc_smoothness_bwd(const float* image, long long ib, long long ic, long long iy, long long ix, const float* flow,
                       long long fb, long long fc, long long fy, long long fx, int N, int H, int W, float edge_constant,
                       const float* scale, float* grad_flow, void* stream) {
  if (!photometric_shape_ok(N, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!image || !flow || !scale || !grad_flow) return RNC_ERR_BAD_POINTER;
  if (!aligned(image, 4) || !aligned(flow, 4) || !aligned(scale, 4) || !aligned(grad_flow, 4)) return RNC_ERR_BAD_POINTER;
  const long long hw = static_cast<long long>(H) * W;
  smoothness_bwd_kernel<<<dim3(static_cast<unsigned>((hw + kWarpThreads - 1) / kWarpThreads), N), kWarpThreads, 0,
                          as_stream(stream)>>>(
      SmoothBwdArgs{{image, ib, ic, iy, ix}, {flow, fb, fc, fy, fx}, scale, grad_flow, H, W, edge_constant});
  return after_launch();
}

}  // extern "C"
