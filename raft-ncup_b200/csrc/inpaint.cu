// Flow-guided video inpainting (the definition: rnc/inpaint.py and DESIGN §3.19): the harmonic fill that completes a field
// inside a hole, the temporal propagation of colours along the completed flows, and SSIM's per-frame partials.
//
// rnc_harmonic_fill, N = A*B images of C channels, image i = (a, b) = (i / B, i % B), in 5 + 2 * sweeps launches:
//   1. known_kernel, a thread per pixel: known = !unknown && every channel finite, into a uint8 map.  Per CTA it counts the
//      unknown pixels of each colour ((x + y) & 1: 0 red, 1 black) and the bounding box of the unknown pixels.
//   2. dist_transform.cuh's column and row passes with the known pixels as sites; the row pass's Out writes every pixel: a known
//      pixel its own values, an unknown one the values of its nearest known pixel, 0 in an image without one.
//   3. list_offsets_kernel, a CTA per image: the exclusive prefix of the CTAs' colour counts, the image's counts, and
//      omega = 2 / (1 + pi_f32 / (L + 1)) from the bounding box's larger side L, each operation rounded once.
//   4. compact_kernel, a thread per pixel: each unknown pixel's index into its image's red list (at the front) or black list
//      (after the red one), in pixel order.  The lists reuse the int map of step 2.
//   5. sweeps times sor_kernel<red> then sor_kernel<black>: a thread per list entry (grid-strided over a fixed grid row per
//      image) updates u += omega (avg - u), avg the in-frame 4-neighbours added up, left, right, down, over their count.  A
//      colour's pixels only read the other colour, so any order of its updates gives the sequential sweep's bits.
// rnc_inpaint_propagate: one launch, a thread per pixel of every frame of every video.  A hole pixel walks its forward and its
// backward chain with the position in registers, takes the masked bilinear colour at each chain's end and combines the two by
// distance; every other pixel copies its colour.
// rnc_ssim_partials: per frame, the fp64 sum of the SSIM map over the 3 channels and the pixels whose 11x11 window is inside,
// and its count, through eval_common.cuh's two fixed-order reductions.
// Every floating-point operation of the three is a __*_rn intrinsic in the order rnc/inpaint.py's host restatements write it,
// so the host gives the same bits (SSIM's fp64 sums agree to their last bits).  No atomics and no host synchronisation.
#include <cmath>

#include "bilinear.cuh"
#include "dist_transform.cuh"
#include "eval_common.cuh"

namespace rnc {
namespace {

constexpr int kFillThreads = 256;
constexpr int kMaxChannels = RNC_HARMONIC_MAX_CHANNELS;
constexpr int kSorRowCtas = 1056;           // the sweep grid's CTAs over all images (8 per SM of an H100 SXM)
constexpr int kPropThreads = 256;
constexpr int kSsimRadius = 5;
constexpr float kPiF32 = 3.14159265358979f;

// image i of the A*B images of a [A][B][C][H][W] view (v the A stride, b the B stride)
template <typename T>
__device__ __forceinline__ T* image_pixel(const VideoView<T>& t, int B, int i, int y, int x) {
  const int ia = i / B, ib = i - ia * B;
  return t.video(ia).pixel(ib, y, x);
}

struct FillBlock {                            // one CTA's part of an image: unknown pixels per colour and their bounding box
  int n[2];
  int x0, x1, y0, y1;
  int pad;
};

struct FillImage {                            // per image: the list lengths per colour and the relaxation factor
  int n[2];
  float omega;
  int pad;
};

struct FillLayout {                           // the workspace
  unsigned char* known;                       // [N][H][W]
  int* map;                                   // [N][H][W]: the distance transform's rows, then the unknown pixels' lists
  FillBlock* blocks;                          // [N][nblk]: counts, then their exclusive prefix
  FillImage* images;                          // [N]
};

FillLayout fill_layout(Carve& ws, int N, int H, int W) {
  const size_t px = static_cast<size_t>(N) * H * W;
  const int nblk = (H * W + kFillThreads - 1) / kFillThreads;
  FillLayout l;
  l.map = ws.take<int>(px);
  l.blocks = ws.take<FillBlock>(static_cast<size_t>(N) * nblk);
  l.images = ws.take<FillImage>(N);
  l.known = ws.take<unsigned char>(px);
  return l;
}

__global__ void __launch_bounds__(kFillThreads) known_kernel(Video in, VideoMask unknown, int B, int C, int H, int W,
                                                             FillLayout l) {
  const int i = blockIdx.y, hw = H * W;
  const int p = blockIdx.x * kFillThreads + threadIdx.x;
  bool unk = false;
  int y = 0, x = 0;
  if (p < hw) {
    y = p / W;
    x = p - y * W;
    bool known = *image_pixel(unknown, B, i, y, x) == 0;
    const float* v = image_pixel(in, B, i, y, x);
    for (int c = 0; c < C; ++c) known = known && finite(v[c * in.c]);
    l.known[static_cast<long long>(i) * hw + p] = known;
    unk = !known;
  }
  const int red = __syncthreads_count(unk && ((x + y) & 1) == 0);
  const int black = __syncthreads_count(unk && ((x + y) & 1) == 1);
  const int x0 = __reduce_min_sync(0xffffffffu, unk ? x : INT_MAX), x1 = __reduce_max_sync(0xffffffffu, unk ? x : -1);
  const int y0 = __reduce_min_sync(0xffffffffu, unk ? y : INT_MAX), y1 = __reduce_max_sync(0xffffffffu, unk ? y : -1);
  __shared__ int4 box[kFillThreads / 32];
  if ((threadIdx.x & 31) == 0) box[threadIdx.x >> 5] = make_int4(x0, x1, y0, y1);
  __syncthreads();
  if (threadIdx.x == 0) {
    FillBlock b{{red, black}, INT_MAX, -1, INT_MAX, -1, 0};
    for (int w = 0; w < kFillThreads / 32; ++w) {
      b.x0 = min(b.x0, box[w].x);
      b.x1 = max(b.x1, box[w].y);
      b.y0 = min(b.y0, box[w].z);
      b.y1 = max(b.y1, box[w].w);
    }
    l.blocks[static_cast<long long>(i) * gridDim.x + blockIdx.x] = b;
  }
}

struct KnownSites {
  const unsigned char* known;
  int hw, W;
  __device__ bool operator()(int i, int y, int x) const { return known[static_cast<long long>(i) * hw + y * W + x] != 0; }
};

struct InitOut {                              // a known pixel keeps its values, an unknown one takes its nearest known pixel's
  static constexpr bool kStores = true;
  Video in;
  VideoView<float> out;
  int B, C;
  __device__ void store(int i, int y, int x, int q, int r) const {
    float* o = image_pixel(out, B, i, y, x);
    if (q < 0) {
      for (int c = 0; c < C; ++c) o[c * out.c] = 0.0f;
      return;
    }
    const float* v = image_pixel(in, B, i, r, q);
    for (int c = 0; c < C; ++c) o[c * out.c] = v[c * in.c];
  }
};

// a CTA per image: blocks[i][*].n becomes its exclusive prefix per colour; the image's totals, its bounding box and omega
__global__ void __launch_bounds__(kFillThreads) list_offsets_kernel(int nblk, FillLayout l) {
  const int i = blockIdx.x, t = threadIdx.x;
  FillBlock* blk = l.blocks + static_cast<long long>(i) * nblk;
  const int per = (nblk + kFillThreads - 1) / kFillThreads, lo = min(t * per, nblk), hi = min(lo + per, nblk);
  int s[2] = {0, 0}, x0 = INT_MAX, x1 = -1, y0 = INT_MAX, y1 = -1;
  for (int k = lo; k < hi; ++k) {
    const FillBlock b = blk[k];
    s[0] += b.n[0];
    s[1] += b.n[1];
    x0 = min(x0, b.x0);
    x1 = max(x1, b.x1);
    y0 = min(y0, b.y0);
    y1 = max(y1, b.y1);
  }
  __shared__ int sums[2][kFillThreads];
  __shared__ int4 box[kFillThreads / 32];
  sums[0][t] = s[0];
  sums[1][t] = s[1];
  x0 = __reduce_min_sync(0xffffffffu, x0);
  x1 = __reduce_max_sync(0xffffffffu, x1);
  y0 = __reduce_min_sync(0xffffffffu, y0);
  y1 = __reduce_max_sync(0xffffffffu, y1);
  if ((t & 31) == 0) box[t >> 5] = make_int4(x0, x1, y0, y1);
  __syncthreads();
  if (t == 0) {                               // the threads' exclusive prefix, serially: integers, any order is exact
    int run[2] = {0, 0};
    for (int k = 0; k < kFillThreads; ++k) {
      for (int c = 0; c < 2; ++c) {
        const int v = sums[c][k];
        sums[c][k] = run[c];
        run[c] += v;
      }
    }
    for (int w = 0; w < kFillThreads / 32; ++w) {
      x0 = min(x0, box[w].x);
      x1 = max(x1, box[w].y);
      y0 = min(y0, box[w].z);
      y1 = max(y1, box[w].w);
    }
    const int L = x1 < 0 ? 0 : max(x1 - x0 + 1, y1 - y0 + 1);
    l.images[i] = {{run[0], run[1]},
                   __fdiv_rn(2.0f, __fadd_rn(1.0f, __fdiv_rn(kPiF32, static_cast<float>(L + 1)))),
                   0};
  }
  __syncthreads();
  int off[2] = {sums[0][t], sums[1][t]};
  for (int k = lo; k < hi; ++k) {
    const int n0 = blk[k].n[0], n1 = blk[k].n[1];
    blk[k].n[0] = off[0];
    blk[k].n[1] = off[1];
    off[0] += n0;
    off[1] += n1;
  }
}

__global__ void __launch_bounds__(kFillThreads) compact_kernel(int H, int W, FillLayout l) {
  const int i = blockIdx.y, hw = H * W;
  const int p = blockIdx.x * kFillThreads + threadIdx.x;
  const int y = p / W, x = p - y * W;
  const bool unk = p < hw && l.known[static_cast<long long>(i) * hw + p] == 0;
  const int colour = (x + y) & 1;
  const unsigned lanes_below = (1u << (threadIdx.x & 31)) - 1u;
  const unsigned in[2] = {__ballot_sync(0xffffffffu, unk && colour == 0), __ballot_sync(0xffffffffu, unk && colour == 1)};
  __shared__ int warp_n[2][kFillThreads / 32];
  if ((threadIdx.x & 31) == 0) {
    warp_n[0][threadIdx.x >> 5] = __popc(in[0]);
    warp_n[1][threadIdx.x >> 5] = __popc(in[1]);
  }
  __syncthreads();
  if (!unk) return;
  int rank = __popc(in[colour] & lanes_below);
  for (int w = 0; w < static_cast<int>(threadIdx.x >> 5); ++w) rank += warp_n[colour][w];
  const FillBlock& b = l.blocks[static_cast<long long>(i) * gridDim.x + blockIdx.x];
  const int base = colour ? l.images[i].n[0] : 0;
  l.map[static_cast<long long>(i) * hw + base + b.n[colour] + rank] = p;
}

template <int Colour>
__global__ void __launch_bounds__(kFillThreads) sor_kernel(VideoView<float> u, int B, int C, int H, int W, FillLayout l) {
  const int i = blockIdx.y, hw = H * W;
  const FillImage im = l.images[i];
  const int n = im.n[Colour];
  const int* list = l.map + static_cast<long long>(i) * hw + (Colour ? im.n[0] : 0);
  for (int e = blockIdx.x * kFillThreads + threadIdx.x; e < n; e += gridDim.x * kFillThreads) {
    const int p = list[e], y = p / W, x = p - y * W;
    float* o = image_pixel(u, B, i, y, x);
    const bool up = y > 0, left = x > 0, right = x < W - 1, down = y < H - 1;
    const int nb = up + left + right + down;
    if (nb == 0) continue;                    // a 1x1 image: no neighbour, the value stays
    const float cnt = static_cast<float>(nb);
    for (int c = 0; c < C; ++c) {
      const long long co = c * u.c;
      float s = -0.0f;                        // -0 + v == v for every v: the first neighbour starts the sum exactly
      if (up) s = __fadd_rn(s, o[co - u.y]);
      if (left) s = __fadd_rn(s, o[co - u.x]);
      if (right) s = __fadd_rn(s, o[co + u.x]);
      if (down) s = __fadd_rn(s, o[co + u.y]);
      const float v = o[co];
      o[co] = __fadd_rn(v, __fmul_rn(im.omega, __fsub_rn(__fdiv_rn(s, cnt), v)));
    }
  }
}

bool fill_shape_ok(int A, int B, int C, int H, int W) {
  return A > 0 && B > 0 && static_cast<long long>(A) * B <= 65535 && C > 0 && C <= kMaxChannels && H > 0 && W > 0 &&
         H <= kSiteMaxSide && W <= kSiteMaxSide;
}

// ------------------------------------------------------------------------------------------------ temporal propagation

struct PropArgs {
  const float* frames;                        // I [V][T][3][H][W]
  long long iv, it, ic, iy, ix;
  const unsigned char* masks;                 // M [V][T][H][W]
  long long mv, mt, my, mx;
  Video flow[2];                              // F~_k, G~_k: b is the pair index k
  VideoMask occ[2];                           // occ~_k on frame k, occ~_bw_k on frame k+1
  float* out;                                 // [V][T][3][H][W] contiguous
  unsigned char* source;                      // [V][T][H][W] contiguous
  int T, H, W, max_distance;
};

__device__ __forceinline__ unsigned char mask_at(const PropArgs& a, int v, int t, int y, int x) {
  return a.masks[v * a.mv + t * a.mt + y * a.my + x * a.mx];
}

// one direction's chain from hole pixel (x, y) of frame t: true with the colour c and distance d of its candidate
template <int Dir>
__device__ __forceinline__ bool chain(const PropArgs& a, int v, int t, float x, float y, float c[3], int& d) {
  const int T = a.T, H = a.H, W = a.W;
  const View fl = a.flow[Dir > 0 ? 0 : 1].video(v);
  const MaskView oc = a.occ[Dir > 0 ? 0 : 1].video(v);
  int k = t;
  d = 0;
  for (;;) {
    if ((Dir > 0 ? k == T - 1 : k == 0) || d == a.max_distance) return false;
    const int pair = Dir > 0 ? k : k - 1;
    if (oc.at(pair, static_cast<int>(rintf(y)), static_cast<int>(rintf(x))) != 0) return false;
    const float nx = __fadd_rn(x, sample(fl, pair, 0, x, y, H, W)), ny = __fadd_rn(y, sample(fl, pair, 1, x, y, H, W));
    if (!inside(nx, ny, H, W)) return false;
    k += Dir;
    ++d;
    x = nx;
    y = ny;
    if (mask_at(a, v, k, static_cast<int>(rintf(y)), static_cast<int>(rintf(x))) == 0) break;
  }
  // the masked bilinear colour of I_k at (x, y): the taps outside the hole, weights and weighted colours added in tap order
  const BilinearTaps tp = bilinear_taps(x, y, H, W);
  const float w[4] = {tp.w(0), tp.w(1), tp.w(2), tp.w(3)};
  float ws = -0.0f, s[3] = {-0.0f, -0.0f, -0.0f};
  const float* img = a.frames + v * a.iv + k * a.it;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int ty = tp.y[j >> 1], tx = tp.x[j & 1];
    if (mask_at(a, v, k, ty, tx) != 0) continue;
    ws = __fadd_rn(ws, w[j]);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) s[ch] = __fadd_rn(s[ch], __fmul_rn(w[j], img[ch * a.ic + ty * a.iy + tx * a.ix]));
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) c[ch] = __fdiv_rn(s[ch], ws);
  return true;
}

__global__ void __launch_bounds__(kPropThreads) propagate_kernel(PropArgs a) {
  const int t = blockIdx.y, v = blockIdx.z, H = a.H, W = a.W, hw = H * W;
  const int p = blockIdx.x * kPropThreads + threadIdx.x;
  if (p >= hw) return;
  const int y = p / W, x = p - y * W;
  const long long vt = static_cast<long long>(v) * a.T + t;
  float* o = a.out + vt * 3 * hw + p;
  unsigned char* src = a.source + vt * hw + p;
  if (mask_at(a, v, t, y, x) == 0) {
    const float* img = a.frames + v * a.iv + t * a.it + y * a.iy + x * a.ix;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) o[ch * hw] = img[ch * a.ic];
    *src = RNC_INPAINT_KNOWN;
    return;
  }
  float cf[3], cb[3];
  int df, db;
  const bool hf = chain<1>(a, v, t, static_cast<float>(x), static_cast<float>(y), cf, df);
  const bool hb = chain<-1>(a, v, t, static_cast<float>(x), static_cast<float>(y), cb, db);
  if (hf && hb) {
    const float wf = static_cast<float>(db), wb = static_cast<float>(df), den = static_cast<float>(df + db);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) o[ch * hw] = __fdiv_rn(__fadd_rn(__fmul_rn(wf, cf[ch]), __fmul_rn(wb, cb[ch])), den);
    *src = RNC_INPAINT_BOTH;
  } else if (hf || hb) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) o[ch * hw] = hf ? cf[ch] : cb[ch];
    *src = hf ? RNC_INPAINT_FORWARD : RNC_INPAINT_BACKWARD;
  } else {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) o[ch * hw] = 0.0f;
    *src = RNC_INPAINT_SPATIAL;
  }
}

bool prop_shape_ok(int V, int T, int H, int W) {
  return V > 0 && V <= 65535 && T >= 2 && T <= 65535 && H > 0 && W > 0 && H <= kSiteMaxSide && W <= kSiteMaxSide;
}

// ------------------------------------------------------------------------------------------------ SSIM

// the 11-tap Gaussian of sigma 1.5, normalised in fp64, as float32
__constant__ float kGauss[2 * kSsimRadius + 1] = {
    1.028380124e-03f, 7.598758209e-03f, 3.600077331e-02f, 1.093606874e-01f, 2.130055428e-01f, 2.660117149e-01f,
    2.130055428e-01f, 1.093606874e-01f, 3.600077331e-02f, 7.598758209e-03f, 1.028380124e-03f};

struct SsimPixel {                            // cta_partials_kernel's pixel (n, y, x): the window centred on (y, x)
  View pred, gt;
  int H, W;
  __device__ void operator()(SumCount& acc, int n, int y, int x) const {
    if (y < kSsimRadius || y >= H - kSsimRadius || x < kSsimRadius || x >= W - kSsimRadius) return;
    constexpr float C1 = 6.5025f, C2 = 58.5225f;          // (0.01 * 255)^2, (0.03 * 255)^2
    for (int c = 0; c < 3; ++c) {
      float m[5];                                         // the filtered x, y, x^2, y^2, xy
      for (int i = 0; i < 2 * kSsimRadius + 1; ++i) {
        const int yy = y - kSsimRadius + i;
        float h[5];
        for (int j = 0; j < 2 * kSsimRadius + 1; ++j) {
          const int xx = x - kSsimRadius + j;
          const float a = pred.at(n, c, yy, xx), b = gt.at(n, c, yy, xx);
          const float q[5] = {a, b, __fmul_rn(a, a), __fmul_rn(b, b), __fmul_rn(a, b)};
#pragma unroll
          for (int k = 0; k < 5; ++k) h[k] = j ? __fadd_rn(h[k], __fmul_rn(kGauss[j], q[k])) : __fmul_rn(kGauss[j], q[k]);
        }
#pragma unroll
        for (int k = 0; k < 5; ++k) m[k] = i ? __fadd_rn(m[k], __fmul_rn(kGauss[i], h[k])) : __fmul_rn(kGauss[i], h[k]);
      }
      const float mx2 = __fmul_rn(m[0], m[0]), my2 = __fmul_rn(m[1], m[1]), mxy = __fmul_rn(m[0], m[1]);
      const float sx = __fsub_rn(m[2], mx2), sy = __fsub_rn(m[3], my2), sxy = __fsub_rn(m[4], mxy);
      const float num = __fmul_rn(__fadd_rn(__fmul_rn(2.0f, mxy), C1), __fadd_rn(__fmul_rn(2.0f, sxy), C2));
      const float den = __fmul_rn(__fadd_rn(__fadd_rn(mx2, my2), C1), __fadd_rn(__fadd_rn(sx, sy), C2));
      acc.sum += static_cast<double>(__fdiv_rn(num, den));
      acc.n += 1;
    }
  }
};

bool ssim_shape_ok(int N, int H, int W) { return eval_shape_ok(N, H, W) && H >= 2 * kSsimRadius + 1 && W >= 2 * kSsimRadius + 1; }

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

size_t rnc_harmonic_fill_workspace_bytes(int A, int B, int C, int H, int W) {
  if (!fill_shape_ok(A, B, C, H, W)) return 0;
  Carve ws{nullptr};
  fill_layout(ws, A * B, H, W);
  return ws.bytes;
}

int rnc_harmonic_fill(const float* values, long long va, long long vb, long long vc, long long vy, long long vx,
                      const unsigned char* unknown, long long ua, long long ub, long long uy, long long ux, int A, int B,
                      int C, int H, int W, int sweeps, float* out, long long oa, long long ob, long long oc, long long oy,
                      long long ox, void* workspace, size_t workspace_bytes, void* stream) {
  if (!fill_shape_ok(A, B, C, H, W) || sweeps < 0) return RNC_ERR_BAD_SHAPE;
  if (!values || !unknown || !out || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(values, 4) || !aligned(out, 4) || !aligned(workspace, 16)) return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_harmonic_fill_workspace_bytes(A, B, C, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const int N = A * B, hw = H * W, nblk = (hw + kFillThreads - 1) / kFillThreads;
  const Video in{values, va, vb, vc, vy, vx};
  const VideoMask unk{unknown, ua, ub, 0, uy, ux};
  const VideoView<float> o{out, oa, ob, oc, oy, ox};
  Carve ws{static_cast<char*>(workspace)};
  const FillLayout l = fill_layout(ws, N, H, W);
  known_kernel<<<dim3(nblk, N), kFillThreads, 0, s>>>(in, unk, B, C, H, W, l);
  if (int st = after_launch()) return st;
  dist2_column_kernel<<<dim3((W + kSiteColThreads - 1) / kSiteColThreads, N), kSiteColThreads, 0, s>>>(
      KnownSites{l.known, hw, W}, H, W, l.map);
  if (int st = after_launch()) return st;
  dist2_row_kernel<<<dim3(H, N), 32, dist2_row_smem(W), s>>>(H, W, l.map, InitOut{in, o, B, C});
  if (int st = after_launch()) return st;
  list_offsets_kernel<<<N, kFillThreads, 0, s>>>(nblk, l);
  if (int st = after_launch()) return st;
  compact_kernel<<<dim3(nblk, N), kFillThreads, 0, s>>>(H, W, l);
  if (int st = after_launch()) return st;
  // a fixed grid row per image, wide enough for a full-frame hole's half and for the whole GPU when there are few images
  const int row = max(1, min((kSorRowCtas + N - 1) / N, (hw / 2 + kFillThreads) / kFillThreads));
  for (int k = 0; k < sweeps; ++k) {
    sor_kernel<0><<<dim3(row, N), kFillThreads, 0, s>>>(o, B, C, H, W, l);
    if (int st = after_launch()) return st;
    sor_kernel<1><<<dim3(row, N), kFillThreads, 0, s>>>(o, B, C, H, W, l);
    if (int st = after_launch()) return st;
  }
  return RNC_OK;
}

int rnc_inpaint_propagate(const float* frames, long long iv, long long it, long long ic, long long iy, long long ix,
                          const unsigned char* masks, long long mv, long long mt, long long my, long long mx,
                          const float* flow, long long fv, long long fk, long long fc, long long fy, long long fx,
                          const float* flow_bw, long long gv, long long gk, long long gc, long long gy, long long gx,
                          const unsigned char* occ, long long ov, long long ok, long long oy, long long ox,
                          const unsigned char* occ_bw, long long pv, long long pk, long long py, long long px, int V, int T,
                          int H, int W, int max_distance, float* out, unsigned char* source, void* stream) {
  if (!prop_shape_ok(V, T, H, W) || max_distance < 1) return RNC_ERR_BAD_SHAPE;
  if (!frames || !masks || !flow || !flow_bw || !occ || !occ_bw || !out || !source) return RNC_ERR_BAD_POINTER;
  if (!aligned(frames, 4) || !aligned(flow, 4) || !aligned(flow_bw, 4) || !aligned(out, 4)) return RNC_ERR_BAD_POINTER;
  const PropArgs a{frames, iv, it, ic, iy, ix, masks, mv, mt, my, mx,
                   {{flow, fv, fk, fc, fy, fx}, {flow_bw, gv, gk, gc, gy, gx}},
                   {{occ, ov, ok, 0, oy, ox}, {occ_bw, pv, pk, 0, py, px}},
                   out, source, T, H, W, max_distance};
  propagate_kernel<<<dim3((H * W + kPropThreads - 1) / kPropThreads, T, V), kPropThreads, 0, as_stream(stream)>>>(a);
  return after_launch();
}

size_t rnc_ssim_partials_workspace_bytes(int N, int H, int W) {
  return ssim_shape_ok(N, H, W) ? static_cast<size_t>(N) * eval_blocks(H, W) * sizeof(SumCount) : 0;
}

int rnc_ssim_partials(const float* pred, long long pn, long long pc, long long py, long long px, const float* gt,
                      long long gn, long long gc, long long gy, long long gx, int N, int H, int W, double* sum,
                      long long* count, void* workspace, size_t workspace_bytes, void* stream) {
  if (!ssim_shape_ok(N, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!pred || !gt || !sum || !count || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(pred, 4) || !aligned(gt, 4) || !aligned(sum, 8) || !aligned(count, 8) || !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_ssim_partials_workspace_bytes(N, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const int nblk = eval_blocks(H, W);
  SumCount* parts = static_cast<SumCount*>(workspace);
  cta_partials_kernel<<<dim3(nblk, N), kEvalThreads, 0, s>>>(SsimPixel{{pred, pn, pc, py, px}, {gt, gn, gc, gy, gx}, H, W},
                                                            H, W, parts);
  if (int st = after_launch()) return st;
  return launch_image_reduce(parts, N, nblk, 1, SumCountStore{sum, count}, s);
}

}  // extern "C"
