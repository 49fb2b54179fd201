// What the evaluation kernels share: the float32 per-pixel arithmetic of the validation metrics, a strided view of an input,
// the host-side checks, and the two fixed-order reductions that make an image's partials the same bits whatever the batch,
// the image's position in it, the rank or the GPU.
//
// A kernel's partials are reduced in two launches.  CTA (x, b) of cta_partials_kernel takes kEvalPerCta pixels of image b
// (kEvalPerThread per thread, strided by the CTA size), accumulates each thread's pixels in order, adds a warp's threads with
// warp_sum and then the CTA's warps in order, and writes one Part per (image, CTA).  image_reduce_kernel then adds each
// (image, cell)'s CTAs with a warp: lane-strided, then warp_sum.  The grid's x extent depends only on H*W, so the order of every
// addition depends only on the image's size.
#pragma once
#include <type_traits>

#include "rnc_common.cuh"

namespace rnc {

// Each value is what torch computes in float32 on the host: dx = flow - gt, epe = sqrt(dx*dx + dy*dy), mag the same from gt,
// outlier = epe > 3 & epe / mag > 0.05 (a Python float compared with a float32 tensor is rounded to float32).  The *_rn
// intrinsics keep nvcc from contracting any of it into an FMA, and IEEE division gives x/0 = inf and 0/0 = NaN, so a
// zero-magnitude ground truth, NaN and inf count as the torch comparisons count them.
struct PixelMetrics {
  float epe, mag;
  bool outlier;
};

__device__ __forceinline__ PixelMetrics pixel_metrics(float f0, float f1, float g0, float g1) {
  const float dx = __fsub_rn(f0, g0), dy = __fsub_rn(f1, g1);
  const float epe = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
  const float mag = __fsqrt_rn(__fadd_rn(__fmul_rn(g0, g0), __fmul_rn(g1, g1)));
  return {epe, mag, static_cast<bool>((epe > 3.0f) & (__fdiv_rn(epe, mag) > 0.05f))};
}

// A tensor through element strides: [B,C,H,W], or a [B,H,W] mask with c unused.
template <typename T>
struct StridedView {
  T* p;
  long long b, c, y, x;
  __device__ __forceinline__ T* pixel(int bi, int yi, int xi) const { return p + bi * b + yi * y + xi * x; }
  __device__ __forceinline__ std::remove_const_t<T> at(int bi, int ci, int yi, int xi) const { return pixel(bi, yi, xi)[ci * c]; }
  __device__ __forceinline__ std::remove_const_t<T> at(int bi, int yi, int xi) const { return *pixel(bi, yi, xi); }
};
using View = StridedView<const float>;
using MaskView = StridedView<const unsigned char>;   // uint8 masks, visible where 0
using OutView = StridedView<float>;
using OutMaskView = StridedView<unsigned char>;

// A stack of such tensors, one per video ([V][B,C,H,W]) through the stride v between videos: video(i) is video i's view.
template <typename T>
struct VideoView {
  T* p;
  long long v, b, c, y, x;
  __device__ __forceinline__ StridedView<T> video(int i) const { return {p + i * v, b, c, y, x}; }
};
using Video = VideoView<const float>;
using VideoMask = VideoView<const unsigned char>;

inline bool aligned(const void* p, uintptr_t n) { return (reinterpret_cast<uintptr_t>(p) & (n - 1)) == 0; }

// the batches the per-image partials accept: B images (one grid row each) of H*W < 2^30 pixels
inline bool eval_shape_ok(int B, int H, int W) {
  return B > 0 && H > 0 && W > 0 && B <= 65535 && static_cast<long long>(H) * W < (1ll << 30);
}

constexpr int kEvalThreads = 256;
constexpr int kEvalWarps = kEvalThreads / 32;
constexpr int kEvalPerThread = 8;
constexpr int kEvalPerCta = kEvalThreads * kEvalPerThread;

inline int eval_blocks(int H, int W) { return (H * W + kEvalPerCta - 1) / kEvalPerCta; }

// A part is zero when value-initialised and adds with +=.  warp_sum gives lane 0 the sum of its warp's parts: floating-point
// values by a fixed xor-shuffle tree, counts (exact in any order) by one warp reduction.
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

constexpr int kMetCounts = 5;         // valid, epe < 1, < 3, < 5, KITTI outliers

struct MetricsPart {                  // the flow metrics' partials of a set of pixels; 32 bytes
  double epe_sum;
  unsigned n[kMetCounts];
  unsigned pad;
  __device__ __forceinline__ MetricsPart& operator+=(const MetricsPart& o) {
    epe_sum += o.epe_sum;
#pragma unroll
    for (int c = 0; c < kMetCounts; ++c) n[c] += o.n[c];
    return *this;
  }
};

__device__ __forceinline__ MetricsPart warp_sum(MetricsPart v) {
  v.epe_sum = warp_sum(v.epe_sum);
#pragma unroll
  for (int c = 0; c < kMetCounts; ++c) v.n[c] = __reduce_add_sync(0xffffffffu, v.n[c]);
  return v;
}

struct SumCount {                     // a set of pixels' fp64 sum and count; 16 bytes
  double sum;
  unsigned n, pad;
  __device__ __forceinline__ SumCount& operator+=(const SumCount& o) {
    sum += o.sum;
    n += o.n;
    return *this;
  }
};

__device__ __forceinline__ SumCount warp_sum(SumCount v) {
  v.sum = warp_sum(v.sum);
  v.n = __reduce_add_sync(0xffffffffu, v.n);
  return v;
}

struct SumCountStore {                // partials of (image, cell) i -> sum [i], count [i]
  double* sum;
  long long* count;
  __device__ void operator()(int i, const SumCount& v) const {
    sum[i] = v.sum;
    count[i] = v.n;
  }
};

template <int N>
struct Counts {                       // N exact counts of a set of pixels
  unsigned n[N];
  __device__ __forceinline__ Counts& operator+=(const Counts& o) {
#pragma unroll
    for (int c = 0; c < N; ++c) n[c] += o.n[c];
    return *this;
  }
};

template <int N>
__device__ __forceinline__ Counts<N> warp_sum(Counts<N> v) {
#pragma unroll
  for (int c = 0; c < N; ++c) v.n[c] = __reduce_add_sync(0xffffffffu, v.n[c]);
  return v;
}

template <int N>
struct CountsStore {                  // partials of (image, cell) i -> counts [i][N]
  long long* counts;
  __device__ void operator()(int i, const Counts<N>& v) const {
#pragma unroll
    for (int c = 0; c < N; ++c) counts[static_cast<long long>(i) * N + c] = v.n[c];
  }
};

struct MetricsStore {                 // partials of (image, cell) i -> counts [i][5], epe_sum [i]
  long long* counts;
  double* epe_sum;
  __device__ void operator()(int i, const MetricsPart& v) const {
    epe_sum[i] = v.epe_sum;
#pragma unroll
    for (int c = 0; c < kMetCounts; ++c) counts[static_cast<long long>(i) * kMetCounts + c] = v.n[c];
  }
};

// grid (eval_blocks(H, W), B): pixel(acc, b, y, x) adds pixel (y, x) of image b into the thread's acc; -> parts [B][nblk]
template <typename Part, typename Pixel>
__global__ void __launch_bounds__(kEvalThreads) cta_partials_kernel(Pixel pixel, int H, int W, Part* __restrict__ parts) {
  const int b = blockIdx.y, hw = H * W;
  Part acc{};
  for (int p = blockIdx.x * kEvalPerCta + threadIdx.x, e = 0; e < kEvalPerThread && p < hw; ++e, p += kEvalThreads) {
    const int y = p / W, x = p - y * W;
    pixel(acc, b, y, x);
  }
  acc = warp_sum(acc);
  __shared__ Part warps[kEvalWarps];
  if ((threadIdx.x & 31) == 0) warps[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    Part out{};
    for (int w = 0; w < kEvalWarps; ++w) out += warps[w];
    parts[static_cast<long long>(b) * gridDim.x + blockIdx.x] = out;
  }
}

// a warp per (image, cell) i < n: parts [n / cells][nblk][cells] -> store(i, sum over the image's CTAs)
template <typename Part, typename Store>
__global__ void __launch_bounds__(kEvalThreads) image_reduce_kernel(const Part* __restrict__ parts, int n, int nblk, int cells,
                                                                    Store store) {
  const int i = blockIdx.x * kEvalWarps + (threadIdx.x >> 5);
  if (i >= n) return;
  const int b = i / cells, cell = i - b * cells;
  Part sum{};
  for (int k = threadIdx.x & 31; k < nblk; k += 32) sum += parts[(static_cast<long long>(b) * nblk + k) * cells + cell];
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) store(i, sum);
}

template <typename Part, typename Store>
int launch_image_reduce(const Part* parts, int n, int nblk, int cells, Store store, cudaStream_t s) {
  image_reduce_kernel<<<(n + kEvalWarps - 1) / kEvalWarps, kEvalThreads, 0, s>>>(parts, n, nblk, cells, store);
  return after_launch();
}

}  // namespace rnc
