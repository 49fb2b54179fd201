// Sparsification curves of a confidence score (the AUSE protocol) for a batch of float32 flows: per image and per fraction
// f_k = k/100, k = 0..99, the number of valid pixels kept and the fp64 sum of their EPE once the floor(k*N/100) valid pixels
// of lowest score are removed, and the same sum when the pixels of largest EPE are removed instead (the ideal curve,
// which the AUSE literature calls the oracle).
//
// Each pixel's EPE is the one rnc_flow_metrics computes: eval_common.cuh's pixel_metrics.
//
// Keys.  Pixel p of image b sits at position b*H*W + p of a device-wide radix sort whose key is (b << 32) | low, so a stable
// sort keeps every image in its own H*W slot, orders it by `low`, and breaks ties by row-major pixel index.  `low` is:
//   score order  : the monotone bits of the score (ascending float order as unsigned order), -0 folded onto +0 (they compare
//                  equal) and every NaN onto 0, below -inf;
//   ideal order  : the complement of the monotone bits of the EPE (descending EPE), every NaN onto 0, above +inf;
//   invalid pixel: 0xffffffff in both, which no valid pixel reaches (+inf's score key is 0xff800000, the largest ideal key
//                  that of +0, 0x7fffffff), so the N valid pixels of image b are the first N of its slot.
// The score sort carries the EPE as its value; the ideal sort is keys-only, since its key holds the EPE's bits.
//
// Sums.  A CTA per (fraction k, image, order) adds the sorted EPEs of [m_k, m_{k+1}) in fp64 in a fixed order (thread-strided,
// then a fixed tree), and a thread per (image, order) adds those range sums from k = 99 down to k = 0.  No atomics.  Each
// image's results depend only on its own slot, so they are bit for bit the same whatever B, its position in the batch or the
// GPU.
#include <cub/device/device_radix_sort.cuh>

#include "eval_common.cuh"

namespace rnc {
namespace {

constexpr int kSpFractions = 100;
constexpr int kSpThreads = 256;
constexpr unsigned kSpInvalid = 0xffffffffu;

struct SparsArgs {
  View flow, gt;
  View valid;                  // p == nullptr: every pixel is valid
  View score;
  int H, W;
};

__device__ __forceinline__ unsigned monotone(float v) {
  const unsigned u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(kSpThreads) spars_keys_kernel(SparsArgs a, unsigned long long* __restrict__ skey,
                                                                float* __restrict__ sval, unsigned long long* __restrict__ okey) {
  const int b = blockIdx.y;
  const int hw = a.H * a.W;
  const int p = blockIdx.x * kSpThreads + threadIdx.x;
  if (p >= hw) return;
  const int y = p / a.W, x = p - y * a.W;
  const float epe = pixel_metrics(a.flow.at(b, 0, y, x), a.flow.at(b, 1, y, x), a.gt.at(b, 0, y, x), a.gt.at(b, 1, y, x)).epe;
  const bool ok = !a.valid.p || a.valid.at(b, y, x) >= 0.5f;
  const float s = a.score.at(b, y, x);
  const unsigned sk = !ok ? kSpInvalid : (s != s) ? 0u : monotone(s == 0.0f ? 0.0f : s);
  const unsigned ek = !ok ? kSpInvalid : (epe != epe) ? 0u : ~monotone(epe);
  const unsigned long long hi = static_cast<unsigned long long>(b) << 32;
  const long long i = static_cast<long long>(b) * hw + p;
  skey[i] = hi | sk;
  sval[i] = epe;
  okey[i] = hi | ek;
}

// the number of valid pixels of image b: the first position of its slot that holds the invalid key
__device__ int valid_count(const unsigned long long* __restrict__ key, long long base, int hw) {
  int lo = 0, hi = hw;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (static_cast<unsigned>(key[base + mid]) == kSpInvalid) hi = mid; else lo = mid + 1;
  }
  return lo;
}

__device__ __forceinline__ long long removed(int k, int n) { return static_cast<long long>(k) * n / kSpFractions; }

// CTA (k, b, order): the fp64 sum of the sorted EPEs of [m_k, m_{k+1}) of image b -> part[order][b][k]; n_valid[b] from (0, b, 0)
__global__ void __launch_bounds__(kSpThreads) spars_range_kernel(const unsigned long long* __restrict__ skey,
                                                                 const float* __restrict__ sval,
                                                                 const unsigned long long* __restrict__ okey, int hw,
                                                                 double* __restrict__ part, int* __restrict__ n_valid) {
  const int k = blockIdx.x, b = blockIdx.y, order = blockIdx.z, B = gridDim.y;
  const long long base = static_cast<long long>(b) * hw;
  __shared__ int s_n;
  __shared__ double s_sum[kSpThreads / 32];
  if (threadIdx.x == 0) s_n = valid_count(skey, base, hw);
  __syncthreads();
  const int n = s_n;
  const long long lo = removed(k, n), hi = removed(k + 1, n);
  double sum = 0.0;
  for (long long i = lo + threadIdx.x; i < hi; i += kSpThreads)
    sum += order == 0 ? static_cast<double>(sval[base + i])
                      : static_cast<double>(__uint_as_float(~static_cast<unsigned>(okey[base + i]) ^ 0x80000000u));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kSpThreads / 32; ++w) t += s_sum[w];
    part[(static_cast<long long>(order) * B + b) * kSpFractions + k] = t;
    if (k == 0 && order == 0) n_valid[b] = n;
  }
}

// thread (b, order): suffix sums of the range sums, k = 99 down to 0, and with order 0 the counts N - m_k
__global__ void spars_suffix_kernel(const double* __restrict__ part, const int* __restrict__ n_valid, int B,
                                    long long* __restrict__ count, double* __restrict__ kept, double* __restrict__ ideal) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * B) return;
  const int order = t / B, b = t - order * B;
  const double* r = part + static_cast<long long>(t) * kSpFractions;
  double* out = (order == 0 ? kept : ideal) + static_cast<long long>(b) * kSpFractions;
  double acc = 0.0;
  for (int k = kSpFractions - 1; k >= 0; --k) {
    acc += r[k];
    out[k] = acc;
  }
  if (order == 0) {
    const int n = n_valid[b];
    for (int k = 0; k < kSpFractions; ++k) count[static_cast<long long>(b) * kSpFractions + k] = n - removed(k, n);
  }
}

// the sort ranks the whole batch with int offsets: B*H*W < 2^31 besides the per-image limits
bool shape_ok(int B, int H, int W) { return eval_shape_ok(B, H, W) && static_cast<long long>(B) * H * W < (1ll << 31); }

size_t up256(size_t x) { return (x + 255) & ~size_t{255}; }

// workspace: score keys x2, score values x2, ideal keys x2, range sums, valid counts, then the radix sort's scratch
struct SparsPlan {
  size_t n, keys, vals, part, nval, scratch, bytes;
  int end_bit;
};

SparsPlan plan(int B, int H, int W) {
  SparsPlan p;
  p.n = static_cast<size_t>(B) * H * W;
  p.keys = up256(p.n * sizeof(unsigned long long));
  p.vals = up256(p.n * sizeof(float));
  p.part = up256(size_t{2} * B * kSpFractions * sizeof(double));
  p.nval = up256(static_cast<size_t>(B) * sizeof(int));
  // the onesweep radix sort needs a few histograms and one look-back word per digit and tile: a fixed bound, checked at run time
  p.scratch = up256((size_t{1} << 20) + p.n * 4);
  p.bytes = 4 * p.keys + 2 * p.vals + p.part + p.nval + p.scratch;
  p.end_bit = 32;
  while (p.end_bit < 64 && (1ll << (p.end_bit - 32)) < B) ++p.end_bit;
  return p;
}

int cuda_status(cudaError_t e) {
  if (e == cudaSuccess) return RNC_OK;
  g_last_cuda_error = static_cast<int>(e);
  return RNC_ERR_CUDA;
}

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

size_t rnc_sparsification_workspace_bytes(int B, int H, int W) { return shape_ok(B, H, W) ? plan(B, H, W).bytes : 0; }

int rnc_sparsification(const float* flow, long long fb, long long fc, long long fy, long long fx, const float* gt, long long gb,
                       long long gc, long long gy, long long gx, const float* valid, long long vb, long long vy, long long vx,
                       const float* score, long long sb, long long sy, long long sx, int B, int H, int W, long long* count,
                       double* kept_epe, double* ideal_epe, void* workspace, size_t workspace_bytes, void* stream) {
  if (!shape_ok(B, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!flow || !gt || !score || !count || !kept_epe || !ideal_epe || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(flow, 4) || !aligned(gt, 4) || !aligned(valid, 4) || !aligned(score, 4) || !aligned(count, 8) ||
      !aligned(kept_epe, 8) || !aligned(ideal_epe, 8) || !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  const SparsPlan p = plan(B, H, W);
  if (workspace_bytes < p.bytes) return RNC_ERR_WORKSPACE;
  char* w = static_cast<char*>(workspace);
  auto* sk0 = reinterpret_cast<unsigned long long*>(w);
  auto* sk1 = reinterpret_cast<unsigned long long*>(w + p.keys);
  auto* ok0 = reinterpret_cast<unsigned long long*>(w + 2 * p.keys);
  auto* ok1 = reinterpret_cast<unsigned long long*>(w + 3 * p.keys);
  auto* sv0 = reinterpret_cast<float*>(w + 4 * p.keys);
  auto* sv1 = reinterpret_cast<float*>(w + 4 * p.keys + p.vals);
  auto* part = reinterpret_cast<double*>(w + 4 * p.keys + 2 * p.vals);
  auto* nval = reinterpret_cast<int*>(w + 4 * p.keys + 2 * p.vals + p.part);
  void* scratch = w + 4 * p.keys + 2 * p.vals + p.part + p.nval;
  const int n = static_cast<int>(p.n);
  cudaStream_t s = as_stream(stream);

  cub::DoubleBuffer<unsigned long long> sk(sk0, sk1), ok(ok0, ok1);
  cub::DoubleBuffer<float> sv(sv0, sv1);
  size_t need_s = 0, need_o = 0;
  if (int st = cuda_status(cub::DeviceRadixSort::SortPairs(nullptr, need_s, sk, sv, n, 0, p.end_bit, s))) return st;
  if (int st = cuda_status(cub::DeviceRadixSort::SortKeys(nullptr, need_o, ok, n, 0, p.end_bit, s))) return st;
  if (need_s > p.scratch || need_o > p.scratch) return RNC_ERR_WORKSPACE;

  const SparsArgs a{{flow, fb, fc, fy, fx}, {gt, gb, gc, gy, gx}, {valid, vb, 0, vy, vx}, {score, sb, 0, sy, sx}, H, W};
  spars_keys_kernel<<<dim3((H * W + kSpThreads - 1) / kSpThreads, B), kSpThreads, 0, s>>>(a, sk0, sv0, ok0);
  if (int st = after_launch()) return st;
  if (int st = cuda_status(cub::DeviceRadixSort::SortPairs(scratch, need_s, sk, sv, n, 0, p.end_bit, s))) return st;
  if (int st = cuda_status(cub::DeviceRadixSort::SortKeys(scratch, need_o, ok, n, 0, p.end_bit, s))) return st;
  spars_range_kernel<<<dim3(kSpFractions, B, 2), kSpThreads, 0, s>>>(sk.Current(), sv.Current(), ok.Current(), H * W, part, nval);
  if (int st = after_launch()) return st;
  spars_suffix_kernel<<<(2 * B + 127) / 128, 128, 0, s>>>(part, nval, B, count, kept_epe, ideal_epe);
  return after_launch();
}

}  // extern "C"
