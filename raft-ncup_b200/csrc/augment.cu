// Training-sample augmentation (core/utils/augmentor.py FlowAugmentor / SparseFlowAugmentor, then the tensor conversion of
// FlowDataset.__getitem__, core/datasets.py:81-90), for a whole batch of samples of different source sizes.
//
// The host draws every random parameter in the reference's order (rnc/augment.py) and uploads them, one rnc_aug_desc per
// sample, with the raw samples.  Four kernels then produce the float NCHW crops:
//   1. contrast statistics: per sample, the integer sum of Pillow's L over the image after the jitter ops that precede
//      contrast (over the stacked pair when the jitter is symmetric);
//   2. eraser statistics: per sample with an eraser, the integer channel sums of the fully jittered img2;
//   3. sparse scatter (SparseFlowAugmentor with a resize): every valid source point writes source index + 1 into an int map
//      of the crop with atomicMax, so the highest source index wins, as numpy's repeated-index assignment does;
//   4. gather: thread = crop pixel.  It undoes crop and flips, finds cv2's INTER_LINEAR taps, jitters and erases exactly
//      the source pixels it reads, and writes images, flow and valid.
// The integer sums are exact, so every output repeats bit for bit.
//
// The arithmetic follows Pillow 12 (Blend.c, Convert.c) and cv2 4.13 (resizeGeneric_) rounding by rounding: float and
// double operations that those libraries do one by one go through the *_rn helpers below, so nvcc never contracts them into
// an FMA.  The helpers are __host__ __device__ so the same per-pixel code can be evaluated on a CPU.
#include "rnc_common.cuh"

namespace rnc {
namespace {

constexpr int kAugThreads = 256;
constexpr int kStatWords = 8;   // per sample: L sums of img1, img2; eraser sums r, g, b; 3 spare

__host__ __device__ __forceinline__ float mul_f(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ float add_f(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ float sub_f(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ float div_f(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
__host__ __device__ __forceinline__ double mul_d(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ double add_d(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ double sub_d(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ double div_d(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

// ---------------------------------------------------------------------------------------------------------------------
// Pillow's 8-bit colour operations

// Image.blend(im1, im2, alpha) on 8-bit bands: (float)(in1 + alpha * (in2 - in1)), clipped, truncated.
__host__ __device__ __forceinline__ int blend8(int in1, int in2, float alpha) {
  const float t = add_f(static_cast<float>(in1), mul_f(alpha, static_cast<float>(in2 - in1)));
  return t <= 0.f ? 0 : (t >= 255.f ? 255 : static_cast<int>(t));
}

// convert("L"): ITU-R 601-2 luma in 16-bit fixed point.
__host__ __device__ __forceinline__ int luma8(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

// convert("HSV"), shift H by `dh` with uint8 wrap-around, convert("RGB")  (torchvision adjust_hue on a PIL image).
__host__ __device__ inline void hue_shift(int& r, int& g, int& b, int dh) {
  const int mx = r > g ? (r > b ? r : b) : (g > b ? g : b);
  const int mn = r < g ? (r < b ? r : b) : (g < b ? g : b);
  if (mx == mn) return;                       // H = S = 0: the shift is lost, grey stays grey
  const float cr = static_cast<float>(mx - mn);
  const float s = div_f(cr, static_cast<float>(mx));
  const float rc = div_f(static_cast<float>(mx - r), cr);
  const float gc = div_f(static_cast<float>(mx - g), cr);
  const float bc = div_f(static_cast<float>(mx - b), cr);
  float h;
  if (r == mx) h = sub_f(bc, gc);
  else if (g == mx) h = static_cast<float>(sub_d(add_d(2.0, rc), bc));
  else h = static_cast<float>(sub_d(add_d(4.0, gc), rc));
  h = static_cast<float>(fmod(add_d(div_d(h, 6.0), 1.0), 1.0));
  int uh = static_cast<int>(mul_d(h, 255.0));
  int us = static_cast<int>(mul_d(s, 255.0));
  uh = uh < 0 ? 0 : (uh > 255 ? 255 : uh);
  us = us < 0 ? 0 : (us > 255 ? 255 : us);
  uh = (uh + dh) & 255;
  const int v = mx;
  if (us == 0) { r = g = b = v; return; }
  const double hf = div_d(mul_d(static_cast<float>(uh), 6.0), 255.0);
  const int i = static_cast<int>(floor(hf));
  const float f = static_cast<float>(sub_d(hf, static_cast<float>(i)));
  const float fs = static_cast<float>(div_d(static_cast<float>(us), 255.0));
  const double vf = static_cast<float>(v);
  int p = static_cast<int>(round(mul_d(vf, sub_d(1.0, fs))));
  int q = static_cast<int>(round(mul_d(vf, sub_d(1.0, mul_f(fs, f)))));
  int t = static_cast<int>(round(mul_d(vf, sub_d(1.0, mul_d(fs, sub_d(1.0, f))))));
  p = p < 0 ? 0 : (p > 255 ? 255 : p);
  q = q < 0 ? 0 : (q > 255 ? 255 : q);
  t = t < 0 ? 0 : (t > 255 ? 255 : t);
  switch (i % 6) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

// torchvision ColorJitter on a PIL image: ops in perm order, 0 brightness, 1 contrast (blend with the mean L `cmean`),
// 2 saturation, 3 hue.  `stop_at_contrast` evaluates only the ops before contrast (the contrast statistics pass).
__host__ __device__ inline void jitter(const rnc_aug_desc& d, int k, int cmean, bool stop_at_contrast, int& r, int& g, int& b) {
  const int p = d.asym ? k : 0;
  for (int i = 0; i < 4; ++i) {
    const int op = d.perm[p][i];
    if (op == 0) {
      const float a = d.factor[p][0];
      r = blend8(0, r, a); g = blend8(0, g, a); b = blend8(0, b, a);
    } else if (op == 1) {
      if (stop_at_contrast) return;
      const float a = d.factor[p][1];
      r = blend8(cmean, r, a); g = blend8(cmean, g, a); b = blend8(cmean, b, a);
    } else if (op == 2) {
      const float a = d.factor[p][2];
      const int l = luma8(r, g, b);
      r = blend8(l, r, a); g = blend8(l, g, a); b = blend8(l, b, a);
    } else {
      hue_shift(r, g, b, d.hue[p]);
    }
  }
}

// ImageEnhance.Contrast's degenerate value: int(mean(L) + 0.5), over the stacked pair when symmetric.
__host__ __device__ __forceinline__ int contrast_mean(const rnc_aug_desc& d, const unsigned long long* st, int k) {
  const double n = static_cast<double>(d.H) * d.W * (d.asym ? 1 : 2);
  const unsigned long long s = d.asym ? st[k] : st[0] + st[1];
  return static_cast<int>(add_d(div_d(static_cast<double>(s), n), 0.5));
}

// Source pixel (y, x) of image k after jitter and (img2) eraser.  cm: contrast mean; ec: eraser colour.
__host__ __device__ __forceinline__ void source_pixel(const rnc_aug_desc& d, const uint8_t* img, int k, int y, int x, int cm,
                                                      const int* ec, int& r, int& g, int& b) {
  if (k == 1) {
    for (int e = 0; e < d.n_erase; ++e) {
      const int* q = d.erase[e];
      if (x >= q[0] && x < q[0] + q[2] && y >= q[1] && y < q[1] + q[3]) { r = ec[0]; g = ec[1]; b = ec[2]; return; }
    }
  }
  const size_t hw = static_cast<size_t>(d.H) * d.W, o = static_cast<size_t>(y) * d.W + x;
  r = img[o]; g = img[hw + o]; b = img[2 * hw + o];
  jitter(d, k, cm, false, r, g, b);
}

// ---------------------------------------------------------------------------------------------------------------------
// cv2 INTER_LINEAR taps (resizeGeneric_): source coordinate (float)((dst + 0.5) * inv - 0.5), floor, fraction.
struct Tap { int s0, s1; float fr; bool clamped; };

// Columns: a coordinate left of 0 or at/after the last column is clamped with its fraction zeroed.
__host__ __device__ __forceinline__ Tap tap_x(int dx, double inv, int n) {
  const float f = static_cast<float>(sub_d(mul_d(add_d(static_cast<double>(dx), 0.5), inv), 0.5));
  int s = static_cast<int>(floorf(f));
  float fr = sub_f(f, static_cast<float>(s));
  bool right = false;
  if (s < 0) { s = 0; fr = 0.f; }
  if (s >= n - 1) { s = n - 1; fr = 0.f; right = true; }
  return {s, s + 1 < n ? s + 1 : n - 1, fr, right};
}
// Rows: the fraction is kept and the two rows are clamped, so border rows blend a row with itself.
__host__ __device__ __forceinline__ Tap tap_y(int dy, double inv, int n) {
  const float f = static_cast<float>(sub_d(mul_d(add_d(static_cast<double>(dy), 0.5), inv), 0.5));
  const int s = static_cast<int>(floorf(f));
  const float fr = sub_f(f, static_cast<float>(s));
  const int s0 = s < 0 ? 0 : (s > n - 1 ? n - 1 : s), s1 = s + 1 < 0 ? 0 : (s + 1 > n - 1 ? n - 1 : s + 1);
  return {s0, s1, fr, false};
}
// Fixed-point coefficients: saturate_cast<short>(c * 2048) of the float weights 1 - fr and fr.
__host__ __device__ __forceinline__ void icoef(float fr, int& c0, int& c1) {
  c0 = static_cast<int>(rintf(mul_f(sub_f(1.f, fr), 2048.f)));
  c1 = static_cast<int>(rintf(mul_f(fr, 2048.f)));
}
// Vertical pass of the 8-bit resize, in the SIMD form cv2 uses for every column: 16-bit mul_hi of the >>4 row sums.
__host__ __device__ __forceinline__ float vmix8(int s0, int s1, int b0, int b1) {
  const int v = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
  return static_cast<float>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

struct Ctx {
  const rnc_aug_desc* desc;
  const uint8_t* src;
  unsigned long long* stats;   // [B][kStatWords]
  int* map;                    // [B][h][w] sparse winner + 1 (0: none)
  float *img1, *img2, *flow, *valid;
  int B, h, w, sparse;
};

// Each block serves one sample: its descriptor is staged in shared memory once.
__device__ __forceinline__ const rnc_aug_desc& stage_desc(const rnc_aug_desc* all, int i) {
  __shared__ rnc_aug_desc sd;
  constexpr int words = sizeof(rnc_aug_desc) / 4;
  static_assert(sizeof(rnc_aug_desc) % 8 == 0, "descriptor size");
  const uint32_t* g = reinterpret_cast<const uint32_t*>(all + i);
  for (int j = threadIdx.x; j < words; j += blockDim.x) reinterpret_cast<uint32_t*>(&sd)[j] = g[j];
  __syncthreads();
  return sd;
}

// ---------------------------------------------------------------------------------------------------------------------
// 1. contrast statistics
__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <int N>
__device__ __forceinline__ void block_add(unsigned long long (&v)[N], unsigned long long* dst) {
  __shared__ unsigned long long part[kAugThreads / 32][N];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = warp_sum(v[i]);
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < N; ++i) part[wid][i] = v[i];
  }
  __syncthreads();
  if (threadIdx.x < N) {
    unsigned long long s = 0;
    for (int i = 0; i < kAugThreads / 32; ++i) s += part[i][threadIdx.x];
    if (s) atomicAdd(dst + threadIdx.x, s);   // integer: exact in any order
  }
}

__global__ void __launch_bounds__(kAugThreads) aug_contrast_stats_kernel(Ctx c) {
  const rnc_aug_desc& d = stage_desc(c.desc, blockIdx.y);
  const long long hw = static_cast<long long>(d.H) * d.W;
  unsigned long long s[2] = {0, 0};
  for (long long i = blockIdx.x * static_cast<long long>(kAugThreads) + threadIdx.x; i < 2 * hw;
       i += static_cast<long long>(gridDim.x) * kAugThreads) {
    const int k = i >= hw;
    const long long o = i - k * hw;
    const uint8_t* img = c.src + (k ? d.img2 : d.img1);
    int r = img[o], g = img[hw + o], b = img[2 * hw + o];
    jitter(d, k, 0, true, r, g, b);
    const unsigned long long l = static_cast<unsigned long long>(luma8(r, g, b));
    if (k) s[1] += l; else s[0] += l;
  }
  block_add<2>(s, c.stats + blockIdx.y * kStatWords);
}

// 2. eraser statistics: channel sums of the jittered img2
__global__ void __launch_bounds__(kAugThreads) aug_eraser_stats_kernel(Ctx c) {
  const rnc_aug_desc& d = stage_desc(c.desc, blockIdx.y);
  if (d.n_erase == 0) return;
  unsigned long long* st = c.stats + blockIdx.y * kStatWords;
  const int cm = contrast_mean(d, st, 1);
  const long long hw = static_cast<long long>(d.H) * d.W;
  const uint8_t* img = c.src + d.img2;
  unsigned long long s[3] = {0, 0, 0};
  for (long long o = blockIdx.x * static_cast<long long>(kAugThreads) + threadIdx.x; o < hw;
       o += static_cast<long long>(gridDim.x) * kAugThreads) {
    int r = img[o], g = img[hw + o], b = img[2 * hw + o];
    jitter(d, 1, cm, false, r, g, b);
    s[0] += r; s[1] += g; s[2] += b;
  }
  block_add<3>(s, st + 2);
}

// 3. sparse scatter (resize_sparse_flow_map, augmentor.py:160-193), straight into crop coordinates
__global__ void __launch_bounds__(kAugThreads) aug_sparse_scatter_kernel(Ctx c) {
  const rnc_aug_desc& d = stage_desc(c.desc, blockIdx.y);
  if (!d.resized) return;
  const long long hw = static_cast<long long>(d.H) * d.W;
  const float* valid = reinterpret_cast<const float*>(c.src + d.valid);
  int* map = c.map + static_cast<size_t>(blockIdx.y) * c.h * c.w;
  for (long long i = blockIdx.x * static_cast<long long>(kAugThreads) + threadIdx.x; i < hw;
       i += static_cast<long long>(gridDim.x) * kAugThreads) {
    if (!(valid[i] >= 1.f)) continue;
    const int y = static_cast<int>(i / d.W), x = static_cast<int>(i - static_cast<long long>(y) * d.W);
    const int xx = static_cast<int>(rint(mul_d(static_cast<double>(x), d.fx)));   // np.round: half to even
    const int yy = static_cast<int>(rint(mul_d(static_cast<double>(y), d.fy)));
    if (!(xx > 0 && xx < d.rw && yy > 0 && yy < d.rh)) continue;                   // the reference drops row and column 0
    const int cx = (d.hflip ? d.rw - 1 - xx : xx) - d.x0, cy = yy - d.y0;
    if (cx < 0 || cx >= c.w || cy < 0 || cy >= c.h) continue;
    atomicMax(map + static_cast<size_t>(cy) * c.w + cx, static_cast<int>(i) + 1);
  }
}

// 4. gather: one thread per crop pixel
__global__ void __launch_bounds__(kAugThreads) aug_gather_kernel(Ctx c) {
  const int bi = blockIdx.y;
  const int n = c.h * c.w;
  const int pix = blockIdx.x * kAugThreads + threadIdx.x;
  const rnc_aug_desc& d = stage_desc(c.desc, bi);
  if (pix >= n) return;
  const int oy = pix / c.w, ox = pix - oy * c.w;
  const unsigned long long* st = c.stats + bi * kStatWords;
  const int cm0 = contrast_mean(d, st, 0), cm1 = contrast_mean(d, st, 1);
  int ec[3] = {0, 0, 0};
  if (d.n_erase) {
    const unsigned long long hw = static_cast<unsigned long long>(d.H) * d.W;
#pragma unroll
    for (int k = 0; k < 3; ++k) ec[k] = static_cast<int>(st[2 + k] / hw);   // float64 mean stored to uint8: truncation
  }
  int ry = d.y0 + oy, rx = d.x0 + ox;
  if (d.vflip) ry = d.rh - 1 - ry;
  if (d.hflip) rx = d.rw - 1 - rx;
  const size_t plane = static_cast<size_t>(n), o = static_cast<size_t>(bi) * 3 * plane + pix;
  const size_t hw = static_cast<size_t>(d.H) * d.W;
  const float* fsrc = reinterpret_cast<const float*>(c.src + d.flow);
  float u, v;
  float vout = 0.f;
  bool have_valid = false;

  if (d.resized) {
    const Tap tx = tap_x(rx, d.ifx, d.W), ty = tap_y(ry, d.ify, d.H);
    int a0, a1, b0, b1;
    icoef(tx.fr, a0, a1);
    icoef(ty.fr, b0, b1);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const uint8_t* img = c.src + (k ? d.img2 : d.img1);
      const int cm = k ? cm1 : cm0;
      int p[2][2][3];
#pragma unroll
      for (int yy = 0; yy < 2; ++yy) {
        const int sy = yy ? ty.s1 : ty.s0;
        if (yy && ty.s1 == ty.s0) { for (int j = 0; j < 2; ++j) for (int ch = 0; ch < 3; ++ch) p[1][j][ch] = p[0][j][ch]; continue; }
        source_pixel(d, img, k, sy, tx.s0, cm, ec, p[yy][0][0], p[yy][0][1], p[yy][0][2]);
        if (a1) source_pixel(d, img, k, sy, tx.s1, cm, ec, p[yy][1][0], p[yy][1][1], p[yy][1][2]);
        else p[yy][1][0] = p[yy][1][1] = p[yy][1][2] = 0;
      }
      float* out = k ? c.img2 : c.img1;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const int s0 = p[0][0][ch] * a0 + p[0][1][ch] * a1, s1 = p[1][0][ch] * a0 + p[1][1][ch] * a1;
        out[o + ch * plane] = vmix8(s0, s1, b0, b1);
      }
    }
    if (!c.sparse) {
      const float fa0 = sub_f(1.f, tx.fr), fa1 = tx.fr, fb0 = sub_f(1.f, ty.fr), fb1 = ty.fr;
      float r2[2][2];
#pragma unroll
      for (int ch = 0; ch < 2; ++ch)
#pragma unroll
        for (int yy = 0; yy < 2; ++yy) {
          const float* row = fsrc + ch * hw + static_cast<size_t>(yy ? ty.s1 : ty.s0) * d.W;
          r2[ch][yy] = tx.clamped ? row[tx.s0] : add_f(mul_f(row[tx.s0], fa0), mul_f(row[tx.s1], fa1));
        }
      const float fu = add_f(mul_f(r2[0][0], fb0), mul_f(r2[0][1], fb1));
      const float fv = add_f(mul_f(r2[1][0], fb0), mul_f(r2[1][1], fb1));
      u = static_cast<float>(mul_d(fu, d.fx));   // flow * [scale_x, scale_y] in float64, then .float()
      v = static_cast<float>(mul_d(fv, d.fy));
    } else {
      const int m = c.map[static_cast<size_t>(bi) * n + pix];
      if (m > 0) {
        u = static_cast<float>(mul_d(fsrc[m - 1], d.fx));
        v = static_cast<float>(mul_d(fsrc[hw + m - 1], d.fy));
        vout = 1.f;
      } else {
        u = v = 0.f;
      }
      have_valid = true;
    }
  } else {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      int r, g, b;
      source_pixel(d, c.src + (k ? d.img2 : d.img1), k, ry, rx, k ? cm1 : cm0, ec, r, g, b);
      float* out = k ? c.img2 : c.img1;
      out[o] = static_cast<float>(r); out[o + plane] = static_cast<float>(g); out[o + 2 * plane] = static_cast<float>(b);
    }
    const size_t so = static_cast<size_t>(ry) * d.W + rx;
    u = fsrc[so];
    v = fsrc[hw + so];
    if (c.sparse) { vout = reinterpret_cast<const float*>(c.src + d.valid)[so]; have_valid = true; }
  }
  if (d.hflip) u = -u;
  if (d.vflip) v = -v;
  if (!have_valid) vout = (fabsf(u) < 1000.f && fabsf(v) < 1000.f) ? 1.f : 0.f;
  const size_t fo = static_cast<size_t>(bi) * 2 * plane + pix;
  c.flow[fo] = u;
  c.flow[fo + plane] = v;
  c.valid[static_cast<size_t>(bi) * plane + pix] = vout;
}

size_t stats_bytes(int B) { return (static_cast<size_t>(B) * kStatWords * sizeof(unsigned long long) + 255) & ~size_t(255); }

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

size_t rnc_augment_workspace_bytes(int B, int crop_h, int crop_w, int sparse) {
  if (B <= 0 || crop_h <= 0 || crop_w <= 0) return 0;
  return stats_bytes(B) + (sparse ? static_cast<size_t>(B) * crop_h * crop_w * sizeof(int) : 0);
}

int rnc_augment(const rnc_aug_desc* desc_host, const rnc_aug_desc* desc_dev, int B, const void* src, size_t src_bytes,
                int crop_h, int crop_w, int sparse, float* img1, float* img2, float* flow, float* valid, void* workspace,
                size_t workspace_bytes, void* stream) {
  if (B <= 0 || crop_h <= 0 || crop_w <= 0 || (sparse != 0 && sparse != 1)) return RNC_ERR_BAD_SHAPE;
  if (!desc_host || !desc_dev || !src || !img1 || !img2 || !flow || !valid || !workspace) return RNC_ERR_BAD_POINTER;
  if ((reinterpret_cast<uintptr_t>(desc_dev) & 7) || (reinterpret_cast<uintptr_t>(src) & 3) || !aligned16(workspace) ||
      (reinterpret_cast<uintptr_t>(img1) & 3) || (reinterpret_cast<uintptr_t>(img2) & 3) ||
      (reinterpret_cast<uintptr_t>(flow) & 3) || (reinterpret_cast<uintptr_t>(valid) & 3))
    return RNC_ERR_BAD_POINTER;
  if (static_cast<long long>(crop_h) * crop_w >= (1ll << 30)) return RNC_ERR_BAD_SHAPE;
  long long max_px = 0;
  for (int i = 0; i < B; ++i) {
    const rnc_aug_desc& d = desc_host[i];
    if (d.H <= 0 || d.W <= 0 || static_cast<long long>(d.H) * d.W >= (1ll << 30)) return RNC_ERR_BAD_SHAPE;
    if (d.rh < crop_h || d.rw < crop_w || d.y0 < 0 || d.x0 < 0 || d.y0 > d.rh - crop_h || d.x0 > d.rw - crop_w)
      return RNC_ERR_BAD_SHAPE;
    if (!d.resized && (d.rh != d.H || d.rw != d.W)) return RNC_ERR_BAD_SHAPE;
    if (d.resized && !(d.fx > 0.0 && d.fy > 0.0 && d.ifx > 0.0 && d.ify > 0.0)) return RNC_ERR_BAD_SHAPE;
    if (sparse && (d.vflip || d.asym)) return RNC_ERR_BAD_SHAPE;
    if ((d.resized | d.hflip | d.vflip | d.asym) & ~1) return RNC_ERR_BAD_SHAPE;
    for (int p = 0; p < 2; ++p) {
      int seen = 0;
      for (int j = 0; j < 4; ++j) {
        if (d.perm[p][j] < 0 || d.perm[p][j] > 3) return RNC_ERR_BAD_SHAPE;
        seen |= 1 << d.perm[p][j];
      }
      if (seen != 15 || d.hue[p] < 0 || d.hue[p] > 255) return RNC_ERR_BAD_SHAPE;
    }
    if (d.n_erase < 0 || d.n_erase > 2) return RNC_ERR_BAD_SHAPE;
    for (int e = 0; e < d.n_erase; ++e)
      if (d.erase[e][0] < 0 || d.erase[e][1] < 0 || d.erase[e][2] < 0 || d.erase[e][3] < 0) return RNC_ERR_BAD_SHAPE;
    const long long hw = static_cast<long long>(d.H) * d.W;
    const long long sb = static_cast<long long>(src_bytes);
    if (d.img1 < 0 || d.img2 < 0 || d.flow < 0 || d.img1 + 3 * hw > sb || d.img2 + 3 * hw > sb || d.flow + 8 * hw > sb)
      return RNC_ERR_BAD_SHAPE;
    if (d.flow & 3) return RNC_ERR_BAD_POINTER;
    if (sparse) {
      if (d.valid < 0 || d.valid + 4 * hw > sb) return RNC_ERR_BAD_SHAPE;
      if (d.valid & 3) return RNC_ERR_BAD_POINTER;
    }
    if (2 * hw > max_px) max_px = 2 * hw;
  }
  if (workspace_bytes < rnc_augment_workspace_bytes(B, crop_h, crop_w, sparse)) return RNC_ERR_WORKSPACE;
  if (B > 65535) return RNC_ERR_BAD_SHAPE;

  cudaStream_t s = as_stream(stream);
  Ctx c;
  c.desc = desc_dev;
  c.src = static_cast<const uint8_t*>(src);
  c.stats = static_cast<unsigned long long*>(workspace);
  c.map = reinterpret_cast<int*>(static_cast<char*>(workspace) + stats_bytes(B));
  c.img1 = img1; c.img2 = img2; c.flow = flow; c.valid = valid;
  c.B = B; c.h = crop_h; c.w = crop_w; c.sparse = sparse;
  cudaError_t e = cudaMemsetAsync(workspace, 0, rnc_augment_workspace_bytes(B, crop_h, crop_w, sparse), s);
  if (e != cudaSuccess) { g_last_cuda_error = static_cast<int>(e); return RNC_ERR_CUDA; }
  // statistics: ~8 pixels per thread
  const int sblocks = static_cast<int>((max_px + 8ll * kAugThreads - 1) / (8ll * kAugThreads));
  aug_contrast_stats_kernel<<<dim3(sblocks, B), kAugThreads, 0, s>>>(c);
  int st = after_launch();
  if (st) return st;
  aug_eraser_stats_kernel<<<dim3((sblocks + 1) / 2, B), kAugThreads, 0, s>>>(c);
  if ((st = after_launch())) return st;
  if (sparse) {
    aug_sparse_scatter_kernel<<<dim3((sblocks + 1) / 2, B), kAugThreads, 0, s>>>(c);
    if ((st = after_launch())) return st;
  }
  aug_gather_kernel<<<dim3((crop_h * crop_w + kAugThreads - 1) / kAugThreads, B), kAugThreads, 0, s>>>(c);
  return after_launch();
}

}  // extern "C"
