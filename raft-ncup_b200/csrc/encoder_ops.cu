// Non-GEMM pieces of the feature/context encoders (core/extractor.py:118-192, BasicEncoder):
//   stem      : image normalisation 2*(x/255)-1 (raft_nc_dbl.py:118-119) fused with conv1 = Conv2d(3,64,7,stride 2,pad 3)
//               (extractor.py:135,171); K = 147 is too thin for tensor cores -> exact fp32 FFMA
//   instnorm  : nn.InstanceNorm2d (no affine, biased variance, eps 1e-5; extractor.py:128-129, 28-33) as a statistics
//               pass (fp64 accumulation) and an apply pass fused with ReLU / residual add / hi-lo re-splitting
//               (ResidualBlock.forward, extractor.py:48-56)
//   pyramid   : 2x2 average pooling of the CL fmap2 (core/corr.py:18-21 applied to features instead of the volume)
// The wide 3x3 / 1x1 convolutions of the encoders run on rnc_conv2d_umma_fwd.
#include <cuda_fp16.h>
#include "rnc_common.cuh"

namespace rnc {

// ---------------------------------------------------------------- stem: 7x7 stride-2 conv on the raw image
constexpr int ST_TX = 32, ST_TY = 8;                 // output tile: 256 px = 64 pixel quads x 4 channel groups = 256 threads
constexpr int ST_IN_W = ST_TX * 2 + 5, ST_IN_H = ST_TY * 2 + 5;
constexpr int ST_PW = ST_IN_W + 1;                   // patch row pitch
constexpr int ST_SMEM = (3 * ST_IN_H * ST_PW + 147 * 64) * 4;   // 17.6 KB patch + 37.6 KB weights (dynamic: > 48 KB)

// weight layout [147 = (c*7+ky)*7+kx][64].  Thread = (4 horizontally adjacent output pixels, 16-channel group): per
// (channel, filter row) the 13 input values of the quad are loaded once and every weight float4 feeds 16 multiply-adds, issued
// as 8 FMA pairs (ffma2: two adjacent output channels) — the kernel is FMA-issue-bound.  In shared
// memory a tap's 64 weights are stored as [quad q][channel group cg][4], so that the four channel groups of a quarter warp
// read four consecutive 16-byte chunks (the plain [64] order put groups 0/2 and 1/3 into the same banks).
__global__ void __launch_bounds__(256)
stem_conv7x7s2_kernel(const float* __restrict__ img, const float* __restrict__ weight, const float* __restrict__ bias,
                      int N, int Hin, int Win, int Ho, int Wo, int relu, float* __restrict__ out_f32,
                      __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  extern __shared__ __align__(16) float st_smem[];
  float* wsm = st_smem;                                // [147][64]
  float* patch = st_smem + 147 * 64;                   // [3][ST_IN_H][ST_PW]
  const int n = blockIdx.z, oy0 = blockIdx.y * ST_TY, ox0 = blockIdx.x * ST_TX;
  const int tid = threadIdx.x;
  for (int i = tid; i < 147 * 64 / 4; i += 256) {                // float4 index i = tap*16 + cg*4 + q  ->  tap*16 + q*4 + cg
    const int tap = i >> 4, cgq = i & 15;
    reinterpret_cast<float4*>(wsm)[tap * 16 + (cgq & 3) * 4 + (cgq >> 2)] = reinterpret_cast<const float4*>(weight)[i];
  }
  const int iy0 = oy0 * 2 - 3, ix0 = ox0 * 2 - 3;
  for (int i = tid; i < 3 * ST_IN_H * ST_IN_W; i += 256) {
    const int c = i / (ST_IN_H * ST_IN_W), r = i % (ST_IN_H * ST_IN_W);
    const int py = r / ST_IN_W, px = r % ST_IN_W;
    const int y = iy0 + py, x = ix0 + px;
    float v = 0.f;                                     // zero padding applies to the NORMALISED image
    if (y >= 0 && y < Hin && x >= 0 && x < Win) v = 2.f * (img[((size_t)(n * 3 + c) * Hin + y) * Win + x] / 255.0f) - 1.0f;
    patch[(c * ST_IN_H + py) * ST_PW + px] = v;
  }
  __syncthreads();
  const int cg = tid & 3, quad = tid >> 2;
  const int ty = quad / (ST_TX / 4), tx = (quad % (ST_TX / 4)) * 4;
  float2 acc2[4][8];                                   // [pixel][channel pair]
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float2 bv = make_float2(bias[cg * 16 + 2 * j], bias[cg * 16 + 2 * j + 1]);
    acc2[0][j] = bv; acc2[1][j] = bv; acc2[2][j] = bv; acc2[3][j] = bv;
  }
  for (int c = 0; c < 3; ++c)
    for (int ky = 0; ky < 7; ++ky) {
      const float* prow = &patch[(c * ST_IN_H + ty * 2 + ky) * ST_PW + tx * 2];
      float2 a[13];
#pragma unroll
      for (int i = 0; i < 13; ++i) { const float v = prow[i]; a[i] = make_float2(v, v); }
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const float4* w4 = reinterpret_cast<const float4*>(&wsm[((c * 7 + ky) * 7 + kx) * 64]) + cg;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 w = w4[q * 4];
          const float2 w01 = make_float2(w.x, w.y), w23 = make_float2(w.z, w.w);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            acc2[i][2 * q] = ffma2(a[2 * i + kx], w01, acc2[i][2 * q]);
            acc2[i][2 * q + 1] = ffma2(a[2 * i + kx], w23, acc2[i][2 * q + 1]);
          }
        }
      }
    }
  float acc[4][16];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc[i][2 * j] = acc2[i][j].x; acc[i][2 * j + 1] = acc2[i][j].y; }
  const int oy = oy0 + ty;
  if (oy >= Ho) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int ox = ox0 + tx + i;
    if (ox >= Wo) continue;
    const size_t base = (((size_t)n * Ho + oy) * Wo + ox) * 64 + cg * 16;
    float v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = relu ? fmaxf(acc[i][j], 0.f) : acc[i][j];
    if (out_f32) {
#pragma unroll
      for (int q = 0; q < 4; ++q) reinterpret_cast<float4*>(out_f32 + base)[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    }
    if (out_hi) {
      __half2 hh[8], ll[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float v0 = fminf(fmaxf(v[2 * j], -65504.f), 65504.f), v1 = fminf(fmaxf(v[2 * j + 1], -65504.f), 65504.f);
        const __half h0 = __float2half_rn(v0), h1 = __float2half_rn(v1);
        hh[j] = __halves2half2(h0, h1);
        ll[j] = __halves2half2(__float2half_rn(v0 - __half2float(h0)), __float2half_rn(v1 - __half2float(h1)));
      }
      reinterpret_cast<uint4*>(out_hi + base)[0] = reinterpret_cast<uint4*>(hh)[0];
      reinterpret_cast<uint4*>(out_hi + base)[1] = reinterpret_cast<uint4*>(hh)[1];
      reinterpret_cast<uint4*>(out_lo + base)[0] = reinterpret_cast<uint4*>(ll)[0];
      reinterpret_cast<uint4*>(out_lo + base)[1] = reinterpret_cast<uint4*>(ll)[1];
    }
  }
}

// ---------------------------------------------------------------- instance norm statistics: sum / sum of squares in fp64
// x CL fp32 [N][P][C] (C <= 128, C % 4 == 0); stats [N][C][2] doubles, zeroed by the caller
__global__ void __launch_bounds__(256)
instnorm_stats_kernel(const float* __restrict__ x, int P, int C, int rows_per_cta, double* __restrict__ stats) {
  __shared__ double ssum[8][128], ssq[8][128];
  const int n = blockIdx.y;
  const int c4 = C >> 2;                         // float4 columns
  const int col = threadIdx.x % c4, rsub = threadIdx.x / c4, nsub = 256 / c4;
  const int r0 = blockIdx.x * rows_per_cta, r1 = min(P, r0 + rows_per_cta);
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = s;
  double ds[4] = {0, 0, 0, 0}, dq[4] = {0, 0, 0, 0};
  int cnt = 0;
  if (rsub < nsub) {
    for (int r = r0 + rsub; r < r1; r += nsub) {
      const float4 v = *reinterpret_cast<const float4*>(x + ((size_t)n * P + r) * C + col * 4);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      q.x = fmaf(v.x, v.x, q.x); q.y = fmaf(v.y, v.y, q.y); q.z = fmaf(v.z, v.z, q.z); q.w = fmaf(v.w, v.w, q.w);
      if (++cnt == 32) {                           // flush short fp32 runs into fp64
        ds[0] += s.x; ds[1] += s.y; ds[2] += s.z; ds[3] += s.w; dq[0] += q.x; dq[1] += q.y; dq[2] += q.z; dq[3] += q.w;
        s = make_float4(0.f, 0.f, 0.f, 0.f); q = s; cnt = 0;
      }
    }
    ds[0] += s.x; ds[1] += s.y; ds[2] += s.z; ds[3] += s.w; dq[0] += q.x; dq[1] += q.y; dq[2] += q.z; dq[3] += q.w;
  }
  // reduce the nsub row-groups through shared memory (nsub <= 16 for C >= 64; use 8-row chunks)
  for (int base = 0; base < nsub; base += 8) {
    if (rsub >= base && rsub < base + 8 && rsub < nsub) {
#pragma unroll
      for (int j = 0; j < 4; ++j) { ssum[rsub - base][col * 4 + j] = ds[j]; ssq[rsub - base][col * 4 + j] = dq[j]; }
    }
    __syncthreads();
    const int lim = min(8, nsub - base);
    if (threadIdx.x < C) {
      double a = 0, b = 0;
      for (int k = 0; k < lim; ++k) { a += ssum[k][threadIdx.x]; b += ssq[k][threadIdx.x]; }
      atomicAdd(&stats[((size_t)n * C + threadIdx.x) * 2 + 0], a);
      atomicAdd(&stats[((size_t)n * C + threadIdx.x) * 2 + 1], b);
    }
    __syncthreads();
  }
}

__global__ void instnorm_finalize_kernel(double* __restrict__ stats, int NC, int P, float eps, float* __restrict__ mean_rstd, int rezero) {
  pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NC) return;
  const double mean = stats[2 * i] / P;
  const double var = fmax(stats[2 * i + 1] / P - mean * mean, 0.0);     // biased variance (F.instance_norm)
  mean_rstd[2 * i] = (float)mean;
  mean_rstd[2 * i + 1] = (float)(1.0 / sqrt(var + (double)eps));
  if (rezero) { stats[2 * i] = 0.0; stats[2 * i + 1] = 0.0; }           // ready for the next accumulating producer
}

// ---------------------------------------------------------------- instance norm apply (+ ReLU / residual / split)
// mode 0: y = norm(x)                         -> out_f32                (downsample branch, extractor.py:44-45)
// mode 1: y = relu(norm(x))                   -> out_hi/lo (+ out_f32)  (extractor.py:50-51)
// mode 2: y = relu(res + relu(norm(x)))       -> out_f32 + out_hi/lo    (extractor.py:51,56)
__global__ void instnorm_apply_kernel(const float* __restrict__ x, const float* __restrict__ mean_rstd, const float* __restrict__ res,
                                      int N, int P, int C, int mode, float* __restrict__ out_f32,
                                      __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  pdl_trigger();
  const int c4 = C >> 2;
  const size_t total = (size_t)N * P * c4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int col = (int)(i % c4);
    const size_t row = i / c4;
    const int n = (int)(row / P);
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    float in[4] = {v.x, v.y, v.z, v.w}, o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 mr = __ldg(reinterpret_cast<const float2*>(mean_rstd) + (size_t)n * C + col * 4 + j);
      o[j] = (in[j] - mr.x) * mr.y;
      if (mode >= 1) o[j] = fmaxf(o[j], 0.f);
    }
    if (mode == 2) {
      const float4 r = reinterpret_cast<const float4*>(res)[i];
      o[0] = fmaxf(o[0] + r.x, 0.f); o[1] = fmaxf(o[1] + r.y, 0.f); o[2] = fmaxf(o[2] + r.z, 0.f); o[3] = fmaxf(o[3] + r.w, 0.f);
    }
    if (out_f32) reinterpret_cast<float4*>(out_f32)[i] = make_float4(o[0], o[1], o[2], o[3]);
    if (out_hi) {
      __half h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float vc = fminf(fmaxf(o[j], -65504.f), 65504.f);
        h[j] = __float2half_rn(vc);
        l[j] = __float2half_rn(vc - __half2float(h[j]));
      }
      reinterpret_cast<uint2*>(out_hi)[i] = *reinterpret_cast<uint2*>(h);
      reinterpret_cast<uint2*>(out_lo)[i] = *reinterpret_cast<uint2*>(l);
    }
  }
}

// y = relu(a + b) on CL fp32 (block tail when the norm is folded into the convolutions), -> fp32 + split
__global__ void add_relu_split_kernel(const float4* __restrict__ a, const float4* __restrict__ b, size_t n4, float4* __restrict__ out_f32,
                                      uint2* __restrict__ out_hi, uint2* __restrict__ out_lo) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    const float4 x = a[i], y = b[i];
    float o[4] = {fmaxf(x.x + y.x, 0.f), fmaxf(x.y + y.y, 0.f), fmaxf(x.z + y.z, 0.f), fmaxf(x.w + y.w, 0.f)};
    if (out_f32) out_f32[i] = make_float4(o[0], o[1], o[2], o[3]);
    __half h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float vc = fminf(o[j], 65504.f);
      h[j] = __float2half_rn(vc);
      l[j] = __float2half_rn(vc - __half2float(h[j]));
    }
    out_hi[i] = *reinterpret_cast<uint2*>(h);
    out_lo[i] = *reinterpret_cast<uint2*>(l);
  }
}

__global__ void pool2_cl_kernel2(const float4* __restrict__ src, float4* __restrict__ dst, int B, int Hs, int Ws, int D4) {
  const int Hd = Hs >> 1, Wd = Ws >> 1;
  const size_t n = (size_t)B * Hd * Wd * D4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int d = (int)(i % D4);
    size_t r = i / D4;
    const int x = (int)(r % Wd); r /= Wd;
    const int y = (int)(r % Hd);
    const int b = (int)(r / Hd);
    const float4* s = src + (((size_t)b * Hs + 2 * y) * Ws + 2 * x) * D4 + d;
    const float4 a = s[0], c = s[D4], e = s[(size_t)Ws * D4], f = s[(size_t)Ws * D4 + D4];
    dst[i] = make_float4(0.25f * ((a.x + c.x) + (e.x + f.x)), 0.25f * ((a.y + c.y) + (e.y + f.y)),
                         0.25f * ((a.z + c.z) + (e.z + f.z)), 0.25f * ((a.w + c.w) + (e.w + f.w)));
  }
}


// Image normalisation 2*(x/255)-1 (raft_nc_dbl.py:118-119) + repack for the tensor-core stem (rnc_conv_umma_desc.win_pitch):
// NCHW fp32 -> zero-padded pixel plane [N][Hin][pitch_px][4] of split halves; pixel p holds image column p - 3 (channels
// 0..2, channel 3 = 0), zero outside the image, so that output column ox's 7 taps start at pixel 2*ox: a 16-byte step.
__global__ void __launch_bounds__(256)
stem_window_prep_kernel(const float* __restrict__ img, int N, int Hin, int Win, int pitch_px, uint2* __restrict__ hi,
                        uint2* __restrict__ lo) {
  const size_t total = static_cast<size_t>(N) * Hin * pitch_px;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int p = static_cast<int>(i % pitch_px);
    const size_t row = i / pitch_px;                       // n * Hin + y
    const int x = p - 3;
    float v[3] = {0.f, 0.f, 0.f};
    if (x >= 0 && x < Win) {
      const size_t n = row / Hin, y = row - n * Hin;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        v[c] = __fsub_rn(__fmul_rn(2.f, __fdiv_rn(img[((n * 3 + c) * Hin + y) * Win + x], 255.f)), 1.f);
    }
    uint2 h, l;
    split_pair(v[0], v[1], h.x, l.x);
    split_pair(v[2], 0.f, h.y, l.y);
    hi[i] = h;
    lo[i] = l;
  }
}

}  // namespace rnc

using namespace rnc;

extern "C" {

int rnc_stem_conv7x7s2_fwd(const float* img, const float* weight, const float* bias, int N, int Hin, int Win, int relu,
                           float* out_f32, void* out_hi, void* out_lo, void* stream) {
  if (N <= 0 || Hin <= 0 || Win <= 0) return RNC_ERR_BAD_SHAPE;
  if (!img || !weight || !bias || (!out_f32 && !out_hi) || (out_hi && !out_lo)) return RNC_ERR_BAD_POINTER;
  if ((out_f32 && !aligned16(out_f32)) || (out_hi && (!aligned16(out_hi) || !aligned16(out_lo))) || !aligned16(weight)) return RNC_ERR_BAD_POINTER;
  const int Ho = (Hin + 1) / 2, Wo = (Win + 1) / 2;            // floor((H + 6 - 7)/2) + 1
  dim3 grid((Wo + ST_TX - 1) / ST_TX, (Ho + ST_TY - 1) / ST_TY, N);
  static unsigned long long done = 0;
  if (int st = ensure_dyn_smem(stem_conv7x7s2_kernel, ST_SMEM, &done)) return st;
  stem_conv7x7s2_kernel<<<grid, 256, ST_SMEM, as_stream(stream)>>>(img, weight, bias, N, Hin, Win, Ho, Wo, relu, out_f32,
                                                            static_cast<__half*>(out_hi), static_cast<__half*>(out_lo));
  return after_launch();
}

int rnc_stem_window_prep(const float* img, int N, int Hin, int Win, int pitch_px, void* out_hi, void* out_lo, void* stream) {
  if (N <= 0 || Hin <= 0 || Win <= 0 || pitch_px < Win + 6 || (pitch_px & 1)) return RNC_ERR_BAD_SHAPE;
  if (!img || !out_hi || !out_lo || !aligned16(out_hi) || !aligned16(out_lo)) return RNC_ERR_BAD_POINTER;
  const size_t total = static_cast<size_t>(N) * Hin * pitch_px;
  const int blocks = static_cast<int>(total / 256 < 132 * 16 ? total / 256 + 1 : 132 * 16);
  stem_window_prep_kernel<<<blocks, 256, 0, as_stream(stream)>>>(img, N, Hin, Win, pitch_px, static_cast<uint2*>(out_hi),
                                                                  static_cast<uint2*>(out_lo));
  return after_launch();
}

int rnc_instnorm_stats(const float* x, int N, int P, int C, float eps, double* stats, float* mean_rstd, void* stream) {
  if (N <= 0 || P <= 0 || C <= 0 || C > 128 || (C & 3)) return RNC_ERR_BAD_SHAPE;
  if (!x || !stats || !mean_rstd || !aligned16(x)) return RNC_ERR_BAD_POINTER;
  cudaError_t e = cudaMemsetAsync(stats, 0, (size_t)N * C * 2 * sizeof(double), as_stream(stream));
  if (e != cudaSuccess) { g_last_cuda_error = (int)e; return RNC_ERR_CUDA; }
  const int rows = 512;
  dim3 grid((P + rows - 1) / rows, N);
  instnorm_stats_kernel<<<grid, 256, 0, as_stream(stream)>>>(x, P, C, rows, stats);
  if (int st = after_launch()) return st;
  instnorm_finalize_kernel<<<(N * C + 127) / 128, 128, 0, as_stream(stream)>>>(stats, N * C, P, eps, mean_rstd, 1);
  return after_launch();
}

int rnc_instnorm_finalize(double* stats, int N, int P, int C, float eps, float* mean_rstd, void* stream) {
  if (N <= 0 || P <= 0 || C <= 0) return RNC_ERR_BAD_SHAPE;
  if (!stats || !mean_rstd) return RNC_ERR_BAD_POINTER;
  instnorm_finalize_kernel<<<(N * C + 127) / 128, 128, 0, as_stream(stream)>>>(stats, N * C, P, eps, mean_rstd, 1);
  return after_launch();
}

int rnc_instnorm_apply(const float* x, const float* mean_rstd, const float* res, int N, int P, int C, int mode,
                       float* out_f32, void* out_hi, void* out_lo, void* stream) {
  if (N <= 0 || P <= 0 || C <= 0 || (C & 3) || mode < 0 || mode > 2) return RNC_ERR_BAD_SHAPE;
  if (!x || !mean_rstd || (mode == 2 && !res) || (!out_f32 && !out_hi) || (out_hi && !out_lo)) return RNC_ERR_BAD_POINTER;
  if (!aligned16(x) || (res && !aligned16(res)) || (out_f32 && !aligned16(out_f32))) return RNC_ERR_BAD_POINTER;
  const size_t total = (size_t)N * P * (C / 4);
  size_t blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  instnorm_apply_kernel<<<(int)blocks, 256, 0, as_stream(stream)>>>(x, mean_rstd, res, N, P, C, mode, out_f32,
                                                                   static_cast<__half*>(out_hi), static_cast<__half*>(out_lo));
  return after_launch();
}

int rnc_add_relu_split(const float* a, const float* b, size_t n, float* out_f32, void* out_hi, void* out_lo, void* stream) {
  if (n == 0 || (n & 3)) return RNC_ERR_BAD_SHAPE;
  if (!a || !b || !out_hi || !out_lo || !aligned16(a) || !aligned16(b)) return RNC_ERR_BAD_POINTER;
  size_t blocks = (n / 4 + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  add_relu_split_kernel<<<(int)blocks, 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(a), reinterpret_cast<const float4*>(b), n / 4,
                                                                    reinterpret_cast<float4*>(out_f32), static_cast<uint2*>(out_hi),
                                                                    static_cast<uint2*>(out_lo));
  return after_launch();
}

int rnc_fmap_pyramid(float* f2_pyr, int B, int D, int H, int W, int levels, void* stream) {
  if (B <= 0 || D <= 0 || (D & 3) || H <= 0 || W <= 0 || levels < 1 || levels > 4) return RNC_ERR_BAD_SHAPE;
  if (!f2_pyr || !aligned16(f2_pyr)) return RNC_ERR_BAD_POINTER;
  for (int l = 1; l < levels; ++l) {
    const float* s = f2_pyr + rnc_pyramid_offset(B, D, H, W, l - 1);
    float* d = f2_pyr + rnc_pyramid_offset(B, D, H, W, l);
    const int Hs = H >> (l - 1), Ws = W >> (l - 1);
    const size_t n = (size_t)B * (Hs >> 1) * (Ws >> 1) * (D / 4);
    if (n == 0) return RNC_ERR_BAD_SHAPE;
    int blocks = (int)((n + 255) / 256);
    if (blocks > 132 * 16) blocks = 132 * 16;
    pool2_cl_kernel2<<<blocks, 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(s), reinterpret_cast<float4*>(d), B, Hs, Ws, D / 4);
    if (int st = after_launch()) return st;
  }
  return RNC_OK;
}

}  // extern "C"
