// Fused NCUP upsampler: zero-stuffing + the 4 live normalized-convolution layers + final scale, one kernel.
// Replaces NConvUpsampler.forward / get_out_tensor (core/upsampler.py:143-177,179-210), NConvUNet.forward
// (core/nconv_modules.py:106-136 — at the shipped config the pooled branch is dead, only
// nconv_in -> nconv_x2[0] -> decoder[0](cat(x1,x1)) -> nconv_out is live, SURVEY.md Appendix A.3) and
// NConv2d.forward (core/nconv_modules.py:164-199):
//     den = conv(c, W), num = conv(x*c, W), y = num / (den + 1e-20), c' = den / sum(W[o])
// and the `8 *` of raft_nc_dbl.py:161.
//
// A CTA produces a 30x30 full-resolution tile of one (batch, channel) plane.  Stage 0 stages the <= 12x12 lattice samples that
// can influence the tile; stage 1 (5x5 over the stride-4 lattice: <= 4 non-zero taps) fills a 36x36 region in shared memory;
// stage 2 (dense 5x5, 2->2 ch) a 32x32 region; stage 3 (3x3 with the folded decoder weights) and stage 4 (1x1) run per output
// pixel.  Positions outside the image hold zeros, which is exactly F.conv2d's zero padding of both the data*conf and the conf
// stream.
//
// The kernel is bound by the FP32 FMA pipe (~300 multiply-adds per output pixel), not by HBM, so it is organised around the
// instruction count: the (data*conf, conf) pair of a position is one float2 and both streams share every weight, so
// num/den accumulate as one FMA pair (ffma2) per tap; threads own 1x4 (stage 2) / 1x2 (stage 3) register tiles and fetch
// their input rows with 128-bit shared-memory loads (8 lanes = 256 contiguous bytes: conflict-free).
// Tile sides are chosen so that stage 2 is exactly one 1x4 item per thread (32 rows x 8 groups = 256).
//
// The stages are device functions templated on the region they fill, shared by three kernels:
//   ncup_fused_kernel       inference: weights in the kernel parameter bank (rnc_ncup_fwd, host weights)
//   ncup_train_fwd_kernel   the same forward with the weights read from device memory (rnc_ncup_train_fwd): no host copy
//                           of the trainable weights per call; bit-identical outputs
//   ncup_bwd_kernel         the backward (rnc_ncup_bwd): recomputes the forward of a 32x32 tile with its halos through the
//                           same stages (bit-identical to the forward), then differentiates the chain in the pair form the
//                           kernel computes.  Each CTA owns the lattice samples of its tile (written once, no atomics) and
//                           writes its weight-gradient partial sums to the workspace; two small kernels reduce them in a
//                           fixed order in fp64, so gradients are bit-identical across calls.
// Each has a twin instantiated from the same code with a compile-time flag that also handles nconv_out's output confidence
// den4 / sum(W4): ncup_fused_conf_kernel and ncup_train_fwd_conf_kernel write it, ncup_conf_bwd_kernel adds its adjoint.  The
// entry points launch a twin only when the caller passes conf_out / g_conf_out; the flag off compiles to the plain kernels.
#include "rnc_common.cuh"

namespace rnc {

constexpr int NT = 30;             // output tile side
constexpr int R1 = NT + 6;         // stage-1 region side (halo 3) = 36
constexpr int R2 = NT + 2;         // stage-2 region side (halo 1) = 32
constexpr int P1 = R1 + 2;         // stage-1 row pitch (float2): a 1x4 item reads columns [4g, 4g + 8) <= 36; 304-byte rows
constexpr int P2 = R2 + 2;         // stage-2 row pitch (float2): 272-byte rows — a 256-byte pitch would put the four rows a warp
                                   // stores at once into the same banks (ncu: LSU data pipe 76 % busy, ahead of the FMA pipe)
constexpr int LT = 12;             // lattice samples per side
constexpr float kEps = 1e-20f;     // nconv_modules.py:149
constexpr int kThreads = 256;

struct NcupWeights {               // lives in the kernel parameter (constant) bank; every weight duplicated for the FMA pairs
  float2 w1[2][25];                // nconv_in   [2,1,5,5]
  float2 w2[2][2][25];             // nconv_x2.0 [2,2,5,5]
  float2 w3[2][2][9];              // decoder.0  [2,4,3,3] folded: W[:, :2] + W[:, 2:]  (input is cat(x1, x1))
  float w4[2];                     // nconv_out  [1,2,1,1]
  float inv_s1[2], inv_s2[2], inv_s3[2];   // 1 / sum over (in,kh,kw) of the UNFOLDED weights (nconv_modules.py:186-190)
};

// (num, den) -> (data * conf, conf) of the layer's output: y = num / (den + eps), c = den / sum(W); the next layer reads y * c
__device__ __forceinline__ float2 nconv_out_pair(float2 nd, float inv_s) {
  const float c = nd.y * inv_s;
  return make_float2(nd.x / (nd.y + kEps) * c, c);
}

// ---- stage 0: lattice samples iy_base.., ix_base.. of one plane.  X[4i+2][4j+2] = x_lowres[i][j], C[4i+2][4j+2] = conf[i][j]
template <int LTN>
__device__ __forceinline__ void stage0_lattice(const float* __restrict__ x_lowres, const float* __restrict__ conf, int plane,
                                               int iy_base, int ix_base, int H4, int W4, float (&lx)[LTN][LTN],
                                               float (&lc)[LTN][LTN]) {
  static_assert(LTN * LTN <= kThreads, "one lattice sample per thread");
  const int idx = threadIdx.x;
  if (idx < LTN * LTN) {
    const int li = idx / LTN, lj = idx - li * LTN;
    const int iy = iy_base + li, ix = ix_base + lj;
    float xv = 0.f, cv = 0.f;
    if (iy >= 0 && iy < H4 && ix >= 0 && ix < W4) {
      xv = x_lowres[((size_t)plane * H4 + iy) * W4 + ix];
      cv = conf[((size_t)plane * H4 + iy) * W4 + ix];
    }
    lx[li][lj] = xv;
    lc[li][lj] = cv;
  }
}

// Layer 1 accumulators (num, den) of both output channels at an in-image position (y, x): at most 2x2 lattice samples fall
// under a 5x5 window of the zero-stuffed lattice
template <int LTN>
__device__ __forceinline__ void stage1_acc(const float (&lx)[LTN][LTN], const float (&lc)[LTN][LTN], int iy_base, int ix_base,
                                           int y, int x, int H4, int W4, const NcupWeights& w, float2& a0, float2& a1) {
  a0 = make_float2(0.f, 0.f);
  a1 = a0;
  for (int iy = max((y - 1) >> 2, 0); iy <= min(y >> 2, H4 - 1); ++iy) {
    const int ky = 4 * iy + 2 - y + 2;
    for (int ix = max((x - 1) >> 2, 0); ix <= min(x >> 2, W4 - 1); ++ix) {
      const int kx = 4 * ix + 2 - x + 2;
      const float cv = lc[iy - iy_base][ix - ix_base];
      const float2 pc = make_float2(lx[iy - iy_base][ix - ix_base] * cv, cv);
      a0 = ffma2(pc, w.w1[0][ky * 5 + kx], a0);
      a1 = ffma2(pc, w.w1[1][ky * 5 + kx], a1);
    }
  }
}

// ---- stage 1: NConv(1->2, 5x5) pairs on the RN x RN region with origin (y0, x0)
template <int LTN, int RN, int PN>
__device__ __forceinline__ void stage1(const float (&lx)[LTN][LTN], const float (&lc)[LTN][LTN], int iy_base, int ix_base, int y0,
                                       int x0, int H, int W, int H4, int W4, const NcupWeights& w, float2 (&s1)[2][RN][PN]) {
  for (int idx = threadIdx.x; idx < RN * RN; idx += kThreads) {
    const int ry = idx / RN, rx = idx - ry * RN;
    const int y = y0 + ry, x = x0 + rx;
    float2 o0 = make_float2(0.f, 0.f), o1 = o0;
    if (y >= 0 && y < H && x >= 0 && x < W) {
      float2 a0, a1;
      stage1_acc(lx, lc, iy_base, ix_base, y, x, H4, W4, w, a0, a1);
      o0 = nconv_out_pair(a0, w.inv_s1[0]);
      o1 = nconv_out_pair(a1, w.inv_s1[1]);
    }
    s1[0][ry][rx] = o0;
    s1[1][ry][rx] = o1;
  }
}

// ---- stage 2: NConv(2->2, 5x5) on the RN x RN region with origin (y0, x0) from the stage-1 region with origin (y0-2, x0-2):
// item = row ry, columns 4g .. 4g+3.  nd (optional) also receives the raw (num, den) accumulators (zeros outside the image).
template <int RIN, int PIN, int RN, int PN>
__device__ __forceinline__ void stage2(const float2 (&s1)[2][RIN][PIN], int y0, int x0, int H, int W, const NcupWeights& w,
                                       float2 (&s2)[2][RN][PN], float2 (*nd)[RN][PN]) {
  static_assert(RN % 4 == 0 && RIN >= RN + 4 && PIN >= RN + 4 && PIN % 2 == 0 && PN % 2 == 0, "stage-2 geometry");
  constexpr int G = RN / 4;
  constexpr bool kOne = RN * G == kThreads;               // the forward's 32x32 region: exactly one item per thread
  for (int item = threadIdx.x; kOne || item < RN * G; item += kThreads) {
    const int ry = item / G, g = item - ry * G;
    float2 acc[4][2];
#pragma unroll
    for (int x = 0; x < 4; ++x) acc[x][0] = acc[x][1] = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int ky = 0; ky < 5; ++ky) {
        float2 row[8];
        const float4* rp = reinterpret_cast<const float4*>(&s1[i][ry + ky][4 * g]);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 v = rp[q];
          row[2 * q] = make_float2(v.x, v.y);
          row[2 * q + 1] = make_float2(v.z, v.w);
        }
#pragma unroll
        for (int kx = 0; kx < 5; ++kx) {
          const float2 wa = w.w2[0][i][ky * 5 + kx], wb = w.w2[1][i][ky * 5 + kx];
#pragma unroll
          for (int x = 0; x < 4; ++x) {
            acc[x][0] = ffma2(row[x + kx], wa, acc[x][0]);
            acc[x][1] = ffma2(row[x + kx], wb, acc[x][1]);
          }
        }
      }
    const int y = y0 + ry;
#pragma unroll
    for (int x = 0; x < 4; x += 2) {           // two positions = one 16-byte store per channel
      float2 o[2][2];
#pragma unroll
      for (int d = 0; d < 2; ++d) {
        const int xx = x0 + 4 * g + x + d;
        const bool in = y >= 0 && y < H && xx >= 0 && xx < W;
        o[d][0] = in ? nconv_out_pair(acc[x + d][0], w.inv_s2[0]) : make_float2(0.f, 0.f);
        o[d][1] = in ? nconv_out_pair(acc[x + d][1], w.inv_s2[1]) : make_float2(0.f, 0.f);
        if (nd != nullptr) {
          nd[0][ry][4 * g + x + d] = in ? acc[x + d][0] : make_float2(0.f, 0.f);
          nd[1][ry][4 * g + x + d] = in ? acc[x + d][1] : make_float2(0.f, 0.f);
        }
      }
      *reinterpret_cast<float4*>(&s2[0][ry][4 * g + x]) = make_float4(o[0][0].x, o[0][0].y, o[1][0].x, o[1][0].y);
      *reinterpret_cast<float4*>(&s2[1][ry][4 * g + x]) = make_float4(o[0][1].x, o[0][1].y, o[1][1].x, o[1][1].y);
    }
    if (kOne) break;
  }
}

// ---- stage 3: NConv(2->2, 3x3, folded decoder weights) on the RN x RN region whose origin is the stage-2 origin + (1, 1):
// item = row oy, columns 2g, 2g+1; epi(oy, g, acc) consumes the raw (num, den) accumulators acc[column][channel]
template <int RIN, int PIN, int RN, class Epi>
__device__ __forceinline__ void stage3(const float2 (&s2)[2][RIN][PIN], const NcupWeights& w, Epi epi) {
  static_assert(RN % 2 == 0 && RIN >= RN + 2 && PIN >= RN + 2, "stage-3 geometry");
  constexpr int G = RN / 2;
  for (int idx = threadIdx.x; idx < RN * G; idx += kThreads) {
    const int oy = idx / G, g = idx - oy * G;
    float2 acc[2][2];
    acc[0][0] = acc[0][1] = acc[1][0] = acc[1][1] = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const float4* rp = reinterpret_cast<const float4*>(&s2[i][oy + ky][2 * g]);
        const float4 v0 = rp[0], v1 = rp[1];
        const float2 row[4] = {make_float2(v0.x, v0.y), make_float2(v0.z, v0.w), make_float2(v1.x, v1.y), make_float2(v1.z, v1.w)};
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float2 wa = w.w3[0][i][ky * 3 + kx], wb = w.w3[1][i][ky * 3 + kx];
#pragma unroll
          for (int x = 0; x < 2; ++x) {
            acc[x][0] = ffma2(row[x + kx], wa, acc[x][0]);
            acc[x][1] = ffma2(row[x + kx], wb, acc[x][1]);
          }
        }
      }
    epi(oy, g, acc);
  }
}

// ---- stage 4: NConv(2->1, 1x1) on the stage-3 pairs -> (num, den); the output is out_scale * num / (den + eps)
__device__ __forceinline__ float2 stage4_nd(float2 a, float2 b, const NcupWeights& w) {
  const float den = fmaf(a.y, w.w4[0], b.y * w.w4[1]);
  const float num = fmaf(a.x, w.w4[0], b.x * w.w4[1]);
  return make_float2(num, den);
}

// The whole forward of one 30x30 output tile.  kConf: also write nconv_out's output confidence den4 / sum(W4) to conf_out
// (same layout as out, no out_scale); without it the instantiation is the plain forward.
template <bool kConf>
__device__ __forceinline__ void ncup_forward_tile(const float* __restrict__ x_lowres, const float* __restrict__ conf,
                                                  const NcupWeights& w, int H4, int W4, float out_scale, float* __restrict__ out,
                                                  float* __restrict__ conf_out) {
  __shared__ float lx[LT][LT], lc[LT][LT];                  // lattice data (flow) and confidence
  __shared__ __align__(16) float2 s1[2][R1][P1];            // stage 1: (data*conf, conf) per channel
  __shared__ __align__(16) float2 s2[2][R2][P2];            // stage 2

  const int plane = blockIdx.z;                             // b*2 + c   (channels_to_batch, upsampler.py:168)
  const int ty0 = blockIdx.y * NT, tx0 = blockIdx.x * NT;
  const int H = 4 * H4, W = 4 * W4;                         // scale 4, samples at offset 2 (upsampler.py:208)
  // first lattice sample that can reach the stage-1 region (rows ty0-3 ..): floor((ty0 - 4) / 4), -1 for the first tile
  const int iy_base = ty0 >= 4 ? (ty0 - 4) >> 2 : -1, ix_base = tx0 >= 4 ? (tx0 - 4) >> 2 : -1;

  stage0_lattice<LT>(x_lowres, conf, plane, iy_base, ix_base, H4, W4, lx, lc);
  __syncthreads();
  stage1<LT, R1, P1>(lx, lc, iy_base, ix_base, ty0 - 3, tx0 - 3, H, W, H4, W4, w, s1);
  __syncthreads();
  stage2<R1, P1, R2, P2>(s1, ty0 - 1, tx0 - 1, H, W, w, s2, nullptr);
  __syncthreads();
  // stage 3 (3x3, folded decoder) + stage 4 (1x1) + scale: thread = row oy, columns 2g, 2g+1 of the 30x30 tile
  stage3<R2, P2, NT>(s2, w, [&](int oy, int g, const float2 (&acc)[2][2]) {
    const int y = ty0 + oy;
    if (y >= H) return;
    float res[2], cres[2];
#pragma unroll
    for (int x = 0; x < 2; ++x) {
      const float2 a = nconv_out_pair(acc[x][0], w.inv_s3[0]), b = nconv_out_pair(acc[x][1], w.inv_s3[1]);   // (y*c, c) pairs
      const float2 nd = stage4_nd(a, b, w);
      res[x] = out_scale * (nd.x / (nd.y + kEps));
      if constexpr (kConf) cres[x] = nd.y / (w.w4[0] + w.w4[1]);    // c' = den / sum(W), nconv_modules.py:186-190
    }
    const int x0 = tx0 + 2 * g;
    const size_t o = ((size_t)plane * H + y) * W + x0;
    if (x0 + 1 < W) {                                         // W = 4*W4 and x0 are even: 8-byte aligned
      *reinterpret_cast<float2*>(out + o) = make_float2(res[0], res[1]);
      if constexpr (kConf) *reinterpret_cast<float2*>(conf_out + o) = make_float2(cres[0], cres[1]);
    } else if (x0 < W) {
      out[o] = res[0];
      if constexpr (kConf) conf_out[o] = cres[0];
    }
  });
}

__global__ void __launch_bounds__(kThreads)
ncup_fused_kernel(const float* __restrict__ x_lowres, const float* __restrict__ conf, const __grid_constant__ NcupWeights w,
                  int H4, int W4, float out_scale, float* __restrict__ out) {
  ncup_forward_tile<false>(x_lowres, conf, w, H4, W4, out_scale, out, nullptr);
}

__global__ void __launch_bounds__(kThreads)
ncup_fused_conf_kernel(const float* __restrict__ x_lowres, const float* __restrict__ conf, const __grid_constant__ NcupWeights w,
                       int H4, int W4, float out_scale, float* __restrict__ out, float* __restrict__ conf_out) {
  ncup_forward_tile<true>(x_lowres, conf, w, H4, W4, out_scale, out, conf_out);
}

// The 224 positive weights (state_dict order) -> NcupWeights, with the same fp32 arithmetic as the host packing of
// rnc_ncup_fwd (sequential sums, IEEE division), so both forwards see bit-identical weights.
__device__ __forceinline__ void load_weights(const float* __restrict__ p, NcupWeights& w) {
  const int tid = threadIdx.x;
  for (int k = tid; k < 50; k += kThreads) { const float v = p[k]; w.w1[k / 25][k % 25] = make_float2(v, v); }
  for (int k = tid; k < 100; k += kThreads) { const float v = p[50 + k]; w.w2[k / 50][(k / 25) % 2][k % 25] = make_float2(v, v); }
  for (int k = tid; k < 36; k += kThreads) {
    const int o = k / 18, i = (k / 9) % 2, t = k % 9;
    const float v = p[150 + (o * 4 + i) * 9 + t] + p[150 + (o * 4 + i + 2) * 9 + t];
    w.w3[o][i][t] = make_float2(v, v);
  }
  if (tid < 2) w.w4[tid] = p[222 + tid];
  if (tid >= 32 && tid < 38) {                              // one thread per normalisation sum
    const int k = tid - 32, o = k & 1;
    float s = 0.f;
    if (k < 2) {
      for (int t = 0; t < 25; ++t) s += p[o * 25 + t];
      w.inv_s1[o] = 1.0f / s;
    } else if (k < 4) {
      for (int i = 0; i < 2; ++i)
        for (int t = 0; t < 25; ++t) s += p[50 + (o * 2 + i) * 25 + t];
      w.inv_s2[o] = 1.0f / s;
    } else {
      for (int i = 0; i < 4; ++i)
        for (int t = 0; t < 9; ++t) s += p[150 + (o * 4 + i) * 9 + t];
      w.inv_s3[o] = 1.0f / s;
    }
  }
}

__global__ void __launch_bounds__(kThreads)
ncup_train_fwd_kernel(const float* __restrict__ x_lowres, const float* __restrict__ conf, const float* __restrict__ wdev,
                      int H4, int W4, float out_scale, float* __restrict__ out) {
  __shared__ NcupWeights w;
  load_weights(wdev, w);
  __syncthreads();
  ncup_forward_tile<false>(x_lowres, conf, w, H4, W4, out_scale, out, nullptr);
}

__global__ void __launch_bounds__(kThreads)
ncup_train_fwd_conf_kernel(const float* __restrict__ x_lowres, const float* __restrict__ conf, const float* __restrict__ wdev,
                           int H4, int W4, float out_scale, float* __restrict__ out, float* __restrict__ conf_out) {
  __shared__ NcupWeights w;
  load_weights(wdev, w);
  __syncthreads();
  ncup_forward_tile<true>(x_lowres, conf, w, H4, W4, out_scale, out, conf_out);
}

// ------------------------------------------------------------------------------------------------------------------ backward
//
// Every layer k < 4 carries the pair P = (y*c, c) with y = num/D, D = den + eps, c = den*inv_s, inv_s = 1/sum(W).  Given the
// upstream (gPx, gPy) at a position:
//   a = dL/dnum = gPx * inv_s * den/D
//   b = dL/dden = inv_s * (gPx * y * eps/D + gPy)           (the eps term carries num: 0 where the confidence is 0)
//   dL/dinv_s  += den * (gPx * y + gPy)                      -> every weight of output o gets -inv_s^2 * that sum
// the layer's inputs receive the transposed convolutions of (a, b), and dL/dW[o,i,t] = sum_p a_o(p) Px_i(p+t) + b_o(p) Py_i(p+t).
// The last layer is out = out_scale * num/D: a = g * out_scale / D, b = -a * y.
//
// A CTA owns a 32x32 tile R of full-resolution positions (8x8 lattice samples).  It recomputes the forward on R+8 (stage 1),
// R+6 (stage 2) and R+5 (stage 3), then runs the chain backwards: (a, b) of layer 3 on R+5, of layer 2 on R+4, of layer 1 on
// R+2, and the lattice gradients on R.  Weight-gradient sums run over the positions of R only, so every position counts once.
constexpr int NB = 32;                   // owned tile side
constexpr int LTB = 13;                  // lattice samples per side reaching the stage-1 region
constexpr int RB1 = NB + 16, PB1 = RB1 + 2;     // stage 1: origin tile - 8
constexpr int RB2 = NB + 12, PB2 = RB2 + 2;     // stage 2: origin tile - 6
constexpr int RB3 = NB + 10;                    // stage 3: origin tile - 5
constexpr int kNPart = 194;              // W1 50 | W2 100 | folded W3 36 | w4 2 | sum(gc*den)-terms 3 x 2
constexpr int kPartLd = 196;             // doubles per CTA partial row
constexpr int kOffW2 = 50, kOffW3 = 150, kOffW4 = 186, kOffS = 188;

struct BwdSmem {
  NcupWeights w;
  float lx[LTB][LTB], lc[LTB][LTB];
  __align__(16) float2 s1[2][RB1][PB1];  // layer-1 pairs
  __align__(16) float2 s2[2][RB2][PB2];  // layer-2 pairs
  __align__(16) float2 nd2[2][RB2][PB2]; // layer-2 (num, den), then its (a, b)
  __align__(16) float2 nd3[2][RB3][RB3]; // layer-3 (num, den), then its (a, b); later layer 1's (a, b) on R+2
  __align__(16) float red[kThreads * 5]; // reduction scratch
  double part[kPartLd];                  // this CTA's partial sums
};

// Gradient of a layer's pair at one position: (gPx, gPy), (num, den) -> (a, b); returns den * (gPx * y + gPy) for dL/dinv_s
__device__ __forceinline__ float pair_bwd(float gpx, float gpy, float2 nd, float inv_s, float2& ab) {
  const float D = nd.y + kEps;
  const float y = nd.x / D;
  ab = make_float2(gpx * inv_s * (nd.y / D), inv_s * fmaf(gpx * y, kEps / D, gpy));
  return nd.y * fmaf(gpx, y, gpy);
}

// Deterministic CTA sum of one float per thread (fixed tree) -> every thread gets the result.
__device__ __forceinline__ double block_sum(float v, float* red) {
  double d = v;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) reinterpret_cast<double*>(red)[threadIdx.x >> 5] = d;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < kThreads / 32; ++k) s += reinterpret_cast<const double*>(red)[k];
  __syncthreads();
  return s;
}

// dL/dW[o][i][ky][kx] over the owned tile: sum_p a_o(p) . in_i(p + (ky, kx) - K/2) for (num, den) pairs.  ab is indexed with
// the tile origin at (oa, oa), in with the tile origin at (oi, oi) minus the K/2 shift (so that in[oi + py + ky][oi + px + kx]
// is the tap (ky, kx)).  Thread = (o, i, ky) x row set; results go to part[off + (o*2 + i)*K*K + ky*K + kx].
template <int K, int PA, int RA, int PI, int RI>
__device__ __forceinline__ void wgrad(const float2 (&ab)[2][RA][PA], int oa, const float2 (&in)[2][RI][PI], int oi, float* red,
                                      double* part, int off) {
  constexpr int NG = 4 * K, NRS = kThreads / NG;
  const int tid = threadIdx.x;
  if (tid < NG * NRS) {
    const int g = tid % NG, rs = tid / NG;
    const int o = g / (2 * K), i = (g / K) % 2, ky = g % K;
    float acc[K];
#pragma unroll
    for (int kx = 0; kx < K; ++kx) acc[kx] = 0.f;
    for (int py = rs; py < NB; py += NRS) {
      const float2* ar = &ab[o][oa + py][oa];
      const float2* ir = &in[i][oi + py + ky][oi];
      for (int px = 0; px < NB; ++px) {
        const float2 a = ar[px];
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
          const float2 v = ir[px + kx];
          acc[kx] = fmaf(a.x, v.x, fmaf(a.y, v.y, acc[kx]));
        }
      }
    }
#pragma unroll
    for (int kx = 0; kx < K; ++kx) red[(rs * NG + g) * K + kx] = acc[kx];
  }
  __syncthreads();
  if (tid < NG * K) {
    double s = 0.0;
    for (int rs = 0; rs < NRS; ++rs) s += red[rs * NG * K + tid];
    const int g = tid / K, kx = tid % K;
    const int o = g / (2 * K), i = (g / K) % 2, ky = g % K;
    part[off + (o * 2 + i) * K * K + ky * K + kx] = s;
  }
  __syncthreads();
}

// dL/dc3[k] of the last layer: the flow's term gy, plus t4 * W4[k] from the confidence when kConf
template <bool kConf>
__device__ __forceinline__ float conf_adjoint(float gy, float t4, float w4) {
  if constexpr (kConf) return fmaf(t4, w4, gy);
  return gy;
}

// kConf: the loss also has the term sum(g_conf_out * conf_out), conf_out = den4 / S4 with S4 = W4[0] + W4[1], and either
// upstream gradient may be NULL.  It enters at layer 4: dL/dc3[k] += g * W4[k] / S4 (the den component of pair k, from where
// the existing chain carries it down) and dL/dW4[k] += g * (c3[k] - den4 / S4) / S4.  Without it the instantiation is the
// plain backward.
template <bool kConf>
__device__ __forceinline__ void ncup_bwd_tile(const float* __restrict__ x_lowres, const float* __restrict__ conf,
                                              const float* __restrict__ wdev, int H4, int W4, float out_scale,
                                              const float* __restrict__ g_out, const float* __restrict__ g_conf_out,
                                              float* __restrict__ g_x, float* __restrict__ g_conf, double* __restrict__ partials) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  BwdSmem& S = *reinterpret_cast<BwdSmem*>(smem_raw);
  const NcupWeights& w = S.w;
  const int tid = threadIdx.x;
  const int plane = blockIdx.z;
  const int ty0 = blockIdx.y * NB, tx0 = blockIdx.x * NB;
  const int H = 4 * H4, W = 4 * W4;
  const int iy_base = (ty0 - 9) >> 2, ix_base = (tx0 - 9) >> 2;      // floor((origin - 1) / 4) of the stage-1 region

  load_weights(wdev, S.w);
  stage0_lattice<LTB>(x_lowres, conf, plane, iy_base, ix_base, H4, W4, S.lx, S.lc);
  __syncthreads();
  // ---- forward recompute (the forward's own stages: bit-identical values)
  stage1<LTB, RB1, PB1>(S.lx, S.lc, iy_base, ix_base, ty0 - 8, tx0 - 8, H, W, H4, W4, w, S.s1);
  __syncthreads();
  stage2<RB1, PB1, RB2, PB2>(S.s1, ty0 - 6, tx0 - 6, H, W, w, S.s2, S.nd2);
  __syncthreads();
  stage3<RB2, PB2, RB3>(S.s2, w, [&](int oy, int g, const float2 (&acc)[2][2]) {
#pragma unroll
    for (int x = 0; x < 2; ++x) {
      S.nd3[0][oy][2 * g + x] = acc[x][0];
      S.nd3[1][oy][2 * g + x] = acc[x][1];
    }
  });
  __syncthreads();

  // ---- layer 4 and layer 3 on R+5: (a3, b3) replace (num3, den3)
  float gw4[2] = {0.f, 0.f}, gs3[2] = {0.f, 0.f};
  [[maybe_unused]] const float inv_s4 = kConf ? 1.0f / (w.w4[0] + w.w4[1]) : 0.f;
  for (int idx = tid; idx < RB3 * RB3; idx += kThreads) {
    const int ry = idx / RB3, rx = idx - ry * RB3;
    const int y = ty0 - 5 + ry, x = tx0 - 5 + rx;
    if (y < 0 || y >= H || x < 0 || x >= W) {
      S.nd3[0][ry][rx] = S.nd3[1][ry][rx] = make_float2(0.f, 0.f);
      continue;
    }
    const bool own = ry >= 5 && ry < 5 + NB && rx >= 5 && rx < 5 + NB;
    const float2 n0 = S.nd3[0][ry][rx], n1 = S.nd3[1][ry][rx];
    const float2 pa = nconv_out_pair(n0, w.inv_s3[0]), pb = nconv_out_pair(n1, w.inv_s3[1]);
    const float2 nd4 = stage4_nd(pa, pb, w);
    const float D4 = nd4.y + kEps;
    const size_t gi = ((size_t)plane * H + y) * W + x;
    const float a4 = (kConf && g_out == nullptr ? 0.f : g_out[gi]) * out_scale / D4;
    const float b4 = -a4 * (nd4.x / D4);
    [[maybe_unused]] const float t4 = kConf && g_conf_out != nullptr ? g_conf_out[gi] * inv_s4 : 0.f;    // g / S4
    float2 ab0, ab1;
    const float s0 = pair_bwd(a4 * w.w4[0], conf_adjoint<kConf>(b4 * w.w4[0], t4, w.w4[0]), n0, w.inv_s3[0], ab0);
    const float s1 = pair_bwd(a4 * w.w4[1], conf_adjoint<kConf>(b4 * w.w4[1], t4, w.w4[1]), n1, w.inv_s3[1], ab1);
    if (own) {
      gw4[0] = fmaf(a4, pa.x, fmaf(b4, pa.y, gw4[0]));
      gw4[1] = fmaf(a4, pb.x, fmaf(b4, pb.y, gw4[1]));
      if constexpr (kConf) {
        const float c4 = nd4.y * inv_s4;
        gw4[0] = fmaf(t4, pa.y - c4, gw4[0]);
        gw4[1] = fmaf(t4, pb.y - c4, gw4[1]);
      }
      gs3[0] += s0;
      gs3[1] += s1;
    }
    S.nd3[0][ry][rx] = ab0;
    S.nd3[1][ry][rx] = ab1;
  }
  __syncthreads();

  // ---- layer 2 on R+4: gP2 = transposed 3x3 of (a3, b3); (a2, b2) replace (num2, den2) at the same position
  float gs2[2] = {0.f, 0.f};
  for (int idx = tid; idx < (NB + 8) * (NB + 8); idx += kThreads) {
    const int ry = idx / (NB + 8), rx = idx - ry * (NB + 8);
    const int y = ty0 - 4 + ry, x = tx0 - 4 + rx;
    if (y < 0 || y >= H || x < 0 || x >= W) {
      S.nd2[0][ry + 2][rx + 2] = S.nd2[1][ry + 2][rx + 2] = make_float2(0.f, 0.f);
      continue;
    }
    float2 gp[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
#pragma unroll
    for (int o = 0; o < 2; ++o)
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float2 ab = S.nd3[o][ry + 2 - ky][rx + 2 - kx];
#pragma unroll
          for (int i = 0; i < 2; ++i) gp[i] = ffma2(ab, w.w3[o][i][ky * 3 + kx], gp[i]);
        }
    const bool own = ry >= 4 && ry < 4 + NB && rx >= 4 && rx < 4 + NB;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float2 ab;
      const float s = pair_bwd(gp[i].x, gp[i].y, S.nd2[i][ry + 2][rx + 2], w.inv_s2[i], ab);
      if (own) gs2[i] += s;
      S.nd2[i][ry + 2][rx + 2] = ab;
    }
  }
  // dL/dW3 (folded): (a3, b3) on R against the layer-2 pairs (reads nd3 and s2 only: no barrier needed before it)
  wgrad<3, RB3, RB3, PB2, RB2>(S.nd3, 5, S.s2, 5, S.red, S.part, kOffW3);

  // ---- layer 1 on R+2: gP1 = transposed 5x5 of (a2, b2); (a1, b1) -> nd3 (free now), origin tile - 2
  float gs1[2] = {0.f, 0.f};
  for (int idx = tid; idx < (NB + 4) * (NB + 4); idx += kThreads) {
    const int ry = idx / (NB + 4), rx = idx - ry * (NB + 4);
    const int y = ty0 - 2 + ry, x = tx0 - 2 + rx;
    if (y < 0 || y >= H || x < 0 || x >= W) {
      S.nd3[0][ry][rx] = S.nd3[1][ry][rx] = make_float2(0.f, 0.f);
      continue;
    }
    float2 gp[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
#pragma unroll
    for (int o = 0; o < 2; ++o)
#pragma unroll
      for (int ky = 0; ky < 5; ++ky)
#pragma unroll
        for (int kx = 0; kx < 5; ++kx) {
          const float2 ab = S.nd2[o][ry + 6 - ky][rx + 6 - kx];
#pragma unroll
          for (int i = 0; i < 2; ++i) gp[i] = ffma2(ab, w.w2[o][i][ky * 5 + kx], gp[i]);
        }
    float2 a0, a1;
    stage1_acc(S.lx, S.lc, iy_base, ix_base, y, x, H4, W4, w, a0, a1);
    const bool own = ry >= 2 && ry < 2 + NB && rx >= 2 && rx < 2 + NB;
    float2 ab0, ab1;
    const float s0 = pair_bwd(gp[0].x, gp[0].y, a0, w.inv_s1[0], ab0);
    const float s1 = pair_bwd(gp[1].x, gp[1].y, a1, w.inv_s1[1], ab1);
    if (own) { gs1[0] += s0; gs1[1] += s1; }
    S.nd3[0][ry][rx] = ab0;
    S.nd3[1][ry][rx] = ab1;
  }
  // dL/dW2: (a2, b2) on R (nd2, origin tile - 6) against the layer-1 pairs (s1, origin tile - 8)
  wgrad<5, PB2, RB2, PB1, RB1>(S.nd2, 6, S.s1, 6, S.red, S.part, kOffW2);   // its barriers also publish layer 1's (a, b)

  // ---- lattice samples of R: gradient of the input pair (X*C, C) -> g_x = gX * C, g_conf = gX * X + gC
  for (int k = tid; k < (NB / 4) * (NB / 4); k += kThreads) {
    const int li = k / (NB / 4), lj = k % (NB / 4);
    const int iy = ty0 / 4 + li, ix = tx0 / 4 + lj;
    if (iy >= H4 || ix >= W4) continue;
    const int qy = 4 * li + 2, qx = 4 * lj + 2;            // relative to the tile origin
    float2 gp = make_float2(0.f, 0.f);
#pragma unroll
    for (int o = 0; o < 2; ++o)
#pragma unroll
      for (int ky = 0; ky < 5; ++ky)
#pragma unroll
        for (int kx = 0; kx < 5; ++kx) gp = ffma2(S.nd3[o][qy + 4 - ky][qx + 4 - kx], w.w1[o][ky * 5 + kx], gp);
    const float xv = S.lx[iy - iy_base][ix - ix_base], cv = S.lc[iy - iy_base][ix - ix_base];
    const size_t gi = ((size_t)plane * H4 + iy) * W4 + ix;
    if (g_x) g_x[gi] = gp.x * cv;
    if (g_conf) g_conf[gi] = fmaf(gp.x, xv, gp.y);
  }
  if (partials == nullptr) return;
  // dL/dW1[o][t]: the layer-1 input is non-zero on lattice samples only; p = q - (t - 2) must lie in R
  if (tid < 50) {
    const int o = tid / 25, ky = (tid % 25) / 5, kx = tid % 5;
    float acc = 0.f;
    for (int li = 0; li < LTB; ++li) {
      const int py = 4 * (iy_base + li) + 2 - (ky - 2) - ty0;
      if (py < 0 || py >= NB) continue;
      for (int lj = 0; lj < LTB; ++lj) {
        const int px = 4 * (ix_base + lj) + 2 - (kx - 2) - tx0;
        if (px < 0 || px >= NB) continue;
        const float cv = S.lc[li][lj];
        const float2 ab = S.nd3[o][py + 2][px + 2];
        acc = fmaf(ab.x, S.lx[li][lj] * cv, fmaf(ab.y, cv, acc));
      }
    }
    S.part[tid] = acc;
  }
  {
    const float v[8] = {gw4[0], gw4[1], gs1[0], gs1[1], gs2[0], gs2[1], gs3[0], gs3[1]};
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const double s = block_sum(v[k], S.red);
      if (tid == 0) S.part[kOffW4 + k] = s;
    }
  }
  __syncthreads();
  double* dst = partials + ((size_t)(blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * kPartLd;
  for (int k = tid; k < kNPart; k += kThreads) dst[k] = S.part[k];
}

__global__ void __launch_bounds__(kThreads)
ncup_bwd_kernel(const float* __restrict__ x_lowres, const float* __restrict__ conf, const float* __restrict__ wdev, int H4, int W4,
                float out_scale, const float* __restrict__ g_out, float* __restrict__ g_x, float* __restrict__ g_conf,
                double* __restrict__ partials) {
  ncup_bwd_tile<false>(x_lowres, conf, wdev, H4, W4, out_scale, g_out, nullptr, g_x, g_conf, partials);
}

__global__ void __launch_bounds__(kThreads)
ncup_conf_bwd_kernel(const float* __restrict__ x_lowres, const float* __restrict__ conf, const float* __restrict__ wdev, int H4,
                     int W4, float out_scale, const float* __restrict__ g_out, const float* __restrict__ g_conf_out,
                     float* __restrict__ g_x, float* __restrict__ g_conf, double* __restrict__ partials) {
  ncup_bwd_tile<true>(x_lowres, conf, wdev, H4, W4, out_scale, g_out, g_conf_out, g_x, g_conf, partials);
}

// Fixed-order fp64 sum of the per-CTA partials: block k reduces column k
__global__ void __launch_bounds__(kThreads)
ncup_bwd_reduce_kernel(const double* __restrict__ partials, int nblocks, double* __restrict__ sums) {
  __shared__ double red[kThreads / 32];
  const int k = blockIdx.x;
  double s = 0.0;
  for (int b = threadIdx.x; b < nblocks; b += kThreads) s += partials[(size_t)b * kPartLd + k];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) t += red[i];
    sums[k] = t;
  }
}

// sums -> dL/dW of the 224 unfolded positive weights: the folded decoder gradient goes to both halves, and every weight of
// output o of layer k gets -inv_s^2 * sum(gc * den) (inv_s from the unfolded weights, in fp64)
__global__ void __launch_bounds__(kThreads)
ncup_bwd_finish_kernel(const double* __restrict__ sums, const float* __restrict__ p, float* __restrict__ g_w) {
  __shared__ double corr[3][2];
  const int tid = threadIdx.x;
  if (tid < 6) {
    const int l = tid / 2, o = tid % 2;
    const int n = l == 0 ? 25 : l == 1 ? 50 : 36, base = l == 0 ? o * 25 : l == 1 ? 50 + o * 50 : 150 + o * 36;
    double s = 0.0;
    for (int t = 0; t < n; ++t) s += p[base + t];
    corr[l][o] = sums[kOffS + 2 * l + o] / (s * s);
  }
  __syncthreads();
  if (tid < 50) g_w[tid] = static_cast<float>(sums[tid] - corr[0][tid / 25]);
  if (tid < 100) g_w[50 + tid] = static_cast<float>(sums[kOffW2 + tid] - corr[1][tid / 50]);
  if (tid < 72) {
    const int o = tid / 36, i = (tid / 9) % 4, t = tid % 9;
    g_w[150 + tid] = static_cast<float>(sums[kOffW3 + (o * 2 + (i & 1)) * 9 + t] - corr[2][o]);
  }
  if (tid < 2) g_w[222 + tid] = static_cast<float>(sums[kOffW4 + tid]);
}

// The grid of tile x tile output tiles (NT for the forwards, NB for the backward) over the B * 2 planes
inline dim3 ncup_grid(int B, int H4, int W4, int tile) {
  return dim3((4 * W4 + tile - 1) / tile, (4 * H4 + tile - 1) / tile, B * 2);
}

// Rejects, before anything is launched, a shape whose ncup_grid(B, H4, W4, tile) exceeds the 65535 limit of grid.y and grid.z
inline int ncup_check_shape(int B, int H4, int W4, int tile) {
  if (B <= 0 || H4 <= 0 || W4 <= 0) return RNC_ERR_BAD_SHAPE;
  if (H4 > (1 << 20) || W4 > (1 << 20) || 2LL * B > 65535 || (4LL * H4 + tile - 1) / tile > 65535) return RNC_ERR_UNSUPPORTED;
  return RNC_OK;
}

}  // namespace rnc

using namespace rnc;

// wts_host: softplus'd weights in state_dict order: nconv_in[2,1,5,5], nconv_x2.0[2,2,5,5], decoder.0[2,4,3,3], nconv_out[1,2,1,1]
static NcupWeights pack_host_weights(const float* wts_host) {
  NcupWeights w;
  const float* p = wts_host;
  for (int o = 0; o < 2; ++o) {
    float s = 0.f;
    for (int t = 0; t < 25; ++t) { w.w1[o][t] = make_float2(p[o * 25 + t], p[o * 25 + t]); s += p[o * 25 + t]; }
    w.inv_s1[o] = 1.0f / s;
  }
  p += 50;
  for (int o = 0; o < 2; ++o) {
    float s = 0.f;
    for (int i = 0; i < 2; ++i)
      for (int t = 0; t < 25; ++t) { const float v = p[(o * 2 + i) * 25 + t]; w.w2[o][i][t] = make_float2(v, v); s += v; }
    w.inv_s2[o] = 1.0f / s;
  }
  p += 100;
  for (int o = 0; o < 2; ++o) {
    float s = 0.f;
    for (int i = 0; i < 4; ++i)
      for (int t = 0; t < 9; ++t) s += p[(o * 4 + i) * 9 + t];
    for (int i = 0; i < 2; ++i)
      for (int t = 0; t < 9; ++t) { const float v = p[(o * 4 + i) * 9 + t] + p[(o * 4 + i + 2) * 9 + t]; w.w3[o][i][t] = make_float2(v, v); }
    w.inv_s3[o] = 1.0f / s;
  }
  p += 72;
  w.w4[0] = p[0]; w.w4[1] = p[1];
  return w;
}

// conf_out NULL launches the plain kernels, non-NULL their confidence twins (ncup_forward_tile<kConf>)
extern "C" int rnc_ncup_fwd(const float* x_lowres, const float* conf, const float* wts_host, int B, int H4, int W4,
                            float out_scale, float* out, float* conf_out, void* stream) {
  if (int st = ncup_check_shape(B, H4, W4, NT)) return st;
  if (!x_lowres || !conf || !wts_host || !out) return RNC_ERR_BAD_POINTER;
  const NcupWeights w = pack_host_weights(wts_host);
  const dim3 grid = ncup_grid(B, H4, W4, NT);
  cudaStream_t s = as_stream(stream);
  if (conf_out)
    ncup_fused_conf_kernel<<<grid, kThreads, 0, s>>>(x_lowres, conf, w, H4, W4, out_scale, out, conf_out);
  else
    ncup_fused_kernel<<<grid, kThreads, 0, s>>>(x_lowres, conf, w, H4, W4, out_scale, out);
  return after_launch();
}

extern "C" int rnc_ncup_train_fwd(const float* x_lowres, const float* conf, const float* weights_dev, int B, int H4, int W4,
                                  float out_scale, float* out, float* conf_out, void* stream) {
  if (int st = ncup_check_shape(B, H4, W4, NT)) return st;
  if (!x_lowres || !conf || !weights_dev || !out) return RNC_ERR_BAD_POINTER;
  const dim3 grid = ncup_grid(B, H4, W4, NT);
  cudaStream_t s = as_stream(stream);
  if (conf_out)
    ncup_train_fwd_conf_kernel<<<grid, kThreads, 0, s>>>(x_lowres, conf, weights_dev, H4, W4, out_scale, out, conf_out);
  else
    ncup_train_fwd_kernel<<<grid, kThreads, 0, s>>>(x_lowres, conf, weights_dev, H4, W4, out_scale, out);
  return after_launch();
}

extern "C" size_t rnc_ncup_bwd_workspace_bytes(int B, int H4, int W4) {
  if (ncup_check_shape(B, H4, W4, NB)) return 0;
  const dim3 g = ncup_grid(B, H4, W4, NB);
  return sizeof(double) * ((size_t)g.x * g.y * g.z * kPartLd + kPartLd);
}

// g_conf_out NULL launches ncup_bwd_kernel, non-NULL ncup_conf_bwd_kernel; then, with g_weights, the fixed-order reduction of
// the per-CTA partials and the finish
extern "C" int rnc_ncup_bwd(const float* x_lowres, const float* conf, const float* weights_dev, int B, int H4, int W4,
                            float out_scale, const float* g_out, const float* g_conf_out, float* g_x_lowres, float* g_conf,
                            float* g_weights, void* workspace, size_t workspace_bytes, void* stream) {
  if (int st = ncup_check_shape(B, H4, W4, NB)) return st;
  if (!x_lowres || !conf || !weights_dev || (!g_out && !g_conf_out) || (!g_x_lowres && !g_conf && !g_weights))
    return RNC_ERR_BAD_POINTER;
  if (g_weights && (!workspace || !aligned16(workspace))) return RNC_ERR_BAD_POINTER;
  if (g_weights && workspace_bytes < rnc_ncup_bwd_workspace_bytes(B, H4, W4)) return RNC_ERR_WORKSPACE;
  static unsigned long long attr_done = 0, attr_done_conf = 0;       // one per kernel
  if (int st = g_conf_out ? ensure_dyn_smem(ncup_conf_bwd_kernel, (int)sizeof(BwdSmem), &attr_done_conf)
                          : ensure_dyn_smem(ncup_bwd_kernel, (int)sizeof(BwdSmem), &attr_done))
    return st;
  const dim3 grid = ncup_grid(B, H4, W4, NB);
  const int nblocks = grid.x * grid.y * grid.z;
  double* partials = g_weights ? static_cast<double*>(workspace) : nullptr;
  cudaStream_t s = as_stream(stream);
  if (g_conf_out)
    ncup_conf_bwd_kernel<<<grid, kThreads, sizeof(BwdSmem), s>>>(x_lowres, conf, weights_dev, H4, W4, out_scale, g_out,
                                                                 g_conf_out, g_x_lowres, g_conf, partials);
  else
    ncup_bwd_kernel<<<grid, kThreads, sizeof(BwdSmem), s>>>(x_lowres, conf, weights_dev, H4, W4, out_scale, g_out, g_x_lowres,
                                                            g_conf, partials);
  if (!g_weights) return after_launch();
  double* sums = partials + (size_t)nblocks * kPartLd;
  ncup_bwd_reduce_kernel<<<kNPart, kThreads, 0, s>>>(partials, nblocks, sums);
  ncup_bwd_finish_kernel<<<1, kThreads, 0, s>>>(sums, weights_dev, g_weights);
  return after_launch(3);
}
