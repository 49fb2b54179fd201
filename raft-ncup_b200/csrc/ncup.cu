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
// num/den accumulate as one FMA pair (ffma2) per tap; threads own 1x4 (stage 2) / 1x2 (stage 3)
// register tiles and fetch their input rows with 128-bit shared-memory loads (8 lanes = 256 contiguous bytes: conflict-free).
// Tile sides are chosen so that stage 2 is exactly one 1x4 item per thread (32 rows x 8 groups = 256).
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

__global__ void __launch_bounds__(256)
ncup_fused_kernel(const float* __restrict__ x_lowres, const float* __restrict__ conf, const __grid_constant__ NcupWeights w,
                  int H4, int W4, float out_scale, float* __restrict__ out) {
  __shared__ float lx[LT][LT], lc[LT][LT];                  // lattice data (flow) and confidence
  __shared__ __align__(16) float2 s1[2][R1][P1];            // stage 1: (data*conf, conf) per channel
  __shared__ __align__(16) float2 s2[2][R2][P2];            // stage 2

  const int tid = threadIdx.x;
  const int plane = blockIdx.z;                             // b*2 + c   (channels_to_batch, upsampler.py:168)
  const int ty0 = blockIdx.y * NT, tx0 = blockIdx.x * NT;
  const int H = 4 * H4, W = 4 * W4;                         // scale 4, samples at offset 2 (upsampler.py:208)
  // first lattice sample that can reach the stage-1 region (rows ty0-3 ..): floor((ty0 - 4) / 4), -1 for the first tile
  const int iy_base = ty0 >= 4 ? (ty0 - 4) >> 2 : -1, ix_base = tx0 >= 4 ? (tx0 - 4) >> 2 : -1;

  // ---- stage 0: lattice samples.  X[4i+2][4j+2] = x_lowres[i][j], C[4i+2][4j+2] = conf[i][j]
  if (tid < LT * LT) {
    const int li = tid / LT, lj = tid - li * LT;
    const int iy = iy_base + li, ix = ix_base + lj;
    float xv = 0.f, cv = 0.f;
    if (iy >= 0 && iy < H4 && ix >= 0 && ix < W4) {
      xv = x_lowres[((size_t)plane * H4 + iy) * W4 + ix];
      cv = conf[((size_t)plane * H4 + iy) * W4 + ix];
    }
    lx[li][lj] = xv;
    lc[li][lj] = cv;
  }
  __syncthreads();

  // ---- stage 1: NConv(1->2, 5x5) on the zero-stuffed lattice: at most 2x2 lattice samples fall under a 5x5 window
  for (int idx = tid; idx < R1 * R1; idx += 256) {
    const int ry = idx / R1, rx = idx - ry * R1;
    const int y = ty0 - 3 + ry, x = tx0 - 3 + rx;
    float2 o0 = make_float2(0.f, 0.f), o1 = o0;
    if (y >= 0 && y < H && x >= 0 && x < W) {
      float2 a0 = make_float2(0.f, 0.f), a1 = a0;
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
      o0 = nconv_out_pair(a0, w.inv_s1[0]);
      o1 = nconv_out_pair(a1, w.inv_s1[1]);
    }
    s1[0][ry][rx] = o0;
    s1[1][ry][rx] = o1;
  }
  __syncthreads();

  // ---- stage 2: NConv(2->2, 5x5): thread = row ry, columns 4g .. 4g+3 of the 32x32 region (exactly 256 items)
  {
    const int ry = tid >> 3, g = tid & 7;
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
    const int y = ty0 - 1 + ry;
#pragma unroll
    for (int x = 0; x < 4; x += 2) {           // two positions = one 16-byte store per channel
      float2 o[2][2];
#pragma unroll
      for (int d = 0; d < 2; ++d) {
        const int xx = tx0 - 1 + 4 * g + x + d;
        const bool in = y >= 0 && y < H && xx >= 0 && xx < W;
        o[d][0] = in ? nconv_out_pair(acc[x + d][0], w.inv_s2[0]) : make_float2(0.f, 0.f);
        o[d][1] = in ? nconv_out_pair(acc[x + d][1], w.inv_s2[1]) : make_float2(0.f, 0.f);
      }
      *reinterpret_cast<float4*>(&s2[0][ry][4 * g + x]) = make_float4(o[0][0].x, o[0][0].y, o[1][0].x, o[1][0].y);
      *reinterpret_cast<float4*>(&s2[1][ry][4 * g + x]) = make_float4(o[0][1].x, o[0][1].y, o[1][1].x, o[1][1].y);
    }
  }
  __syncthreads();

  // ---- stage 3 (3x3, folded decoder) + stage 4 (1x1) + scale: thread = row oy, columns 2g, 2g+1 of the 30x30 tile
  for (int idx = tid; idx < NT * (NT / 2); idx += 256) {
    const int oy = idx / (NT / 2), g = idx - oy * (NT / 2);
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
    const int y = ty0 + oy;
    if (y >= H) continue;
    float res[2];
#pragma unroll
    for (int x = 0; x < 2; ++x) {
      const float2 a = nconv_out_pair(acc[x][0], w.inv_s3[0]), b = nconv_out_pair(acc[x][1], w.inv_s3[1]);   // (y*c, c) pairs
      const float den = fmaf(a.y, w.w4[0], b.y * w.w4[1]);
      const float num = fmaf(a.x, w.w4[0], b.x * w.w4[1]);
      res[x] = out_scale * (num / (den + kEps));
    }
    const int x0 = tx0 + 2 * g;
    float* op = out + ((size_t)plane * H + y) * W + x0;
    if (x0 + 1 < W) *reinterpret_cast<float2*>(op) = make_float2(res[0], res[1]);     // W = 4*W4 and x0 are even: 8-byte aligned
    else if (x0 < W) op[0] = res[0];
  }
}

}  // namespace rnc

using namespace rnc;

extern "C" int rnc_ncup_fwd(const float* x_lowres, const float* conf, const float* wts_host, int B, int H4, int W4,
                            float out_scale, float* out, void* stream) {
  if (B <= 0 || H4 <= 0 || W4 <= 0) return RNC_ERR_BAD_SHAPE;
  if (!x_lowres || !conf || !wts_host || !out) return RNC_ERR_BAD_POINTER;
  // wts_host: softplus'd weights in state_dict order: nconv_in[2,1,5,5], nconv_x2.0[2,2,5,5], decoder.0[2,4,3,3], nconv_out[1,2,1,1]
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
  const int H = 4 * H4, W = 4 * W4;
  dim3 grid((W + NT - 1) / NT, (H + NT - 1) / NT, B * 2);
  ncup_fused_kernel<<<grid, 256, 0, as_stream(stream)>>>(x_lowres, conf, w, H4, W4, out_scale, out);
  return after_launch();
}
