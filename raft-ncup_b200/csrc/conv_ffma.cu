// Channel-last implicit-GEMM convolution with the update block's fusions as epilogues — exact-fp32 CUDA-core
// version (v1).  Replaces every nn.Conv2d + activation + torch.cat + GRU gate arithmetic of
// core/update.py:33-60 (SepConvGRU), :79-97 (BasicMotionEncoder), :6-14 (FlowHead), :123-126 (mask head) and the
// 3x3 layers of core/interp_weights_est.py:10-47.
//
// GEMM view: M = B*H*W pixels, N = Cout, K = KH*KW*Cin.  CTA tile 128 x 64, K chunks of 16 channels of one
// filter tap; zero padding is realised by zero-filling out-of-image source pixels while staging the A tile.
#include "rnc_common.cuh"

namespace rnc {

constexpr int BM = 128, BN = 64, BK = 16, CT = 128;  // CT threads, each an 8x8 micro tile
constexpr int APAD = 4;

struct ConvParams {
  rnc_conv_desc d;
  int M, cin, coutpad, nchunk_per_tap;
};

__device__ __forceinline__ float apply_act(float v, int epi) {
  if (epi == RNC_EPI_RELU || epi == RNC_EPI_RELU_FLOW) return fmaxf(v, 0.f);
  if (epi == RNC_EPI_SIGMOID) return sigmoidf_(v);
  return v;
}

__global__ void __launch_bounds__(CT)
conv_cl_ffma_kernel(const ConvParams p) {
  __shared__ __align__(16) float As[2][BK][BM + APAD];
  __shared__ __align__(16) float Bs[2][BK][BN];

  const rnc_conv_desc& d = p.d;
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int HW = d.H * d.W;

  // ---- A staging: thread loads 4 pixels x one float4 (4 channels) per chunk
  const int lq = tid & 3;
  int lm[4], ly[4], lx[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    lm[i] = m0 + (tid >> 2) + 32 * i;
    const int r = lm[i] % HW;
    ly[i] = r / d.W;
    lx[i] = r - ly[i] * d.W;
  }
  // ---- B staging: 16 rows x 64 floats = 256 float4, 2 per thread
  const int bk0 = tid >> 4, bn4 = (tid & 15) * 4;   // rows bk0 and bk0+8

  const int ntaps = d.kh * d.kw;
  const int nchunks = ntaps * p.nchunk_per_tap;
  const int ph = d.kh / 2, pw = d.kw / 2;

  float4 ra[4], rb[2];
  auto load_chunk = [&](int kc) {
    const int tap = kc / p.nchunk_per_tap;
    const int ci0 = (kc - tap * p.nchunk_per_tap) * BK;
    const int dy = tap / d.kw - ph, dx = tap % d.kw - pw;
    const int ci = ci0 + 4 * lq;
    const float* base; int ld, cc;
    if (ci < d.c0) { base = d.in0; ld = d.ld0; cc = ci; } else { base = d.in1; ld = d.ld1; cc = ci - d.c0; }
    const bool cok = ci < p.cin;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int y = ly[i] + dy, x = lx[i] + dx;
      const bool ok = cok && lm[i] < p.M && y >= 0 && y < d.H && x >= 0 && x < d.W;
      ra[i] = ok ? *reinterpret_cast<const float4*>(base + (size_t)(lm[i] + dy * d.W + dx) * ld + cc)
                 : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int k = ci0 + bk0 + 8 * i;
      rb[i] = k < p.cin ? *reinterpret_cast<const float4*>(d.weight + ((size_t)tap * p.cin + k) * p.coutpad + n0 + bn4)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_chunk = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = (tid >> 2) + 32 * i;
      As[buf][4 * lq + 0][m] = ra[i].x;
      As[buf][4 * lq + 1][m] = ra[i].y;
      As[buf][4 * lq + 2][m] = ra[i].z;
      As[buf][4 * lq + 3][m] = ra[i].w;
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) *reinterpret_cast<float4*>(&Bs[buf][bk0 + 8 * i][bn4]) = rb[i];
  };

  const int tx = tid & 7, ty = tid >> 3;
  // accumulators as pairs of adjacent output columns (same IEEE fma per element: bit-identical to the scalar form)
  float2 acc2[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc2[i][j] = make_float2(0.f, 0.f);

  load_chunk(0);
  store_chunk(0);
  __syncthreads();
  for (int kc = 0; kc < nchunks; ++kc) {
    const int buf = kc & 1;
    if (kc + 1 < nchunks) load_chunk(kc + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8 + 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 8]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 8 + 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float2 bv2[4] = {make_float2(b0.x, b0.y), make_float2(b0.z, b0.w), make_float2(b1.x, b1.y), make_float2(b1.z, b1.w)};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float2 ai = make_float2(av[i], av[i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc2[i][j] = ffma2(ai, bv2[j], acc2[i][j]);
      }
    }
    if (kc + 1 < nchunks) store_chunk(buf ^ 1);
    __syncthreads();
  }

  // ---- epilogue
  const int epi = d.epilogue;
  const int nb = n0 + tx * 8;
  float bias[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) bias[j] = d.bias[nb + j];   // bias is padded to CoutPad
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[i][2 * j] = acc2[i][j].x; acc[i][2 * j + 1] = acc2[i][j].y; }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + ty * 8 + i;
    if (m >= p.M) continue;
    if (epi == RNC_EPI_GRU_ZR) {
      const int C = d.cout >> 1;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int n = nb + j;
        if (n >= d.cout) continue;
        const float v = sigmoidf_(acc[i][j] + bias[j]);
        if (n < C) d.aux0[(size_t)m * d.ldaux + n] = v;
        else d.out[(size_t)m * d.ldo + (n - C)] = v * d.h[(size_t)m * d.ldh + (n - C)];
      }
    } else if (epi == RNC_EPI_GRU_Q) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int n = nb + j;
        if (n >= d.cout) continue;
        const float q = tanhf(acc[i][j] + bias[j]);
        const float z = d.aux0[(size_t)m * d.ldaux + n];
        const float hv = d.h[(size_t)m * d.ldh + n];
        d.h[(size_t)m * d.ldh + n] = (1.f - z) * hv + z * q;
      }
    } else {
      float* o = d.out + (size_t)m * d.ldo + nb;
      if (nb + 8 <= d.cout && (d.ldo & 3) == 0 && aligned16_dev(d.out)) {
        float4 v0, v1;
        v0.x = apply_act(acc[i][0] + bias[0], epi); v0.y = apply_act(acc[i][1] + bias[1], epi);
        v0.z = apply_act(acc[i][2] + bias[2], epi); v0.w = apply_act(acc[i][3] + bias[3], epi);
        v1.x = apply_act(acc[i][4] + bias[4], epi); v1.y = apply_act(acc[i][5] + bias[5], epi);
        v1.z = apply_act(acc[i][6] + bias[6], epi); v1.w = apply_act(acc[i][7] + bias[7], epi);
        *reinterpret_cast<float4*>(o) = v0;
        *reinterpret_cast<float4*>(o + 4) = v1;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (nb + j < d.cout) o[j] = apply_act(acc[i][j] + bias[j], epi);
      }
      if (epi == RNC_EPI_RELU_FLOW && nb <= d.cout && d.cout < nb + 8) {
        // append flow = coords1 - grid as channels [cout, cout+2)   (update.py:97: cat([out, flow]))
        const int r = m % HW, b = m / HW;
        const int y = r / d.W, x = r - y * d.W;
        const float* c1 = d.aux0 + (size_t)b * 2 * HW + r;
        d.out[(size_t)m * d.ldo + d.cout] = c1[0] - (float)x;
        d.out[(size_t)m * d.ldo + d.cout + 1] = c1[HW] - (float)y;
      }
    }
  }
}

}  // namespace rnc

using namespace rnc;

extern "C" int rnc_conv2d_cl_fwd(const rnc_conv_desc* desc, void* stream) {
  if (!desc) return RNC_ERR_BAD_POINTER;
  const rnc_conv_desc& d = *desc;
  if (d.B <= 0 || d.H <= 0 || d.W <= 0 || d.cout <= 0 || d.c0 <= 0 || d.c1 < 0) return RNC_ERR_BAD_SHAPE;
  if (d.kh < 1 || d.kw < 1 || !(d.kh & 1) || !(d.kw & 1) || d.kh * d.kw > 49) return RNC_ERR_BAD_SHAPE;
  if ((d.c0 & 3) || (d.c1 & 3) || (d.ld0 & 3) || d.ld0 < d.c0) return RNC_ERR_BAD_SHAPE;
  if (d.c1 > 0 && ((d.c0 % BK) != 0 || (d.ld1 & 3) || d.ld1 < d.c1)) return RNC_ERR_BAD_SHAPE;
  if (!d.in0 || (d.c1 > 0 && !d.in1) || !d.weight || !d.bias) return RNC_ERR_BAD_POINTER;
  if (!aligned16(d.in0) || (d.c1 > 0 && !aligned16(d.in1)) || !aligned16(d.weight)) return RNC_ERR_BAD_POINTER;
  switch (d.epilogue) {
    case RNC_EPI_LINEAR: case RNC_EPI_RELU: case RNC_EPI_SIGMOID:
      if (!d.out || d.ldo < d.cout) return RNC_ERR_BAD_POINTER;
      break;
    case RNC_EPI_RELU_FLOW:
      if (!d.out || !d.aux0 || d.ldo < d.cout + 2) return RNC_ERR_BAD_POINTER;
      break;
    case RNC_EPI_GRU_ZR:
      if (!d.out || !d.aux0 || !d.h || (d.cout & 1) || d.ldo < d.cout / 2 || d.ldaux < d.cout / 2 || d.ldh < d.cout / 2)
        return RNC_ERR_BAD_POINTER;
      break;
    case RNC_EPI_GRU_Q:
      if (!d.aux0 || !d.h || d.ldaux < d.cout || d.ldh < d.cout) return RNC_ERR_BAD_POINTER;
      break;
    default: return RNC_ERR_UNSUPPORTED;
  }
  ConvParams p;
  p.d = d;
  p.M = d.B * d.H * d.W;
  p.cin = d.c0 + d.c1;
  p.coutpad = (d.cout + BN - 1) / BN * BN;
  p.nchunk_per_tap = (p.cin + BK - 1) / BK;
  dim3 grid((p.M + BM - 1) / BM, p.coutpad / BN);
  conv_cl_ffma_kernel<<<grid, CT, 0, as_stream(stream)>>>(p);
  return after_launch();
}
