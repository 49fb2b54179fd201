// Thin-channel layers of the update block / weights net and the convex upsampler.
//   conv_flow7x7 : BasicMotionEncoder.convf1 (core/update.py:83,92) — Conv2d(2,128,7,pad 3)+ReLU on flow
//   flow_head2   : FlowHead.conv2 (core/update.py:10,14) fused with coords1 += delta (raft_nc_dbl.py:157)
//   conf_head    : Simple.out + sigmoid (core/interp_weights_est.py:37,47; core/upsampler.py:44-46)
//   ncup_guidance: nearest-x2 of flow and of the guidance (raft_nc_dbl.py:110, upsampler.py:150,155)
//   convex       : RAFT.upsample_flow (core/raft.py:73-84)
#include <cuda_fp16.h>
#include "rnc_common.cuh"

namespace rnc {

// ---------------------------------------------------------------- convf1: 7x7, Cin = 2
constexpr int F7_PX = 16;   // pixels (along x) per CTA
__global__ void __launch_bounds__(128)
conv_flow7x7_kernel(const float* __restrict__ coords1, const float* __restrict__ weight, const float* __restrict__ bias,
                    int B, int H, int W, int cout, float* __restrict__ out, int ldo) {
  __shared__ float patch[2][7][F7_PX + 6];
  const int b = blockIdx.z, y = blockIdx.y, x0 = blockIdx.x * F7_PX;
  const int HW = H * W;
  for (int i = threadIdx.x; i < 2 * 7 * (F7_PX + 6); i += blockDim.x) {
    const int c = i / (7 * (F7_PX + 6)), r = i % (7 * (F7_PX + 6));
    const int ty = r / (F7_PX + 6), tx = r % (F7_PX + 6);
    const int yy = y + ty - 3, xx = x0 + tx - 3;
    float v = 0.f;
    if (yy >= 0 && yy < H && xx >= 0 && xx < W)
      v = coords1[((size_t)b * 2 + c) * HW + yy * W + xx] - (c == 0 ? (float)xx : (float)yy);
    patch[c][ty][tx] = v;
  }
  __syncthreads();
  for (int co = threadIdx.x; co < cout; co += blockDim.x) {
    float acc[F7_PX];
    const float bv = bias[co];
#pragma unroll
    for (int i = 0; i < F7_PX; ++i) acc[i] = bv;
    for (int ky = 0; ky < 7; ++ky)
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const float w0 = weight[((ky * 7 + kx) * 2 + 0) * cout + co];
        const float w1 = weight[((ky * 7 + kx) * 2 + 1) * cout + co];
#pragma unroll
        for (int i = 0; i < F7_PX; ++i) {
          acc[i] = fmaf(patch[0][ky][i + kx], w0, acc[i]);
          acc[i] = fmaf(patch[1][ky][i + kx], w1, acc[i]);
        }
      }
#pragma unroll
    for (int i = 0; i < F7_PX; ++i)
      if (x0 + i < W) out[((size_t)b * HW + y * W + x0 + i) * ldo + co] = fmaxf(acc[i], 0.f);
  }
}

// ---------------------------------------------------------------- FlowHead.conv2: 3x3, Cout = 2, + coords update
__global__ void __launch_bounds__(256)
flow_head2_kernel(const float* __restrict__ in, int cin, int ldi, const float* __restrict__ weight,
                  const float* __restrict__ bias, int B, int H, int W, float* __restrict__ delta,
                  float* __restrict__ coords1) {
  extern __shared__ __align__(16) float wsm[];   // [9][cin][2]
  for (int i = threadIdx.x; i < 9 * cin * 2; i += blockDim.x) wsm[i] = weight[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int HW = H * W, M = B * HW;
  for (int m = blockIdx.x * nwarp + warp; m < M; m += gridDim.x * nwarp) {
    const int b = m / HW, r = m - b * HW, y = r / W, x = r - y * W;
    float s0 = 0.f, s1 = 0.f;
    for (int t = 0; t < 9; ++t) {
      const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;   // warp-uniform
      const float* src = in + (size_t)(m + (t / 3 - 1) * W + (t % 3 - 1)) * ldi;
      for (int c = lane * 4; c < cin; c += 128) {
        const float4 v = *reinterpret_cast<const float4*>(src + c);
        const float4 wa = *reinterpret_cast<const float4*>(&wsm[(t * cin + c) * 2]);       // (c,0)(c,1)(c+1,0)(c+1,1)
        const float4 wb = *reinterpret_cast<const float4*>(&wsm[(t * cin + c) * 2 + 4]);
        s0 = fmaf(v.x, wa.x, s0); s1 = fmaf(v.x, wa.y, s1);
        s0 = fmaf(v.y, wa.z, s0); s1 = fmaf(v.y, wa.w, s1);
        s0 = fmaf(v.z, wb.x, s0); s1 = fmaf(v.z, wb.y, s1);
        s0 = fmaf(v.w, wb.z, s0); s1 = fmaf(v.w, wb.w, s1);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, o);
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    }
    if (lane < 2) {
      const float dv = (lane == 0 ? s0 : s1) + bias[lane];
      const size_t idx = ((size_t)b * 2 + lane) * HW + r;
      if (delta) delta[idx] = dv;
      coords1[idx] += dv;
    }
  }
}

// ---------------------------------------------------------------- Simple.out (1x1, Cout = 2) + sigmoid -> NCHW
__global__ void conf_head_kernel(const float* __restrict__ in, int cin, int ldi, const float* __restrict__ weight,
                                 const float* __restrict__ bias, int B, int HW, float* __restrict__ conf) {
  const int M = B * HW;
  for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < M; m += gridDim.x * blockDim.x) {
    const float* src = in + (size_t)m * ldi;
    float s0 = bias[0], s1 = bias[1];
    for (int c = 0; c < cin; c += 4) {
      const float4 v = *reinterpret_cast<const float4*>(src + c);
      s0 = fmaf(v.x, weight[2 * c + 0], s0); s1 = fmaf(v.x, weight[2 * c + 1], s1);
      s0 = fmaf(v.y, weight[2 * c + 2], s0); s1 = fmaf(v.y, weight[2 * c + 3], s1);
      s0 = fmaf(v.z, weight[2 * c + 4], s0); s1 = fmaf(v.z, weight[2 * c + 5], s1);
      s0 = fmaf(v.w, weight[2 * c + 6], s0); s1 = fmaf(v.w, weight[2 * c + 7], s1);
    }
    const int b = m / HW, r = m - b * HW;
    conf[((size_t)b * 2 + 0) * HW + r] = sigmoidf_(s0);
    conf[((size_t)b * 2 + 1) * HW + r] = sigmoidf_(s1);
  }
}

// ---------------------------------------------------------------- nearest x2 of flow = coords1 - grid (raft_nc_dbl.py:110)
__global__ void flow_x2_kernel(const float* __restrict__ coords1, int B, int H8, int W8, float* __restrict__ x4) {
  const int H4 = 2 * H8, W4 = 2 * W8;
  const int n = B * 2 * H4 * W4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int x = i % W4, y = (i / W4) % H4, pl = i / (W4 * H4);
    const int ys = y >> 1, xs = x >> 1;
    x4[i] = coords1[((size_t)pl * H8 + ys) * W8 + xs] - ((pl & 1) == 0 ? (float)xs : (float)ys);
  }
}

// ---------------------------------------------------------------- weights-net input: cat(x_lowres, x2(net)) at 1/4 res
__global__ void ncup_guidance_kernel(const float* __restrict__ x_lowres, const float* __restrict__ net, int ldg, int C,
                                     int B, int H8, int W8, float* __restrict__ out, int ldo) {
  const int H4 = 2 * H8, W4 = 2 * W8;
  const size_t n = (size_t)B * H4 * W4 * ldo;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % ldo);
    size_t r = i / ldo;
    const int x = (int)(r % W4); r /= W4;
    const int y = (int)(r % H4);
    const int b = (int)(r / H4);
    float v = 0.f;
    if (c < 2) v = x_lowres[(((size_t)b * 2 + c) * H4 + y) * W4 + x];
    else if (c < 2 + C) v = net[(((size_t)b * H8 + (y >> 1)) * W8 + (x >> 1)) * ldg + (c - 2)];   // 'area' x2 == replicate
    out[i] = v;
  }
}

// Same staging, written directly as the hi/lo split halves planes the tensor-core weights net consumes (no fp32 round trip):
// thread = one pixel x 8 channels, one 16-byte store per plane.
__global__ void ncup_guidance_split_kernel(const float* __restrict__ x_lowres, const float* __restrict__ net, int ldg, int C,
                                           int B, int H8, int W8, __half* __restrict__ out_hi, __half* __restrict__ out_lo, int ldo) {
  const int H4 = 2 * H8, W4 = 2 * W8, groups = ldo >> 3;
  const long long n = static_cast<long long>(B) * H4 * W4 * groups;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    long long r = i / groups;
    const int x = static_cast<int>(r % W4); r /= W4;
    const int y = static_cast<int>(r % H4);
    const int b = static_cast<int>(r / H4);
    const float* np = net + ((static_cast<size_t>(b) * H8 + (y >> 1)) * W8 + (x >> 1)) * ldg;   // 'area' x2 == replicate
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = 8 * g + j;
      v[j] = c < 2 ? x_lowres[((static_cast<size_t>(b) * 2 + c) * H4 + y) * W4 + x] : c < 2 + C ? __ldg(np + c - 2) : 0.f;
    }
    uint32_t hh[4], ll[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split_pair(v[2 * j], v[2 * j + 1], hh[j], ll[j]);
    const size_t o = ((static_cast<size_t>(b) * H4 + y) * W4 + x) * ldo + 8 * g;
    *reinterpret_cast<uint4*>(out_hi + o) = make_uint4(hh[0], hh[1], hh[2], hh[3]);
    *reinterpret_cast<uint4*>(out_lo + o) = make_uint4(ll[0], ll[1], ll[2], ll[3]);
  }
}

// ---------------------------------------------------------------- fp32 CL -> exact hi/lo halves planes
__global__ void f32_to_split_kernel(const float* __restrict__ src, int lds, int C, long long M, __half* __restrict__ hi,
                                    __half* __restrict__ lo, int ldd, int ch_off) {
  const long long n = M * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / C;
    const int c = (int)(i - m * C);
    // the epilogues' split (split_pair): beyond 65504 lo carries the excess up to 131008, and a NaN stays a NaN
    uint32_t h, l;
    split_pair(src[m * lds + c], 0.f, h, l);
    hi[m * ldd + ch_off + c] = __ushort_as_half(static_cast<unsigned short>(h & 0xffffu));
    lo[m * ldd + ch_off + c] = __ushort_as_half(static_cast<unsigned short>(l & 0xffffu));
  }
}

// ---------------------------------------------------------------- fp32 CL -> TF32 hi/lo planes (training-path tensor-core layers)
__global__ void f32_to_tf32_split_kernel(const float* __restrict__ src, int lds, int C, long long M, float* __restrict__ hi,
                                         float* __restrict__ lo, int ldd, int ch_off) {
  const long long n = M * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / C;
    const int c = (int)(i - m * C);
    const float v = src[m * lds + c];
    uint32_t t;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(v));
    const float h = __uint_as_float(t);
    hi[m * ldd + ch_off + c] = h;
    lo[m * ldd + ch_off + c] = v - h;
  }
}

// ---------------------------------------------------------------- convex upsampling (raft.py:73-84)
__global__ void __launch_bounds__(256)
convex_upsample_kernel(const float* __restrict__ flow, const float* __restrict__ mask, int ldm, int B, int H8, int W8,
                       float* __restrict__ out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int HW = H8 * W8, M = B * HW;
  const int H = 8 * H8, W = 8 * W8;
  for (int m = blockIdx.x * nwarp + warp; m < M; m += gridDim.x * nwarp) {
    const int b = m / HW, r = m - b * HW, y = r / W8, x = r - y * W8;
    // 9 neighbours of 8*flow, zero outside (F.unfold padding=1)
    float fx[9], fy[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
      const bool ok = yy >= 0 && yy < H8 && xx >= 0 && xx < W8;
      fx[k] = ok ? 8.f * flow[((size_t)b * 2 + 0) * HW + yy * W8 + xx] : 0.f;
      fy[k] = ok ? 8.f * flow[((size_t)b * 2 + 1) * HW + yy * W8 + xx] : 0.f;
    }
    const float* mp = mask + (size_t)m * ldm;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int s = lane + 32 * half;   // sub-pixel sy*8+sx
      float l[9], mx = -INFINITY;
#pragma unroll
      for (int k = 0; k < 9; ++k) { l[k] = mp[k * 64 + s]; mx = fmaxf(mx, l[k]); }
      float den = 0.f, ax = 0.f, ay = 0.f;
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const float e = expf(l[k] - mx);
        den += e; ax = fmaf(e, fx[k], ax); ay = fmaf(e, fy[k], ay);
      }
      const int oy = 8 * y + (s >> 3), ox = 8 * x + (s & 7);
      out[(((size_t)b * 2 + 0) * H + oy) * W + ox] = ax / den;
      out[(((size_t)b * 2 + 1) * H + oy) * W + ox] = ay / den;
    }
  }
}

// FlowHead.conv2 as "1x1 conv per tap + shifted sum": P[q][2*tap + o] = W[o][:, tap] . in[q] was produced by a 1x1
// tensor-core convolution (K = cin instead of 9*cin for two real output channels); the 3x3 convolution with zero padding is
// out[o](y,x) = bias[o] + sum_tap P[(y+ky-1, x+kx-1)][2*tap + o] over the in-image neighbours.  Fused with
// `coords1 = coords1 + delta_flow` (raft_nc_dbl.py:157).
__global__ void flow_tap_gather_kernel(const float* __restrict__ P, int ldp, const float* __restrict__ bias, int B, int H, int W,
                                       float* __restrict__ coords1, float* __restrict__ delta) {
  pdl_trigger();
  const int HW = H * W;
  const long long M = static_cast<long long>(B) * HW;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < M; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / HW), r = static_cast<int>(i - static_cast<long long>(b) * HW);
    const int y = r / W, x = r - y * W;
    float d0 = bias[0], d1 = bias[1];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int yy = y + ky - 1;
      if (yy < 0 || yy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int xx = x + kx - 1;
        if (xx < 0 || xx >= W) continue;
        const float2 v = __ldg(reinterpret_cast<const float2*>(P + (static_cast<size_t>(b) * HW + yy * W + xx) * ldp + 2 * (ky * 3 + kx)));
        d0 += v.x; d1 += v.y;
      }
    }
    const size_t i0 = static_cast<size_t>(b) * 2 * HW + r;
    coords1[i0] += d0;
    coords1[i0 + HW] += d1;
    if (delta) { delta[i0] = d0; delta[i0 + HW] = d1; }
  }
}

// convf1 = Conv2d(2, 128, 7, padding=3) on flow = coords1 - grid (update.py:83,93-94), first half of the tensor-core
// formulation: the 7x7x2 neighbourhood of every pixel as one K-major row of 98 (+30 zero) split halves, k = 2*(7*ky+kx)+c,
// which a 1x1 tensor-core layer then multiplies by the [128][98] weight.  One thread = one pixel x 8 consecutive k.
__global__ void flow_im2col7_kernel(const float* __restrict__ coords1, int B, int H, int W, __half* __restrict__ out_hi,
                                    __half* __restrict__ out_lo, int ld) {
  pdl_trigger();
  const int HW = H * W;
  const long long total = static_cast<long long>(B) * HW * 16;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i & 15);
    const long long pix = i >> 4;
    const int b = static_cast<int>(pix / HW), r = static_cast<int>(pix - static_cast<long long>(b) * HW);
    const int y = r / W, x = r - y * W;
    const float* cx = coords1 + static_cast<size_t>(b) * 2 * HW;
    float v[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int tap = g * 4 + j;                 // 4 taps x 2 components per thread
      const int ky = tap / 7, kx = tap - ky * 7;
      const int yy = y + ky - 3, xx = x + kx - 3;
      const bool in = tap < 49 && yy >= 0 && yy < H && xx >= 0 && xx < W;
      v[2 * j] = in ? __ldg(cx + yy * W + xx) - static_cast<float>(xx) : 0.f;
      v[2 * j + 1] = in ? __ldg(cx + HW + yy * W + xx) - static_cast<float>(yy) : 0.f;
    }
    __half2 hh[4], ll[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = fminf(fmaxf(v[2 * j], -65504.f), 65504.f), c = fminf(fmaxf(v[2 * j + 1], -65504.f), 65504.f);
      hh[j] = __floats2half2_rn(a, c);
      const float2 back = __half22float2(hh[j]);
      ll[j] = __floats2half2_rn(a - back.x, c - back.y);
    }
    *reinterpret_cast<uint4*>(out_hi + pix * ld + g * 8) = *reinterpret_cast<uint4*>(hh);
    *reinterpret_cast<uint4*>(out_lo + pix * ld + g * 8) = *reinterpret_cast<uint4*>(ll);
  }
}

}  // namespace rnc

using namespace rnc;

extern "C" {

int rnc_conv_flow7x7_fwd(const float* coords1, const float* weight, const float* bias, int B, int H, int W,
                         int cout, float* out, int ldo, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || cout <= 0 || ldo < cout) return RNC_ERR_BAD_SHAPE;
  if (!coords1 || !weight || !bias || !out) return RNC_ERR_BAD_POINTER;
  dim3 grid((W + F7_PX - 1) / F7_PX, H, B);
  conv_flow7x7_kernel<<<grid, 128, 0, as_stream(stream)>>>(coords1, weight, bias, B, H, W, cout, out, ldo);
  return after_launch();
}

int rnc_flow_head2_fwd(const float* in, int cin, int ldi, const float* weight, const float* bias,
                       int B, int H, int W, float* delta, float* coords1, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || cin <= 0 || (cin & 3) || (ldi & 3) || ldi < cin || cin > 512) return RNC_ERR_BAD_SHAPE;
  if (!in || !weight || !bias || !coords1 || !aligned16(in) || !aligned16(weight)) return RNC_ERR_BAD_POINTER;
  const int M = B * H * W;
  int blocks = (M + 7) / 8;
  if (blocks > 132 * 4) blocks = 132 * 4;
  const size_t smem = (size_t)9 * cin * 2 * sizeof(float);
  flow_head2_kernel<<<blocks, 256, smem, as_stream(stream)>>>(in, cin, ldi, weight, bias, B, H, W, delta, coords1);
  return after_launch();
}

int rnc_flow_im2col7_split_fwd(const float* coords1, int B, int H, int W, void* out_hi, void* out_lo, int ld, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || ld < 128 || (ld & 7)) return RNC_ERR_BAD_SHAPE;
  if (!coords1 || !out_hi || !out_lo || !aligned16(out_hi) || !aligned16(out_lo)) return RNC_ERR_BAD_POINTER;
  const long long total = static_cast<long long>(B) * H * W * 16;
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  flow_im2col7_kernel<<<static_cast<int>(blocks), 256, 0, as_stream(stream)>>>(coords1, B, H, W, static_cast<__half*>(out_hi),
                                                                              static_cast<__half*>(out_lo), ld);
  return after_launch();
}

int rnc_flow_tap_gather_fwd(const float* taps, int ldt, const float* bias, int B, int H, int W, float* delta, float* coords1,
                            void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || ldt < 18 || (ldt & 1)) return RNC_ERR_BAD_SHAPE;
  if (!taps || !bias || !coords1 || (reinterpret_cast<uintptr_t>(taps) & 7)) return RNC_ERR_BAD_POINTER;
  const long long M = static_cast<long long>(B) * H * W;
  long long blocks = (M + 127) / 128;
  if (blocks > 132 * 16) blocks = 132 * 16;
  flow_tap_gather_kernel<<<static_cast<int>(blocks), 128, 0, as_stream(stream)>>>(taps, ldt, bias, B, H, W, coords1, delta);
  return after_launch();
}

int rnc_conf_head_fwd(const float* in, int cin, int ldi, const float* weight, const float* bias,
                      int B, int H4, int W4, float* conf, void* stream) {
  if (B <= 0 || H4 <= 0 || W4 <= 0 || cin <= 0 || (cin & 3) || (ldi & 3) || ldi < cin) return RNC_ERR_BAD_SHAPE;
  if (!in || !weight || !bias || !conf || !aligned16(in)) return RNC_ERR_BAD_POINTER;
  const int M = B * H4 * W4;
  int blocks = (M + 255) / 256;
  conf_head_kernel<<<blocks, 256, 0, as_stream(stream)>>>(in, cin, ldi, weight, bias, B, H4 * W4, conf);
  return after_launch();
}

int rnc_f32_to_split(const float* src, int lds, int C, long long M, void* dst_hi, void* dst_lo, int ldd, int ch_off,
                     void* stream) {
  if (C <= 0 || M <= 0 || lds < C || ldd < C + ch_off || ch_off < 0) return RNC_ERR_BAD_SHAPE;
  if (!src || !dst_hi || !dst_lo) return RNC_ERR_BAD_POINTER;
  long long blocks = (M * C + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  f32_to_split_kernel<<<(int)blocks, 256, 0, as_stream(stream)>>>(src, lds, C, M, static_cast<__half*>(dst_hi),
                                                                 static_cast<__half*>(dst_lo), ldd, ch_off);
  return after_launch();
}

int rnc_f32_to_tf32_split(const float* src, int lds, int C, long long M, float* dst_hi, float* dst_lo, int ldd, int ch_off,
                          void* stream) {
  if (C <= 0 || M <= 0 || lds < C || ldd < C + ch_off || ch_off < 0) return RNC_ERR_BAD_SHAPE;
  if (!src || !dst_hi || !dst_lo) return RNC_ERR_BAD_POINTER;
  long long blocks = (M * C + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  f32_to_tf32_split_kernel<<<(int)blocks, 256, 0, as_stream(stream)>>>(src, lds, C, M, dst_hi, dst_lo, ldd, ch_off);
  return after_launch();
}

int rnc_flow_x2_fwd(const float* coords1, int B, int H8, int W8, float* x4, void* stream) {
  if (B <= 0 || H8 <= 0 || W8 <= 0) return RNC_ERR_BAD_SHAPE;
  if (!coords1 || !x4) return RNC_ERR_BAD_POINTER;
  const int n = B * 2 * 4 * H8 * W8;
  flow_x2_kernel<<<(n + 255) / 256, 256, 0, as_stream(stream)>>>(coords1, B, H8, W8, x4);
  return after_launch();
}

int rnc_ncup_guidance_fwd(const float* x_lowres, const float* net, int ldg, int C, int B, int H8, int W8,
                          float* out, int ldo, void* stream) {
  if (B <= 0 || H8 <= 0 || W8 <= 0 || C <= 0 || ldg < C || ldo < C + 2) return RNC_ERR_BAD_SHAPE;
  if (!x_lowres || !net || !out) return RNC_ERR_BAD_POINTER;
  const size_t n = (size_t)B * 4 * H8 * W8 * ldo;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 32) blocks = 132 * 32;
  ncup_guidance_kernel<<<blocks, 256, 0, as_stream(stream)>>>(x_lowres, net, ldg, C, B, H8, W8, out, ldo);
  return after_launch();
}

int rnc_ncup_guidance_split_fwd(const float* x_lowres, const float* net, int ldg, int C, int B, int H8, int W8,
                                void* out_hi, void* out_lo, int ldo, void* stream) {
  if (B <= 0 || H8 <= 0 || W8 <= 0 || C <= 0 || ldg < C || ldo < C + 2 || (ldo & 7)) return RNC_ERR_BAD_SHAPE;
  if (!x_lowres || !net || !out_hi || !out_lo || !aligned16(out_hi) || !aligned16(out_lo)) return RNC_ERR_BAD_POINTER;
  const long long n = static_cast<long long>(B) * 4 * H8 * W8 * (ldo >> 3);
  long long blocks = (n + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  ncup_guidance_split_kernel<<<static_cast<int>(blocks), 256, 0, as_stream(stream)>>>(
      x_lowres, net, ldg, C, B, H8, W8, static_cast<__half*>(out_hi), static_cast<__half*>(out_lo), ldo);
  return after_launch();
}

int rnc_convex_upsample_fwd(const float* flow, const float* mask, int ldm, int B, int H8, int W8,
                            float* out, void* stream) {
  if (B <= 0 || H8 <= 0 || W8 <= 0 || ldm < 576) return RNC_ERR_BAD_SHAPE;
  if (!flow || !mask || !out) return RNC_ERR_BAD_POINTER;
  const int M = B * H8 * W8;
  int blocks = (M + 7) / 8;
  if (blocks > 132 * 8) blocks = 132 * 8;
  convex_upsample_kernel<<<blocks, 256, 0, as_stream(stream)>>>(flow, mask, ldm, B, H8, W8, out);
  return after_launch();
}

}  // extern "C"
