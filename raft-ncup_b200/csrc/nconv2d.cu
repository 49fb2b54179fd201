// One normalized-convolution layer, forward and backward: the operator seam NConv2d.forward
// (core/nconv_modules.py:164-199) and the per-layer form the training path differentiates through.
//
//   den[o] = conv(conf, W)[o]          num[o] = conv(data * conf, W)[o]        (zero padding k/2, stride 1)
//   y[o]   = num[o] / (den[o] + eps)   conf_out[o] = den[o] / sum_{i,ky,kx} W[o,i,ky,kx]
//
// W is the already-positive kernel (softplus_{beta=10}(weight_p), nconv_modules.py:250-264, applied by the caller);
// bias is not supported (no reference script enables it).  NCHW fp32 tensors, thin channel counts (<= 4): thread = pixel,
// weights in shared memory.  The inference path does not use this file: it runs the fused chain of ncup.cu.
//
// Backward (quotient rule; SURVEY.md Appendix G).  With D = den + eps, s_o = sum W[o]:
//   a_o = dL/dnum_o = gy_o / D_o          b_o = dL/dden_o = -gy_o * y_o / D_o + gc_o / s_o
//   A_i(q) = sum_{o,t} a_o(q - t) W[o,i,t]     B_i(q) = sum_{o,t} b_o(q - t) W[o,i,t]
//   g_data_i = A_i * conf_i                     g_conf_i = A_i * data_i + B_i
//   g_W[o,i,t] = sum_p a_o(p) (data*conf)_i(p+t) + b_o(p) conf_i(p+t)  -  (1/s_o^2) sum_p gc_o(p) den_o(p)
#include "rnc_common.cuh"

namespace rnc {
namespace nconv {

constexpr int kMaxC = 4;      // channels in / out
constexpr int kMaxK = 7;      // kernel side

__global__ void __launch_bounds__(256)
nconv2d_fwd_kernel(const float* __restrict__ data, const float* __restrict__ conf, const float* __restrict__ weight,
                   int N, int Cin, int Cout, int H, int W, int kh, int kw, float eps,
                   float* __restrict__ y, float* __restrict__ conf_out) {
  __shared__ float wsm[kMaxC * kMaxC * kMaxK * kMaxK];
  __shared__ float inv_s[kMaxC];
  const int nw = Cout * Cin * kh * kw;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) wsm[i] = weight[i];
  __syncthreads();
  if (threadIdx.x < Cout) {
    float s = 0.f;
    for (int i = 0; i < Cin * kh * kw; ++i) s += wsm[threadIdx.x * Cin * kh * kw + i];
    inv_s[threadIdx.x] = 1.0f / s;
  }
  __syncthreads();
  const int HW = H * W, ph = kh / 2, pw = kw / 2;
  const long long total = static_cast<long long>(N) * HW;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(idx / HW), r = static_cast<int>(idx - static_cast<long long>(n) * HW);
    const int py = r / W, px = r - py * W;
    float num[kMaxC], den[kMaxC];
#pragma unroll
    for (int o = 0; o < kMaxC; ++o) num[o] = den[o] = 0.f;
    for (int i = 0; i < Cin; ++i) {
      const float* dp = data + (static_cast<size_t>(n) * Cin + i) * HW;
      const float* cp = conf + (static_cast<size_t>(n) * Cin + i) * HW;
      for (int ky = 0; ky < kh; ++ky) {
        const int yy = py + ky - ph;
        if (yy < 0 || yy >= H) continue;
        for (int kx = 0; kx < kw; ++kx) {
          const int xx = px + kx - pw;
          if (xx < 0 || xx >= W) continue;
          const float c = __ldg(cp + yy * W + xx), xc = __ldg(dp + yy * W + xx) * c;
#pragma unroll
          for (int o = 0; o < kMaxC; ++o)
            if (o < Cout) {
              const float w = wsm[((o * Cin + i) * kh + ky) * kw + kx];
              den[o] = fmaf(c, w, den[o]);
              num[o] = fmaf(xc, w, num[o]);
            }
        }
      }
    }
#pragma unroll
    for (int o = 0; o < kMaxC; ++o)
      if (o < Cout) {
        const size_t oi = (static_cast<size_t>(n) * Cout + o) * HW + r;
        y[oi] = num[o] / (den[o] + eps);
        conf_out[oi] = den[o] * inv_s[o];
      }
  }
}

// a, b planes of the backward (see the header comment); also accumulates sum_p gc_o(p) * den_o(p) per output channel.
__global__ void __launch_bounds__(256)
nconv2d_bwd_ab_kernel(const float* __restrict__ y, const float* __restrict__ conf_out, const float* __restrict__ gy,
                      const float* __restrict__ gc, const float* __restrict__ weight, int N, int Cin, int Cout, int HW,
                      int ktaps, float eps, float* __restrict__ a, float* __restrict__ b, double* __restrict__ gs) {
  __shared__ float s_sum[kMaxC];
  if (threadIdx.x < Cout) {
    float s = 0.f;
    for (int i = 0; i < Cin * ktaps; ++i) s += weight[threadIdx.x * Cin * ktaps + i];
    s_sum[threadIdx.x] = s;
  }
  __syncthreads();
  const long long total = static_cast<long long>(N) * Cout * HW;
  double local[kMaxC] = {0.0, 0.0, 0.0, 0.0};
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int o = static_cast<int>((idx / HW) % Cout);
    const float s = s_sum[o];
    const float den = conf_out[idx] * s, D = den + eps;
    const float g = gy ? gy[idx] : 0.f, gcv = gc ? gc[idx] : 0.f;
    a[idx] = g / D;
    b[idx] = -g * y[idx] / D + gcv / s;
#pragma unroll
    for (int k = 0; k < kMaxC; ++k)
      if (k == o) local[k] += static_cast<double>(gcv) * den;
  }
  if (gs != nullptr) {
#pragma unroll
    for (int k = 0; k < kMaxC; ++k) {
      double v = local[k];
      for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if ((threadIdx.x & 31) == 0 && k < Cout && v != 0.0) atomicAdd(gs + k, v);
    }
  }
}

__global__ void __launch_bounds__(256)
nconv2d_bwd_data_kernel(const float* __restrict__ data, const float* __restrict__ conf, const float* __restrict__ a,
                        const float* __restrict__ b, const float* __restrict__ weight, int N, int Cin, int Cout, int H, int W,
                        int kh, int kw, float* __restrict__ g_data, float* __restrict__ g_conf) {
  __shared__ float wsm[kMaxC * kMaxC * kMaxK * kMaxK];
  const int nw = Cout * Cin * kh * kw;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) wsm[i] = weight[i];
  __syncthreads();
  const int HW = H * W, ph = kh / 2, pw = kw / 2;
  const long long total = static_cast<long long>(N) * HW;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(idx / HW), r = static_cast<int>(idx - static_cast<long long>(n) * HW);
    const int qy = r / W, qx = r - qy * W;
    float A[kMaxC], Bv[kMaxC];
#pragma unroll
    for (int i = 0; i < kMaxC; ++i) A[i] = Bv[i] = 0.f;
    for (int o = 0; o < Cout; ++o) {
      const float* ap = a + (static_cast<size_t>(n) * Cout + o) * HW;
      const float* bp = b + (static_cast<size_t>(n) * Cout + o) * HW;
      for (int ky = 0; ky < kh; ++ky) {
        const int yy = qy - (ky - ph);            // output pixel p = q - t
        if (yy < 0 || yy >= H) continue;
        for (int kx = 0; kx < kw; ++kx) {
          const int xx = qx - (kx - pw);
          if (xx < 0 || xx >= W) continue;
          const float av = __ldg(ap + yy * W + xx), bv = __ldg(bp + yy * W + xx);
#pragma unroll
          for (int i = 0; i < kMaxC; ++i)
            if (i < Cin) {
              const float w = wsm[((o * Cin + i) * kh + ky) * kw + kx];
              A[i] = fmaf(av, w, A[i]);
              Bv[i] = fmaf(bv, w, Bv[i]);
            }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < kMaxC; ++i)
      if (i < Cin) {
        const size_t ii = (static_cast<size_t>(n) * Cin + i) * HW + r;
        if (g_data) g_data[ii] = A[i] * conf[ii];
        if (g_conf) g_conf[ii] = fmaf(A[i], data[ii], Bv[i]);
      }
  }
}

// g_W: blockIdx.y = (i, ky); every thread keeps [kw][Cout] partial sums over its pixels, reduced in fp64.
__global__ void __launch_bounds__(256)
nconv2d_bwd_weight_kernel(const float* __restrict__ data, const float* __restrict__ conf, const float* __restrict__ a,
                          const float* __restrict__ b, int N, int Cin, int Cout, int H, int W, int kh, int kw,
                          double* __restrict__ gw) {
  const int i = blockIdx.y / kh, ky = blockIdx.y - i * kh;
  const int HW = H * W, ph = kh / 2, pw = kw / 2;
  float acc[kMaxK][kMaxC];
#pragma unroll
  for (int kx = 0; kx < kMaxK; ++kx)
#pragma unroll
    for (int o = 0; o < kMaxC; ++o) acc[kx][o] = 0.f;
  const long long total = static_cast<long long>(N) * HW;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(idx / HW), r = static_cast<int>(idx - static_cast<long long>(n) * HW);
    const int py = r / W, px = r - py * W;
    const int yy = py + ky - ph;
    if (yy < 0 || yy >= H) continue;
    float av[kMaxC], bv[kMaxC];
#pragma unroll
    for (int o = 0; o < kMaxC; ++o) {
      av[o] = o < Cout ? a[(static_cast<size_t>(n) * Cout + o) * HW + r] : 0.f;
      bv[o] = o < Cout ? b[(static_cast<size_t>(n) * Cout + o) * HW + r] : 0.f;
    }
    const float* dp = data + (static_cast<size_t>(n) * Cin + i) * HW + yy * W;
    const float* cp = conf + (static_cast<size_t>(n) * Cin + i) * HW + yy * W;
#pragma unroll
    for (int kx = 0; kx < kMaxK; ++kx) {
      const int xx = px + kx - pw;
      if (kx < kw && xx >= 0 && xx < W) {
        const float c = __ldg(cp + xx), xc = __ldg(dp + xx) * c;
#pragma unroll
        for (int o = 0; o < kMaxC; ++o) acc[kx][o] = fmaf(av[o], xc, fmaf(bv[o], c, acc[kx][o]));
      }
    }
  }
#pragma unroll
  for (int kx = 0; kx < kMaxK; ++kx)
#pragma unroll
    for (int o = 0; o < kMaxC; ++o) {
      if (kx >= kw || o >= Cout) continue;       // uniform
      double v = acc[kx][o];
      for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if ((threadIdx.x & 31) == 0) atomicAdd(gw + ((o * Cin + i) * kh + ky) * kw + kx, v);
    }
}

// g_W (fp32) = gw (fp64 sums) - gs[o] / s_o^2; then the fp64 scratch is zeroed for the next call.
__global__ void nconv2d_bwd_weight_finish_kernel(double* __restrict__ gw, double* __restrict__ gs, const float* __restrict__ weight,
                                                 int Cin, int Cout, int ktaps, float* __restrict__ g_weight) {
  __shared__ double corr[kMaxC];
  if (threadIdx.x < Cout) {
    double s = 0.0;
    for (int i = 0; i < Cin * ktaps; ++i) s += weight[threadIdx.x * Cin * ktaps + i];
    corr[threadIdx.x] = gs[threadIdx.x] / (s * s);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < Cout * Cin * ktaps; k += blockDim.x) {
    g_weight[k] = static_cast<float>(gw[k] - corr[k / (Cin * ktaps)]);
    gw[k] = 0.0;
  }
  __syncthreads();
  if (threadIdx.x < kMaxC) gs[threadIdx.x] = 0.0;
}

inline int grid_for(long long total) {
  long long g = (total + 255) / 256;
  if (g > 132 * 8) g = 132 * 8;
  return static_cast<int>(g < 1 ? 1 : g);
}

inline int check_shape(int N, int Cin, int Cout, int H, int W, int kh, int kw) {
  if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return RNC_ERR_BAD_SHAPE;
  if (Cin > kMaxC || Cout > kMaxC || kh > kMaxK || kw > kMaxK || kh < 1 || kw < 1 || !(kh & 1) || !(kw & 1)) return RNC_ERR_UNSUPPORTED;
  return RNC_OK;
}

}  // namespace nconv
}  // namespace rnc

using namespace rnc;

extern "C" int rnc_nconv2d_fwd(const float* data, const float* conf, const float* weight, int N, int Cin, int Cout, int H, int W,
                               int kh, int kw, float eps, float* y, float* conf_out, void* stream) {
  if (int st = nconv::check_shape(N, Cin, Cout, H, W, kh, kw)) return st;
  if (!data || !conf || !weight || !y || !conf_out) return RNC_ERR_BAD_POINTER;
  nconv::nconv2d_fwd_kernel<<<nconv::grid_for(static_cast<long long>(N) * H * W), 256, 0, as_stream(stream)>>>(
      data, conf, weight, N, Cin, Cout, H, W, kh, kw, eps, y, conf_out);
  return after_launch();
}

extern "C" size_t rnc_nconv2d_bwd_workspace_bytes(int N, int Cout, int H, int W) {
  // a, b planes + fp64 scratch for the weight gradient (Cout*Cin*kh*kw <= 4*4*49) and the sum(W) term
  return 2 * sizeof(float) * static_cast<size_t>(N) * Cout * H * W + sizeof(double) * (4 * 4 * 49 + 8);
}

extern "C" int rnc_nconv2d_bwd(const float* data, const float* conf, const float* weight, const float* y, const float* conf_out,
                               const float* g_y, const float* g_conf_out, int N, int Cin, int Cout, int H, int W, int kh, int kw,
                               float eps, float* g_data, float* g_conf, float* g_weight, void* workspace, size_t workspace_bytes,
                               void* stream) {
  if (int st = nconv::check_shape(N, Cin, Cout, H, W, kh, kw)) return st;
  if (!data || !conf || !weight || !y || !conf_out || !workspace || (!g_y && !g_conf_out)) return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_nconv2d_bwd_workspace_bytes(N, Cout, H, W) || !aligned16(workspace)) return RNC_ERR_WORKSPACE;
  const size_t plane = static_cast<size_t>(N) * Cout * H * W;
  // fp64 scratch first (keeps it 16-byte aligned); it must be zero on entry: the finish kernel re-zeroes it, and the very
  // first use zeroes it here (the caller hands over a zero-initialised workspace: torch.zeros)
  double* gw = static_cast<double*>(workspace);
  double* gs = gw + 4 * 4 * 49;
  float* a = reinterpret_cast<float*>(gs + 8);
  float* b = a + plane;
  cudaStream_t s = as_stream(stream);
  const int ktaps = kh * kw;
  nconv::nconv2d_bwd_ab_kernel<<<nconv::grid_for(static_cast<long long>(plane)), 256, 0, s>>>(
      y, conf_out, g_y, g_conf_out, weight, N, Cin, Cout, H * W, ktaps, eps, a, b, g_weight ? gs : nullptr);
  int launches = 1;
  if (g_data || g_conf) {
    nconv::nconv2d_bwd_data_kernel<<<nconv::grid_for(static_cast<long long>(N) * H * W), 256, 0, s>>>(
        data, conf, a, b, weight, N, Cin, Cout, H, W, kh, kw, g_data, g_conf);
    ++launches;
  }
  if (g_weight) {
    dim3 grid(nconv::grid_for(static_cast<long long>(N) * H * W / 8), Cin * kh);
    nconv::nconv2d_bwd_weight_kernel<<<grid, 256, 0, s>>>(data, conf, a, b, N, Cin, Cout, H, W, kh, kw, gw);
    nconv::nconv2d_bwd_weight_finish_kernel<<<1, 256, 0, s>>>(gw, gs, weight, Cin, Cout, ktaps, g_weight);
    launches += 2;
  }
  return after_launch(launches);
}
