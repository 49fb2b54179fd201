// Normalized-convolution layers, forward and backward: the operator seam NConv2d.forward (core/nconv_modules.py:164-199),
// the per-layer form the training path differentiates through, and the per-level chain that runs every NConvUNet
// configuration other than the shipped one (whose fused chain is ncup.cu).
//
//   den[o] = conv(conf, W)[o]          num[o] = conv(data * conf, W)[o]        (zero padding k/2, stride 1)
//   y[o]   = (num[o] / (den[o] + eps) + bias[o]) * y_scale      conf_out[o] = den[o] / sum_{i,ky,kx} W[o,i,ky,kx]
//
// W is the already-positive kernel (softplus_{beta=10}(weight_p), nconv_modules.py:250-264, applied by the caller).  The
// input is the channel concatenation of an optional "up" source [N][Cup][Hup][Wup], read at full resolution through
// PyTorch's nearest-neighbour index map (F.interpolate(mode='nearest'), the decoder's upsample, nconv_modules.py:129-131),
// and the full-resolution source [N][Cin][H][W].  NCHW fp32 tensors, thin channel counts (Cup + Cin <= 8, Cout <= 4):
// thread = pixel, weights in shared memory.
//
// Backward (quotient rule; SURVEY.md Appendix G).  With D = den + eps, s_o = sum W[o], yq = y - bias (the quotient):
//   a_o = dL/dnum_o = gy_o / D_o          b_o = dL/dden_o = -gy_o * yq_o / D_o + gc_o / s_o
//   A_i(q) = sum_{o,t} a_o(q - t) W[o,i,t]     B_i(q) = sum_{o,t} b_o(q - t) W[o,i,t]
//   g_data_i = A_i * conf_i                     g_conf_i = A_i * data_i + B_i
//   g_W[o,i,t] = sum_p a_o(p) (data*conf)_i(p+t) + b_o(p) conf_i(p+t)  -  (1/s_o^2) sum_p gc_o(p) den_o(p)
//   g_bias[o] = sum_p gy_o(p)
// Up-source channels sum A_i, B_i over the full-resolution pixels that map to each coarse pixel, in row-major order.
// Every reduction runs in a fixed order (per-block fp64 partials, summed block by block), so gradients are bit-identical
// from call to call.
//
// Pooling (NConvUNet.downsample_data_conf, nconv_modules.py:94-104): 2x2/2 max-pool of the confidence (floor mode, first
// maximum in row-major window order as F.max_pool2d), divided by 4; the data is gathered at the confidence argmax
// (conf_based) or max-pooled on its own (max_pooling).  The backward routes each gradient to its argmax; windows do not
// overlap, so every input pixel is written by one thread.
#include "rnc_common.cuh"

namespace rnc {
namespace nconv {

constexpr int kMaxCout = 4;   // channels out
constexpr int kMaxCin = 8;    // channels in (up + full resolution)
constexpr int kMaxK = 7;      // kernel side
constexpr int kThreads = 256;

// F.interpolate(mode='nearest', size=out) source index: min(floor(dst * (in / out)), in - 1) with a float scale.
__device__ __forceinline__ int nearest_src(int dst, float scale, int in) {
  return min(static_cast<int>(floorf(static_cast<float>(dst) * scale)), in - 1);
}

// Input channel i of the virtual concatenation [up (Cup channels, read through the index map), full-resolution (Cin)].
struct Src {
  const float* data; const float* conf; int Cin;
  const float* up_data; const float* up_conf; int Cup, Hup, Wup;
  float sy, sx;   // Hup / H, Wup / W
  int H, W;
  __device__ __forceinline__ const float* dptr(int i) const { return i < Cup ? up_data : data; }
  __device__ __forceinline__ const float* cptr(int i) const { return i < Cup ? up_conf : conf; }
};

// Fixed-order block sum of per-thread fp64 values (one per output channel) -> part[kMaxCout].
__device__ __forceinline__ void block_sum(double (&v)[kMaxCout], double* part) {
  __shared__ double red[kThreads / 32][kMaxCout];
#pragma unroll
  for (int k = 0; k < kMaxCout; ++k) {
    double x = v[k];
    for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = x;
  }
  __syncthreads();
  if (threadIdx.x < kMaxCout) {
    double s = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) s += red[w][threadIdx.x];
    part[threadIdx.x] = s;
  }
}

__global__ void __launch_bounds__(kThreads)
nconv2d_fwd_kernel(Src src, const float* __restrict__ weight, const float* __restrict__ bias, int N, int Cout, int kh,
                   int kw, float eps, float y_scale, float* __restrict__ y, float* __restrict__ conf_out) {
  __shared__ float wsm[kMaxCout * kMaxCin * kMaxK * kMaxK];
  __shared__ float inv_s[kMaxCout];
  const int Cin = src.Cup + src.Cin, H = src.H, W = src.W;
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
    float num[kMaxCout], den[kMaxCout];
#pragma unroll
    for (int o = 0; o < kMaxCout; ++o) num[o] = den[o] = 0.f;
    for (int i = 0; i < Cin; ++i) {
      const bool up = i < src.Cup;
      const int Hs = up ? src.Hup : H, Ws = up ? src.Wup : W;
      const size_t plane = up ? (static_cast<size_t>(n) * src.Cup + i) * Hs * Ws
                              : (static_cast<size_t>(n) * src.Cin + (i - src.Cup)) * HW;
      const float* dp = (up ? src.up_data : src.data) + plane;
      const float* cp = (up ? src.up_conf : src.conf) + plane;
      for (int ky = 0; ky < kh; ++ky) {
        const int yy = py + ky - ph;
        if (yy < 0 || yy >= H) continue;
        const int ys = up ? nearest_src(yy, src.sy, Hs) : yy;
        for (int kx = 0; kx < kw; ++kx) {
          const int xx = px + kx - pw;
          if (xx < 0 || xx >= W) continue;
          const int p = ys * Ws + (up ? nearest_src(xx, src.sx, Ws) : xx);
          const float c = __ldg(cp + p), xc = __ldg(dp + p) * c;
#pragma unroll
          for (int o = 0; o < kMaxCout; ++o)
            if (o < Cout) {
              const float w = wsm[((o * Cin + i) * kh + ky) * kw + kx];
              den[o] = fmaf(c, w, den[o]);
              num[o] = fmaf(xc, w, num[o]);
            }
        }
      }
    }
#pragma unroll
    for (int o = 0; o < kMaxCout; ++o)
      if (o < Cout) {
        const size_t oi = (static_cast<size_t>(n) * Cout + o) * HW + r;
        float v = num[o] / (den[o] + eps);
        if (bias) v += bias[o];
        y[oi] = v * y_scale;
        conf_out[oi] = den[o] * inv_s[o];
      }
  }
}

// a, b planes of the backward (see the header comment), and per-block partial sums of gc_o * den_o and gy_o.
__global__ void __launch_bounds__(kThreads)
nconv2d_bwd_ab_kernel(const float* __restrict__ y, const float* __restrict__ conf_out, const float* __restrict__ gy,
                      const float* __restrict__ gc, const float* __restrict__ weight, const float* __restrict__ bias, int N,
                      int Cin, int Cout, int HW, int ktaps, float eps, float* __restrict__ a, float* __restrict__ b,
                      double* __restrict__ gs_part, double* __restrict__ gb_part) {
  __shared__ float s_sum[kMaxCout];
  if (threadIdx.x < Cout) {
    float s = 0.f;
    for (int i = 0; i < Cin * ktaps; ++i) s += weight[threadIdx.x * Cin * ktaps + i];
    s_sum[threadIdx.x] = s;
  }
  __syncthreads();
  const long long total = static_cast<long long>(N) * Cout * HW;
  double lgs[kMaxCout] = {0.0, 0.0, 0.0, 0.0}, lgb[kMaxCout] = {0.0, 0.0, 0.0, 0.0};
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int o = static_cast<int>((idx / HW) % Cout);
    const float s = s_sum[o];
    const float den = conf_out[idx] * s, D = den + eps;
    const float g = gy ? gy[idx] : 0.f, gcv = gc ? gc[idx] : 0.f;
    const float yq = bias ? y[idx] - bias[o] : y[idx];
    a[idx] = g / D;
    b[idx] = -g * yq / D + gcv / s;
#pragma unroll
    for (int k = 0; k < kMaxCout; ++k)
      if (k == o) {
        lgs[k] += static_cast<double>(gcv) * den;
        lgb[k] += g;
      }
  }
  if (gs_part != nullptr) {
    block_sum(lgs, gs_part + blockIdx.x * kMaxCout);
    __syncthreads();
    block_sum(lgb, gb_part + blockIdx.x * kMaxCout);
  }
}

// A, B of every input channel at every full-resolution pixel q.  Full-resolution channels get their data / confidence
// gradients here; up-source channels leave A, B in the scratch planes ab_up [2][N][Cup][H][W] for the gather kernel.
template <int MAXC>
__global__ void __launch_bounds__(kThreads)
nconv2d_bwd_data_kernel(Src src, const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ weight,
                        int N, int Cout, int kh, int kw, float* __restrict__ g_data, float* __restrict__ g_conf,
                        float* __restrict__ ab_up) {
  __shared__ float wsm[kMaxCout * kMaxCin * kMaxK * kMaxK];
  const int Cin = src.Cup + src.Cin, H = src.H, W = src.W;
  const int nw = Cout * Cin * kh * kw;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) wsm[i] = weight[i];
  __syncthreads();
  const int HW = H * W, ph = kh / 2, pw = kw / 2;
  const long long total = static_cast<long long>(N) * HW;
  const size_t up_plane = static_cast<size_t>(N) * src.Cup * HW;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(idx / HW), r = static_cast<int>(idx - static_cast<long long>(n) * HW);
    const int qy = r / W, qx = r - qy * W;
    float A[MAXC], Bv[MAXC];
#pragma unroll
    for (int i = 0; i < MAXC; ++i) A[i] = Bv[i] = 0.f;
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
          for (int i = 0; i < MAXC; ++i)
            if (i < Cin) {
              const float w = wsm[((o * Cin + i) * kh + ky) * kw + kx];
              A[i] = fmaf(av, w, A[i]);
              Bv[i] = fmaf(bv, w, Bv[i]);
            }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < MAXC; ++i) {
      if (i >= Cin) continue;
      if (i < src.Cup) {
        const size_t ui = (static_cast<size_t>(n) * src.Cup + i) * HW + r;
        ab_up[ui] = A[i];
        ab_up[up_plane + ui] = Bv[i];
        continue;
      }
      const size_t ii = (static_cast<size_t>(n) * src.Cin + (i - src.Cup)) * HW + r;
      if (g_data) g_data[ii] = A[i] * src.conf[ii];
      if (g_conf) g_conf[ii] = fmaf(A[i], src.data[ii], Bv[i]);
    }
  }
}

// Up-source gradients: each coarse pixel sums its full-resolution preimage (rows, then columns, ascending).
__global__ void __launch_bounds__(kThreads)
nconv2d_bwd_up_kernel(Src src, const float* __restrict__ ab_up, int N, float* __restrict__ g_up_data,
                      float* __restrict__ g_up_conf) {
  const int H = src.H, W = src.W, Hup = src.Hup, Wup = src.Wup, HW = H * W;
  const long long total = static_cast<long long>(N) * src.Cup * Hup * Wup;
  const size_t up_plane = static_cast<size_t>(N) * src.Cup * HW;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(idx % Wup), yc = static_cast<int>((idx / Wup) % Hup);
    const long long nc = idx / (static_cast<long long>(Hup) * Wup);
    const float d = src.up_data[idx], c = src.up_conf[idx];
    // the index map is non-decreasing: start a little before the proportional position and scan forward
    int y0 = max(0, static_cast<int>(static_cast<long long>(yc) * H / Hup) - 2);
    while (y0 < H && nearest_src(y0, src.sy, Hup) < yc) ++y0;
    int x0 = max(0, static_cast<int>(static_cast<long long>(x) * W / Wup) - 2);
    while (x0 < W && nearest_src(x0, src.sx, Wup) < x) ++x0;
    float gd = 0.f, gcf = 0.f;
    for (int yy = y0; yy < H && nearest_src(yy, src.sy, Hup) == yc; ++yy)
      for (int xx = x0; xx < W && nearest_src(xx, src.sx, Wup) == x; ++xx) {
        const size_t q = static_cast<size_t>(nc) * HW + static_cast<size_t>(yy) * W + xx;
        const float A = ab_up[q], B = ab_up[up_plane + q];
        gd += A * c;
        gcf += fmaf(A, d, B);
      }
    if (g_up_data) g_up_data[idx] = gd;
    if (g_up_conf) g_up_conf[idx] = gcf;
  }
}

// g_W partials: blockIdx.y = (i, ky); every thread keeps [kw][Cout] partial sums over its pixels; one fp64 partial per
// block and weight, summed in block order by the finish kernel.
__global__ void __launch_bounds__(kThreads)
nconv2d_bwd_weight_kernel(Src src, const float* __restrict__ a, const float* __restrict__ b, int N, int Cout, int kh, int kw,
                          double* __restrict__ gw_part) {
  __shared__ double red[kThreads / 32][kMaxK * kMaxCout];
  const int i = blockIdx.y / kh, ky = blockIdx.y - i * kh;
  const int H = src.H, W = src.W, HW = H * W, ph = kh / 2, pw = kw / 2;
  const float* dsrc = src.dptr(i);
  const float* csrc = src.cptr(i);
  float acc[kMaxK][kMaxCout];
#pragma unroll
  for (int kx = 0; kx < kMaxK; ++kx)
#pragma unroll
    for (int o = 0; o < kMaxCout; ++o) acc[kx][o] = 0.f;
  const long long total = static_cast<long long>(N) * HW;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(idx / HW), r = static_cast<int>(idx - static_cast<long long>(n) * HW);
    const int py = r / W, px = r - py * W;
    const int yy = py + ky - ph;
    if (yy < 0 || yy >= H) continue;
    float av[kMaxCout], bv[kMaxCout];
#pragma unroll
    for (int o = 0; o < kMaxCout; ++o) {
      av[o] = o < Cout ? a[(static_cast<size_t>(n) * Cout + o) * HW + r] : 0.f;
      bv[o] = o < Cout ? b[(static_cast<size_t>(n) * Cout + o) * HW + r] : 0.f;
    }
    const bool up = i < src.Cup;
    const int Ws = up ? src.Wup : W;
    const size_t row = up ? ((static_cast<size_t>(n) * src.Cup + i) * src.Hup + nearest_src(yy, src.sy, src.Hup)) * Ws
                          : ((static_cast<size_t>(n) * src.Cin + (i - src.Cup)) * H + yy) * W;
#pragma unroll
    for (int kx = 0; kx < kMaxK; ++kx) {
      const int xx = px + kx - pw;
      if (kx < kw && xx >= 0 && xx < W) {
        const size_t off = row + (up ? nearest_src(xx, src.sx, Ws) : xx);
        const float c = __ldg(csrc + off), xc = __ldg(dsrc + off) * c;
#pragma unroll
        for (int o = 0; o < kMaxCout; ++o) acc[kx][o] = fmaf(av[o], xc, fmaf(bv[o], c, acc[kx][o]));
      }
    }
  }
#pragma unroll
  for (int kx = 0; kx < kMaxK; ++kx)
#pragma unroll
    for (int o = 0; o < kMaxCout; ++o) {
      double v = acc[kx][o];
      for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][kx * kMaxCout + o] = v;
    }
  __syncthreads();
  if (threadIdx.x < kMaxK * kMaxCout) {
    double s = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) s += red[w][threadIdx.x];
    gw_part[(static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x) * (kMaxK * kMaxCout) + threadIdx.x] = s;
  }
}

// g_W (fp32) = sum of the weight partials - gs[o] / s_o^2, g_bias = sum of the gy partials; all sums in block order.
__global__ void nconv2d_bwd_weight_finish_kernel(const double* __restrict__ gw_part, int gx, const double* __restrict__ gs_part,
                                                 const double* __restrict__ gb_part, int gab, const float* __restrict__ weight,
                                                 int Cin, int Cout, int kh, int kw, float* __restrict__ g_weight,
                                                 float* __restrict__ g_bias) {
  __shared__ double corr[kMaxCout];
  const int ktaps = kh * kw;
  if (threadIdx.x < Cout) {
    double s = 0.0;
    for (int i = 0; i < Cin * ktaps; ++i) s += weight[threadIdx.x * Cin * ktaps + i];
    double gs = 0.0, gb = 0.0;
    for (int blk = 0; blk < gab; ++blk) {
      gs += gs_part[blk * kMaxCout + threadIdx.x];
      gb += gb_part[blk * kMaxCout + threadIdx.x];
    }
    corr[threadIdx.x] = gs / (s * s);
    if (g_bias) g_bias[threadIdx.x] = static_cast<float>(gb);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < Cout * Cin * ktaps; k += blockDim.x) {
    const int o = k / (Cin * ktaps), t = k - o * Cin * ktaps;
    const int i = t / ktaps, ky = (t - i * ktaps) / kw, kx = t - i * ktaps - ky * kw;
    const double* p = gw_part + static_cast<size_t>(i * kh + ky) * gx * (kMaxK * kMaxCout) + kx * kMaxCout + o;
    double v = 0.0;
    for (int blk = 0; blk < gx; ++blk) v += p[static_cast<size_t>(blk) * (kMaxK * kMaxCout)];
    g_weight[k] = static_cast<float>(v - corr[o]);
  }
}

__global__ void __launch_bounds__(kThreads)
nconv_pool2_fwd_kernel(const float* __restrict__ data, const float* __restrict__ conf, int NC, int H, int W, int max_data,
                       float* __restrict__ data_out, float* __restrict__ conf_out, int* __restrict__ idx) {
  const int Ho = H / 2, Wo = W / 2;
  const long long total = static_cast<long long>(NC) * Ho * Wo;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int xo = static_cast<int>(t % Wo), yo = static_cast<int>((t / Wo) % Ho);
    const size_t plane = static_cast<size_t>(t / (static_cast<long long>(Ho) * Wo)) * H * W;
    const float* cp = conf + plane;
    const float* dp = data + plane;
    int ci = (2 * yo) * W + 2 * xo, di = ci;
    float cm = -INFINITY, dm = -INFINITY;
#pragma unroll
    for (int k = 0; k < 4; ++k) {                     // row-major window order; the first maximum wins (F.max_pool2d)
      const int p = (2 * yo + (k >> 1)) * W + 2 * xo + (k & 1);
      const float c = cp[p];
      if (c > cm || isnan(c)) { cm = c; ci = p; }
      const float d = dp[p];
      if (d > dm || isnan(d)) { dm = d; di = p; }
    }
    if (!max_data) di = ci;
    conf_out[t] = cm / 4.0f;
    data_out[t] = dp[di];
    idx[t] = ci;
    idx[total + t] = di;
  }
}

__global__ void __launch_bounds__(kThreads)
nconv_pool2_bwd_kernel(const int* __restrict__ idx, const float* __restrict__ g_data_out, const float* __restrict__ g_conf_out,
                       int NC, int H, int W, float* __restrict__ g_data, float* __restrict__ g_conf) {
  const int Ho = H / 2, Wo = W / 2;
  const long long total = static_cast<long long>(NC) * H * W, pooled = static_cast<long long>(NC) * Ho * Wo;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(t % W), y = static_cast<int>((t / W) % H);
    const long long nc = t / (static_cast<long long>(H) * W);
    float gd = 0.f, gcv = 0.f;
    if (y / 2 < Ho && x / 2 < Wo) {
      const long long o = (nc * Ho + y / 2) * Wo + x / 2;
      const int p = y * W + x;
      if (g_conf_out && idx[o] == p) gcv = g_conf_out[o] / 4.0f;
      if (g_data_out && idx[pooled + o] == p) gd = g_data_out[o];
    }
    if (g_data) g_data[t] = gd;
    if (g_conf) g_conf[t] = gcv;
  }
}

inline int grid_for(long long total) {
  long long g = (total + kThreads - 1) / kThreads;
  if (g > 132 * 8) g = 132 * 8;
  return static_cast<int>(g < 1 ? 1 : g);
}

inline int check_shape(int N, int Cin, int Cup, int Cout, int H, int W, int kh, int kw, int Hup, int Wup) {
  if (N <= 0 || H <= 0 || W <= 0 || Cin < 0 || Cup < 0 || Cin + Cup <= 0 || Cout <= 0) return RNC_ERR_BAD_SHAPE;
  if (Cup > 0 && (Hup <= 0 || Wup <= 0)) return RNC_ERR_BAD_SHAPE;
  if (Cin + Cup > kMaxCin || Cout > kMaxCout || kh > kMaxK || kw > kMaxK || kh < 1 || kw < 1 || !(kh & 1) || !(kw & 1))
    return RNC_ERR_UNSUPPORTED;
  return RNC_OK;
}

inline Src make_src(const float* data, const float* conf, int Cin, const float* up_data, const float* up_conf, int Cup,
                    int Hup, int Wup, int H, int W) {
  Src s{data, conf, Cin, up_data, up_conf, Cup, Hup, Wup, 0.f, 0.f, H, W};
  if (Cup > 0) {
    s.sy = static_cast<float>(Hup) / static_cast<float>(H);
    s.sx = static_cast<float>(Wup) / static_cast<float>(W);
  }
  return s;
}

struct BwdLayout {
  size_t gw, gab, ab, up;   // element counts: weight partials, ab-kernel partials (per array), a/b planes, up scratch
  int gx, gridab;
};

inline BwdLayout bwd_layout(int N, int Cin, int Cup, int Cout, int H, int W, int kh) {
  BwdLayout l;
  const long long pix = static_cast<long long>(N) * H * W;
  l.gx = grid_for(pix / 8);   // each thread's fp32 partial sums cover the same pixels as before the fixed-order reduction
  l.gridab = grid_for(pix * Cout);
  l.gw = static_cast<size_t>(l.gx) * (Cin + Cup) * kh * kMaxK * kMaxCout;
  l.gab = static_cast<size_t>(l.gridab) * kMaxCout;
  l.ab = static_cast<size_t>(pix) * Cout;
  l.up = static_cast<size_t>(pix) * Cup;
  return l;
}

}  // namespace nconv
}  // namespace rnc

using namespace rnc;

extern "C" int rnc_nconv2d_fwd(const float* data, const float* conf, const float* weight, const float* bias, int N, int Cin,
                               int Cout, int H, int W, int kh, int kw, float eps, const float* up_data, const float* up_conf,
                               int Cup, int Hup, int Wup, float y_scale, float* y, float* conf_out, void* stream) {
  if (int st = nconv::check_shape(N, Cin, Cup, Cout, H, W, kh, kw, Hup, Wup)) return st;
  if ((Cin > 0 && (!data || !conf)) || (Cup > 0 && (!up_data || !up_conf)) || !weight || !y || !conf_out)
    return RNC_ERR_BAD_POINTER;
  const nconv::Src src = nconv::make_src(data, conf, Cin, up_data, up_conf, Cup, Hup, Wup, H, W);
  nconv::nconv2d_fwd_kernel<<<nconv::grid_for(static_cast<long long>(N) * H * W), nconv::kThreads, 0, as_stream(stream)>>>(
      src, weight, bias, N, Cout, kh, kw, eps, y_scale, y, conf_out);
  return after_launch();
}

extern "C" size_t rnc_nconv2d_bwd_workspace_bytes(int N, int Cin, int Cup, int Cout, int H, int W, int kh) {
  if (nconv::check_shape(N, Cin, Cup, Cout, H, W, kh, 1, 1, 1)) return 0;
  const nconv::BwdLayout l = nconv::bwd_layout(N, Cin, Cup, Cout, H, W, kh);
  return sizeof(double) * (l.gw + 2 * l.gab) + sizeof(float) * (2 * l.ab + 2 * l.up);
}

extern "C" int rnc_nconv2d_bwd(const float* data, const float* conf, const float* weight, const float* bias, const float* y,
                               const float* conf_out, const float* g_y, const float* g_conf_out, int N, int Cin, int Cout,
                               int H, int W, int kh, int kw, float eps, const float* up_data, const float* up_conf, int Cup,
                               int Hup, int Wup, float* g_data, float* g_conf, float* g_up_data, float* g_up_conf,
                               float* g_weight, float* g_bias, void* workspace, size_t workspace_bytes, void* stream) {
  if (int st = nconv::check_shape(N, Cin, Cup, Cout, H, W, kh, kw, Hup, Wup)) return st;
  if ((Cin > 0 && (!data || !conf)) || (Cup > 0 && (!up_data || !up_conf)) || !weight || !y || !conf_out || !workspace ||
      (!g_y && !g_conf_out) || (g_bias && !g_weight))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_nconv2d_bwd_workspace_bytes(N, Cin, Cup, Cout, H, W, kh) || !aligned16(workspace))
    return RNC_ERR_WORKSPACE;
  const nconv::BwdLayout l = nconv::bwd_layout(N, Cin, Cup, Cout, H, W, kh);
  double* gw_part = static_cast<double*>(workspace);
  double* gs_part = gw_part + l.gw;
  double* gb_part = gs_part + l.gab;
  float* a = reinterpret_cast<float*>(gb_part + l.gab);
  float* b = a + l.ab;
  float* ab_up = b + l.ab;
  const nconv::Src src = nconv::make_src(data, conf, Cin, up_data, up_conf, Cup, Hup, Wup, H, W);
  cudaStream_t s = as_stream(stream);
  const int Ct = Cin + Cup;
  nconv::nconv2d_bwd_ab_kernel<<<l.gridab, nconv::kThreads, 0, s>>>(y, conf_out, g_y, g_conf_out, weight, bias, N, Ct, Cout,
                                                                     H * W, kh * kw, eps, a, b, g_weight ? gs_part : nullptr,
                                                                     gb_part);
  int launches = 1;
  const bool want_up = Cup > 0 && (g_up_data || g_up_conf);
  if (g_data || g_conf || want_up) {
    const int grid = nconv::grid_for(static_cast<long long>(N) * H * W);
    if (Ct <= 4)
      nconv::nconv2d_bwd_data_kernel<4><<<grid, nconv::kThreads, 0, s>>>(src, a, b, weight, N, Cout, kh, kw, g_data, g_conf, ab_up);
    else
      nconv::nconv2d_bwd_data_kernel<8><<<grid, nconv::kThreads, 0, s>>>(src, a, b, weight, N, Cout, kh, kw, g_data, g_conf, ab_up);
    ++launches;
    if (want_up) {
      nconv::nconv2d_bwd_up_kernel<<<nconv::grid_for(static_cast<long long>(N) * Cup * Hup * Wup), nconv::kThreads, 0, s>>>(
          src, ab_up, N, g_up_data, g_up_conf);
      ++launches;
    }
  }
  if (g_weight) {
    nconv::nconv2d_bwd_weight_kernel<<<dim3(l.gx, Ct * kh), nconv::kThreads, 0, s>>>(src, a, b, N, Cout, kh, kw, gw_part);
    nconv::nconv2d_bwd_weight_finish_kernel<<<1, nconv::kThreads, 0, s>>>(gw_part, l.gx, gs_part, gb_part, l.gridab, weight,
                                                                          Ct, Cout, kh, kw, g_weight, g_bias);
    launches += 2;
  }
  return after_launch(launches);
}

extern "C" int rnc_nconv_pool2_fwd(const float* data, const float* conf, int N, int C, int H, int W, int max_pool_data,
                                   float* data_out, float* conf_out, int* idx, void* stream) {
  if (N <= 0 || C <= 0 || H < 2 || W < 2) return RNC_ERR_BAD_SHAPE;
  if (max_pool_data != 0 && max_pool_data != 1) return RNC_ERR_UNSUPPORTED;
  if (!data || !conf || !data_out || !conf_out || !idx) return RNC_ERR_BAD_POINTER;
  const long long pooled = static_cast<long long>(N) * C * (H / 2) * (W / 2);
  nconv::nconv_pool2_fwd_kernel<<<nconv::grid_for(pooled), nconv::kThreads, 0, as_stream(stream)>>>(
      data, conf, N * C, H, W, max_pool_data, data_out, conf_out, idx);
  return after_launch();
}

extern "C" int rnc_nconv_pool2_bwd(const int* idx, const float* g_data_out, const float* g_conf_out, int N, int C, int H, int W,
                                   float* g_data, float* g_conf, void* stream) {
  if (N <= 0 || C <= 0 || H < 2 || W < 2) return RNC_ERR_BAD_SHAPE;
  if (!idx || (!g_data && !g_conf)) return RNC_ERR_BAD_POINTER;
  nconv::nconv_pool2_bwd_kernel<<<nconv::grid_for(static_cast<long long>(N) * C * H * W), nconv::kThreads, 0,
                                  as_stream(stream)>>>(idx, g_data_out, g_conf_out, N * C, H, W, g_data, g_conf);
  return after_launch();
}
