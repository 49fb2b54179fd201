// Backward kernels of the training path (SURVEY.md §8f-3, Appendix G; north-star config #5), exact fp32 on CUDA cores:
//   rnc_corr_lookup_bwd    gradient of CorrBlock.__call__ (core/corr.py:23-44) w.r.t. fmap1 / the fmap2 pyramid — the reference
//                          back-propagates through the stored 4-D pyramid; here the volume never exists
//   rnc_pyramid_pool_bwd   adjoint of the 2x2 average pooling that builds the pyramid (core/corr.py:18-21, on features)
//   rnc_conv2d_cl_wgrad_det weight / bias gradient of a channel-last convolution (every nn.Conv2d of core/update.py,
//                          core/extractor.py, core/interp_weights_est.py); the data gradient reuses rnc_conv2d_cl_fwd with
//                          flipped, transposed weights
// The forward of the same ops in training mode runs the exact fp32 kernels (corr_lookup.cu, conv_ffma.cu, nconv2d.cu).
// rnc_corr_lookup_bwd_det is the atomic-free form of rnc_corr_lookup_bwd (torch.use_deterministic_algorithms): the same
// products, summed in a fixed order.  The weight gradient has only a fixed-order form.  Identical inputs give bit-identical
// gradients.
#include <cub/device/device_radix_sort.cuh>

#include "rnc_common.cuh"

namespace rnc {
namespace train {

constexpr int kR = 4, kS = 9, kG = 10, kD = 256;

// ------------------------------------------------------------------------------------------------ correlation lookup, backward
// Forward (Appendix A.1): out[l*81 + i*9 + j] = sum_{corners} w * G[i + di][j + dj],  G[a][c] = <f1(p), f2^l(ix0 + a, iy0 + c)> / 16.
// coords are detached (raft_nc_dbl.py:149): the bilinear weights are constants.  warp = pixel, lane = 8 channels.
//   gG[a][c]   = w00 g[a][c] + w10 g[a-1][c] + w01 g[a][c-1] + w11 g[a-1][c-1]          (g = d loss / d out, zero outside 0..8)
//   g_f1[p]   += (1/16) sum_{a,c} gG[a][c] f2^l(pos)          g_f2^l[pos] += (1/16) gG[a][c] f1[p]   (vector atomics)
// DET: instead of the g_f2 atomics, each pixel stages gG at stage[(l * B*H*W + pix) * 100 + a * 10 + c] and its window-origin
// cell key (LookupCells) at keys[l * B*H*W + pix], with vals[] = its staging row; lookup_gather_kernel then sums d fmap2.
struct LookupCells {
  int levels, total;            // total = number of cells over all levels = the sentinel key
  int off[4], wc[4], hc[4];     // level l: cells (ix0 + 9, iy0 + 9) in [0, wc) x [0, hc) per image, keys from off[l]
};

template <bool DET>
__global__ void __launch_bounds__(256)
corr_lookup_bwd_kernel(const float* __restrict__ f1_cl, const float* __restrict__ f2_pyr, const float* __restrict__ coords,
                       const float* __restrict__ g_out, int ldg, int B, int H, int W, int levels, float scale,
                       float* __restrict__ g_f1, float* __restrict__ g_f2, LookupCells cells, float* __restrict__ stage,
                       unsigned* __restrict__ keys, unsigned* __restrict__ vals) {
  __shared__ float gG[8][kG * kG + 4];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int HW = H * W;
  const long long total = static_cast<long long>(B) * HW;
  for (long long pix = static_cast<long long>(blockIdx.x) * 8 + warp; pix < total; pix += static_cast<long long>(gridDim.x) * 8) {
    const int b = static_cast<int>(pix / HW), r = static_cast<int>(pix - static_cast<long long>(b) * HW);
    float cx = coords[(static_cast<size_t>(b) * 2 + 0) * HW + r], cy = coords[(static_cast<size_t>(b) * 2 + 1) * HW + r];
    cx = fminf(fmaxf(cx, -1.0e6f), 1.0e6f);
    cy = fminf(fmaxf(cy, -1.0e6f), 1.0e6f);
    const float4* f1p = reinterpret_cast<const float4*>(f1_cl + static_cast<size_t>(pix) * kD);
    const float4 a0 = __ldg(f1p + lane), a1 = __ldg(f1p + 32 + lane);
    float4 acc0 = make_float4(0.f, 0.f, 0.f, 0.f), acc1 = acc0;
    size_t lvl_off = 0;
    float inv = 1.f;
    for (int l = 0; l < levels; ++l) {
      const int Hl = H >> l, Wl = W >> l;
      const float sx = cx * inv, sy = cy * inv;
      inv *= 0.5f;
      const float fx0 = floorf(sx), fy0 = floorf(sy), ax = sx - fx0, ay = sy - fy0;
      const int ix0 = static_cast<int>(fx0) - kR, iy0 = static_cast<int>(fy0) - kR;
      const float w00 = (1.f - ax) * (1.f - ay), w10 = ax * (1.f - ay), w01 = (1.f - ax) * ay, w11 = ax * ay;
      const float* go = g_out + static_cast<size_t>(pix) * ldg + l * kS * kS;
      __syncwarp();
      for (int t = lane; t < kG * kG; t += 32) {
        const int a = t / kG, c = t - a * kG;
        float v = 0.f;
        if (a < kS && c < kS) v = fmaf(w00, go[a * kS + c], v);
        if (a >= 1 && c < kS) v = fmaf(w10, go[(a - 1) * kS + c], v);
        if (a < kS && c >= 1) v = fmaf(w01, go[a * kS + c - 1], v);
        if (a >= 1 && c >= 1) v = fmaf(w11, go[(a - 1) * kS + c - 1], v);
        gG[warp][t] = v * scale;
        if (DET) stage[(static_cast<size_t>(l) * total + pix) * (kG * kG) + t] = v * scale;
      }
      if (DET && lane == 0) {
        const bool hit = ix0 >= -(kG - 1) && ix0 < Wl && iy0 >= -(kG - 1) && iy0 < Hl;
        const size_t row = static_cast<size_t>(l) * total + pix;
        keys[row] = hit ? static_cast<unsigned>(cells.off[l] + (b * cells.hc[l] + iy0 + kG - 1) * cells.wc[l] + ix0 + kG - 1)
                        : static_cast<unsigned>(cells.total);
        vals[row] = static_cast<unsigned>(row);
      }
      __syncwarp();
      const float* f2l = f2_pyr + lvl_off + static_cast<size_t>(b) * Hl * Wl * kD;
      float* g2l = g_f2 + lvl_off + static_cast<size_t>(b) * Hl * Wl * kD;
      lvl_off += static_cast<size_t>(B) * Hl * Wl * kD;
      for (int c = 0; c < kG; ++c) {
        const int Y = iy0 + c;
        if (Y < 0 || Y >= Hl) continue;                               // warp-uniform
        for (int a = 0; a < kG; ++a) {
          const int X = ix0 + a;
          if (X < 0 || X >= Wl) continue;
          const float gv = gG[warp][a * kG + c];
          if (gv == 0.f) continue;
          const size_t pos = (static_cast<size_t>(Y) * Wl + X) * kD;
          const float4* q = reinterpret_cast<const float4*>(f2l + pos);
          const float4 b0 = __ldg(q + lane), b1 = __ldg(q + 32 + lane);
          acc0.x = fmaf(gv, b0.x, acc0.x); acc0.y = fmaf(gv, b0.y, acc0.y); acc0.z = fmaf(gv, b0.z, acc0.z); acc0.w = fmaf(gv, b0.w, acc0.w);
          acc1.x = fmaf(gv, b1.x, acc1.x); acc1.y = fmaf(gv, b1.y, acc1.y); acc1.z = fmaf(gv, b1.z, acc1.z); acc1.w = fmaf(gv, b1.w, acc1.w);
          if (!DET) {
            float4* gq = reinterpret_cast<float4*>(g2l + pos);
            atomicAdd(gq + lane, make_float4(gv * a0.x, gv * a0.y, gv * a0.z, gv * a0.w));
            atomicAdd(gq + 32 + lane, make_float4(gv * a1.x, gv * a1.y, gv * a1.z, gv * a1.w));
          }
        }
      }
    }
    float4* g1 = reinterpret_cast<float4*>(g_f1 + static_cast<size_t>(pix) * kD);
    g1[lane] = acc0;
    g1[32 + lane] = acc1;
  }
}

// Sorted cell keys -> start[k] = first sorted row of cell k, for k in [0, total]; start[total] = number of in-grid rows.
// Every entry is written by exactly one thread: the row where the key sequence passes it.
__global__ void cell_start_kernel(const unsigned* __restrict__ keys, int n, int total, int* __restrict__ start) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int k = static_cast<int>(keys[i]);
    const int kp = i == 0 ? -1 : static_cast<int>(keys[i - 1]);
    for (int kk = kp + 1; kk <= k && kk <= total; ++kk) start[kk] = i;
    if (i == n - 1)
      for (int kk = k + 1; kk <= total; ++kk) start[kk] = n;
  }
}

// d fmap2 at level l, one warp per pyramid position (b, Y, X), lane = 8 channels: the windows that cover the position have
// their origin cell at (X - a, Y - c), a, c in 0..9.  Cells in the forward kernel's (c, a) loop order, each cell's pixels in
// ascending index; every term is the atomic kernel's product gv * f1[p] (rounded on its own), added in that fixed order.
__global__ void __launch_bounds__(256)
lookup_gather_kernel(const float* __restrict__ f1_cl, const float* __restrict__ stage, const unsigned* __restrict__ rows,
                     const int* __restrict__ start, int B, int Hl, int Wl, int key_off, int wc, int hc, size_t row_off,
                     float* __restrict__ g2l) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long npos = static_cast<long long>(B) * Hl * Wl;
  for (long long q = static_cast<long long>(blockIdx.x) * 8 + warp; q < npos; q += static_cast<long long>(gridDim.x) * 8) {
    const int b = static_cast<int>(q / (static_cast<long long>(Hl) * Wl));
    const int r = static_cast<int>(q - static_cast<long long>(b) * Hl * Wl);
    const int Y = r / Wl, X = r - Y * Wl;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int c = 0; c < kG; ++c) {
      const int cy = Y - c + kG - 1;                               // in [0, hc): the cell always exists
      for (int a = 0; a < kG; ++a) {
        const int key = key_off + (b * hc + cy) * wc + X - a + kG - 1;
        const int s0 = __ldg(start + key), s1 = __ldg(start + key + 1);
        for (int i = s0; i < s1; ++i) {
          const size_t row = __ldg(rows + i);
          const float gv = __ldg(stage + row * (kG * kG) + a * kG + c);
          if (gv == 0.f) continue;
          const float4* fp = reinterpret_cast<const float4*>(f1_cl + (row - row_off) * kD);
          const float4 u0 = __ldg(fp + lane), u1 = __ldg(fp + 32 + lane);
          const float u[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = __fadd_rn(acc[j], __fmul_rn(gv, u[j]));
        }
      }
    }
    float4* g = reinterpret_cast<float4*>(g2l + static_cast<size_t>(q) * kD);
    g[lane] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    g[32 + lane] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  }
}

// g_l[b, y, x, :] += 0.25 * g_{l+1}[b, y/2, x/2, :] where (y/2, x/2) exists (floor-mode pooling drops odd rows / columns)
__global__ void pool2_adjoint_kernel(float4* __restrict__ fine, const float4* __restrict__ coarse, int B, int Hf, int Wf, int D4) {
  const int Hc = Hf >> 1, Wc = Wf >> 1;
  const size_t n = static_cast<size_t>(B) * Hf * Wf * D4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % D4);
    size_t r = i / D4;
    const int x = static_cast<int>(r % Wf); r /= Wf;
    const int y = static_cast<int>(r % Hf);
    const int b = static_cast<int>(r / Hf);
    if ((y >> 1) >= Hc || (x >> 1) >= Wc) continue;
    const float4 g = coarse[((static_cast<size_t>(b) * Hc + (y >> 1)) * Wc + (x >> 1)) * D4 + c];
    float4 v = fine[i];
    v.x = fmaf(0.25f, g.x, v.x); v.y = fmaf(0.25f, g.y, v.y); v.z = fmaf(0.25f, g.z, v.z); v.w = fmaf(0.25f, g.w, v.w);
    fine[i] = v;
  }
}

// ------------------------------------------------------------------------------------------------ convolution weight gradient
// gw[tap][ci][co] = sum_p x[(p shifted by tap), ci] * gy[p, co];   gb[co] = sum_p gy[p, co]
// GEMM view: M = Cin, N = Cout, K = output pixels, split across blockIdx.z.  Block z writes its partial sums to
// part + z * taps * cin * cout ([tap][ci][co]) and its bias partials to part_bias + z * cout; wgrad_reduce_kernel adds them in
// ascending z.
constexpr int WT = 64;       // tile side (ci and co)
constexpr int WK = 16;       // pixels per step
__global__ void __launch_bounds__(64)
conv_wgrad_kernel(const float* __restrict__ x, int ldx, int cin, const float* __restrict__ gy, int ldg, int cout, int B, int Hin,
                  int Win, int Ho, int Wo, int kh, int kw, int stride, int dil, int px_per_block, float* __restrict__ part,
                  float* __restrict__ part_bias) {
  float* const gw = part + static_cast<size_t>(blockIdx.z) * kh * kw * cin * cout;
  float* const gb = part_bias ? part_bias + static_cast<size_t>(blockIdx.z) * cout : nullptr;
  __shared__ __align__(16) float Xs[WK][WT + 4];
  __shared__ __align__(16) float Gs[WK][WT + 4];
  const int tid = threadIdx.x;
  const int ntc = (cout + WT - 1) / WT;
  const int ci0 = (blockIdx.x / ntc) * WT, co0 = (blockIdx.x % ntc) * WT;
  const int tap = blockIdx.y, ky = tap / kw, kx = tap - ky * kw;
  const int ph = kh / 2 * dil, pw = kw / 2 * dil;
  const long long P = static_cast<long long>(B) * Ho * Wo;
  const long long p0 = static_cast<long long>(blockIdx.z) * px_per_block;
  const long long p1 = p0 + px_per_block < P ? p0 + px_per_block : P;
  const int ty = tid >> 3, tx = tid & 7;        // thread = 8 (ci) x 8 (co) micro tile
  float2 acc2[8][4];                              // pairs of adjacent output channels (ffma2)
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc2[i][j] = make_float2(0.f, 0.f);
  float bsum[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const bool do_bias = gb != nullptr && tap == 0 && ci0 == 0 && ty == 0;
  // staging: 16 px x 64 ch = 256 float4 per operand, 4 per thread: pixel = (tid >> 4) + 4 * i, channel quad = tid & 15.
  // Register double buffering: the global loads of step k+1 are issued before the FMAs of step k.
  const int sq = tid & 15;
  float4 xr[4], gr[4];
  auto fetch = [&](long long pb) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int sp = (tid >> 4) + 4 * i;
      const long long p = pb + sp;
      float4 xv = make_float4(0.f, 0.f, 0.f, 0.f), gv = xv;
      if (p < p1) {
        const int b = static_cast<int>(p / (Ho * Wo)), r = static_cast<int>(p - static_cast<long long>(b) * Ho * Wo);
        const int yo = r / Wo, xo = r - yo * Wo;
        const int yi = yo * stride + ky * dil - ph, xi = xo * stride + kx * dil - pw;
        if (yi >= 0 && yi < Hin && xi >= 0 && xi < Win && ci0 + 4 * sq < cin)
          xv = __ldg(reinterpret_cast<const float4*>(x + ((static_cast<size_t>(b) * Hin + yi) * Win + xi) * ldx + ci0 + 4 * sq));
        if (co0 + 4 * sq < cout) {
          const float* gp = gy + static_cast<size_t>(p) * ldg + co0 + 4 * sq;
          if (co0 + 4 * sq + 4 <= cout) gv = __ldg(reinterpret_cast<const float4*>(gp));
          else { gv.x = gp[0]; if (co0 + 4 * sq + 1 < cout) gv.y = gp[1]; if (co0 + 4 * sq + 2 < cout) gv.z = gp[2]; }
        }
      }
      xr[i] = xv; gr[i] = gv;
    }
  };
  fetch(p0);
  for (long long pb = p0; pb < p1; pb += WK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int sp = (tid >> 4) + 4 * i;
      *reinterpret_cast<float4*>(&Xs[sp][4 * sq]) = xr[i];
      *reinterpret_cast<float4*>(&Gs[sp][4 * sq]) = gr[i];
    }
    __syncthreads();
    if (pb + WK < p1) fetch(pb + WK);
#pragma unroll
    for (int k = 0; k < WK; ++k) {
      const float4 x0 = *reinterpret_cast<const float4*>(&Xs[k][ty * 8]), x1 = *reinterpret_cast<const float4*>(&Xs[k][ty * 8 + 4]);
      const float4 g0 = *reinterpret_cast<const float4*>(&Gs[k][tx * 8]), g1 = *reinterpret_cast<const float4*>(&Gs[k][tx * 8 + 4]);
      const float xa[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
      const float ga[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float2 g2[4] = {make_float2(g0.x, g0.y), make_float2(g0.z, g0.w), make_float2(g1.x, g1.y), make_float2(g1.z, g1.w)};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float2 xi = make_float2(xa[i], xa[i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc2[i][j] = ffma2(xi, g2[j], acc2[i][j]);
      }
      if (do_bias) {
#pragma unroll
        for (int j = 0; j < 8; ++j) bsum[j] += ga[j];
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int ci = ci0 + ty * 8 + i;
    if (ci >= cin) continue;
    const float acc[8] = {acc2[i][0].x, acc2[i][0].y, acc2[i][1].x, acc2[i][1].y, acc2[i][2].x, acc2[i][2].y, acc2[i][3].x, acc2[i][3].y};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int co = co0 + tx * 8 + j;
      if (co < cout) gw[(static_cast<size_t>(tap) * cin + ci) * cout + co] = acc[j];
    }
  }
  if (do_bias) {
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (co0 + tx * 8 + j < cout) gb[co0 + tx * 8 + j] = bsum[j];
  }
}

// gw[tap][ci][co] = sum over z ascending of part[z][tap][ci][co], from 0, in fp32; the bias rows follow the weight rows:
// part[nsplit * n + z * cout + co].
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int nsplit, int taps_cin, int cout, float* __restrict__ gw,
                                    int ldw, float* __restrict__ gb) {
  const size_t n = static_cast<size_t>(taps_cin) * cout;
  const size_t total = n + (gb ? cout : 0);
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const bool bias = i >= n;
    const float* p = bias ? part + nsplit * n + (i - n) : part + i;
    const size_t step = bias ? cout : n;
    float s = 0.f;
    for (int z = 0; z < nsplit; ++z) s = __fadd_rn(s, __ldg(p + z * step));
    if (bias) gb[i - n] = s;
    else gw[(i / cout) * ldw + i % cout] = s;
  }
}

}  // namespace train
}  // namespace rnc

using namespace rnc;

extern "C" int rnc_corr_lookup_bwd(const float* f1_cl, const float* f2_pyr, const float* coords, const float* g_out, int ldg,
                                   int B, int D, int H, int W, int levels, int radius, float* g_f1, float* g_f2_pyr, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || levels < 1 || levels > 4 || (H >> (levels - 1)) < 1 || (W >> (levels - 1)) < 1) return RNC_ERR_BAD_SHAPE;
  if (D != train::kD || radius != train::kR || ldg < levels * train::kS * train::kS) return RNC_ERR_UNSUPPORTED;
  if (!f1_cl || !f2_pyr || !coords || !g_out || !g_f1 || !g_f2_pyr) return RNC_ERR_BAD_POINTER;
  if (!aligned16(f1_cl) || !aligned16(f2_pyr) || !aligned16(g_f1) || !aligned16(g_f2_pyr)) return RNC_ERR_BAD_POINTER;
  const long long total = static_cast<long long>(B) * H * W;
  long long blocks = (total + 7) / 8;
  if (blocks > 132 * 8) blocks = 132 * 8;
  train::corr_lookup_bwd_kernel<false><<<static_cast<int>(blocks), 256, 0, as_stream(stream)>>>(
      f1_cl, f2_pyr, coords, g_out, ldg, B, H, W, levels, 1.0f / sqrtf(static_cast<float>(D)), g_f1, g_f2_pyr, {}, nullptr,
      nullptr, nullptr);
  return after_launch();
}

namespace {
// Workspace of rnc_corr_lookup_bwd_det, 256-byte aligned parts: stage [levels][B*H*W][100] floats, keys / rows twice (radix
// sort double buffers) [levels * B*H*W], start [cells + 1], then the radix sort's scratch.
struct LookupPlan {
  train::LookupCells cells;
  size_t n, stage, keys, start, sort_scratch, bytes;
  int end_bit;
};

size_t up256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

bool lookup_plan(int B, int H, int W, int levels, LookupPlan* p) {
  if (B <= 0 || H <= 0 || W <= 0 || levels < 1 || levels > 4 || (H >> (levels - 1)) < 1 || (W >> (levels - 1)) < 1) return false;
  long long total = 0;
  p->cells.levels = levels;
  for (int l = 0; l < 4; ++l) {
    const int Hl = l < levels ? H >> l : 0, Wl = l < levels ? W >> l : 0;
    p->cells.off[l] = static_cast<int>(total);
    p->cells.wc[l] = Wl + train::kG - 1;
    p->cells.hc[l] = Hl + train::kG - 1;
    if (l < levels) total += static_cast<long long>(B) * p->cells.wc[l] * p->cells.hc[l];
  }
  const long long n = static_cast<long long>(levels) * B * H * W;
  if (total >= (1LL << 31) - 1 || n * train::kG * train::kG >= (1LL << 40) || n >= (1LL << 31)) return false;
  p->cells.total = static_cast<int>(total);
  p->end_bit = 1;
  while ((1LL << p->end_bit) <= total) ++p->end_bit;
  p->n = static_cast<size_t>(n);
  p->stage = up256(p->n * train::kG * train::kG * sizeof(float));
  p->keys = up256(p->n * sizeof(unsigned));
  p->start = up256((static_cast<size_t>(total) + 1) * sizeof(int));
  // the onesweep radix sort needs a few histograms and one look-back word per digit and tile: a fixed bound, checked at run time
  p->sort_scratch = up256((size_t{1} << 20) + p->n * 4);
  p->bytes = p->stage + 4 * p->keys + p->start + p->sort_scratch;
  return true;
}
}  // namespace

extern "C" size_t rnc_corr_lookup_bwd_workspace_bytes(int B, int H, int W, int levels) {
  LookupPlan p;
  return lookup_plan(B, H, W, levels, &p) ? p.bytes : 0;
}

extern "C" int rnc_corr_lookup_bwd_det(const float* f1_cl, const float* f2_pyr, const float* coords, const float* g_out, int ldg,
                                       int B, int D, int H, int W, int levels, int radius, float* g_f1, float* g_f2_pyr,
                                       void* workspace, size_t workspace_bytes, void* stream) {
  LookupPlan p;
  if (!lookup_plan(B, H, W, levels, &p)) return RNC_ERR_BAD_SHAPE;
  if (D != train::kD || radius != train::kR || ldg < levels * train::kS * train::kS) return RNC_ERR_UNSUPPORTED;
  if (!f1_cl || !f2_pyr || !coords || !g_out || !g_f1 || !g_f2_pyr || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned16(f1_cl) || !aligned16(f2_pyr) || !aligned16(g_f1) || !aligned16(g_f2_pyr) || !aligned16(workspace))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < p.bytes) return RNC_ERR_WORKSPACE;
  char* w = static_cast<char*>(workspace);
  float* stage = reinterpret_cast<float*>(w);
  unsigned* k0 = reinterpret_cast<unsigned*>(w + p.stage);
  unsigned* k1 = reinterpret_cast<unsigned*>(w + p.stage + p.keys);
  unsigned* v0 = reinterpret_cast<unsigned*>(w + p.stage + 2 * p.keys);
  unsigned* v1 = reinterpret_cast<unsigned*>(w + p.stage + 3 * p.keys);
  int* start = reinterpret_cast<int*>(w + p.stage + 4 * p.keys);
  void* scratch = w + p.stage + 4 * p.keys + p.start;
  const cudaStream_t s = as_stream(stream);
  const long long total = static_cast<long long>(B) * H * W;
  long long blocks = (total + 7) / 8;
  if (blocks > 132 * 8) blocks = 132 * 8;
  // pass 1: g_f1 and the staged gG / origin cells
  train::corr_lookup_bwd_kernel<true><<<static_cast<int>(blocks), 256, 0, s>>>(
      f1_cl, f2_pyr, coords, g_out, ldg, B, H, W, levels, 1.0f / sqrtf(static_cast<float>(D)), g_f1, g_f2_pyr, p.cells, stage,
      k0, v0);
  if (int st = after_launch()) return st;
  // pass 2: stable sort of the staging rows by cell (rows enter ascending, so each cell lists its pixels in ascending order)
  cub::DoubleBuffer<unsigned> dk(k0, k1), dv(v0, v1);
  size_t need = 0;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, need, dk, dv, static_cast<int>(p.n), 0, p.end_bit, s);
  if (e != cudaSuccess) { g_last_cuda_error = static_cast<int>(e); return RNC_ERR_CUDA; }
  if (need > p.sort_scratch) return RNC_ERR_WORKSPACE;
  e = cub::DeviceRadixSort::SortPairs(scratch, need, dk, dv, static_cast<int>(p.n), 0, p.end_bit, s);
  if (e != cudaSuccess) { g_last_cuda_error = static_cast<int>(e); return RNC_ERR_CUDA; }
  const int nb = static_cast<int>(p.n / 256 + 1 < 132 * 8 ? p.n / 256 + 1 : 132 * 8);
  train::cell_start_kernel<<<nb, 256, 0, s>>>(dk.Current(), static_cast<int>(p.n), p.cells.total, start);
  if (int st = after_launch()) return st;
  // pass 3: every pyramid position gathers its d fmap2
  size_t lvl_off = 0;
  for (int l = 0; l < levels; ++l) {
    const int Hl = H >> l, Wl = W >> l;
    long long gb = (static_cast<long long>(B) * Hl * Wl + 7) / 8;
    if (gb > 132 * 8) gb = 132 * 8;
    train::lookup_gather_kernel<<<static_cast<int>(gb), 256, 0, s>>>(f1_cl, stage, dv.Current(), start, B, Hl, Wl, p.cells.off[l],
                                                                     p.cells.wc[l], p.cells.hc[l], static_cast<size_t>(l) * total,
                                                                     g_f2_pyr + lvl_off);
    lvl_off += static_cast<size_t>(B) * Hl * Wl * train::kD;
  }
  return after_launch(levels);
}

extern "C" int rnc_pyramid_pool_bwd(float* g_f2_pyr, int B, int D, int H, int W, int levels, void* stream) {
  if (B <= 0 || D <= 0 || (D & 3) || H <= 0 || W <= 0 || levels < 1 || levels > 4) return RNC_ERR_BAD_SHAPE;
  if (!g_f2_pyr || !aligned16(g_f2_pyr)) return RNC_ERR_BAD_POINTER;
  int launches = 0;
  for (int l = levels - 2; l >= 0; --l) {
    float* fine = g_f2_pyr + rnc_pyramid_offset(B, D, H, W, l);
    const float* coarse = g_f2_pyr + rnc_pyramid_offset(B, D, H, W, l + 1);
    const int Hf = H >> l, Wf = W >> l;
    const size_t n = static_cast<size_t>(B) * Hf * Wf * (D / 4);
    size_t blocks = (n + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    train::pool2_adjoint_kernel<<<static_cast<int>(blocks), 256, 0, as_stream(stream)>>>(
        reinterpret_cast<float4*>(fine), reinterpret_cast<const float4*>(coarse), B, Hf, Wf, D / 4);
    ++launches;
  }
  return after_launch(launches);
}

namespace {
bool wgrad_shape_ok(int cin, int cout, int B, int Hin, int Win, int kh, int kw, int stride) {
  return B > 0 && Hin > 0 && Win > 0 && cin > 0 && cout > 0 && !(cin & 3) && kh >= 1 && kw >= 1 && (kh & 1) && (kw & 1) &&
         kh * kw <= 49 && (stride == 1 || stride == 2);
}

// K split of the weight gradient, from the shape alone: enough blocks to fill the machine a few times over (at most
// 132 * 24 of them), every block a multiple of WK pixels.  The partials of one split are one (ci, co) tile per tap and block, so
// all splits together hold at most 132 * 24 * 64 * 64 floats (52 MB) whatever the layer.  Returns 0 if too many splits.
int wgrad_split(int cin, int cout, int B, int Hin, int Win, int kh, int kw, int stride, long long* per_out) {
  const int Ho = (Hin + stride - 1) / stride, Wo = (Win + stride - 1) / stride;
  const long long P = static_cast<long long>(B) * Ho * Wo;
  const int tiles = ((cin + train::WT - 1) / train::WT) * ((cout + train::WT - 1) / train::WT);
  const int taps = kh * kw;
  long long want = (132LL * 24 + tiles * taps - 1) / (static_cast<long long>(tiles) * taps);
  if (want < 1) want = 1;
  long long per = (P + want - 1) / want;
  per = (per + train::WK - 1) / train::WK * train::WK;
  if (per < 4 * train::WK) per = 4 * train::WK;
  const long long ksplit = (P + per - 1) / per;
  if (ksplit > 65535 || per > (1LL << 30)) return 0;
  *per_out = per;
  return static_cast<int>(ksplit);
}
}  // namespace

extern "C" size_t rnc_conv2d_cl_wgrad_workspace_bytes(int cin, int cout, int B, int Hin, int Win, int kh, int kw, int stride) {
  if (!wgrad_shape_ok(cin, cout, B, Hin, Win, kh, kw, stride)) return 0;
  long long per = 0;
  const int ksplit = wgrad_split(cin, cout, B, Hin, Win, kh, kw, stride, &per);
  return static_cast<size_t>(ksplit) * (static_cast<size_t>(kh) * kw * cin * cout + cout) * sizeof(float);
}

static int wgrad_det(const float* x, int ldx, int cin, const float* gy, int ldg, int cout, int B, int Hin, int Win, int kh, int kw,
                     int stride, int dil, float* gw, int ldw, float* gb, void* workspace, size_t workspace_bytes, void* stream) {
  if (!wgrad_shape_ok(cin, cout, B, Hin, Win, kh, kw, stride) || (ldx & 3) || ldx < cin || ldg < cout || ldw < cout)
    return RNC_ERR_BAD_SHAPE;
  if (!x || !gy || !gw || !workspace || !aligned16(x) || !aligned16(gy) || (ldg & 3)) return RNC_ERR_BAD_POINTER;
  const int Ho = (Hin + stride - 1) / stride, Wo = (Win + stride - 1) / stride;
  long long per = 0;
  const int ksplit = wgrad_split(cin, cout, B, Hin, Win, kh, kw, stride, &per);
  if (ksplit == 0) return RNC_ERR_BAD_SHAPE;
  const size_t n = static_cast<size_t>(kh) * kw * cin * cout;
  if (workspace_bytes < static_cast<size_t>(ksplit) * (n + cout) * sizeof(float)) return RNC_ERR_WORKSPACE;
  float* part = static_cast<float*>(workspace);
  const int tiles = ((cin + train::WT - 1) / train::WT) * ((cout + train::WT - 1) / train::WT);
  dim3 grid(tiles, kh * kw, ksplit);
  train::conv_wgrad_kernel<<<grid, 64, 0, as_stream(stream)>>>(x, ldx, cin, gy, ldg, cout, B, Hin, Win, Ho, Wo, kh, kw, stride,
                                                                dil, static_cast<int>(per), part,
                                                                gb ? part + static_cast<size_t>(ksplit) * n : nullptr);
  if (int st = after_launch()) return st;
  const size_t total = n + (gb ? cout : 0);
  const int blocks = static_cast<int>(total / 256 + 1 < 132 * 16 ? total / 256 + 1 : 132 * 16);
  train::wgrad_reduce_kernel<<<blocks, 256, 0, as_stream(stream)>>>(part, ksplit, kh * kw * cin, cout, gw, ldw, gb);
  return after_launch();
}

extern "C" int rnc_conv2d_cl_wgrad_det(const float* x, int ldx, int cin, const float* gy, int ldg, int cout, int B, int Hin,
                                       int Win, int kh, int kw, int stride, float* gw, int ldw, float* gb, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  return wgrad_det(x, ldx, cin, gy, ldg, cout, B, Hin, Win, kh, kw, stride, 1, gw, ldw, gb, workspace, workspace_bytes, stream);
}

// Stride 1 with dilation dil: the same tiles, K split and workspace as the undilated layer of that shape.
extern "C" size_t rnc_conv2d_cl_wgrad_dil_workspace_bytes(int cin, int cout, int B, int Hin, int Win, int kh, int kw, int dil) {
  return dil >= 1 && dil <= 8 ? rnc_conv2d_cl_wgrad_workspace_bytes(cin, cout, B, Hin, Win, kh, kw, 1) : 0;
}

extern "C" int rnc_conv2d_cl_wgrad_dil_det(const float* x, int ldx, int cin, const float* gy, int ldg, int cout, int B, int Hin,
                                           int Win, int kh, int kw, int dil, float* gw, int ldw, float* gb, void* workspace,
                                           size_t workspace_bytes, void* stream) {
  if (dil < 1 || dil > 8) return RNC_ERR_BAD_SHAPE;
  return wgrad_det(x, ldx, cin, gy, ldg, cout, B, Hin, Win, kh, kw, 1, dil, gw, ldw, gb, workspace, workspace_bytes, stream);
}
