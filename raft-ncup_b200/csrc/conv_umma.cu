// wgmma implicit-GEMM convolution: persistent CTAs, TMA-staged 128B-swizzled operand rings fed by one producer warp, two
// consumer warpgroups that each issue wgmma (M64 x N<=256 x K16) for 64 of the tile's 128 rows and keep the fp32
// accumulators in registers, then run the epilogue of the tile themselves.
// Replaces: core/update.py:33-60 (SepConvGRU), :79-97 (BasicMotionEncoder), :6-14 (FlowHead), :123-126 (mask head), the 3x3
// layers of core/interp_weights_est.py:10-47 and (stride 1/2, residual epilogue) the convolutions of
// core/extractor.py:6-56,118-192.
//
// fp32-faithful on fp16 tensor cores: every activation x and weight w is an exact-sum pair of halves (x = x_hi + x_lo;
// weights pre-scaled by a power of two so w_lo stays normal) and each K step issues x_hi*w_hi + x_hi*w_lo + x_lo*w_hi
// (3 MMAs): plain TF32/bf16 operands miss the 1e-3 EPE bar by 17-60x (SURVEY.md Appendix D).
//
// GEMM view: M = 128 output pixels, N = Cout tile, K = taps x 64-channel blocks.  Zero padding is free: A tiles are
// 4-D TMA boxes whose out-of-image elements are zero-filled.  Three A-staging modes cut the L2->SM traffic of the taps:
//   TAP      one 128-row box per filter tap (any geometry, strides 1 and 2 via TMA element strides)
//   ROWHALO  tile = 1 image row x 128 px: one (128 + 8)-row box per (ky, channel block); the kw horizontal taps are
//            operand descriptors shifted by kx rows
//   COLHALO  kw == 1: tile = 8 x 16 px with a vertical halo, the kh taps are descriptors shifted by ky*16 rows
// A fourth input form, RNC_CONV_WINDOW, reads in0 through a sliding-window tensor map (dimension 1 steps fewer bytes than
// dimension 0 spans): the TMA unit builds im2col rows of a small-Cin layer (the encoders' 7x7/2 stem) without a copy.
// Epilogue: registers -> a staged accumulator tile (thread = pixel) -> per-warp swizzled staging in shared memory ->
// cp.async.bulk.tensor stores (split halves, fp32 outputs, the GRU state); fused InstanceNorm sums read the staged chunk column-wise.
#include "umma_ptx.cuh"

namespace rnc {
namespace umma {

constexpr int kThreads = 288;        // warps 0-7: two consumer warpgroups (wgmma on 64 rows each + epilogue), warp 8: TMA producer
constexpr int kBM = 128;
constexpr int kBK = 64;
constexpr int kMaxSA = 4, kMaxSB = 12;
constexpr int kStageWarp = 4096;     // epilogue staging per consumer warp: 32 px x 32 ch as [hi 2 KB | lo 2 KB] halves or 4 KB of fp32
constexpr int kStageBytes = 8 * kStageWarp;
constexpr int kAccCols = 64;         // accumulator columns staged in shared memory per epilogue pass
constexpr int kAccStride = kAccCols + 4;    // floats per staged pixel row: conflict-free 16-byte reads of a pixel's chunk
constexpr int kAccBytes = kBM * kAccStride * 4;
constexpr int kSmemFixed = 1024 + 512 + 8192 + 1024 + kAccBytes + kStageBytes;   // alignment, barriers, statistics, staging
constexpr int kSmemMax = 226 * 1024;      // 227 KB per block, less the 1 KB the system reserves on sm_90
constexpr int kRingBudget = kSmemMax - kSmemFixed;   // A + B rings
enum { MODE_TAP = 0, MODE_ROWHALO = 1, MODE_COLHALO = 2 };

struct Params {
  int B, H, W;                        // output geometry
  int TW, TH, tiles_x, tiles_y, ntiles, ntn;
  int mode, kh, kw, ph, pw, stride;   // stride: y (and x unless sx overrides)
  int sx;                             // x stride (1 for a window view, whose positions already step by the stride)
  int nblk0, nblk;                    // K blocks (128 bytes of channels: 64 halves or 32 TF32 words) in segment 0 / total
  int bk;                             // channels per K block: 64 (fp16 hi/lo operands) or 32 (TF32 hi/lo operands)
  int tf32;                           // operands are fp32 planes consumed as TF32 (wgmma .tf32): training-path layers
  int a_plane, SA, SB;                // bytes per A half-plane stage (rows*128, 1024-aligned), ring depths
  int resident_b;                     // the layer's whole weight matrix fits the B ring: loaded once per CTA, never released
  int probe_nob;                      // developer probe (RNC_CONV_PROBE_NOB=1): skip the weight loads after the first ring fill
  int cout, epilogue;
  float unscale;
  const float* bias;
  float* out_f32; int ldo_f32;
  __half* out_hi; __half* out_lo; int ldo_split;
  float* h; int ldh;
  float* aux0; int ldaux;
  const float* res; int ldres;
  const float* add; int ldadd;        // optional fp32 addend of the pre-activation, [pixel][ldadd]
  int aux_blocked, out_blocked;       // aux0 + add / out_f32 in the tile-blocked layout [tile][channel][128 px] (coalesced for thread = pixel)
  double* stats;                      // [B][cout][2]: per-(image, channel) sum / sum of squares of the outputs, accumulated
};

// exact hi/lo split of 8 floats into two 16-byte vectors of halves
__device__ __forceinline__ void split8(const float* v, uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) split_pair(v[2 * i], v[2 * i + 1], h[i], l[i]);
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

template <int BN>
struct Cfg {
  static constexpr int kBTile = BN * kBK * 2;                     // bytes per half-plane of weights
  static constexpr int kChunksN = BN / 32;                        // 32-channel epilogue chunks
  static constexpr int kPasses = (BN + kAccCols - 1) / kAccCols;  // epilogue passes over the staged accumulator tile
};

// Each thread's accumulators of one 64-row half of the tile: `main` (d[0, BN/2)) takes the x_hi*w_hi products, `corr`
// (d[BN/2, BN)) the two 2^-11-smaller cross terms.  The tensor core truncates on every accumulate, so the error grows with the
// number of full-magnitude adds; keeping the cross terms out of `main` cuts it 3x (measured: 4.8e-5 -> 1.7e-5 on a 3x3x256
// layer).  All three instructions have the same shape, so their accumulator accesses are ordered without a fence.
template <int BN, bool TF32>
__device__ __forceinline__ void mma_block(float* d, uint64_t ah, uint64_t al, uint64_t bh, uint64_t bl, int first) {
  constexpr int kSteps = 4;          // 128 bytes of K per block: 4 x (16 halves | 8 TF32 words)
#pragma unroll
  for (int k = 0; k < kSteps; ++k) {
    const int acc = (first && k == 0) ? 0 : 1;
    wgmma<BN, TF32>(d, ah + 2 * k, bh + 2 * k, acc);
    wgmma<BN, TF32>(d + BN / 2, ah + 2 * k, bl + 2 * k, acc);
    wgmma<BN, TF32>(d + BN / 2, al + 2 * k, bh + 2 * k, 1);
  }
}

// Columns [P*64, P*64 + 64) of main + corr (already summed into d[0, BN/2)) -> the staged accumulator tile [128 px][kAccStride] (rows of this warpgroup)
template <int BN, int P>
__device__ __forceinline__ void stash_acc(const float* d, float* acc_tile, int row0, int lane) {
  constexpr int j0 = P * kAccCols / 8, j1 = (P + 1) * kAccCols / 8 < BN / 8 ? (P + 1) * kAccCols / 8 : BN / 8;
  const int c0 = 2 * (lane & 3);
#pragma unroll
  for (int j = j0; j < j1; ++j) {
    const int col = 8 * j + c0 - P * kAccCols;
    *reinterpret_cast<float2*>(acc_tile + row0 * kAccStride + col) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(acc_tile + (row0 + 8) * kAccStride + col) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

// EC: epilogue class, compiled separately so that a launch carries only its own epilogue code (the union of all epilogues
// costs the gate layers instruction-cache misses and registers): 0 = plain layers (linear / relu / sigmoid), 1 = GRU z|r
// gates, 2 = GRU q, 3 = the rest (flow append, residual tail, tanh|relu head, coords update, fused InstanceNorm sums).
enum { EC_PLAIN = 0, EC_GRU_ZR = 1, EC_GRU_Q = 2, EC_MISC = 3 };

// 9 warps: the SM sub-partition holding three of them caps the kernel at 168 registers per thread
template <int BN, int EC>
__global__ void __launch_bounds__(kThreads, 1)
conv_umma_kernel(const __grid_constant__ CUtensorMap mA0h, const __grid_constant__ CUtensorMap mA0l,
                 const __grid_constant__ CUtensorMap mA1h, const __grid_constant__ CUtensorMap mA1l,
                 const __grid_constant__ CUtensorMap mBh, const __grid_constant__ CUtensorMap mBl,
                 const __grid_constant__ CUtensorMap mOh, const __grid_constant__ CUtensorMap mOl,
                 const __grid_constant__ CUtensorMap mOf, const Params p) {
  using C = Cfg<BN>;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int a_stage = 2 * p.a_plane;
  constexpr int kBStageBytes = 2 * C::kBTile;                   // [w_hi | w_lo] rows of one K block
  unsigned char* sA = smem;
  unsigned char* sB = smem + p.SA * a_stage;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + p.SB * kBStageBytes);
  uint64_t* a_full = bars;
  uint64_t* a_empty = a_full + kMaxSA;
  uint64_t* b_full = a_empty + kMaxSA;
  uint64_t* b_empty = b_full + kMaxSB;
  double* stat_acc = reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(bars) + 512);   // [8 warps][passes][32 lanes][2]
  // epilogue staging (TMA-store source), 1024-aligned so the 64B / 128B swizzle patterns are functions of the buffer offset,
  // then the staged accumulator tile
  unsigned char* stage_base = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(bars) + 512 + 8192 + 1023) & ~uintptr_t(1023));
  float* acc_tile = reinterpret_cast<float*>(stage_base + kStageBytes);

  pdl_trigger();                       // the next kernel in the stream may begin its prologue on SMs this grid has left
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tpi = p.tiles_x * p.tiles_y;
  const int G = p.mode == MODE_TAP ? p.kh * p.kw : p.mode == MODE_ROWHALO ? p.kh : 1;     // A-stage groups per channel block
  const int T = p.mode == MODE_TAP ? 1 : p.mode == MODE_ROWHALO ? p.kw : p.kh;            // taps sharing one A stage
  const int items = p.ntiles * p.ntn;                                                     // (pixel tile, column tile)
  const int item0 = static_cast<int>(blockIdx.x), item_step = static_cast<int>(gridDim.x);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.SA; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 8); }
    for (int s = 0; s < p.SB; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();                          // everything above overlapped the predecessor's tail; its results are visible from here

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer
    // The whole warp runs the loop so that addresses / coordinates stay in uniform registers; one elected lane issues.
    // Ring positions are (slot, parity) counters: a runtime modulo per stage costs ~100 cycles of dependent integer code.
    int sa_n = 0, pa_n = 0, sb_n = 0, pb_n = 0, b_it = 0;
    for (int item = item0; item < items; item += item_step) {
      const int tile = item / p.ntn, n0 = (item - tile * p.ntn) * BN;
      const int b = tile / tpi, tr = tile - b * tpi;
      const int y0 = (tr / p.tiles_x) * p.TH, x0 = (tr % p.tiles_x) * p.TW;
      for (int g = 0; g < G; ++g) {
        int cx, cy;
        if (p.mode == MODE_TAP) { cx = x0 * p.sx + g % p.kw - p.pw; cy = y0 * p.stride + g / p.kw - p.ph; }
        else if (p.mode == MODE_ROWHALO) { cx = x0 - p.pw; cy = y0 + g - p.ph; }
        else { cx = x0; cy = y0 - p.ph; }
        for (int cb = 0; cb < p.nblk; ++cb) {
          const int sa = sa_n, pa = pa_n;
          if (++sa_n == p.SA) { sa_n = 0; pa_n ^= 1; }
          mbar_wait(&a_empty[sa], pa ^ 1);
          const bool seg0 = cb < p.nblk0;
          const int c = (seg0 ? cb : cb - p.nblk0) * p.bk;
          if (elect_one()) {
            mbar_expect_tx(&a_full[sa], a_stage);
            tma_load_4d(sA + sa * a_stage, seg0 ? &mA0h : &mA1h, &a_full[sa], c, cx, cy, b);
            tma_load_4d(sA + sa * a_stage + p.a_plane, seg0 ? &mA0l : &mA1l, &a_full[sa], c, cx, cy, b);
          }
          __syncwarp();
          for (int t = 0; t < T; ++t) {
            const int tap = p.mode == MODE_TAP ? g : p.mode == MODE_ROWHALO ? g * p.kw + t : t;
            const int sb = sb_n, pb = pb_n;
            if (++sb_n == p.SB) { sb_n = 0; pb_n ^= 1; }
            ++b_it;
            if (p.resident_b && item != item0) continue;     // weights already resident
            mbar_wait(&b_empty[sb], pb ^ 1);
            const int kcol = (tap * p.nblk + cb) * p.bk;
            if (elect_one()) {
              if (p.probe_nob && b_it > p.SB) {
                mbar_arrive(&b_full[sb]);
              } else {
                mbar_expect_tx(&b_full[sb], kBStageBytes);
                tma_load_2d(sB + sb * kBStageBytes, &mBh, &b_full[sb], kcol, n0);
                tma_load_2d(sB + sb * kBStageBytes + C::kBTile, &mBl, &b_full[sb], kcol, n0);
              }
            }
            __syncwarp();
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: wgmma main loop, then the epilogue
  const int wg = warp >> 2;                        // warpgroup: rows [64 wg, 64 wg + 64) of the tile
  const int row0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);   // accumulator rows row0, row0 + 8 of this thread
  float d[BN];                                     // main | corr
  const uint32_t sA_u = smem_u32(sA), sB_u = smem_u32(sB);
  const uint32_t t_rows = p.mode == MODE_ROWHALO ? 1u : p.mode == MODE_COLHALO ? static_cast<uint32_t>(p.TW) : 0u;   // tap shift in rows

  // epilogue: thread = pixel; warp w takes lane group w & 3 (pixels 32 (w & 3) + lane), half h = w >> 2 takes the chunks
  // 2 * pass + h of the staged accumulator columns
  const int lg = warp & 3, hsel = warp >> 2;
  const int ml = lg * 32 + lane;
  const int epi = p.epilogue;
  const bool use_stats = EC == EC_MISC && p.stats != nullptr;
  double* my_acc = stat_acc + (static_cast<size_t>(warp) * C::kPasses * 32 + lane) * 2;   // [pass] stride 64 doubles
  int acc_b = -1, acc_n0 = 0;
  auto flush_stats = [&]() {
    if (acc_b < 0) return;
    for (int ci = 0; ci < C::kPasses; ++ci) {
      const int ch = acc_n0 + (2 * ci + hsel) * 32 + lane;
      if (2 * ci + hsel < C::kChunksN && ch < p.cout) {
        double* dst = p.stats + (static_cast<size_t>(acc_b) * p.cout + ch) * 2;
        atomicAdd(dst, my_acc[ci * 64]);
        atomicAdd(dst + 1, my_acc[ci * 64 + 1]);
      }
      my_acc[ci * 64] = 0.0; my_acc[ci * 64 + 1] = 0.0;
    }
  };
  if (use_stats) {
    for (int ci = 0; ci < C::kPasses; ++ci) { my_acc[ci * 64] = 0.0; my_acc[ci * 64 + 1] = 0.0; }
  }
  // Outputs leave through shared memory and TMA stores: a warp's 32 px x 32 ch chunk is one box of the output tensor
  // (full 64- / 128-byte rows per pixel instead of 16-byte pieces per thread; image borders are clipped by the TMA unit).
  // The staging rows are written with the map's swizzle (64B for halves, 128B for fp32): conflict-free.
  unsigned char* stg = stage_base + warp * kStageWarp;
  bool stg_busy = false;                           // warp-uniform: a TMA store may still be reading the staging buffer
  const int lgx = (lg * 32) % p.TW, lgy = (lg * 32) / p.TW;
  int bx = 0, by = 0, bb = 0;                      // box origin of this warp's lane group in the current tile
  auto stage_free = [&]() {
    if (stg_busy) { if (lane == 0) bulk_wait_read0(); __syncwarp(); stg_busy = false; }
  };
  auto store_split = [&](const float* v, int ch) {           // hi/lo halves of v[0..32) -> channels [ch, ch+32) of out_hi / out_lo
    stage_free();
    uint4* sh = reinterpret_cast<uint4*>(stg + lane * 64);
    uint4* sl = reinterpret_cast<uint4*>(stg + 2048 + lane * 64);
    const int sw = (lane >> 1) & 3;
#pragma unroll
    for (int q = 0; q < 4; ++q) split8(v + 8 * q, sh[q ^ sw], sl[q ^ sw]);
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) {
      tma_store_4d(&mOh, stg, ch, bx, by, bb);
      tma_store_4d(&mOl, stg + 2048, ch, bx, by, bb);
      bulk_commit();
    }
    stg_busy = true;
  };
  auto store_f32 = [&](const float* v, int ch) {             // fp32 v[0..32) -> channels [ch, ch+32) of h (q gate) / out_f32
    stage_free();
    float4* sf = reinterpret_cast<float4*>(stg + lane * 128);
    const int sw = lane & 7;
#pragma unroll
    for (int q = 0; q < 8; ++q) sf[q ^ sw] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) { tma_store_4d(&mOf, stg, ch, bx, by, bb); bulk_commit(); }
    stg_busy = true;
  };

  int sa_n = 0, pa_n = 0, sb_n = 0, pb_n = 0;
  for (int item = item0; item < items; item += item_step) {
    const int tile = item / p.ntn, n0 = (item - tile * p.ntn) * BN;
    // ---- main loop: K = taps x channel blocks, one wgmma batch per weight stage
    int first = 1;
    for (int g = 0; g < G; ++g)
      for (int cb = 0; cb < p.nblk; ++cb) {
        const int sa = sa_n, pa = pa_n;
        if (++sa_n == p.SA) { sa_n = 0; pa_n ^= 1; }
        mbar_wait(&a_full[sa], pa);
        for (int t = 0; t < T; ++t) {
          const int sb = sb_n, pb = pb_n;
          if (++sb_n == p.SB) { sb_n = 0; pb_n ^= 1; }
          mbar_wait(&b_full[sb], p.resident_b ? 0 : pb);
          // A rows of this warpgroup, shifted by the tap (ROWHALO: kx rows, COLHALO: ky image rows of TW pixels)
          const uint32_t a_addr = sA_u + sa * a_stage + (64u * wg + t * t_rows) * 128u;
          // no base_offset: with 1024-byte aligned stages the swizzle is a function of the absolute address
          const uint64_t ah = smem_desc_sw128(a_addr);
          const uint64_t al = ah + (static_cast<uint32_t>(p.a_plane) >> 4);
          const uint64_t bh = smem_desc_sw128(sB_u + sb * kBStageBytes), bl = bh + (C::kBTile >> 4);
          wgmma_fence();
          if (p.tf32) mma_block<BN, true>(d, ah, al, bh, bl, first); else mma_block<BN, false>(d, ah, al, bh, bl, first);
          wgmma_commit();
          wgmma_wait<0>();
          first = 0;
          __syncwarp();
          if (!p.resident_b && lane == 0) mbar_arrive(&b_empty[sb]);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&a_empty[sa]);
      }
#pragma unroll
    for (int i = 0; i < BN; ++i) reg_fence(d[i]);
    // main + corr once, so that only half of the accumulator registers stay live through the epilogue passes
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) d[i] += d[BN / 2 + i];

    // ---- epilogue
    const int b = tile / tpi, tr = tile - b * tpi;
    if (use_stats && (b != acc_b || n0 != acc_n0)) { flush_stats(); acc_b = b; acc_n0 = n0; }
    const int ty0 = (tr / p.tiles_x) * p.TH, tx0 = (tr % p.tiles_x) * p.TW;
    const int y = ty0 + ml / p.TW, x = tx0 + ml % p.TW;
    const bool valid = y < p.H && x < p.W;
    bx = tx0 + lgx; by = ty0 + lgy; bb = b;
    // tile-blocked tensors (p.aux_blocked / p.out_blocked): element (tile, channel c, row ml) at ((tile * ld + c) * 128 + ml),
    // so a warp's 32 pixels are contiguous per channel
    const size_t pix = (static_cast<size_t>(b) * p.H + y) * p.W + x;
    auto chunk = [&](int pass, int cc) {
      const int n = n0 + cc * 32;
        float v[32];
        const float4* sv = reinterpret_cast<const float4*>(acc_tile + ml * kAccStride + (cc - 2 * pass) * 32);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 bv = __ldg(reinterpret_cast<const float4*>(p.bias + n) + q), s = sv[q];
          v[4 * q + 0] = fmaf(s.x, p.unscale, bv.x);
          v[4 * q + 1] = fmaf(s.y, p.unscale, bv.y);
          v[4 * q + 2] = fmaf(s.z, p.unscale, bv.z);
          v[4 * q + 3] = fmaf(s.w, p.unscale, bv.w);
        }
        if (p.add != nullptr && valid) {
          // hoisted part of the layer (input channels that are constant across calls), computed once by another launch
          if (p.aux_blocked) {
            const float* ap = p.add + (static_cast<size_t>(tile) * p.ldadd + n) * kBM + ml;
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] += __ldg(ap + static_cast<size_t>(j) * kBM);
          } else {
            const float4* ap = reinterpret_cast<const float4*>(p.add + pix * p.ldadd + n);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              const float4 a = __ldg(ap + q);
              v[4 * q] += a.x; v[4 * q + 1] += a.y; v[4 * q + 2] += a.z; v[4 * q + 3] += a.w;
            }
          }
        }
        if (use_stats) {
          // InstanceNorm statistics of this layer's output (extractor.py:128-129), fused here instead of a pass over the fp32
          // tensor.  The chunk is staged in shared memory for its TMA store anyway ([pixel][32 ch], 128B-swizzled), which is
          // the transposition the reduction over pixels needs: lane = channel walks its column (conflict-free: a row's 32
          // words are a permutation of the 32 banks), fp32 partial sums over the warp's 32 pixels, accumulated in fp64 per
          // lane in shared memory across the CTA's tiles and flushed with fp64 atomics when the image changes.  Pixels beyond
          // the image are staged as zeros (the TMA store clips them).
          if (!valid) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = 0.f;
          }
          store_f32(v, n);                       // stats layers are RNC_EPI_LINEAR with a channel-last fp32 output (host check)
          float s1 = 0.f, s2 = 0.f;
          const int cw = lane >> 2, ce = lane & 3;
#pragma unroll
          for (int px = 0; px < 32; ++px) {
            const float x = *reinterpret_cast<const float*>(stg + px * 128 + ((cw ^ (px & 7)) << 4) + ce * 4);
            s1 += x;
            s2 = fmaf(x, x, s2);
          }
          my_acc[pass * 64] += static_cast<double>(s1);
          my_acc[pass * 64 + 1] += static_cast<double>(s2);
          return;
        }
        if (EC == EC_GRU_ZR) {
          const int Ch = p.cout >> 1;
          if (n < Ch) {            // z gate -> fp32 aux buffer
            if (valid) {
              if (p.aux_blocked) {
                float* dst = p.aux0 + (static_cast<size_t>(tile) * p.ldaux + n) * kBM + ml;
#pragma unroll
                for (int j = 0; j < 32; ++j) dst[static_cast<size_t>(j) * kBM] = sigmoid_fast(v[j]);
              } else {
                float4* dst = reinterpret_cast<float4*>(p.aux0 + pix * p.ldaux + n);
#pragma unroll
                for (int q = 0; q < 8; ++q)
                  dst[q] = make_float4(sigmoid_fast(v[4 * q]), sigmoid_fast(v[4 * q + 1]), sigmoid_fast(v[4 * q + 2]), sigmoid_fast(v[4 * q + 3]));
              }
            }
          } else {                 // r gate -> r*h as split halves
            const float4* hp = reinterpret_cast<const float4*>(p.h + pix * p.ldh + (n - Ch));
            float4 hreg[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) hreg[q] = valid ? __ldg(hp + q) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              const float4 hv = hreg[q];
              v[4 * q + 0] = sigmoid_fast(v[4 * q + 0]) * hv.x; v[4 * q + 1] = sigmoid_fast(v[4 * q + 1]) * hv.y;
              v[4 * q + 2] = sigmoid_fast(v[4 * q + 2]) * hv.z; v[4 * q + 3] = sigmoid_fast(v[4 * q + 3]) * hv.w;
            }
            store_split(v, n - Ch);
          }
          return;
        }
        if (EC == EC_MISC && epi == RNC_EPI_FLOW_DELTA) {
          // FlowHead.conv2 + `coords1 = coords1 + delta_flow` (update.py:14, raft_nc_dbl.py:157); only channels 0,1 are real
          if (valid) {
            const int HW = p.H * p.W;
            const size_t i0 = static_cast<size_t>(b) * 2 * HW + y * p.W + x;
            p.aux0[i0] += v[0];
            p.aux0[i0 + HW] += v[1];
            if (p.out_f32) { p.out_f32[i0] = v[0]; p.out_f32[i0 + HW] = v[1]; }
          }
          return;
        }
        bool want_f32 = p.out_f32 != nullptr;
        if (EC == EC_GRU_Q) {
          const float4* hp = reinterpret_cast<const float4*>(p.h + pix * p.ldh + n);
          float4 zreg[8], hreg[8];
          if (!valid) {
#pragma unroll
            for (int q = 0; q < 8; ++q) { zreg[q] = make_float4(0.f, 0.f, 0.f, 0.f); hreg[q] = zreg[q]; }
          } else {
            if (p.aux_blocked) {
              const float* zb = p.aux0 + (static_cast<size_t>(tile) * p.ldaux + n) * kBM + ml;
#pragma unroll
              for (int q = 0; q < 8; ++q)
                zreg[q] = make_float4(__ldg(zb + static_cast<size_t>(4 * q) * kBM), __ldg(zb + static_cast<size_t>(4 * q + 1) * kBM),
                                      __ldg(zb + static_cast<size_t>(4 * q + 2) * kBM), __ldg(zb + static_cast<size_t>(4 * q + 3) * kBM));
            } else {
              const float4* zp = reinterpret_cast<const float4*>(p.aux0 + pix * p.ldaux + n);
#pragma unroll
              for (int q = 0; q < 8; ++q) zreg[q] = __ldg(zp + q);
            }
            // plain loads: h is rewritten by this kernel (each chunk is read before its own TMA store is issued)
#pragma unroll
            for (int q = 0; q < 8; ++q) hreg[q] = hp[q];
          }
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 z = zreg[q], hv = hreg[q];
            v[4 * q + 0] = (1.f - z.x) * hv.x + z.x * tanh_fast(v[4 * q + 0]);
            v[4 * q + 1] = (1.f - z.y) * hv.y + z.y * tanh_fast(v[4 * q + 1]);
            v[4 * q + 2] = (1.f - z.z) * hv.z + z.z * tanh_fast(v[4 * q + 2]);
            v[4 * q + 3] = (1.f - z.w) * hv.w + z.w * tanh_fast(v[4 * q + 3]);
          }
          store_f32(v, n);
        } else if (EC == EC_PLAIN) {
          if (epi == RNC_EPI_RELU) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
          } else if (epi == RNC_EPI_SIGMOID) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = sigmoid_fast(v[j]);
          }
        } else if (EC != EC_MISC) {
          // (not reached: the z|r class left the chunk above)
        } else if (epi == RNC_EPI_RELU_FLOW) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
          if (n <= p.cout && p.cout < n + 32 && valid) {
            // append flow = coords1 - grid as channels [cout, cout+2)  (update.py:97)
            const int HW = p.H * p.W;
            const float* c1 = p.aux0 + static_cast<size_t>(b) * 2 * HW + y * p.W + x;
            const float fx = c1[0] - static_cast<float>(x), fy = c1[HW] - static_cast<float>(y);
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              if (n + j == p.cout) v[j] = fx;
              if (n + j == p.cout + 1) v[j] = fy;
            }
          }
        } else if (epi == RNC_EPI_RELU_ADD_RELU) {
          // residual block tail (extractor.py:55): relu(x + relu(norm(conv(.)))) with the norm folded into the weights
          const float4* rp = reinterpret_cast<const float4*>(p.res + pix * p.ldres + n);
          float4 rreg[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) rreg[q] = valid ? __ldg(rp + q) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            v[4 * q + 0] = fmaxf(rreg[q].x + fmaxf(v[4 * q + 0], 0.f), 0.f);
            v[4 * q + 1] = fmaxf(rreg[q].y + fmaxf(v[4 * q + 1], 0.f), 0.f);
            v[4 * q + 2] = fmaxf(rreg[q].z + fmaxf(v[4 * q + 2], 0.f), 0.f);
            v[4 * q + 3] = fmaxf(rreg[q].w + fmaxf(v[4 * q + 3], 0.f), 0.f);
          }
        } else if (epi == RNC_EPI_TANH_RELU) {
          // context encoder head (raft_nc_dbl.py:138-140): first half tanh -> net, second half relu -> inp
          if (n < (p.cout >> 1)) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = tanh_fast(v[j]);
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
            want_f32 = false;
          }
        }
        if (want_f32) {
          if (p.out_blocked) {
            if (valid) {
              float* dst = p.out_f32 + (static_cast<size_t>(tile) * p.ldo_f32 + n) * kBM + ml;
#pragma unroll
              for (int j = 0; j < 32; ++j) dst[static_cast<size_t>(j) * kBM] = v[j];
            }
          } else {
            store_f32(v, n);
          }
        }
        if (p.out_hi) store_split(v, n);
    };
#pragma unroll 1
    for (int pass = 0; pass < C::kPasses; ++pass) {
      named_bar_sync(1, 256);                      // every consumer warp is done with the staged tile of the previous pass
      if (pass == 0) stash_acc<BN, 0>(d, acc_tile, row0, lane);
      else if (C::kPasses > 1) stash_acc<BN, (C::kPasses > 1 ? 1 : 0)>(d, acc_tile, row0, lane);
      named_bar_sync(1, 256);
      const int cc = 2 * pass + hsel;
      if (cc < C::kChunksN && n0 + cc * 32 < p.cout + (EC == EC_MISC && epi == RNC_EPI_RELU_FLOW ? 2 : 0)) chunk(pass, cc);
    }
  }
  if (use_stats) flush_stats();
  if (lane == 0) bulk_wait_all0();                 // the staging buffer must outlive its TMA stores; their writes complete here
}

// ---------------------------------------------------------------------------------------------- host side
// activation plane [B][Hin][Win][ld] halves: 4-D map {C, Win, Hin, B}; the box spans bw x bh input elements and is
// traversed with element strides (sx, sy) -> (bw/sx) x (bh/sy) rows of 64 channels in shared memory
static bool make_in_map(CUtensorMap* m, const void* base, int C, int ld, int B, int Hin, int Win, int bw, int bh, int sx, int sy, bool tf32,
                        long long row_pitch = 0) {
  const cuuint64_t esz = tf32 ? 4 : 2;                        // 128-byte rows: 32 fp32 words or 64 halves
  const cuuint64_t pitch = row_pitch > 0 ? (cuuint64_t)row_pitch : (cuuint64_t)Win * ld;     // elements between image rows
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)Win, (cuuint64_t)Hin, (cuuint64_t)B};
  // window view (RNC_CONV_WINDOW): ld < C, i.e. consecutive positions overlap -- the TMA unit walks plain strides
  const cuuint64_t strides[3] = {(cuuint64_t)ld * esz, pitch * esz, (cuuint64_t)Hin * pitch * esz};
  const cuuint32_t box[4] = {tf32 ? 32u : 64u, (cuuint32_t)(bw * sx), (cuuint32_t)(bh * sy), 1};
  const cuuint32_t es[4] = {1, (cuuint32_t)sx, (cuuint32_t)sy, 1};
  return encode_fn()(m, tf32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// weight plane [CoutPad][Ktot] halves: 2-D map {Ktot, CoutPad}, box {64, BN}
static bool make_w_map(CUtensorMap* m, const void* base, int ktot, int coutpad, int bn, bool tf32) {
  const cuuint64_t dims[2] = {(cuuint64_t)ktot, (cuuint64_t)coutpad};
  const cuuint64_t strides[1] = {(cuuint64_t)ktot * (tf32 ? 4 : 2)};
  const cuuint32_t box[2] = {tf32 ? 32u : 64u, (cuuint32_t)bn};
  const cuuint32_t es[2] = {1, 1};
  return encode_fn()(m, tf32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// output plane [B][H][W][ld] (halves or fp32): 4-D map {C, W, H, B}, box = 32 channels x one lane group's bw x bh pixels,
// rows swizzled (64B for halves, 128B for fp32) to match the epilogue's conflict-free staging writes
static bool make_out_map(CUtensorMap* m, const void* base, int C, int ld, int B, int H, int W, int bw, int bh, bool f32) {
  const cuuint64_t esz = f32 ? 4 : 2;
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)ld * esz, (cuuint64_t)W * ld * esz, (cuuint64_t)H * W * ld * esz};
  const cuuint32_t box[4] = {32u, (cuuint32_t)bw, (cuuint32_t)bh, 1};
  const cuuint32_t es[4] = {1, 1, 1, 1};
  return encode_fn()(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, f32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

template <int BN, int EC>
static int launch(const CUtensorMap* maps, Params& p, cudaStream_t stream, int max_sa, int max_sb) {
  using C = Cfg<BN>;
  const int a_stage = 2 * p.a_plane;
  // ring depths within kRingBudget: both rings hide the same TMA latency, so deepen A (up to 4) while B keeps >= 2 stages
  const int budget = kRingBudget, b_stage = 2 * C::kBTile;
  const int sa_cap = max_sa > 0 && max_sa < kMaxSA ? max_sa : kMaxSA;      // debug knobs (rnc_conv_umma_desc.flags bits 8-15)
  p.SA = 2;
  while (p.SA < sa_cap && budget - (p.SA + 1) * a_stage >= 2 * b_stage) ++p.SA;
  int sb = (budget - p.SA * a_stage) / b_stage;
  p.SB = sb > 8 ? 8 : sb < 2 ? 2 : sb;
  if (max_sb > 0 && p.SB > max_sb) p.SB = max_sb;
  // Small layers (64 -> 64 3x3: 9 stages of 16 KB): keep the whole weight matrix in the ring for the CTA's lifetime instead
  // of re-streaming it for every pixel tile.
  p.resident_b = 0;
  {
    const int nb = p.kh * p.kw * p.nblk;
    if (p.ntn == 1 && nb <= kMaxSB && nb > p.SB && max_sb == 0 && 2 * a_stage + nb * b_stage <= kRingBudget) {
      p.resident_b = 1; p.SB = nb; p.SA = (kRingBudget - nb * b_stage) / a_stage;
      if (p.SA > kMaxSA) p.SA = kMaxSA;
    }
  }
  const int smem = p.SA * a_stage + p.SB * b_stage + kSmemFixed;
  if (smem > kSmemMax) return RNC_ERR_UNSUPPORTED;
  static unsigned long long done = 0;
  if (int st = ensure_dyn_smem(conv_umma_kernel<BN, EC>, kSmemMax, &done)) return st;
  const int items = p.ntiles * p.ntn;
  const int grid = items < sm_count() ? items : sm_count();
  cudaError_t e = launch_pdl(conv_umma_kernel<BN, EC>, dim3(grid), dim3(kThreads), smem, stream, maps[0], maps[1], maps[2], maps[3],
                             maps[4], maps[5], maps[6], maps[7], maps[8], p);
  if (e != cudaSuccess) { cudaGetLastError(); g_last_cuda_error = static_cast<int>(e); return RNC_ERR_CUDA; }
  return after_launch();
}

template <int EC>
static int launch_bn(int bn, const CUtensorMap* maps, Params& p, cudaStream_t s, int msa, int msb) {
  switch (bn) {
    case 32: return launch<32, EC>(maps, p, s, msa, msb);
    case 64: return launch<64, EC>(maps, p, s, msa, msb);
    default: return launch<128, EC>(maps, p, s, msa, msb);
  }
}

}  // namespace umma
}  // namespace rnc

using namespace rnc;

// Pixel-tile shape of a layer (the A-staging mode decides it): row halo -> 128x1, column halo -> 16x8, per-tap -> TW x 128/TW.
static void tile_shape(int kh, int kw, int stride, int H, int W, int flags, int& TW, int& TH) {
  if (stride == 1 && (flags & RNC_CONV_NO_HALO) == 0 && kw > 1 && W > 64) { TW = 128; TH = 1; }
  else if (stride == 1 && (flags & RNC_CONV_NO_HALO) == 0 && kw == 1 && kh > 1 && W >= 16 && H >= 8) { TW = 16; TH = 8; }
  else { TW = 8; while (TW < W && TW < umma::kBM) TW <<= 1; TH = umma::kBM / TW; }
}

extern "C" long long rnc_conv_umma_tiles(int kh, int kw, int stride, int B, int H, int W, int flags) {
  if (kh <= 0 || kw <= 0 || stride <= 0 || B <= 0 || H <= 0 || W <= 0) return 0;
  int TW, TH;
  tile_shape(kh, kw, stride, H, W, flags, TW, TH);
  return static_cast<long long>(B) * ((W + TW - 1) / TW) * ((H + TH - 1) / TH);
}

// Column-tile width.  The widest tile that divides coutpad is the default; a narrower one (more, smaller work items per
// pixel tile) wins when the grid is under-filled (small batches: 56 pixel tiles on 132 SMs) or when the tile count just
// misses a multiple of the SM count.  Tiles are at most 128 columns: the main and correction accumulators of a 128-column
// tile already take 128 registers per consumer thread.  Cost model in K-step units: per K-step 1.0 / 0.68 / 0.57 for
// 128 / 64 / 32 columns (operand bytes per K-step: the A tile plus the weight tile), + 0.5 per item, x1.08 when the A tile
// is loaded more than once.
static int choose_bn(const rnc_conv_umma_desc& d, int bn_max, int stride) {
  if (d.flags & RNC_CONV_SPLIT_N) return bn_max;
  const int bkc = (d.flags & RNC_CONV_TF32) ? 32 : 64;
  const int taps = d.kh * d.kw, ksteps = taps * ((d.c0 + bkc - 1) / bkc + (d.c1 + bkc - 1) / bkc);
  int TW, TH;
  tile_shape(d.kh, d.kw, stride, d.H, d.W, d.flags, TW, TH);
  const long ntiles = static_cast<long>(d.B) * ((d.W + TW - 1) / TW) * ((d.H + TH - 1) / TH);
  static const int cand[3] = {128, 64, 32};
  static const float per_k[3] = {1.0f, 0.68f, 0.57f};
  const long slots = umma::sm_count();
  int best = bn_max;
  float best_cost = 1e30f;
  for (int i = 0; i < 3; ++i) {
    const int bn = cand[i];
    if (bn > bn_max || d.coutpad % bn != 0) continue;
    if ((d.epilogue == RNC_EPI_TANH_RELU || d.epilogue == RNC_EPI_GRU_ZR) && bn < 64) continue;
    const int ntn = d.coutpad / bn;
    const long rounds = (ntiles * ntn + slots - 1) / slots;
    float item = ksteps * per_k[i] + 0.5f;
    if (ntn > 1) item *= 1.08f;
    const float cost = rounds * item;
    if (cost < best_cost * 0.97f) { best_cost = cost; best = bn; }     // wider wins near-ties
  }
  return best;
}

extern "C" int rnc_conv2d_umma_fwd(const rnc_conv_umma_desc* desc, void* stream) {
  using namespace rnc::umma;
  if (!desc) return RNC_ERR_BAD_POINTER;
  const rnc_conv_umma_desc& d = *desc;
  const int stride = d.stride <= 0 ? 1 : d.stride;
  const int Hin = d.hin > 0 ? d.hin : d.H, Win = d.win > 0 ? d.win : d.W;
  if (d.B <= 0 || d.H <= 0 || d.W <= 0 || d.cout <= 0 || d.c0 <= 0 || d.c1 < 0 || stride > 2) return RNC_ERR_BAD_SHAPE;
  if (d.kh < 1 || d.kw < 1 || !(d.kh & 1) || !(d.kw & 1) || d.kh * d.kw > 49) return RNC_ERR_BAD_SHAPE;
  const bool tf32 = (d.flags & RNC_CONV_TF32) != 0;
  const int bk = tf32 ? 32 : kBK, ldmask = tf32 ? 3 : 7;      // operand rows are 16-byte multiples
  if (tf32 && (d.out_hi || d.epilogue == RNC_EPI_RELU_FLOW || d.epilogue == RNC_EPI_GRU_ZR || d.epilogue == RNC_EPI_TANH_RELU))
    return RNC_ERR_UNSUPPORTED;                                // TF32 layers write fp32 outputs only
  const bool window = (d.flags & RNC_CONV_WINDOW) != 0;
  if (window && (tf32 || d.c1 > 0 || d.kw != 1 || stride != 2 || d.win <= 0 || d.hin <= 0 || d.win_pitch < d.win * d.ld0 ||
                 (d.win_pitch & 7)))
    return RNC_ERR_BAD_SHAPE;
  if ((d.ld0 & ldmask) || (d.ld0 < d.c0 && !window) || (d.c1 > 0 && ((d.c0 % bk) != 0 || (d.ld1 & ldmask) || d.ld1 < d.c1))) return RNC_ERR_BAD_SHAPE;
  if (!d.in0_hi || !d.in0_lo || (d.c1 > 0 && (!d.in1_hi || !d.in1_lo)) || !d.w_hi || !d.w_lo || !d.bias) return RNC_ERR_BAD_POINTER;
  if (!aligned16(d.in0_hi) || !aligned16(d.in0_lo) || !aligned16(d.w_hi) || !aligned16(d.w_lo) || !aligned16(d.bias)) return RNC_ERR_BAD_POINTER;
  if (d.c1 > 0 && (!aligned16(d.in1_hi) || !aligned16(d.in1_lo))) return RNC_ERR_BAD_POINTER;
  const int nblk0 = (d.c0 + bk - 1) / bk, nblk1 = (d.c1 + bk - 1) / bk, nblk = nblk0 + nblk1;
  const int ntaps = d.kh * d.kw;
  if (d.ktot != ntaps * nblk * bk) return RNC_ERR_BAD_SHAPE;           // weight planes are [coutpad][taps * blocks * bk]
  const int bn0 = d.coutpad <= 32 ? 32 : d.coutpad <= 64 ? 64 : 128;
  int bn = bn0;
  while (bn > 32 && d.coutpad % bn != 0) bn >>= 1;            // the widest column tile that divides coutpad
  if (d.coutpad % bn != 0) bn = bn0;
  if (d.coutpad % bn == 0 && d.epilogue != RNC_EPI_RELU_FLOW && d.epilogue != RNC_EPI_FLOW_DELTA)
    bn = choose_bn(d, bn, stride);
  if (d.coutpad % bn != 0 || d.coutpad < d.cout) return RNC_ERR_BAD_SHAPE;
  if (d.epilogue == RNC_EPI_RELU_FLOW && (d.coutpad < d.cout + 2 || !d.aux0 || !d.out_hi)) return RNC_ERR_BAD_SHAPE;
  if (d.out_hi && (!d.out_lo || (d.ldo_split & 7) || !aligned16(d.out_hi) || !aligned16(d.out_lo))) return RNC_ERR_BAD_POINTER;
  if (d.out_f32 && ((d.ldo_f32 & 3) || !aligned16(d.out_f32))) return RNC_ERR_BAD_POINTER;
  if (d.add && ((d.ldadd & 3) || d.ldadd < d.coutpad || !aligned16(d.add))) return RNC_ERR_BAD_POINTER;
  if (d.stats && (d.epilogue != RNC_EPI_LINEAR || !d.out_f32 || d.out_hi || d.coutpad > 128)) return RNC_ERR_UNSUPPORTED;
  switch (d.epilogue) {
    case RNC_EPI_RELU_ADD_RELU:
      if (!d.res || (d.ldres & 3) || !aligned16(d.res)) return RNC_ERR_BAD_POINTER;
      /* fall through */
    case RNC_EPI_LINEAR: case RNC_EPI_RELU: case RNC_EPI_SIGMOID: case RNC_EPI_RELU_FLOW: case RNC_EPI_TANH_RELU:
      if (!d.out_f32 && !d.out_hi) return RNC_ERR_BAD_POINTER;
      if ((d.cout % 32) != 0 && d.epilogue != RNC_EPI_RELU_FLOW) {
        // the epilogue stores whole 32-channel chunks: the destination must have room for the padded tail
        const int cpad = (d.cout + 31) / 32 * 32;
        if ((d.out_f32 && d.ldo_f32 < cpad) || (d.out_hi && d.ldo_split < cpad)) return RNC_ERR_BAD_SHAPE;
      }
      if (d.epilogue == RNC_EPI_TANH_RELU && (d.cout % 64) != 0) return RNC_ERR_BAD_SHAPE;
      break;
    case RNC_EPI_FLOW_DELTA:
      if (!d.aux0 || d.cout != 2 || d.out_hi) return RNC_ERR_BAD_SHAPE;
      break;
    case RNC_EPI_GRU_ZR:
      if (!d.out_hi || !d.aux0 || !d.h || (d.cout % 64) != 0 || (d.ldaux & 3) || (d.ldh & 3)) return RNC_ERR_BAD_POINTER;
      break;
    case RNC_EPI_GRU_Q:
      if (!d.aux0 || !d.h || (d.cout % 32) != 0 || (d.ldaux & 3) || (d.ldh & 3)) return RNC_ERR_BAD_POINTER;
      break;
    default: return RNC_ERR_UNSUPPORTED;
  }
  if (!encode_fn()) return RNC_ERR_UNSUPPORTED;

  // ---- tile shape and A-staging mode
  Params p;
  p.B = d.B; p.H = d.H; p.W = d.W;
  p.kh = d.kh; p.kw = d.kw; p.ph = d.kh / 2; p.pw = d.kw / 2; p.stride = stride; p.sx = window ? 1 : stride;
  int mode = MODE_TAP;
  if (stride == 1 && (d.flags & RNC_CONV_NO_HALO) == 0) {
    if (d.kw > 1 && d.W > 64) mode = MODE_ROWHALO;                 // one image row x 128 px per tile
    else if (d.kw == 1 && d.kh > 1 && d.W >= 16 && d.H >= 8) mode = MODE_COLHALO;
  }
  int TW, TH, box_w, box_h;
  if (mode == MODE_ROWHALO) { TW = 128; TH = 1; box_w = 136; box_h = 1; }
  else if (mode == MODE_COLHALO) { TW = 16; TH = 8; box_w = 16; box_h = TH + 2 * p.ph; }
  else {
    TW = 8;
    while (TW < d.W && TW < kBM) TW <<= 1;
    TH = kBM / TW; box_w = TW; box_h = TH;
  }
  if (box_w * box_h > 256 - 8 && mode == MODE_COLHALO) return RNC_ERR_UNSUPPORTED;   // kh <= 9
  p.mode = mode; p.TW = TW; p.TH = TH;
  {
    static const char* env = getenv("RNC_CONV_PROBE_NOB");
    p.probe_nob = env != nullptr && env[0] == '1';
  }
  p.tiles_x = (d.W + TW - 1) / TW; p.tiles_y = (d.H + TH - 1) / TH;
  p.ntiles = d.B * p.tiles_x * p.tiles_y; p.ntn = d.coutpad / bn;
  p.a_plane = box_w * box_h * 128;
  // tall halo boxes (COLHALO, kh >= 5) beside 128-column weight stages leave no room for two stages of each ring
  while (bn > 32 && 2 * 2 * p.a_plane + 2 * 2 * bn * bk * (tf32 ? 4 : 2) > kRingBudget && d.coutpad % (bn >> 1) == 0) bn >>= 1;
  p.ntn = d.coutpad / bn;
  p.nblk0 = nblk0; p.nblk = nblk; p.bk = bk; p.tf32 = tf32 ? 1 : 0;
  p.cout = d.cout; p.epilogue = d.epilogue; p.unscale = d.unscale; p.bias = d.bias;
  p.out_f32 = d.out_f32; p.ldo_f32 = d.ldo_f32;
  p.out_hi = static_cast<__half*>(d.out_hi); p.out_lo = static_cast<__half*>(d.out_lo); p.ldo_split = d.ldo_split;
  p.h = d.h; p.ldh = d.ldh; p.aux0 = d.aux0; p.ldaux = d.ldaux; p.res = d.res; p.ldres = d.ldres;
  p.stats = d.stats;
  p.add = d.add; p.ldadd = d.ldadd;
  p.aux_blocked = (d.flags & RNC_CONV_AUX_BLOCKED) ? 1 : 0;
  p.out_blocked = (d.flags & RNC_CONV_OUT_BLOCKED) ? 1 : 0;
  if (p.out_blocked && (d.epilogue != RNC_EPI_LINEAR || d.out_hi || d.stats)) return RNC_ERR_UNSUPPORTED;
  if (p.aux_blocked && d.epilogue != RNC_EPI_GRU_ZR && d.epilogue != RNC_EPI_GRU_Q) return RNC_ERR_UNSUPPORTED;

  CUtensorMap maps[9];
  const long long pitch0 = window ? d.win_pitch : 0;
  bool ok = make_in_map(&maps[0], d.in0_hi, d.c0, d.ld0, d.B, Hin, Win, box_w, box_h, p.sx, stride, tf32, pitch0) &&
            make_in_map(&maps[1], d.in0_lo, d.c0, d.ld0, d.B, Hin, Win, box_w, box_h, p.sx, stride, tf32, pitch0);
  if (d.c1 > 0) {
    ok = ok && make_in_map(&maps[2], d.in1_hi, d.c1, d.ld1, d.B, Hin, Win, box_w, box_h, stride, stride, tf32) &&
         make_in_map(&maps[3], d.in1_lo, d.c1, d.ld1, d.B, Hin, Win, box_w, box_h, stride, stride, tf32);
  } else {
    maps[2] = maps[0]; maps[3] = maps[1];
  }
  ok = ok && make_w_map(&maps[4], d.w_hi, d.ktot, d.coutpad, bn, tf32) &&
       make_w_map(&maps[5], d.w_lo, d.ktot, d.coutpad, bn, tf32);
  // epilogue stores: out_hi / out_lo (and h for the q gate) as boxes of 32 channels x one epilogue warp's 32 pixels
  {
    const int obw = TW < 32 ? TW : 32, obh = 32 / obw;
    const int flow2 = d.epilogue == RNC_EPI_RELU_FLOW ? 2 : 0;
    const int cw = d.epilogue == RNC_EPI_GRU_ZR ? d.cout / 2 : (d.cout + flow2 + 31) / 32 * 32;
    if (d.out_hi) {
      if ((d.ldo_split & 7) || !aligned16(d.out_hi) || !aligned16(d.out_lo) || d.ldo_split < cw) return RNC_ERR_BAD_POINTER;
      ok = ok && make_out_map(&maps[6], d.out_hi, cw, d.ldo_split, d.B, d.H, d.W, obw, obh, false) &&
           make_out_map(&maps[7], d.out_lo, cw, d.ldo_split, d.B, d.H, d.W, obw, obh, false);
    } else {
      maps[6] = maps[0]; maps[7] = maps[0];
    }
    if (d.epilogue == RNC_EPI_GRU_Q) {
      if (!aligned16(d.h) || d.ldh < d.cout || d.out_f32) return RNC_ERR_BAD_POINTER;
      ok = ok && make_out_map(&maps[8], d.h, d.cout, d.ldh, d.B, d.H, d.W, obw, obh, true);
    } else if (d.out_f32 && !p.out_blocked && d.epilogue != RNC_EPI_FLOW_DELTA) {
      const int cf = d.epilogue == RNC_EPI_TANH_RELU ? d.cout / 2 : (d.cout + 31) / 32 * 32;   // TANH_RELU: only the tanh half
      if (d.ldo_f32 < cf) return RNC_ERR_BAD_SHAPE;
      ok = ok && make_out_map(&maps[8], d.out_f32, cf, d.ldo_f32, d.B, d.H, d.W, obw, obh, true);
    } else {
      maps[8] = maps[0];
    }
  }
  if (!ok) return RNC_ERR_BAD_SHAPE;

  cudaStream_t s = as_stream(stream);
  const int msa = (d.flags >> 8) & 15, msb = (d.flags >> 12) & 15;
  const bool plain = (d.epilogue == RNC_EPI_LINEAR || d.epilogue == RNC_EPI_RELU || d.epilogue == RNC_EPI_SIGMOID) && !d.stats;
  const int ec = d.epilogue == RNC_EPI_GRU_ZR ? EC_GRU_ZR : d.epilogue == RNC_EPI_GRU_Q ? EC_GRU_Q : plain ? EC_PLAIN : EC_MISC;
  switch (ec) {
    case EC_GRU_ZR: return launch_bn<EC_GRU_ZR>(bn, maps, p, s, msa, msb);
    case EC_GRU_Q: return launch_bn<EC_GRU_Q>(bn, maps, p, s, msa, msb);
    case EC_MISC: return launch_bn<EC_MISC>(bn, maps, p, s, msa, msb);
    default: return launch_bn<EC_PLAIN>(bn, maps, p, s, msa, msb);
  }
}
