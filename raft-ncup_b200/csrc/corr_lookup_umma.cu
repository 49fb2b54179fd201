// Tensor-core fused correlation lookup (v2 of corr_lookup.cu; same math, SURVEY.md Appendix A.1; replaces
// core/corr.py:7-55 + core/utils/utils.py:59-73).  The 4-D volume is never built: per tile of 8x16 query pixels the
// kernel computes, with wgmma, the dot products of the tile's 128 fmap1 vectors against a bounding box of fmap2^l
// positions that covers every pixel's 10x10 lattice window, then each pixel gathers its own window from the
// accumulator and blends it bilinearly.
//
//   A  = fmap1 tile      [128 px][256 ch] halves, TMA box {64,16,8,1} x 4 K-blocks, resident while its levels are processed
//   B  = fmap2^l box     chunks of <= 128 positions x 256 ch streamed through a ring of 16 KB stages as TMA boxes of the
//                        needed rows {64, BW, rows, 1}; only the box rows some window needs are loaded and multiplied (N is
//                        set per chunk); out-of-image positions are zero-filled by TMA = the reference's zero padding
//                        (grid_sample padding_mode='zeros')
//   D  = [128][<=128] fp32 in the registers of one warpgroup (two M = 64 halves), staged to shared memory per chunk
//
// Persistent CTAs (one per SM) walk work units (tile, level); a producer warp and the consumer warpgroup are decoupled by
// mbarrier rings, so the loads of the next chunks and units overlap the MMAs and the epilogue of the current one.
//
// Epilogue (thread = pixel): the chunk's accumulator is staged as [pixel][129 words] (odd pitch: the gather's scalar loads
// of 32 pixels hit distinct banks); each pixel reads the 10 lattice values of its window row, interpolates in x, combines
// with the previous row in y -> 9 outputs (fixed j, i = 0..8), which are split into hi/lo halves (the tensor-core
// convolutions' operand format) and stored straight into the level's output tile in shared memory; the tile leaves with one
// TMA store per plane and warp.
//
// Output channel order inside a level (kLvlStride = 88 channels; consumed only by convc1, whose weights are permuted to
// match at pack time — the reference order k = i*9 + j exists only in the seam API, corr_lookup.cu):
//     tap (i, j), i < 8  ->  j*8 + i          tap (8, j)  ->  72 + j          81..87 = zero pads
// so the 8 values a thread produces per window row are ONE aligned 16-byte store per plane instead of 9 scattered words,
// and no second pass re-reads / re-packs the level.
//
// Units whose windows do not fit the fixed boxes (incoherent flow) are flagged and recomputed exactly in fp32 by the same
// CTA after its tensor-core units (exact_unit), so the result never depends on the coherence assumption.
//
// Precision: fmaps are rounded once to fp16 (fp32 accumulate): 2.4e-4 EPE after 32 iterations in SURVEY.md Appendix D.
#include <type_traits>

#include "umma_ptx.cuh"

namespace rnc {
namespace lookup_umma {

using namespace rnc::umma;

constexpr int kThreads = 160;            // warps 0-3: consumer warpgroup (wgmma + epilogue, thread = pixel), warp 4: TMA producer
constexpr int kTY = 8, kTX = 16;         // query tile (level-0 pixels)
constexpr int kD = 256;                  // feature channels
constexpr int kKB = kD / 64;             // K blocks of 64 halves
constexpr int kLevels = 4;
constexpr int kS = 9, kG = 10, kR = 4;
// per-level box: width, rows per chunk, chunks.  Union boxes seen on the benchmark stimuli at iteration 31: 28x24, 19x17,
// 15x14, 13x12; anything larger is handled by the exact fallback.  Chunks of <= 128 MMA columns (the accumulator of 128
// pixels x 128 columns is 128 registers per consumer thread): 4x32, 4x24, 8x16, 8x16 positions; boxes 32x24, 24x24, 16x24.
__host__ __device__ constexpr int box_w(int l) { return l == 0 ? 32 : l == 1 ? 24 : 16; }
__host__ __device__ constexpr int chunk_rows(int l) { return l <= 1 ? 4 : 8; }
__host__ __device__ constexpr int n_chunks(int l) { return l <= 1 ? 6 : 3; }
__host__ __device__ constexpr int box_h(int l) { return chunk_rows(l) * n_chunks(l); }
__host__ __device__ constexpr int chunk_n(int l) { return box_w(l) * chunk_rows(l); }
constexpr int kChunkN = 128;
static_assert(chunk_n(0) <= kChunkN && chunk_n(1) <= kChunkN && chunk_n(2) <= kChunkN, "chunk wider than the accumulator");
constexpr int kStages = 3;               // B ring
constexpr int kATile = 128 * 64 * 2;     // 16 KB per K block
constexpr int kBStage = kChunkN * 64 * 2;    // 16 KB: 128 positions x 64 halves
constexpr int kLvlStride = 88;           // channels per level in the output row (81 taps + 7 zero pads): 16-byte groups
constexpr int kTiRing = 4;               // unit records in flight between the producer and the consumers (power of two)
constexpr int kTiShift = 2;
constexpr int kSmemA = kKB * kATile;                         // 64 KB
constexpr int kSmemB = kStages * kBStage;                    // 48 KB
// output tile of one (tile, level) unit: [plane hi | lo][128 px][88 halves], dense = the TMA store's box {88, 16, 2} per warp
constexpr int kStgPlane = 128 * kLvlStride * 2;              // 22 KB
constexpr int kSmemStage = 2 * kStgPlane;                    // 44 KB
constexpr int kAccPitch = kChunkN + 1;                       // words per pixel of the staged accumulator chunk
constexpr int kSmemAcc = 128 * kAccPitch * 4;                // 64.5 KB
static_assert((32 * kLvlStride * 2) % 128 == 0, "TMA store sources must be 128-byte aligned");
constexpr int kSmemTotal = kSmemA + kSmemB + kSmemStage + kSmemAcc + 1024 + 512;

struct Params {
  const float* f1_cl; const float* f2_pyr;   // fp32 originals: exact path of the units whose windows do not fit the boxes
  const float* coords;                 // [B][2][H][W]
  __half* out_hi; __half* out_lo; int ldo;
  int* flags;                          // [tiles][4 levels]: 1 = recompute this tile with the exact kernel
  int B, H, W, tiles_x, tiles_y;
  int tile_major;                      // unit schedule: 0 level-major, 1 tile-major, 2 hybrid (see unit_at)
  float scale;
};

// fmap2^l boxes of every even row count up to the chunk height per level: the rows a chunk needs are ONE TMA operation
constexpr int kBoxKinds = 4;
static_assert(2 * kBoxKinds >= chunk_rows(0) && 2 * kBoxKinds >= chunk_rows(2), "a box kind per even row count of a chunk");
struct LevelMaps { CUtensorMap m[kLevels][kBoxKinds]; };

struct TileInfo {                      // shared: origin of the unit's union box (0,0 when no window is live), the box rows
  int bx0, by0, overflow, nrows;       // actually needed (even, <= box_h; 0 = no live window): only those are loaded / multiplied
};

// Window origin of one pixel at one level (shared by the producer's box computation and the epilogue's gather).
__device__ __forceinline__ bool window_origin(float cx, float cy, float inv, int Hl, int Wl, int& ix0, int& iy0) {
  ix0 = static_cast<int>(floorf(cx * inv)) - kR;
  iy0 = static_cast<int>(floorf(cy * inv)) - kR;
  return !(ix0 + kG - 1 < 0 || ix0 > Wl - 1 || iy0 + kG - 1 < 0 || iy0 > Hl - 1);   // false: window fully outside -> zeros
}

__device__ __forceinline__ float clamp_coord(float v) { return fminf(fmaxf(v, -1.0e6f), 1.0e6f); }

// The consumer warpgroup's view of the operand rings and of the staged accumulator.
struct MmaCtx {
  uint32_t a_base, b_base;
  uint64_t* a_full; uint64_t* a_empty; uint64_t* b_full; uint64_t* b_empty;
  float* acc;                          // [128 px][kAccPitch]
  int it, na;                          // B ring position, A tile uses
};

struct EpiCtx {
  const Params& p; const TileInfo* ti; __half* stage;
  int b, y0, x0, lg, ml, lane; bool valid; float cx, cy;
  bool load_a, free_a;                 // the unit's first chunk waits for the A tile / its last chunk releases it
};

// Accumulator rows of one chunk: N columns = the positions of the rows the chunk holds (two M = 64 halves), K = 256.
template <int N>
__device__ __forceinline__ void chunk_mma(MmaCtx& m, float* d0, float* d1, bool wait_a, bool free_a) {
  for (int kb = 0; kb < kKB; ++kb, ++m.it) {
    const int s = m.it % kStages, ph = (m.it / kStages) & 1;
    if (wait_a) mbar_wait(&m.a_full[kb], m.na & 1);
    mbar_wait(&m.b_full[s], ph);
    const uint64_t ad = smem_desc_sw128(m.a_base + kb * kATile), bd = smem_desc_sw128(m.b_base + s * kBStage);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      wgmma<N, false>(d0, ad + 2 * kk, bd + 2 * kk, (kb | kk) != 0);
      wgmma<N, false>(d1, ad + (64 * 128 >> 4) + 2 * kk, bd + 2 * kk, (kb | kk) != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {
      mbar_arrive(&m.b_empty[s]);
      if (free_a) mbar_arrive(&m.a_empty[kb]);   // this K block of A is free for the next tile
    }
  }
}

// One chunk: MMAs into registers, then the accumulator -> shared memory [pixel][column] (every consumer thread first waits
// until all have finished reading the previous chunk).
__device__ __forceinline__ void chunk_acc(MmaCtx& m, int nn, bool wait_a, bool free_a) {
  float d0[kChunkN / 2], d1[kChunkN / 2];
  switch (nn) {
    case 32: chunk_mma<32>(m, d0, d1, wait_a, free_a); break;
    case 48: chunk_mma<48>(m, d0, d1, wait_a, free_a); break;
    case 64: chunk_mma<64>(m, d0, d1, wait_a, free_a); break;
    case 96: chunk_mma<96>(m, d0, d1, wait_a, free_a); break;
    default: chunk_mma<128>(m, d0, d1, wait_a, free_a); break;
  }
#pragma unroll
  for (int i = 0; i < kChunkN / 2; ++i) { reg_fence(d0[i]); reg_fence(d1[i]); }
  named_bar_sync(1, 128);
  const int lane = threadIdx.x & 31, r = 16 * (threadIdx.x >> 5) + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < kChunkN / 8; ++j) {
    if (8 * j >= nn) break;
    float* p0 = m.acc + r * kAccPitch + 8 * j + c;
    p0[0] = d0[4 * j]; p0[1] = d0[4 * j + 1];
    p0[8 * kAccPitch] = d0[4 * j + 2]; p0[8 * kAccPitch + 1] = d0[4 * j + 3];
    float* p1 = p0 + 64 * kAccPitch;
    p1[0] = d1[4 * j]; p1[1] = d1[4 * j + 1];
    p1[8 * kAccPitch] = d1[4 * j + 2]; p1[8 * kAccPitch + 1] = d1[4 * j + 3];
  }
  named_bar_sync(1, 128);
}

// Rows of one level (box width BW columns) for the warp's 32 pixels, two box rows per step, so that two independent
// gather -> interpolate chains are in flight.
template <int BW>
__device__ __forceinline__ void lookup_level_rows(const EpiCtx& c, MmaCtx& m, int l, bool live, int ox, int oy, float ax, float ay) {
  const Params& p = c.p;
  const int cr = chunk_rows(l);
  __half* sth = c.stage + c.ml * kLvlStride;                  // this pixel's row of the level's output tile, hi plane
  __half* stl = sth + 128 * kLvlStride;                       // lo plane
  // window row j of this pixel is complete: taps (0..7, j) -> one 16-byte store per plane, tap (8, j) -> the tail
  auto emit = [&](int j, const float (&o)[kS]) {
    uint32_t hh[4], ll[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) split_pair(o[2 * q], o[2 * q + 1], hh[q], ll[q]);
    *reinterpret_cast<uint4*>(sth + j * 8) = make_uint4(hh[0], hh[1], hh[2], hh[3]);
    *reinterpret_cast<uint4*>(stl + j * 8) = make_uint4(ll[0], ll[1], ll[2], ll[3]);
    uint32_t h8, l8;
    split_pair(o[8], 0.f, h8, l8);
    reinterpret_cast<unsigned short*>(sth)[72 + j] = static_cast<unsigned short>(h8 & 0xffffu);
    reinterpret_cast<unsigned short*>(stl)[72 + j] = static_cast<unsigned short>(l8 & 0xffffu);
  };
  const float wx1 = ax * p.scale, wx0 = p.scale - wx1, wy0 = 1.f - ay;   // the 1/sqrt(D) scale rides on the x weights
  // warp-uniform range of box rows that any pixel of this warp (2 tile rows) actually needs
  const int row_lo = __reduce_min_sync(0xffffffffu, live ? oy : 0x7fffffff);
  const int row_hi = __reduce_max_sync(0xffffffffu, live ? oy + kG - 1 : -1);
  float hprev[kS];
#pragma unroll
  for (int i = 0; i < kS; ++i) hprev[i] = 0.f;
  const float* gbase = m.acc + c.ml * kAccPitch + (live ? ox : 0);

  // one step: chunk rows r, r + 1 (TWO); cidx = lattice row of the pixel's window held by box row `row`
  auto step = [&](int r, int row, auto two_tag) {
    constexpr bool TWO = decltype(two_tag)::value;
    const float* gp = gbase + r * BW;
    const int cidx = row - oy;
    float g0[kG], g1[kG], h0[kS], h1[kS];
#pragma unroll
    for (int a = 0; a < kG; ++a) g0[a] = gp[a];
    if (TWO) {
#pragma unroll
      for (int a = 0; a < kG; ++a) g1[a] = gp[BW + a];
    }
#pragma unroll
    for (int i = 0; i < kS; ++i) h0[i] = wx0 * g0[i] + wx1 * g0[i + 1];
    if (TWO) {
#pragma unroll
      for (int i = 0; i < kS; ++i) h1[i] = wx0 * g1[i] + wx1 * g1[i + 1];
    }
    if (live && cidx >= 1 && cidx < kG) {
      float o[kS];
#pragma unroll
      for (int i = 0; i < kS; ++i) o[i] = wy0 * hprev[i] + ay * h0[i];
      emit(cidx - 1, o);
    }
    if (TWO && live && cidx >= 0 && cidx < kG - 1) {
      float o[kS];
#pragma unroll
      for (int i = 0; i < kS; ++i) o[i] = wy0 * h0[i] + ay * h1[i];
      emit(cidx, o);
    }
#pragma unroll
    for (int i = 0; i < kS; ++i) hprev[i] = TWO ? h1[i] : h0[i];
  };

  const int nch = (c.ti->nrows + cr - 1) / cr;
  for (int cc = 0; cc < nch; ++cc) {
    const int nn = min(cr, c.ti->nrows - cc * cr) * BW;
    chunk_acc(m, nn, cc == 0 && c.load_a, cc == nch - 1 && c.free_a);
    const int r0 = max(0, row_lo - cc * cr), r1 = min(cr - 1, row_hi - cc * cr);   // rows of this chunk the warp needs
    for (int r = r0; r <= r1; r += 2) {
      if (r + 1 <= r1) step(r, cc * cr + r, std::true_type{}); else step(r, cc * cr + r, std::false_type{});
    }
  }
}

// Epilogue of one warp (thread = pixel) for one unit = (tile, level l): rows into the output tile, then one TMA store per
// plane of the warp's 2 x 16 pixels (the TMA unit clips pixels beyond the image).
__device__ __forceinline__ void lookup_epilogue(const EpiCtx& c, MmaCtx& m, int l, const CUtensorMap* map_hi, const CUtensorMap* map_lo) {
  const Params& p = c.p;
  __half* sth = c.stage + c.ml * kLvlStride;
  __half* stl = sth + 128 * kLvlStride;
  const float inv = 1.f / static_cast<float>(1 << l);
  const float sx = c.cx * inv, sy = c.cy * inv;
  const float ax = sx - floorf(sx), ay = sy - floorf(sy);
  int ix0, iy0;
  const bool empty = !window_origin(c.cx, c.cy, inv, p.H >> l, p.W >> l, ix0, iy0);
  const int ox = ix0 - c.ti->bx0, oy = iy0 - c.ti->by0;
  const bool live = c.valid && !empty;
  // the previous unit's TMA stores have finished READING this lane group's rows of the output tile
  if (c.lane == 0) bulk_wait_read0();
  __syncwarp();
  if (!live) {                                 // window fully outside the level image (or pixel outside the frame): zeros
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int q = 0; q < 10; ++q) {
      *reinterpret_cast<uint4*>(sth + q * 8) = z;
      *reinterpret_cast<uint4*>(stl + q * 8) = z;
    }
    reinterpret_cast<unsigned short*>(sth)[80] = 0;
    reinterpret_cast<unsigned short*>(stl)[80] = 0;
  }
  if (l == 0) lookup_level_rows<box_w(0)>(c, m, l, live, ox, oy, ax, ay);
  else if (l == 1) lookup_level_rows<box_w(1)>(c, m, l, live, ox, oy, ax, ay);
  else lookup_level_rows<box_w(2)>(c, m, l, live, ox, oy, ax, ay);
  static_assert(box_w(2) == box_w(3), "levels 2 and 3 share the row code");
  fence_proxy_async();                         // this thread's shared-memory writes are visible to the TMA unit
  __syncwarp();
  if (c.lane == 0) {
    const __half* src = c.stage + c.lg * 32 * kLvlStride;
    tma_store_4d(map_hi, src, l * kLvlStride, c.x0, c.y0 + 2 * c.lg, c.b);
    tma_store_4d(map_lo, src + 128 * kLvlStride, l * kLvlStride, c.x0, c.y0 + 2 * c.lg, c.b);
    bulk_commit();
  }
}

// Work units.  A unit is (tile, level): up to 6, 6, 3, 3 accumulator chunks.  Schedules (Params.tile_major):
//   0  level-major: units listed level-major (all level-0 units first = longest first) and dealt to the CTAs in snake order
//      (round k runs left-to-right for even k, right-to-left for odd k); every unit loads its own A tile
//   1  tile-major: the four levels of a tile back to back on one CTA, A loaded once per tile (4x less A traffic, no A reload
//      bubble between levels), but whole tiles balance badly (B=8: 448 tiles on 132 CTAs -> the busiest CTA gets 4)
//   2  hybrid (default): the complete rounds of tiles (floor(ntiles / CTAs) per CTA) tile-major, the remaining tiles
//      level-major over all CTAs.  B=8: 3 tile-major rounds, then 52 tiles' units over all CTAs, with a quarter of the
//      A loads; a single image (56 tiles < 132 CTAs) is all level-major and still fills the SMs.
// Returns the k-th unit of this CTA as (tile-major flag << 30) | (level * ntiles + tile), or -1 (none in round k).
constexpr int kUnitTm = 1 << 30;
__device__ __forceinline__ int unit_id(int u) { return u & (kUnitTm - 1); }
__device__ __forceinline__ bool unit_tm(int u) { return (u & kUnitTm) != 0; }
__device__ __forceinline__ int unit_at(int k, int ntiles, int mode) {
  const int G = gridDim.x, c = blockIdx.x;
  const int full = mode == 0 ? 0 : mode == 1 ? (ntiles + G - 1) / G : ntiles / G;      // tile-major rounds
  if (k < full * kLevels) {
    const int tile = (k / kLevels) * G + c;
    return tile < ntiles ? kUnitTm | ((k % kLevels) * ntiles + tile) : -1;
  }
  if (mode == 1) return -1;
  const int kk = k - full * kLevels, done = full * G, rem = ntiles - done;             // remaining tiles, level-major snake
  const int g = kk * G + ((kk & 1) ? G - 1 - c : c);
  if (g >= rem * kLevels) return -1;
  const int l = g / rem;
  return l * ntiles + done + (g - l * rem);
}
__device__ __forceinline__ int unit_rounds(int ntiles, int mode) {
  const int G = gridDim.x;
  if (mode == 1) return ((ntiles + G - 1) / G) * kLevels;
  const int full = mode == 0 ? 0 : ntiles / G;
  return full * kLevels + ((ntiles - full * G) * kLevels + G - 1) / G;
}

// Exact fp32 recomputation of one (tile, level) unit whose windows did not fit the fixed box (incoherent flow, e.g. a motion
// boundary): warp = pixel, the 100 lattice dot products of the pixel's window straight from the fp32 feature maps (lane = 8
// channels, positions outside the level image contribute 0 = grid_sample's zero padding), then the bilinear blend of
// SURVEY.md Appendix A.1 and the same hi/lo split output in the resident channel order.  Runs on all warps of the CTA after
// its tensor-core units: results never depend on a coherence assumption, and there is no second kernel launch.
__device__ __noinline__ void exact_unit(const Params& p, int l, int tile, float* gsm, int warp, int lane, int nwarps) {
  const int tpi = p.tiles_x * p.tiles_y, HW = p.H * p.W;
  const int b = tile / tpi, tr = tile - b * tpi;
  const int y0 = (tr / p.tiles_x) * kTY, x0 = (tr % p.tiles_x) * kTX;
  const int Hl = p.H >> l, Wl = p.W >> l;
  size_t off = 0;
  for (int k = 0; k < l; ++k) off += static_cast<size_t>(p.B) * (p.H >> k) * (p.W >> k) * kD;
  const float* f2l = p.f2_pyr + off + static_cast<size_t>(b) * Hl * Wl * kD;
  const float inv = 1.f / static_cast<float>(1 << l);
  float* g = gsm + warp * 104;
  for (int px = warp; px < kTY * kTX; px += nwarps) {
    const int qy = y0 + (px >> 4), qx = x0 + (px & 15);
    if (qy >= p.H || qx >= p.W) continue;                       // warp-uniform
    const float cx = clamp_coord(__ldg(p.coords + (static_cast<size_t>(b) * 2 + 0) * HW + qy * p.W + qx));
    const float cy = clamp_coord(__ldg(p.coords + (static_cast<size_t>(b) * 2 + 1) * HW + qy * p.W + qx));
    const float sx = cx * inv, sy = cy * inv;
    const float fx0 = floorf(sx), fy0 = floorf(sy), ax = sx - fx0, ay = sy - fy0;
    const int ix0 = static_cast<int>(fx0) - kR, iy0 = static_cast<int>(fy0) - kR;
    const float4* f1p = reinterpret_cast<const float4*>(p.f1_cl + (static_cast<size_t>(b) * HW + qy * p.W + qx) * kD);
    const float4 a0 = __ldg(f1p + lane), a1 = __ldg(f1p + 32 + lane);
    // lattice (a = x offset, c = y offset) -> g[a*10 + c]; five positions per pass so that their loads are in flight together
    for (int c = 0; c < kG; ++c) {
      const int Y = iy0 + c;
      const bool rowin = Y >= 0 && Y < Hl;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        float4 b0[5], b1[5];
#pragma unroll
        for (int u = 0; u < 5; ++u) {
          const int X = ix0 + half * 5 + u;
          const bool in = rowin && X >= 0 && X < Wl;              // warp-uniform
          const float4* q = reinterpret_cast<const float4*>(f2l + (static_cast<size_t>(in ? Y : 0) * Wl + (in ? X : 0)) * kD);
          b0[u] = in ? __ldg(q + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
          b1[u] = in ? __ldg(q + 32 + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < 5; ++u) {
          float d = a0.x * b0[u].x;
          d = fmaf(a0.y, b0[u].y, d); d = fmaf(a0.z, b0[u].z, d); d = fmaf(a0.w, b0[u].w, d);
          d = fmaf(a1.x, b1[u].x, d); d = fmaf(a1.y, b1[u].y, d); d = fmaf(a1.z, b1[u].z, d); d = fmaf(a1.w, b1[u].w, d);
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
          if (lane == 0) g[(half * 5 + u) * kG + c] = d * p.scale;
        }
      }
    }
    __syncwarp();
    const size_t base = (static_cast<size_t>(b) * HW + qy * p.W + qx) * p.ldo + l * kLvlStride;
    for (int t = lane; t < kS * kS; t += 32) {
      const int i = t / kS, j = t - i * kS;
      const float* gp = g + i * kG + j;
      const float v = (1.f - ax) * (1.f - ay) * gp[0] + ax * (1.f - ay) * gp[kG] + (1.f - ax) * ay * gp[1] + ax * ay * gp[kG + 1];
      uint32_t hh, ll;
      split_pair(v, 0.f, hh, ll);
      const size_t k = base + (i < 8 ? j * 8 + i : 72 + j);
      reinterpret_cast<unsigned short*>(p.out_hi)[k] = static_cast<unsigned short>(hh & 0xffffu);
      reinterpret_cast<unsigned short*>(p.out_lo)[k] = static_cast<unsigned short>(ll & 0xffffu);
    }
    if (lane < kLvlStride - kS * kS) {                          // the level's zero pads
      reinterpret_cast<unsigned short*>(p.out_hi)[base + kS * kS + lane] = 0;
      reinterpret_cast<unsigned short*>(p.out_lo)[base + kS * kS + lane] = 0;
    }
    __syncwarp();
  }
}

// Persistent kernel: one CTA per SM walks its work units.  The producer warp runs ahead of the consumers through mbarrier
// rings, so the TMA loads of the next chunks (and of the next unit) overlap the MMAs and the epilogue of the current one:
//   warp 4      producer: loads the tile's coords, reduces the per-level union boxes, publishes them (ti ring), then streams
//               A (per K block, as soon as the previous tile's last chunk released it) and the B chunks
//   warps 0-3   consumer warpgroup: wgmma per chunk, accumulator -> shared memory, gather + bilinear blend + store
__global__ void __launch_bounds__(kThreads, 1)
corr_lookup_umma_kernel(const __grid_constant__ CUtensorMap mF1, const __grid_constant__ LevelMaps mLv,
                        const __grid_constant__ CUtensorMap mOutHi,
                        const __grid_constant__ CUtensorMap mOutLo, const Params p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // 1024-aligned, stays in the shared window
  unsigned char* sA = smem;
  unsigned char* sB = smem + kSmemA;
  __half* stage = reinterpret_cast<__half*>(smem + kSmemA + kSmemB);
  float* acc = reinterpret_cast<float*>(smem + kSmemA + kSmemB + kSmemStage);
  unsigned char* tail = smem + kSmemTotal - 1024 - 512;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(tail);       // [kKB]
  uint64_t* a_empty = a_full + kKB;                           // [kKB]
  uint64_t* b_full = a_empty + kKB;
  uint64_t* b_empty = b_full + kStages;
  uint64_t* ti_full = b_empty + kStages;                      // [kTiRing]
  uint64_t* ti_empty = ti_full + kTiRing;                     // [kTiRing]
  int* ov_count = reinterpret_cast<int*>(ti_empty + kTiRing); // units of this CTA that overflowed their box
  TileInfo* ti = reinterpret_cast<TileInfo*>(ov_count + 2);   // [kTiRing]

  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tpi = p.tiles_x * p.tiles_y;
  const int ntiles = p.B * tpi;
  const int HW = p.H * p.W;

  if (threadIdx.x == 0) {
    *ov_count = 0;
    for (int kb = 0; kb < kKB; ++kb) { mbar_init(&a_full[kb], 1); mbar_init(&a_empty[kb], 4); }
    for (int s = 0; s < kStages; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 4); }
    for (int i = 0; i < kTiRing; ++i) { mbar_init(&ti_full[i], 1); mbar_init(&ti_empty[i], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();                          // coords1 of the previous iteration's flow update is visible from here

  const int sched = p.tile_major;
  const int rounds = unit_rounds(ntiles, sched);

  if (warp == 4) {
    // ------------------------------------------------------------------ producer (warp-uniform loops, one elected lane issues)
    // lane owns pixels lane, lane+32, lane+64, lane+96 of the tile for the box reduction
    float pcx[4], pcy[4];
    auto load_coords = [&](int tile, float (&ox)[4], float (&oy)[4]) {
      const int b = tile / tpi, tr = tile - b * tpi;
      const int y0 = (tr / p.tiles_x) * kTY, x0 = (tr % p.tiles_x) * kTX;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int ml = lane + 32 * j, py = y0 + (ml >> 4), px = x0 + (ml & 15);
        const bool v = py < p.H && px < p.W;
        ox[j] = v ? clamp_coord(__ldg(p.coords + (static_cast<size_t>(b) * 2 + 0) * HW + py * p.W + px)) : __int_as_float(0x7fc00000);
        oy[j] = v ? clamp_coord(__ldg(p.coords + (static_cast<size_t>(b) * 2 + 1) * HW + py * p.W + px)) : 0.f;
      }
    };
    // record of one unit: union box origin, rows needed, overflow
    struct Rec { int bx0, by0, nrows, ov; };
    auto make_rec = [&](int unit, const float (&ux)[4], const float (&uy)[4]) {
      const int l = unit_id(unit) / ntiles;
      const float inv = 1.f / static_cast<float>(1 << l);
      int lx0 = 0x7fffffff, ly0 = 0x7fffffff, lx1 = -0x7fffffff, ly1 = -0x7fffffff;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int ix0, iy0;
        if (ux[j] == ux[j] && window_origin(ux[j], uy[j], inv, p.H >> l, p.W >> l, ix0, iy0)) {   // NaN marks a pixel outside the image
          lx0 = min(lx0, ix0); ly0 = min(ly0, iy0); lx1 = max(lx1, ix0 + kG - 1); ly1 = max(ly1, iy0 + kG - 1);
        }
      }
      lx0 = __reduce_min_sync(0xffffffffu, lx0); ly0 = __reduce_min_sync(0xffffffffu, ly0);
      lx1 = __reduce_max_sync(0xffffffffu, lx1); ly1 = __reduce_max_sync(0xffffffffu, ly1);
      const bool any = lx1 >= lx0;
      Rec r;
      r.ov = any && (lx1 - lx0 + 1 > box_w(l) || ly1 - ly0 + 1 > box_h(l)) ? 1 : 0;
      r.bx0 = any ? lx0 : 0; r.by0 = any ? ly0 : 0;
      r.nrows = any ? min((ly1 - ly0 + 2) & ~1, box_h(l)) : 0;
      return r;
    };
    int n = 0;
    auto publish = [&](int unit, const Rec& r) {
      const int slot = n & (kTiRing - 1);
      mbar_wait(&ti_empty[slot], ((n >> kTiShift) & 1) ^ 1);
      if (lane == 0) {
        ti[slot].bx0 = r.bx0; ti[slot].by0 = r.by0; ti[slot].overflow = r.ov; ti[slot].nrows = r.nrows;
        const int l = unit_id(unit) / ntiles;
        p.flags[(unit_id(unit) - l * ntiles) * kLevels + l] = r.ov;
        if (r.ov) *ov_count += 1;
        mbar_arrive(&ti_full[slot]);         // release: the unit record is visible to the waiters
      }
      __syncwarp();
      ++n;
    };
    // The record of unit k+1 is computed and published while unit k's loads are in flight (after its first kStages B
    // loads, when the ring is full and this warp would only wait), from coords fetched one unit earlier: nothing but
    // barrier waits sits between the last load of a unit and the first load of the next.
    // (a CTA's units are consecutive k: tile-major rounds first, then at most a run of remainder rounds)
    int unit = unit_at(0, ntiles, sched), next = -1;
    Rec cur = {0, 0, 0, 0}, nxt = {0, 0, 0, 0};
    int kfirst = 0;
    while (unit < 0 && kfirst + 1 < rounds) unit = unit_at(++kfirst, ntiles, sched);
    auto next_unit = [&](int& kk) {              // first valid unit after round kk (rounds with no unit for this CTA are skipped)
      int u = -1;
      while (u < 0 && kk + 1 < rounds) u = unit_at(++kk, ntiles, sched);
      return u;
    };
    int knext = kfirst;
    if (unit >= 0) {
      load_coords(unit_id(unit) % ntiles, pcx, pcy);
      cur = make_rec(unit, pcx, pcy);
      publish(unit, cur);
      next = next_unit(knext);
      if (next >= 0) load_coords(unit_id(next) % ntiles, pcx, pcy);
    }
    int it = 0, na = 0;
    while (unit >= 0) {
      const bool tm = unit_tm(unit);
      const int l = unit_id(unit) / ntiles, tile = unit_id(unit) - l * ntiles;
      const int b = tile / tpi, tr = tile - b * tpi;
      const int y0 = (tr / p.tiles_x) * kTY, x0 = (tr % p.tiles_x) * kTX;
      const int bx0 = cur.bx0, by0 = cur.by0, nrows = cur.nrows;
      const bool skip = cur.ov || nrows == 0;    // overflow: the exact kernel recomputes this tile; no rows: all-zero level
      const bool load_a = tm ? l == 0 : !skip;
      if (load_a) {
#pragma unroll
        for (int kb = 0; kb < kKB; ++kb) {
          mbar_wait(&a_empty[kb], (na & 1) ^ 1);
          if (elect_one()) {
            mbar_expect_tx(&a_full[kb], kATile);
            tma_load_4d(sA + kb * kATile, &mF1, &a_full[kb], kb * 64, x0, y0, b);
          }
          __syncwarp();
        }
        ++na;
      }
      bool ahead_done = false;
      int after = -1;
      auto ahead = [&]() {
        if (ahead_done) return;
        ahead_done = true;
        if (next >= 0) {
          nxt = make_rec(next, pcx, pcy);
          publish(next, nxt);
          after = next_unit(knext);
          if (after >= 0) load_coords(unit_id(after) % ntiles, pcx, pcy);
        }
      };
      if (!skip) {
        // B: only the box rows some window needs, as one TMA box of the chunk's (even) row count
        const CUtensorMap* map = &mLv.m[l][0];
        const int cr = chunk_rows(l), bw = box_w(l);
        int issued = 0;
        for (int c = 0; c * cr < nrows; ++c) {
          const int rows = min(cr, nrows - c * cr);
          for (int kb = 0; kb < kKB; ++kb, ++it) {
            const int s = it % kStages, ph = (it / kStages) & 1;
            mbar_wait(&b_empty[s], ph ^ 1);
            if (elect_one()) {
              mbar_expect_tx(&b_full[s], rows * bw * 128);
              tma_load_4d(sB + s * kBStage, map + (rows >> 1) - 1, &b_full[s], kb * 64, bx0, by0 + c * cr, b);   // rows is even
            }
            __syncwarp();
            if (++issued == kStages) ahead();
          }
        }
      }
      ahead();
      unit = next; cur = nxt; next = after;
    }
  } else {
    // ------------------------------------------------------------------ consumers: MMA + gather + bilinear blend + store
    // thread = pixel = accumulator row
    const int lg = warp, ml = lg * 32 + lane;
    MmaCtx m{smem_u32(sA), smem_u32(sB), a_full, a_empty, b_full, b_empty, acc, 0, 0};
    auto load_coord = [&](int tile, float& ox, float& oy, bool& v) {
      const int b = tile / tpi, tr = tile - b * tpi;
      const int py = (tr / p.tiles_x) * kTY + (ml >> 4), px = (tr % p.tiles_x) * kTX + (ml & 15);
      v = py < p.H && px < p.W;
      ox = v ? clamp_coord(__ldg(p.coords + (static_cast<size_t>(b) * 2 + 0) * HW + py * p.W + px)) : 0.f;
      oy = v ? clamp_coord(__ldg(p.coords + (static_cast<size_t>(b) * 2 + 1) * HW + py * p.W + px)) : 0.f;
    };
    float cx = 0.f, cy = 0.f, ncx = 0.f, ncy = 0.f;
    bool valid = false, nvalid = false;
    {                                          // the 7 pad channels of this pixel's output rows stay zero for the whole kernel
      const uint4 z = make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(stage + ml * kLvlStride + 80) = z;
      *reinterpret_cast<uint4*>(stage + (128 + ml) * kLvlStride + 80) = z;
    }
    int unit = unit_at(0, ntiles, sched);
    if (unit >= 0) load_coord(unit_id(unit) % ntiles, ncx, ncy, nvalid);
    int n = 0;
    for (int k = 0; k < rounds; ++k) {
      const int cur = unit;
      cx = ncx; cy = ncy; valid = nvalid;
      unit = k + 1 < rounds ? unit_at(k + 1, ntiles, sched) : -1;
      if (unit >= 0) load_coord(unit_id(unit) % ntiles, ncx, ncy, nvalid);
      if (cur < 0) continue;
      const bool tm = unit_tm(cur);
      const int l = unit_id(cur) / ntiles, tile = unit_id(cur) - l * ntiles;
      const int b = tile / tpi, tr = tile - b * tpi;
      const int y0 = (tr / p.tiles_x) * kTY, x0 = (tr % p.tiles_x) * kTX;
      const int slot = n & (kTiRing - 1);
      mbar_wait(&ti_full[slot], (n >> kTiShift) & 1);
      const int ov = ti[slot].overflow, nrows = ti[slot].nrows;
      const bool skip = ov || nrows == 0;
      const bool load_a = tm ? l == 0 : !skip, free_a = tm ? l == kLevels - 1 : !skip;
      if (skip) {                              // tile-major order: the A tile's barriers still turn over once per tile
        if (load_a)
          for (int kb = 0; kb < kKB; ++kb) mbar_wait(&a_full[kb], m.na & 1);
        __syncwarp();
        if (free_a && lane == 0)
          for (int kb = 0; kb < kKB; ++kb) mbar_arrive(&a_empty[kb]);
      }
      if (!ov) {
        EpiCtx c{p, &ti[slot], stage, b, y0, x0, lg, ml, lane, valid, cx, cy, load_a, free_a};
        lookup_epilogue(c, m, l, &mOutHi, &mOutLo);
      }
      if (load_a) ++m.na;
      __syncwarp();
      if (lane == 0) mbar_arrive(&ti_empty[slot]);
      ++n;
    }
    if (lane == 0) bulk_wait_all0();           // the output tile must outlive its TMA stores
  }

  __syncthreads();
  // ---- units of this CTA that overflowed their box (flagged by this CTA's own producer warp): exact path, all warps
  if (*ov_count == 0) return;                  // the common case: nothing to redo
  for (int k = 0; k < rounds; ++k) {
    const int unit = unit_at(k, ntiles, sched);
    if (unit < 0) continue;
    const int l = unit_id(unit) / ntiles, tile = unit_id(unit) - l * ntiles;
    if (p.flags[tile * kLevels + l] != 0) exact_unit(p, l, tile, acc, warp, lane, kThreads / 32);
  }
}

__global__ void f32_to_f16_kernel(const float4* __restrict__ src, uint2* __restrict__ dst, size_t n4) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 v = src[i];
    __half2 a = __floats2half2_rn(v.x, v.y), c = __floats2half2_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&a);
    o.y = *reinterpret_cast<uint32_t*>(&c);
    dst[i] = o;
  }
}

}  // namespace lookup_umma
}  // namespace rnc

using namespace rnc;

extern "C" int rnc_f32_to_f16(const float* src, void* dst, size_t n, void* stream) {
  if (n == 0 || (n & 3)) return RNC_ERR_BAD_SHAPE;
  if (!src || !dst || !aligned16(src) || (reinterpret_cast<uintptr_t>(dst) & 7)) return RNC_ERR_BAD_POINTER;
  size_t blocks = (n / 4 + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  lookup_umma::f32_to_f16_kernel<<<static_cast<int>(blocks), 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(src), static_cast<uint2*>(dst), n / 4);
  return after_launch();
}

extern "C" size_t rnc_corr_lookup_umma_workspace_bytes(int B, int H, int W) {
  using namespace lookup_umma;
  return static_cast<size_t>(B) * ((H + kTY - 1) / kTY) * ((W + kTX - 1) / kTX) * kLevels * sizeof(int);
}

static int sm_count() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached = n;
  }
  return cached;
}

extern "C" int rnc_corr_lookup_umma_fwd(const void* f1h_cl, const void* f2h_pyr, const float* f1_cl, const float* f2_pyr,
                                        const float* coords, int B, int D, int H, int W, int levels, int radius,
                                        void* out_hi, void* out_lo, int ldo, int lvl_stride, void* workspace,
                                        size_t workspace_bytes, void* stream) {
  using namespace lookup_umma;
  using namespace rnc::umma;
  if (B <= 0 || H <= 0 || W <= 0) return RNC_ERR_BAD_SHAPE;
  if (D != kD || levels != kLevels || radius != kR) return RNC_ERR_UNSUPPORTED;
  if ((H >> (levels - 1)) < 1 || (W >> (levels - 1)) < 1 || ldo < levels * kLvlStride || (ldo & 7) || lvl_stride != kLvlStride) return RNC_ERR_BAD_SHAPE;
  if (!f1h_cl || !f2h_pyr || !f1_cl || !f2_pyr || !coords || !out_hi || !out_lo || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned16(f1h_cl) || !aligned16(f2h_pyr) || !aligned16(workspace) || !aligned16(out_hi) || !aligned16(out_lo)) return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_corr_lookup_umma_workspace_bytes(B, H, W)) return RNC_ERR_WORKSPACE;
  if (!encode_fn()) return RNC_ERR_UNSUPPORTED;

  Params p;
  p.f1_cl = f1_cl; p.f2_pyr = f2_pyr;
  p.coords = coords;
  p.out_hi = static_cast<__half*>(out_hi); p.out_lo = static_cast<__half*>(out_lo); p.ldo = ldo;
  p.flags = static_cast<int*>(workspace);
  p.B = B; p.H = H; p.W = W;
  p.tiles_x = (W + kTX - 1) / kTX; p.tiles_y = (H + kTY - 1) / kTY;
  p.scale = 1.0f / sqrtf(static_cast<float>(D));
  {
    // Hybrid order by default (see unit_at); RNC_LOOKUP_SCHED=level|tile select the pure orders (developer override).
    static const char* env = getenv("RNC_LOOKUP_SCHED");
    p.tile_major = env == nullptr ? 2 : env[0] == 't' ? 1 : env[0] == 'l' ? 0 : 2;
  }

  CUtensorMap maps[7];
  LevelMaps lv;
  bool ok = make_act_map(&maps[0], f1h_cl, kD, kD, B, H, W, kTX, kTY);
  // output planes [B][H][W][ldo] halves: un-swizzled store boxes of one level (88 channels) x 16 x 2 pixels
  ok = ok && make_plain_map(&maps[5], out_hi, ldo, ldo, B, H, W, kLvlStride, kTX, 2);
  ok = ok && make_plain_map(&maps[6], out_lo, ldo, ldo, B, H, W, kLvlStride, kTX, 2);
  size_t off = 0;
  for (int l = 0; l < kLevels; ++l) {
    const int Hl = H >> l, Wl = W >> l;
    for (int q = 0; q < kBoxKinds; ++q)
      ok = ok && make_act_map(&lv.m[l][q], static_cast<const __half*>(f2h_pyr) + off, kD, kD, B, Hl, Wl, box_w(l), 2 * (q + 1));
    off += static_cast<size_t>(B) * Hl * Wl * kD;
  }
  if (!ok) return RNC_ERR_BAD_SHAPE;

  static unsigned long long done = 0;
  if (int st = ensure_dyn_smem(corr_lookup_umma_kernel, kSmemTotal, &done)) return st;
  const int ntiles = B * p.tiles_x * p.tiles_y;
  const int grid = ntiles * kLevels < sm_count() ? ntiles * kLevels : sm_count();   // persistent: one CTA per SM
  cudaError_t e = launch_pdl(corr_lookup_umma_kernel, dim3(grid), dim3(kThreads), kSmemTotal, as_stream(stream), maps[0], lv, maps[5], maps[6], p);
  if (e != cudaSuccess) { g_last_cuda_error = static_cast<int>(e); return RNC_ERR_CUDA; }
  return after_launch();
}
