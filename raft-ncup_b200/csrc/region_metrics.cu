// Per-region validation metrics: the Sintel benchmark's matched / unmatched, occlusion-boundary distance and speed regions, and
// KITTI 2015's background / foreground and non-occluded regions (the definitions: rnc/metrics.py and DESIGN §3.14).
//
// rnc_boundary_dist2: the exact squared Euclidean distance of every pixel to the nearest occlusion-boundary pixel of its image
// (a pixel with a 4-neighbour inside the image whose label differs), as a separable transform in integers (Felzenszwalb and
// Huttenlocher, "Distance Transforms of Sampled Functions", 2012):
//   1. dist2_column_kernel, a thread per column of one image: the boundary test, then a downward and an upward sweep give
//      g(y, x), the distance to the nearest boundary pixel in the same column (RNC_DIST2_NONE if the column has none).
//   2. dist2_row_kernel, a warp per row: d2(y, x) = min_q g(y, q)^2 + (x - q)^2.  Lane 0 builds the lower envelope of the
//      parabolas q -> g(y, q)^2 + (x - q)^2, comparing intersections by cross-multiplying in int64 (no division, so every
//      comparison is exact); then each lane finds, by binary search on the same comparisons, the parabola of each of its pixels.
//   The row pass reads its row of g into shared memory before it writes d2 over it, so d2 holds g in between and no workspace
//   is needed.  No atomics, no host synchronisation; each pixel's value is an exact integer.
//
// rnc_region_metrics: per image and per cell (one joint label of a pixel; Sintel 2 occlusion x 4 distance x 4 speed classes,
// KITTI 2 noc x 2 fg) the five counts and the fp64 EPE sum of rnc_flow_metrics, from the same per-pixel float32 arithmetic
// (pixel_metrics.cuh).  CTA (x, b) covers the 2048 pixels of image b that rnc_flow_metrics' CTA x covers.  Each warp takes its
// 32 pixels at a time; for each cell present among them (a ballot loop) it counts with ballots and adds the members' EPE with
// a fixed xor-shuffle tree (non-members add 0.0, which changes no sum), into the warp's own per-cell accumulator in shared
// memory.  The CTA adds its 8 warps in order, and a second kernel adds each (image, cell)'s CTAs in a fixed order (a warp per
// pair: lane-strided sums, then a fixed shuffle tree).  The order depends only on H*W and the cell count: an image's results
// do not depend on B, on its position in the batch or on the GPU, and no floating-point atomics are used.
#include "pixel_metrics.cuh"
#include "rnc_common.cuh"

namespace rnc {
namespace {

constexpr int kNone = RNC_DIST2_NONE;
constexpr int kMaxSide = 4096;          // H, W of rnc_boundary_dist2; the row pass keeps 6 W bytes of shared memory
constexpr int kColThreads = 128;

__global__ void __launch_bounds__(kColThreads) dist2_column_kernel(const float* __restrict__ occ, long long ob, long long oy,
                                                                   long long ox, int H, int W, int* __restrict__ d2) {
  const int b = blockIdx.y;
  const int x = blockIdx.x * kColThreads + threadIdx.x;
  if (x >= W) return;
  const float* base = occ + b * ob + x * ox;
  int* col = d2 + static_cast<long long>(b) * H * W + x;
  // downward: distance to the nearest boundary pixel at or above y
  bool up = false, cur = base[0] >= 0.5f;
  int last = -1;
#pragma unroll 4
  for (int y = 0; y < H; ++y) {
    const float* r = base + y * oy;
    const bool down = y + 1 < H ? r[oy] >= 0.5f : cur;
    const bool left = x > 0 ? r[-ox] >= 0.5f : cur;
    const bool right = x + 1 < W ? r[ox] >= 0.5f : cur;
    if ((y > 0 && up != cur) || down != cur || left != cur || right != cur) last = y;
    col[static_cast<long long>(y) * W] = last < 0 ? kNone : y - last;
    up = cur;
    cur = down;
  }
  // upward: the nearest boundary pixel at or below y (a boundary pixel holds 0)
  int next = -1;
  for (int y = H - 1; y >= 0; --y) {
    int* c = col + static_cast<long long>(y) * W;
    const int g = *c;
    if (g == 0) {
      next = y;
    } else if (next >= 0 && next - y < g) {
      *c = next - y;
    }
  }
}

__global__ void __launch_bounds__(32) dist2_row_kernel(int H, int W, int* __restrict__ d2) {
  extern __shared__ int smem[];
  int* F = smem;                                                  // F[q] = g(q)^2 + q^2; -1: the column has no boundary
  unsigned short* v = reinterpret_cast<unsigned short*>(F + W);  // the lower envelope's parabolas, left to right
  const int lane = threadIdx.x;
  int* row = d2 + (static_cast<long long>(blockIdx.y) * H + blockIdx.x) * W;
  for (int q = lane; q < W; q += 32) {
    const int g = row[q];
    F[q] = g == kNone ? -1 : g * g + q * q;
  }
  __syncwarp();
  int n = 0;
  if (lane == 0) {
    for (int q = 0; q < W; ++q) {
      const int fq = F[q];
      if (fq < 0) continue;
      // with s(a, b) = (F_b - F_a) / (2 (b - a)) where the parabolas of a < b meet: drop the top p while q overtakes it no
      // later than p overtook the one below it, r: s(p, q) <= s(r, p)
      while (n > 1) {
        const int p = v[n - 1], r = v[n - 2];
        const int fp = F[p], fr = F[r];
        if (static_cast<long long>(fq - fp) * (p - r) <= static_cast<long long>(fp - fr) * (q - p)) {
          --n;
        } else {
          break;
        }
      }
      v[n++] = static_cast<unsigned short>(q);
    }
  }
  __syncwarp();
  n = __shfl_sync(0xffffffffu, n, 0);
  for (int x = lane; x < W; x += 32) {
    if (n == 0) {                          // no boundary in the image
      row[x] = kNone;
      continue;
    }
    // the last k with k == 0 or x >= s(v[k-1], v[k]); on a tie both parabolas give the same value
    int lo = 0, hi = n - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      const int a = v[mid - 1], c = v[mid];
      if (2ll * x * (c - a) >= static_cast<long long>(F[c] - F[a])) {
        lo = mid;
      } else {
        hi = mid - 1;
      }
    }
    const int q = v[lo];
    row[x] = F[q] - q * q + (x - q) * (x - q);
  }
}

constexpr int kRegThreads = 256;
constexpr int kRegWarps = kRegThreads / 32;
constexpr int kRegPerThread = 8;
constexpr int kRegPerCta = kRegThreads * kRegPerThread;
constexpr int kRegCounts = 5;         // valid, epe < 1, < 3, < 5, KITTI outliers
constexpr int kMaxCells = RNC_REGION_CELLS_SINTEL;

struct RegionPart {                   // one (CTA, cell)'s partials; 32 bytes
  double epe_sum;
  unsigned n[kRegCounts];
  unsigned pad;
};

struct Plane {
  const float* p;
  long long b, y, x;
};

struct RegionArgs {
  const float* flow;
  long long fb, fc, fy, fx;
  const float* gt;
  long long gb, gc, gy, gx;
  Plane valid;                        // p == nullptr: every pixel is valid
  Plane mask;                         // Sintel: occ; KITTI: noc
  const int* d2;                      // Sintel: [B][H][W]
  Plane fg;                           // KITTI; p == nullptr: every pixel is background
  int H, W, kind, cells;
};

__device__ __forceinline__ float at(const Plane& q, int b, int y, int x) { return q.p[b * q.b + y * q.y + x * q.x]; }

__device__ __forceinline__ int sintel_cell(bool occluded, int d2, float mag) {
  const int d = d2 < 100 ? 0 : d2 < 3600 ? 1 : d2 < 19600 ? 2 : 3;
  const int s = mag < 10.0f ? 0 : mag < 40.0f ? 1 : mag >= 40.0f ? 2 : 3;     // NaN: no speed bin
  return (occluded ? 16 : 0) + d * 4 + s;
}

__global__ void __launch_bounds__(kRegThreads) region_part_kernel(RegionArgs a, RegionPart* __restrict__ parts) {
  __shared__ RegionPart acc[kRegWarps][kMaxCells];
  const int b = blockIdx.y;
  const int hw = a.H * a.W;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  acc[warp][lane] = RegionPart{};
  __syncwarp();
  for (int p = blockIdx.x * kRegPerCta + threadIdx.x, e = 0; e < kRegPerThread; ++e, p += kRegThreads) {
    bool has = p < hw;
    int cell = 0;
    PixelMetrics m{};
    if (has) {
      const int y = p / a.W, x = p - y * a.W;
      has = !a.valid.p || at(a.valid, b, y, x) >= 0.5f;
      if (has) {
        const float* f = a.flow + b * a.fb + y * a.fy + x * a.fx;
        const float* g = a.gt + b * a.gb + y * a.gy + x * a.gx;
        m = pixel_metrics(f[0], f[a.fc], g[0], g[a.gc]);
        if (a.kind == RNC_REGIONS_SINTEL) {
          cell = sintel_cell(at(a.mask, b, y, x) >= 0.5f, a.d2[static_cast<long long>(b) * hw + p], m.mag);
        } else {
          cell = (at(a.mask, b, y, x) >= 0.5f ? 0 : 2) + ((a.fg.p && at(a.fg, b, y, x) >= 0.5f) ? 1 : 0);
        }
      }
    }
    for (unsigned todo = __ballot_sync(0xffffffffu, has); todo;) {
      const int c = __shfl_sync(0xffffffffu, cell, __ffs(todo) - 1);
      const bool in = has && cell == c;
      const unsigned members = __ballot_sync(0xffffffffu, in);
      todo &= ~members;
      const unsigned n1 = __popc(__ballot_sync(0xffffffffu, in && m.epe < 1.0f));
      const unsigned n2 = __popc(__ballot_sync(0xffffffffu, in && m.epe < 3.0f));
      const unsigned n3 = __popc(__ballot_sync(0xffffffffu, in && m.epe < 5.0f));
      const unsigned n4 = __popc(__ballot_sync(0xffffffffu, in && m.outlier));
      double s = in ? static_cast<double>(m.epe) : 0.0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) {
        RegionPart& r = acc[warp][c];
        r.epe_sum += s;
        r.n[0] += __popc(members);
        r.n[1] += n1;
        r.n[2] += n2;
        r.n[3] += n3;
        r.n[4] += n4;
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < a.cells) {
    RegionPart out{};
    for (int w = 0; w < kRegWarps; ++w) {
      const RegionPart& r = acc[w][threadIdx.x];
      out.epe_sum += r.epe_sum;
#pragma unroll
      for (int c = 0; c < kRegCounts; ++c) out.n[c] += r.n[c];
    }
    parts[(static_cast<long long>(b) * gridDim.x + blockIdx.x) * a.cells + threadIdx.x] = out;
  }
}

// a warp per (image, cell): parts [B][nblk][cells] -> counts [B][cells][5], epe_sum [B][cells]
__global__ void __launch_bounds__(kRegThreads) region_reduce_kernel(const RegionPart* __restrict__ parts, int B, int nblk,
                                                                    int cells, long long* __restrict__ counts,
                                                                    double* __restrict__ epe_sum) {
  const int i = blockIdx.x * kRegWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= B * cells) return;
  const int b = i / cells, cell = i - b * cells;
  double sum = 0.0;
  unsigned long long n[kRegCounts] = {0, 0, 0, 0, 0};
  for (int k = lane; k < nblk; k += 32) {
    const RegionPart& q = parts[(static_cast<long long>(b) * nblk + k) * cells + cell];
    sum += q.epe_sum;
#pragma unroll
    for (int c = 0; c < kRegCounts; ++c) n[c] += q.n[c];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
#pragma unroll
    for (int c = 0; c < kRegCounts; ++c) n[c] += __shfl_xor_sync(0xffffffffu, n[c], o);
  }
  if (lane == 0) {
    epe_sum[i] = sum;
#pragma unroll
    for (int c = 0; c < kRegCounts; ++c) counts[static_cast<long long>(i) * kRegCounts + c] = static_cast<long long>(n[c]);
  }
}

bool dist2_shape_ok(int B, int H, int W) {
  return B > 0 && H > 0 && W > 0 && B <= 65535 && H <= kMaxSide && W <= kMaxSide;
}

int region_cells(int kind) {
  return kind == RNC_REGIONS_SINTEL ? RNC_REGION_CELLS_SINTEL : kind == RNC_REGIONS_KITTI ? RNC_REGION_CELLS_KITTI : 0;
}

bool region_shape_ok(int B, int H, int W) {
  return B > 0 && H > 0 && W > 0 && B <= 65535 && static_cast<long long>(H) * W < (1ll << 30);
}

int region_blocks(int H, int W) { return (H * W + kRegPerCta - 1) / kRegPerCta; }

bool aligned(const void* p, uintptr_t n) { return (reinterpret_cast<uintptr_t>(p) & (n - 1)) == 0; }

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

int rnc_boundary_dist2(const float* occ, long long ob, long long oy, long long ox, int B, int H, int W, int* d2,
                       void* stream) {
  if (!dist2_shape_ok(B, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!occ || !d2 || !aligned(occ, 4) || !aligned(d2, 4)) return RNC_ERR_BAD_POINTER;
  cudaStream_t s = as_stream(stream);
  dist2_column_kernel<<<dim3((W + kColThreads - 1) / kColThreads, B), kColThreads, 0, s>>>(occ, ob, oy, ox, H, W, d2);
  if (int st = after_launch()) return st;
  const size_t smem = static_cast<size_t>(W) * (sizeof(int) + sizeof(unsigned short));
  dist2_row_kernel<<<dim3(H, B), 32, smem, s>>>(H, W, d2);
  return after_launch();
}

size_t rnc_region_metrics_workspace_bytes(int kind, int B, int H, int W) {
  const int cells = region_cells(kind);
  return cells && region_shape_ok(B, H, W) ? static_cast<size_t>(B) * region_blocks(H, W) * cells * sizeof(RegionPart) : 0;
}

int rnc_region_metrics(int kind, const float* flow, long long fb, long long fc, long long fy, long long fx, const float* gt,
                       long long gb, long long gc, long long gy, long long gx, const float* valid, long long vb, long long vy,
                       long long vx, const float* mask, long long mb, long long my, long long mx, const int* d2,
                       const float* fg, long long qb, long long qy, long long qx, int B, int H, int W, long long* counts,
                       double* epe_sum, void* workspace, size_t workspace_bytes, void* stream) {
  const int cells = region_cells(kind);
  if (!cells) return RNC_ERR_UNSUPPORTED;
  if (!region_shape_ok(B, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!flow || !gt || !mask || !counts || !epe_sum || !workspace) return RNC_ERR_BAD_POINTER;
  if (kind == RNC_REGIONS_SINTEL ? (!d2 || fg) : d2 != nullptr) return RNC_ERR_BAD_POINTER;
  if (!aligned(flow, 4) || !aligned(gt, 4) || !aligned(valid, 4) || !aligned(mask, 4) || !aligned(d2, 4) ||
      !aligned(fg, 4) || !aligned(counts, 8) || !aligned(epe_sum, 8) || !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_region_metrics_workspace_bytes(kind, B, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const RegionArgs a{flow, fb, fc, fy, fx, gt, gb, gc, gy, gx, {valid, vb, vy, vx}, {mask, mb, my, mx}, d2, {fg, qb, qy, qx},
                     H, W, kind, cells};
  const int nblk = region_blocks(H, W);
  RegionPart* parts = static_cast<RegionPart*>(workspace);
  region_part_kernel<<<dim3(nblk, B), kRegThreads, 0, s>>>(a, parts);
  if (int st = after_launch()) return st;
  region_reduce_kernel<<<(B * cells + kRegWarps - 1) / kRegWarps, kRegThreads, 0, s>>>(parts, B, nblk, cells, counts,
                                                                                      epe_sum);
  return after_launch();
}

}  // extern "C"
