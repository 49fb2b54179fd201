// The exact nearest "site" of every pixel of a batch of images, as a separable transform in integers (Felzenszwalb and
// Huttenlocher, "Distance Transforms of Sampled Functions", 2012).  Shared by rnc_boundary_dist2 (region_metrics.cu: the sites
// are occlusion-boundary pixels, the output the squared distance) and rnc_interpolate (interp.cu: the sites are the pixels that
// received a splatted motion, the output the index of the nearest one, a feature transform), and by segment.cu
// (rnc_propagate_labels: the voted pixels, the output their label; rnc_segmentation_counts: mask boundaries, squared distances).
//   1. dist2_column_kernel<Sites>, a thread per column of one image: a downward and an upward sweep give the row of the nearest
//      site in the same column (the upper one on a tie; -1 if the column has none).
//   2. dist2_row_kernel<Out>, a warp per row: with g(q) the distance from (y, q) to column q's nearest site, the nearest site
//      of (y, x) minimises g(q)^2 + (x - q)^2 over q.  Lane 0 builds the lower envelope of those parabolas, comparing
//      intersections by cross-multiplying in int64 (no division, so every comparison is exact); then each lane finds, by binary
//      search on the same comparisons, the parabola of each of its pixels.  Of parabolas that tie at x the smallest q wins (a
//      parabola the envelope drops is never the only nor the leftmost minimum), so the site is the nearest one in exact squared
//      Euclidean distance, ties to the smallest column and then the smallest row.
//   The row pass reads its row of the column pass's output into shared memory before it writes over it, so no workspace is
//   needed.  No atomics, no host synchronisation; every value is an exact integer.
//
// Sites: `__device__ bool operator()(int image, int y, int x) const`, true at a site.  Out: `none`, written in an image without
// a site, and `__device__ int operator()(int y, int x, int q, int r, int fq) const`, the value of pixel (y, x) whose nearest site
// is (r, q), with fq = (y - r)^2 + q^2.  Images are [images][H][W] contiguous in the int map; 1 <= H, W <= kSiteMaxSide.
// An Out with `static constexpr bool kStores = true` writes each pixel's result itself instead, through
// `__device__ void store(int image, int y, int x, int q, int r) const` (q = r = -1 in an image without a site), and the row
// pass leaves the int map as the column pass wrote it (rnc_propagate_labels: the site's label, gathered into a uint8 map).
#pragma once
#include <type_traits>

namespace rnc {

template <class Out, class = void>
struct out_stores : std::false_type {};
template <class Out>
struct out_stores<Out, std::void_t<decltype(Out::kStores)>> : std::bool_constant<Out::kStores> {};

constexpr int kSiteMaxSide = 4096;        // the row pass keeps 8 W bytes of shared memory and 16-bit column / row indices
constexpr int kSiteColThreads = 128;

template <class Sites>
__global__ void __launch_bounds__(kSiteColThreads) dist2_column_kernel(Sites sites, int H, int W, int* __restrict__ out) {
  const int b = blockIdx.y;
  const int x = blockIdx.x * kSiteColThreads + threadIdx.x;
  if (x >= W) return;
  int* col = out + static_cast<long long>(b) * H * W + x;
  // downward: the nearest site at or above y
  int last = -1;
#pragma unroll 4
  for (int y = 0; y < H; ++y) {
    if (sites(b, y, x)) last = y;
    col[static_cast<long long>(y) * W] = last;
  }
  // upward: the nearest site at or below y, where it is strictly nearer (a site holds its own row)
  int next = -1;
  for (int y = H - 1; y >= 0; --y) {
    int* c = col + static_cast<long long>(y) * W;
    const int r = *c;
    if (r == y) {
      next = y;
    } else if (next >= 0 && (r < 0 || next - y < y - r)) {
      *c = next;
    }
  }
}

template <class Out>
__global__ void __launch_bounds__(32) dist2_row_kernel(int H, int W, int* __restrict__ out, Out o) {
  extern __shared__ int smem[];
  int* F = smem;                                                  // F[q] = g(q)^2 + q^2; -1: the column has no site
  unsigned short* R = reinterpret_cast<unsigned short*>(F + W);   // R[q]: the row of column q's nearest site
  unsigned short* v = R + W;                                      // the lower envelope's parabolas, left to right
  const int lane = threadIdx.x;
  const int y = blockIdx.x;
  int* row = out + (static_cast<long long>(blockIdx.y) * H + y) * W;
  for (int q = lane; q < W; q += 32) {
    const int r = row[q];
    F[q] = r < 0 ? -1 : (y - r) * (y - r) + q * q;
    R[q] = static_cast<unsigned short>(r);
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
    if (n == 0) {                          // no site in the image
      if constexpr (out_stores<Out>::value) {
        o.store(blockIdx.y, y, x, -1, -1);
      } else {
        row[x] = o.none;
      }
      continue;
    }
    // the last k with k == 0 or x > s(v[k-1], v[k]): on a tie the left parabola, the smaller column, is kept
    int lo = 0, hi = n - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      const int a = v[mid - 1], c = v[mid];
      if (2ll * x * (c - a) > static_cast<long long>(F[c] - F[a])) {
        lo = mid;
      } else {
        hi = mid - 1;
      }
    }
    const int q = v[lo];
    if constexpr (out_stores<Out>::value) {
      o.store(blockIdx.y, y, x, q, R[q]);
    } else {
      row[x] = o(y, x, q, R[q], F[q]);
    }
  }
}

inline size_t dist2_row_smem(int W) { return static_cast<size_t>(W) * (sizeof(int) + 2 * sizeof(unsigned short)); }

}  // namespace rnc
