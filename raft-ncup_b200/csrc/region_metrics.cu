// Per-region validation metrics: the Sintel benchmark's matched / unmatched, occlusion-boundary distance and speed regions, and
// KITTI 2015's background / foreground and non-occluded regions (the definitions: rnc/metrics.py and DESIGN §3.14).
//
// rnc_boundary_dist2: the exact squared Euclidean distance of every pixel to the nearest occlusion-boundary pixel of its image
// (a pixel with a 4-neighbour inside the image whose label differs), as a separable transform in integers (Felzenszwalb and
// Huttenlocher, "Distance Transforms of Sampled Functions", 2012): dist_transform.cuh's column pass, with the boundary test as
// its sites, then its row pass writing d2(y, x) = min_q g(y, q)^2 + (x - q)^2.  d2 holds the column pass's nearest rows in
// between, so no workspace is needed.  No atomics, no host synchronisation; each pixel's value is an exact integer.
//
// rnc_region_metrics: per image and per cell (one joint label of a pixel; Sintel 2 occlusion x 4 distance x 4 speed classes,
// KITTI 2 noc x 2 fg) the five counts and the fp64 EPE sum of rnc_flow_metrics, from the same per-pixel float32 arithmetic
// (eval_common.cuh's pixel_metrics).  CTA (x, b) covers the kEvalPerCta pixels of image b that rnc_flow_metrics' CTA x covers.
// Each warp takes its 32 pixels at a time; for each cell present among them (a ballot loop) it counts with ballots and adds
// the members' EPE with a fixed xor-shuffle tree (non-members add 0.0, which changes no sum), into the warp's own per-cell
// accumulator in shared memory.  The CTA adds its warps in order, and eval_common.cuh's image_reduce_kernel adds each (image,
// cell)'s CTAs in a fixed order.  The order depends only on H*W and the cell count: an image's results do not depend on B, on
// its position in the batch or on the GPU, and no floating-point atomics are used.
#include "dist_transform.cuh"
#include "eval_common.cuh"

namespace rnc {
namespace {

constexpr int kNone = RNC_DIST2_NONE;

// the sites of rnc_boundary_dist2: pixels with a 4-neighbour inside the image whose label (occluded where >= 0.5) differs
struct BoundarySites {
  const float* occ;
  long long ob, oy, ox;
  int H, W;
  __device__ bool operator()(int b, int y, int x) const {
    const float* r = occ + b * ob + y * oy + x * ox;
    const bool cur = r[0] >= 0.5f;
    return (y > 0 && (r[-oy] >= 0.5f) != cur) || (y + 1 < H && (r[oy] >= 0.5f) != cur) ||
           (x > 0 && (r[-ox] >= 0.5f) != cur) || (x + 1 < W && (r[ox] >= 0.5f) != cur);
  }
};

constexpr int kMaxCells = RNC_REGION_CELLS_SINTEL;

struct RegionArgs {
  View flow, gt;
  View valid;                         // p == nullptr: every pixel is valid
  View mask;                          // Sintel: occ; KITTI: noc
  const int* d2;                      // Sintel: [B][H][W]
  View fg;                            // KITTI; p == nullptr: every pixel is background
  int H, W, kind, cells;
};

__device__ __forceinline__ int sintel_cell(bool occluded, int d2, float mag) {
  const int d = d2 < 100 ? 0 : d2 < 3600 ? 1 : d2 < 19600 ? 2 : 3;
  const int s = mag < 10.0f ? 0 : mag < 40.0f ? 1 : mag >= 40.0f ? 2 : 3;     // NaN: no speed bin
  return (occluded ? 16 : 0) + d * 4 + s;
}

__global__ void __launch_bounds__(kEvalThreads) region_part_kernel(RegionArgs a, MetricsPart* __restrict__ parts) {
  __shared__ MetricsPart acc[kEvalWarps][kMaxCells];
  const int b = blockIdx.y;
  const int hw = a.H * a.W;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  acc[warp][lane] = MetricsPart{};
  __syncwarp();
  for (int p = blockIdx.x * kEvalPerCta + threadIdx.x, e = 0; e < kEvalPerThread; ++e, p += kEvalThreads) {
    bool has = p < hw;
    int cell = 0;
    PixelMetrics m{};
    if (has) {
      const int y = p / a.W, x = p - y * a.W;
      has = !a.valid.p || a.valid.at(b, y, x) >= 0.5f;
      if (has) {
        m = pixel_metrics(a.flow.at(b, 0, y, x), a.flow.at(b, 1, y, x), a.gt.at(b, 0, y, x), a.gt.at(b, 1, y, x));
        if (a.kind == RNC_REGIONS_SINTEL) {
          cell = sintel_cell(a.mask.at(b, y, x) >= 0.5f, a.d2[static_cast<long long>(b) * hw + p], m.mag);
        } else {
          cell = (a.mask.at(b, y, x) >= 0.5f ? 0 : 2) + ((a.fg.p && a.fg.at(b, y, x) >= 0.5f) ? 1 : 0);
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
        MetricsPart& r = acc[warp][c];
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
    MetricsPart out{};
    for (int w = 0; w < kEvalWarps; ++w) out += acc[w][threadIdx.x];
    parts[(static_cast<long long>(b) * gridDim.x + blockIdx.x) * a.cells + threadIdx.x] = out;
  }
}

bool dist2_shape_ok(int B, int H, int W) {
  return B > 0 && H > 0 && W > 0 && B <= 65535 && H <= kSiteMaxSide && W <= kSiteMaxSide;
}

int region_cells(int kind) {
  return kind == RNC_REGIONS_SINTEL ? RNC_REGION_CELLS_SINTEL : kind == RNC_REGIONS_KITTI ? RNC_REGION_CELLS_KITTI : 0;
}

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

int rnc_boundary_dist2(const float* occ, long long ob, long long oy, long long ox, int B, int H, int W, int* d2,
                       void* stream) {
  if (!dist2_shape_ok(B, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!occ || !d2 || !aligned(occ, 4) || !aligned(d2, 4)) return RNC_ERR_BAD_POINTER;
  cudaStream_t s = as_stream(stream);
  dist2_column_kernel<<<dim3((W + kSiteColThreads - 1) / kSiteColThreads, B), kSiteColThreads, 0, s>>>(
      BoundarySites{occ, ob, oy, ox, H, W}, H, W, d2);
  if (int st = after_launch()) return st;
  dist2_row_kernel<<<dim3(H, B), 32, dist2_row_smem(W), s>>>(H, W, d2, Dist2<kNone>{});
  return after_launch();
}

size_t rnc_region_metrics_workspace_bytes(int kind, int B, int H, int W) {
  const int cells = region_cells(kind);
  return cells && eval_shape_ok(B, H, W) ? static_cast<size_t>(B) * eval_blocks(H, W) * cells * sizeof(MetricsPart) : 0;
}

int rnc_region_metrics(int kind, const float* flow, long long fb, long long fc, long long fy, long long fx, const float* gt,
                       long long gb, long long gc, long long gy, long long gx, const float* valid, long long vb, long long vy,
                       long long vx, const float* mask, long long mb, long long my, long long mx, const int* d2,
                       const float* fg, long long qb, long long qy, long long qx, int B, int H, int W, long long* counts,
                       double* epe_sum, void* workspace, size_t workspace_bytes, void* stream) {
  const int cells = region_cells(kind);
  if (!cells) return RNC_ERR_UNSUPPORTED;
  if (!eval_shape_ok(B, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!flow || !gt || !mask || !counts || !epe_sum || !workspace) return RNC_ERR_BAD_POINTER;
  if (kind == RNC_REGIONS_SINTEL ? (!d2 || fg) : d2 != nullptr) return RNC_ERR_BAD_POINTER;
  if (!aligned(flow, 4) || !aligned(gt, 4) || !aligned(valid, 4) || !aligned(mask, 4) || !aligned(d2, 4) ||
      !aligned(fg, 4) || !aligned(counts, 8) || !aligned(epe_sum, 8) || !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_region_metrics_workspace_bytes(kind, B, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const RegionArgs a{{flow, fb, fc, fy, fx}, {gt, gb, gc, gy, gx}, {valid, vb, 0, vy, vx}, {mask, mb, 0, my, mx}, d2,
                     {fg, qb, 0, qy, qx}, H, W, kind, cells};
  const int nblk = eval_blocks(H, W);
  MetricsPart* parts = static_cast<MetricsPart*>(workspace);
  region_part_kernel<<<dim3(nblk, B), kEvalThreads, 0, s>>>(a, parts);
  if (int st = after_launch()) return st;
  return launch_image_reduce(parts, B * cells, nblk, cells, MetricsStore{counts, epe_sum}, s);
}

}  // extern "C"
