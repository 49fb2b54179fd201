// Video object segmentation by label propagation along the backward flows (the definition: rnc/segment.py and DESIGN §3.18),
// and the DAVIS semi-supervised metrics J and F of a predicted label map as exact integer counts.
//
// rnc_propagate_labels, one step k -> k+1 for V videos, in three launches and no host synchronisation:
//   1. vote_kernel, a thread per pixel p of frame k+1: u = G_k(p) at the pixel itself and p' = p + u.  A pixel with a finite u,
//      occ_bw_k(p) == 0 and p' in the frame is matched (bilinear.cuh's follow) and writes the bilinear vote of L_k at p' (bilinear.cuh's taps and
//      weights; per distinct label the weights of its taps added in tap order; the largest sum wins, ties to the smaller
//      label).  Any other pixel writes kUnmatched (255, never a label), so the output is also the site map of the fill.
//   2. dist_transform.cuh's column pass, with the matched pixels as sites, into the int workspace.
//   3. its row pass, whose Out stores into every unmatched pixel the label of its nearest matched pixel (exact squared
//      distance, ties to the smallest column, then the smallest row), or 0 in a frame without one.  A matched pixel is its own
//      nearest site and is not written, so the pass only reads the pixels it gathers from.
// Every floating-point operation is a __*_rn intrinsic in the order rnc/segment.py:host_propagate_step writes it, so the host
// restatement gives the same labels.  No atomics: a video's labels depend only on its own inputs.
//
// rnc_segmentation_counts: per (frame n, object o), with void = gt == 255, M = pred == o & !void and G = gt == o: |M & G|,
// |M | G|, the sizes of their boundary maps (the DAVIS toolkit's seg2bmap) and how many boundary pixels of each have one of
// the other within the tolerance r.  dist_transform.cuh's passes give every pixel's squared distance to each boundary, with
// the boundary test as the column pass's sites (boundary pixels are those at distance 0); eval_common.cuh's two fixed-order
// reductions count.  The counts are exact, so they do not depend on N, the frame's position or the GPU.
#include <cmath>

#include "bilinear.cuh"
#include "dist_transform.cuh"
#include "eval_common.cuh"

namespace rnc {
namespace {

constexpr int kVoteThreads = 256;
constexpr unsigned char kUnmatched = 255;
constexpr int kSegCounts = RNC_SEGMENT_COUNTS;

struct PropagateArgs {
  MaskView labels;                      // L_k [V][H][W]
  View flow;                            // G_k [V][2][H][W]
  MaskView occ;                         // occ_bw_k [V][H][W]
  unsigned char* out;                   // L_{k+1} through (ov, oy, ox)
  long long ov, oy, ox;
  int H, W;
};

__global__ void __launch_bounds__(kVoteThreads) vote_kernel(PropagateArgs a) {
  const int v = blockIdx.y, H = a.H, W = a.W;
  const int p = blockIdx.x * kVoteThreads + threadIdx.x;
  if (p >= H * W) return;
  const int y = p / W, x = p - y * W;
  float px, py;
  unsigned char label = kUnmatched;
  if (follow(a.flow, a.occ, v, y, x, H, W, px, py)) {
    const BilinearTaps t = bilinear_taps(px, py, H, W);
    const float w[4] = {t.w(0), t.w(1), t.w(2), t.w(3)};
    unsigned char l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) l[i] = a.labels.at(v, t.y[i >> 1], t.x[i & 1]);
    float best = -1.0f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      bool first = true;                // tap i is its label's first tap: the label's sum starts here
#pragma unroll
      for (int j = 0; j < i; ++j) first = first && l[j] != l[i];
      float s = w[i];
#pragma unroll
      for (int j = i + 1; j < 4; ++j) s = l[j] == l[i] ? __fadd_rn(s, w[j]) : s;
      if (first && (s > best || (s == best && l[i] < label))) {
        best = s;
        label = l[i];
      }
    }
  }
  a.out[v * a.ov + y * a.oy + x * a.ox] = label;
}

struct MatchedSites {                   // the pixels the vote labelled
  const unsigned char* out;
  long long ov, oy, ox;
  __device__ bool operator()(int v, int y, int x) const { return out[v * ov + y * oy + x * ox] != kUnmatched; }
};

struct FillOut {                        // an unmatched pixel takes its nearest matched pixel's label; 0 in a frame without one
  static constexpr bool kStores = true;
  unsigned char* out;
  long long ov, oy, ox;
  __device__ void store(int v, int y, int x, int q, int r) const {
    if (q == x && r == y) return;       // a matched pixel keeps its vote
    unsigned char* img = out + v * ov;
    img[y * oy + x * ox] = q < 0 ? 0 : img[r * oy + q * ox];
  }
};

// --------------------------------------------------------------------------------------------- J and F counts

// Image i of the boundary transforms is (side, n, o) = (i / NK, (i % NK) / K, i % K + 1): side 0 the prediction's mask M, side 1
// the ground truth's G.  Image i of the counts is (n, o) = (i / K, i % K + 1).
struct SegMasks {
  MaskView pred, gt;
  int K, H, W;
  __device__ __forceinline__ bool at(int side, int n, int o, int y, int x) const {
    const unsigned char g = gt.at(n, y, x);
    return side ? g == o : g != kUnmatched && pred.at(n, y, x) == o;
  }
};

struct BoundarySites {                  // seg2bmap at full resolution
  SegMasks m;
  int nk;                               // N*K: images [0, nk) are side 0, [nk, 2 nk) side 1
  __device__ bool operator()(int i, int y, int x) const {
    const int side = i >= nk, j = i - side * nk, n = j / m.K, o = j - n * m.K + 1;
    const int H = m.H, W = m.W;
    if (y == H - 1 && x == W - 1) return false;
    const bool s = m.at(side, n, o, y, x);
    if (y == H - 1) return s != m.at(side, n, o, y, x + 1);
    if (x == W - 1) return s != m.at(side, n, o, y + 1, x);
    return s != m.at(side, n, o, y, x + 1) || s != m.at(side, n, o, y + 1, x) || s != m.at(side, n, o, y + 1, x + 1);
  }
};

using SegPart = Counts<kSegCounts>;     // the counts of RNC_SEGMENT_COUNTS over a set of pixels

struct SegPixelCounts {                 // cta_partials_kernel's pixel (i, y, x): object o of frame n at (y, x)
  SegMasks m;
  const int* d2;                        // [2][N*K][H][W]: the distances to M's and G's boundaries
  long long side_stride;
  int r2;
  __device__ void operator()(SegPart& acc, int i, int y, int x) const {
    const int n = i / m.K, o = i - n * m.K + 1;
    const bool fg = m.at(0, n, o, y, x), gt = m.at(1, n, o, y, x);
    const long long px = (static_cast<long long>(i) * m.H + y) * m.W + x;
    const int dfg = d2[px], dgt = d2[side_stride + px];
    acc.n[0] += fg && gt;
    acc.n[1] += fg || gt;
    acc.n[2] += dfg == 0;
    acc.n[3] += dgt == 0;
    acc.n[4] += dfg == 0 && dgt <= r2;
    acc.n[5] += dgt == 0 && dfg <= r2;
  }
};

bool side_ok(int H, int W) { return H > 0 && W > 0 && H <= kSiteMaxSide && W <= kSiteMaxSide; }

bool propagate_shape_ok(int V, int H, int W) { return V > 0 && V <= 65535 && side_ok(H, W); }

// N frames of K objects: 2 N K images in one grid row each
bool counts_shape_ok(int N, int K, int H, int W) {
  return N > 0 && K > 0 && K <= 254 && 2ll * N * K <= 65535 && side_ok(H, W);
}

size_t d2_bytes(int N, int K, int H, int W) { return 2 * static_cast<size_t>(N) * K * H * W * sizeof(int); }

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

size_t rnc_propagate_labels_workspace_bytes(int V, int H, int W) {
  return propagate_shape_ok(V, H, W) ? static_cast<size_t>(V) * H * W * sizeof(int) : 0;
}

int rnc_propagate_labels(const unsigned char* labels, long long lv, long long ly, long long lx, const float* flow_bw,
                         long long gv, long long gc, long long gy, long long gx, const unsigned char* occ_bw, long long ov,
                         long long oy, long long ox, int V, int H, int W, unsigned char* out, long long qv, long long qy,
                         long long qx, void* workspace, size_t workspace_bytes, void* stream) {
  if (!propagate_shape_ok(V, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!labels || !flow_bw || !occ_bw || !out || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(flow_bw, 4) || !aligned(workspace, 16)) return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_propagate_labels_workspace_bytes(V, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const PropagateArgs a{{labels, lv, 0, ly, lx}, {flow_bw, gv, gc, gy, gx}, {occ_bw, ov, 0, oy, ox}, out, qv, qy, qx, H, W};
  vote_kernel<<<dim3((H * W + kVoteThreads - 1) / kVoteThreads, V), kVoteThreads, 0, s>>>(a);
  if (int st = after_launch()) return st;
  int* rows = static_cast<int*>(workspace);
  dist2_column_kernel<<<dim3((W + kSiteColThreads - 1) / kSiteColThreads, V), kSiteColThreads, 0, s>>>(
      MatchedSites{out, qv, qy, qx}, H, W, rows);
  if (int st = after_launch()) return st;
  dist2_row_kernel<<<dim3(H, V), 32, dist2_row_smem(W), s>>>(H, W, rows, FillOut{out, qv, qy, qx});
  return after_launch();
}

size_t rnc_segmentation_counts_workspace_bytes(int N, int K, int H, int W) {
  return counts_shape_ok(N, K, H, W)
             ? d2_bytes(N, K, H, W) + static_cast<size_t>(N) * K * eval_blocks(H, W) * sizeof(SegPart)
             : 0;
}

int rnc_segmentation_counts(const unsigned char* pred, long long pn, long long py, long long px, const unsigned char* gt,
                            long long gn, long long gy, long long gx, int N, int K, int H, int W, long long* counts,
                            void* workspace, size_t workspace_bytes, void* stream) {
  if (!counts_shape_ok(N, K, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!pred || !gt || !counts || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(counts, 8) || !aligned(workspace, 16)) return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_segmentation_counts_workspace_bytes(N, K, H, W)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const SegMasks m{{pred, pn, 0, py, px}, {gt, gn, 0, gy, gx}, K, H, W};
  const int nk = N * K;
  int* d2 = static_cast<int*>(workspace);
  dist2_column_kernel<<<dim3((W + kSiteColThreads - 1) / kSiteColThreads, 2 * nk), kSiteColThreads, 0, s>>>(
      BoundarySites{m, nk}, H, W, d2);
  if (int st = after_launch()) return st;
  dist2_row_kernel<<<dim3(H, 2 * nk), 32, dist2_row_smem(W), s>>>(H, W, d2, Dist2<RNC_DIST2_NONE>{});
  if (int st = after_launch()) return st;
  // DAVIS's tolerance: ceil(0.008 * the frame diagonal), the diagonal as numpy's norm computes it
  const int r = static_cast<int>(std::ceil(0.008 * std::sqrt(static_cast<double>(H) * H + static_cast<double>(W) * W)));
  const int nblk = eval_blocks(H, W);
  SegPart* parts = reinterpret_cast<SegPart*>(static_cast<char*>(workspace) + d2_bytes(N, K, H, W));
  cta_partials_kernel<<<dim3(nblk, nk), kEvalThreads, 0, s>>>(
      SegPixelCounts{m, d2, static_cast<long long>(nk) * H * W, r * r}, H, W, parts);
  if (int st = after_launch()) return st;
  return launch_image_reduce(parts, nk, nblk, 1, CountsStore<kSegCounts>{counts}, s);
}

}  // extern "C"
