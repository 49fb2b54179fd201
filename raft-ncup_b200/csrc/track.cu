// Point tracking through video by chaining the bidirectional flows (the definition: rnc/track.py and DESIGN §3.17), and the
// TAP-Vid metrics of the tracks as exact per-video counts.
//
// rnc_track: one launch, grid (N / 256, V), a thread per query point.  The thread keeps its position and its lost flag in
// registers and walks from the query frame forward through F_k / occ_k to frame T-1, then backward through G_k / occ_bw_k to
// frame 0, writing each frame's position and visible flag.  The flows and masks are read through strided views of the stacked
// [V][T-1] tensors, so they need no copy.  The bilinear sample is bilinear.cuh's (interp.cu's), and every floating-point
// operation is a __*_rn intrinsic in the order rnc/track.py:host_track writes it, so the kernel and the host give the same
// bits.  No atomics: a point's outputs depend only on its own video.
//
// rnc_track_metrics: per video, the integer counts TAP-Vid's metrics are ratios of, through eval_common.cuh's two fixed-order
// reductions over the video's (point, frame) pairs.  Counts add exactly in any order, so they do not depend on V, the
// video's position in the batch or the GPU.
#include "bilinear.cuh"
#include "eval_common.cuh"

namespace rnc {
namespace {

constexpr int kTrackThreads = 256;
constexpr int kThresholds = RNC_TRACK_THRESHOLDS;       // delta = 1, 2, 4, 8, 16 (in 256x256 pixels)
constexpr int kTrackCounts = RNC_TRACK_COUNTS;

struct TrackArgs {
  Video flow[2];                        // F_k (frame k -> k+1), G_k (frame k+1 -> k): b is the pair index k
  VideoMask occ[2];                     // occ_k on frame k, occ_bw_k on frame k+1: b is k
  const float* queries;                 // [V][N][3]: (t, x, y)
  float2* tracks;                       // [V][N][T]: (x, y)
  unsigned char* visible;               // [V][N][T]
  int V, N, T, H, W;
};

// One direction of the rule from the query frame tq: with Dir = +1 steps k = tq .. T-2 through F_k / occ_k, each giving frame
// k + 1; with Dir = -1 steps k = tq-1 .. 0 through G_k / occ_bw_k, each giving frame k.  While the point is not lost its
// position lies in the frame, so rint of it indexes the mask without a clamp.
template <int Dir>
__device__ __forceinline__ void chain(const View& f, const MaskView& m, float x, float y, int tq, int T, int H, int W,
                                      float2* tr, unsigned char* vis) {
  bool lost = false;
  const int steps = Dir > 0 ? T - 1 - tq : tq;
  for (int s = 0; s < steps; ++s) {
    const int k = Dir > 0 ? tq + s : tq - 1 - s;
    const float ux = sample(f, k, 0, x, y, H, W), uy = sample(f, k, 1, x, y, H, W);
    const bool fin = finite(ux) && finite(uy);
    if (!lost) lost = !fin || m.at(k, static_cast<int>(rintf(y)), static_cast<int>(rintf(x))) != 0;
    if (fin) {
      x = __fadd_rn(x, ux);
      y = __fadd_rn(y, uy);
    }
    lost = lost || !inside(x, y, H, W);
    const int t = Dir > 0 ? k + 1 : k;
    tr[t] = make_float2(x, y);
    vis[t] = !lost;
  }
}

__global__ void __launch_bounds__(kTrackThreads) track_kernel(TrackArgs a) {
  const int v = blockIdx.y, n = blockIdx.x * kTrackThreads + threadIdx.x;
  if (n >= a.N) return;
  const int T = a.T, H = a.H, W = a.W;
  const long long pt = static_cast<long long>(v) * a.N + n;
  const float qt = a.queries[pt * 3], qx = a.queries[pt * 3 + 1], qy = a.queries[pt * 3 + 2];
  float2* tr = a.tracks + pt * T;
  unsigned char* vis = a.visible + pt * T;
  if (!(qt >= 0.0f && qt <= static_cast<float>(T - 1) && qt == floorf(qt)) || !inside(qx, qy, H, W)) {
    for (int t = 0; t < T; ++t) {       // a query rnc/track.py rejects before the launch: no track
      tr[t] = make_float2(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000));
      vis[t] = 0;
    }
    return;
  }
  const int tq = static_cast<int>(qt);
  tr[tq] = make_float2(qx, qy);
  vis[tq] = 1;
  chain<1>(a.flow[0].video(v), a.occ[0].video(v), qx, qy, tq, T, H, W, tr, vis);
  chain<-1>(a.flow[1].video(v), a.occ[1].video(v), qx, qy, tq, T, H, W, tr, vis);
}

// counts of a set of (point, frame) pairs, in the order of RNC_TRACK_COUNTS: evaluated, occlusion agreements, gt visible, then
// per threshold within & gt visible, then per threshold true positives, then per threshold false positives
using TrackPart = Counts<kTrackCounts>;

// x * 256 / size, rounded once: the multiplication by a power of two is exact
__device__ __forceinline__ float to_256(float x, float size) { return __fdiv_rn(__fmul_rn(x, 256.0f), size); }

struct TrackPairCounts {                // cta_partials_kernel's pixel (v, n, t): point n of video v at frame t
  const float2* pred;
  const unsigned char* pred_vis;
  const float2* gt;
  const unsigned char* gt_vis;
  const float* queries;
  int N, T;
  float H, W;
  __device__ void operator()(TrackPart& acc, int v, int n, int t) const {
    const long long pt = static_cast<long long>(v) * N + n;
    if (static_cast<float>(t) == queries[pt * 3]) return;       // the query frame is not evaluated
    const long long i = pt * T + t;
    const bool gv = gt_vis[i] != 0, pv = pred_vis[i] != 0;
    const float2 p = pred[i], g = gt[i];
    const float dx = __fsub_rn(to_256(p.x, W), to_256(g.x, W)), dy = __fsub_rn(to_256(p.y, H), to_256(g.y, H));
    const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
    acc.n[0] += 1;
    acc.n[1] += gv == pv;
    acc.n[2] += gv;
#pragma unroll
    for (int j = 0; j < kThresholds; ++j) {
      const float d = static_cast<float>(1 << j);
      const bool w = d2 < d * d;        // delta^2 is exact
      acc.n[3 + j] += w && gv;
      acc.n[3 + kThresholds + j] += w && gv && pv;
      acc.n[3 + 2 * kThresholds + j] += pv && (!gv || !w);
    }
  }
};

// V videos of N points over T >= 2 frames of H x W: a grid row per video, N*T < 2^30 (pairs indexed in int), and sides whose
// pixel coordinates are exact in float32
bool track_shape_ok(int V, int N, int T, int H, int W) {
  return eval_shape_ok(V, N, T) && T >= 2 && H > 0 && W > 0 && H <= (1 << 24) && W <= (1 << 24);
}

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

int rnc_track(const float* flow, long long fv, long long fk, long long fc, long long fy, long long fx, const float* flow_bw,
              long long gv, long long gk, long long gc, long long gy, long long gx, const unsigned char* occ, long long ov,
              long long ok, long long oy, long long ox, const unsigned char* occ_bw, long long pv, long long pk, long long py,
              long long px, const float* queries, int V, int N, int T, int H, int W, float* tracks, unsigned char* visible,
              void* stream) {
  if (!track_shape_ok(V, N, T, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!flow || !flow_bw || !occ || !occ_bw || !queries || !tracks || !visible) return RNC_ERR_BAD_POINTER;
  if (!aligned(flow, 4) || !aligned(flow_bw, 4) || !aligned(queries, 4) || !aligned(tracks, 8)) return RNC_ERR_BAD_POINTER;
  TrackArgs a{{{flow, fv, fk, fc, fy, fx}, {flow_bw, gv, gk, gc, gy, gx}},
              {{occ, ov, ok, 0, oy, ox}, {occ_bw, pv, pk, 0, py, px}},
              queries,
              reinterpret_cast<float2*>(tracks),
              visible,
              V, N, T, H, W};
  track_kernel<<<dim3((N + kTrackThreads - 1) / kTrackThreads, V), kTrackThreads, 0, as_stream(stream)>>>(a);
  return after_launch();
}

size_t rnc_track_metrics_workspace_bytes(int V, int N, int T) {
  return track_shape_ok(V, N, T, 1, 1) ? static_cast<size_t>(V) * eval_blocks(N, T) * sizeof(TrackPart) : 0;
}

int rnc_track_metrics(const float* tracks, const unsigned char* visible, const float* gt_tracks,
                      const unsigned char* gt_visible, const float* queries, int V, int N, int T, int H, int W,
                      long long* counts, void* workspace, size_t workspace_bytes, void* stream) {
  if (!track_shape_ok(V, N, T, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!tracks || !visible || !gt_tracks || !gt_visible || !queries || !counts || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(tracks, 8) || !aligned(gt_tracks, 8) || !aligned(queries, 4) || !aligned(counts, 8) || !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  if (workspace_bytes < rnc_track_metrics_workspace_bytes(V, N, T)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const int nblk = eval_blocks(N, T);
  TrackPart* parts = static_cast<TrackPart*>(workspace);
  cta_partials_kernel<<<dim3(nblk, V), kEvalThreads, 0, s>>>(
      TrackPairCounts{reinterpret_cast<const float2*>(tracks), visible, reinterpret_cast<const float2*>(gt_tracks), gt_visible,
                      queries, N, T, static_cast<float>(H), static_cast<float>(W)},
      N, T, parts);
  if (int st = after_launch()) return st;
  return launch_image_reduce(parts, V, nblk, 1, CountsStore<kTrackCounts>{counts}, s);
}

}  // extern "C"
