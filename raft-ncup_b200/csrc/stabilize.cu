// Video stabilization (the definition: rnc/stabilize.py and DESIGN §3.21): a robust homography fit of each pair's camera
// motion to its forward flow, the smoothed camera path of Matsushita et al. (PAMI 2006) with its crop, and the warp.
//
// rnc_homography_fit, N pairs, in 5 + 2 (refine + 1) launches:
//   1. count_kernel, a thread per grid point p = (s/2 + j s, s/2 + i s) of frame k: p is matched when F(p) is finite and
//      q = p + F(p) (fp64) lies in [0, W-1] x [0, H-1]; a CTA of 256 raster-order points writes its count;
//   2. scan_kernel, a thread per pair: the exclusive scan of the CTA counts and n, the matched count;
//   3. write_kernel: the matched points written at their raster rank, in normalized fp64 coordinates (x^, y^, u^, v^), list L;
//   4. hyp_kernel, a CTA per (pair, 64 hypotheses), a thread per hypothesis: 4 indices by splitmix64, the degeneracy tests,
//      the 8x8 DLT solve (a thread's matrix is a column of shared memory) and the integer inlier count over L, tiled through
//      shared memory 256 points at a time;
//   5. argmax_kernel, a CTA per pair: the most inliers, ties to the smaller h; FEW and the identity when n < 4 or no
//      hypothesis is non-degenerate;
//   6. per round r = 0..refine: chunk_kernel, a CTA per (pair, 256 consecutive points of L), marks the inliers of the current
//      H (every point in round 0 when hypotheses = 0) and sums their 36 normal-matrix entries, 8 right-hand sides and count,
//      each in point order; then solve_kernel, one thread per pair, adds the chunks in order and, for r < refine and at least
//      4 inliers, refits H by the same elimination (a singular refit keeps H).  Round `refine` only counts: the output
//      inliers are the final H's, and it de-normalizes H to pixels.
// rnc_stabilize_path: a CTA per video, a thread per frame: S_t from the chained A's and their adjugate inverses, alpha_t in
//   closed form, the video's minimum by a fixed tree, then M_t = Z S_t (crop) and M_t^-1.
// rnc_stabilize_warp: a thread per output pixel: q = M^-1 u in fp64, rounded once to fp32, bilinear.cuh's sample per channel.
// Every float operation is a __*_rn intrinsic in the order rnc/stabilize.py's host restatements write it, so the host gives the
// same bits.  No atomics, no host synchronisation, no transcendental function.
#include <cmath>

#include "bilinear.cuh"
#include "homography.cuh"

namespace rnc {
namespace {

constexpr int kPts = 256;                     // points per compaction CTA and per refit chunk
constexpr int kHyp = 64;                      // hypotheses per hyp_kernel CTA
constexpr int kSums = 45;                     // 36 upper-triangle normal-matrix entries, 8 right-hand sides, the count
constexpr int kPathThreads = 128;
constexpr int kWarpThreads = 256;
constexpr int kMaxSide = 4096;
constexpr double kPivotMin = 1e-12;
constexpr double kCollinear = 1e-9;
constexpr double kShrink = 1.0 - 1.0 / 68719476736.0;   // 1 - 2^-36: the crop's margin against rounding
constexpr int kOk = RNC_HOMOGRAPHY_OK, kFew = RNC_HOMOGRAPHY_FEW;

// grid points along a side of n pixels at stride s: s/2, s/2 + s, ... < n
__host__ __device__ __forceinline__ int grid_side(int n, int s) { return s / 2 < n ? (n - 1 - s / 2) / s + 1 : 0; }

struct FitLayout {                            // the workspace
  double* L;                                  // [N][G][4]: x^, y^, u^, v^ of the matched points, in raster order
  double* chunk;                              // [N][nch][kSums]
  double* hyp;                                // [N][K][8]
  double* cur;                                // [N][8]: the current H (h33 = 1)
  int* hcount;                                // [N][K]: inliers, -1 for a degenerate hypothesis
  int* bcount;                                // [N][nch]: matched points per compaction CTA, then their exclusive scan
  int* npts;                                  // [N]
  int* status;                                // [N]
};

struct FitDims {
  int N, H, W, stride, K, gw, G, nch;
  double cx, cy, nu, nu2, tau2;
};

FitDims fit_dims(int N, int H, int W, int stride, int K, double tau) {
  FitDims d;
  d.N = N, d.H = H, d.W = W, d.stride = stride, d.K = K;
  d.gw = grid_side(W, stride);
  d.G = d.gw * grid_side(H, stride);
  d.nch = (d.G + kPts - 1) / kPts;
  d.cx = (W - 1) * 0.5, d.cy = (H - 1) * 0.5, d.nu = (H > W ? H : W) * 0.5;
  d.nu2 = d.nu * d.nu, d.tau2 = tau * tau;     // exact and correctly rounded on the host: no contraction possible
  return d;
}

FitLayout fit_layout(Carve& ws, const FitDims& d) {
  const size_t N = d.N, G = d.G, nch = d.nch, K = d.K;
  FitLayout l;
  l.L = ws.take<double>(N * G * 4);
  l.chunk = ws.take<double>(N * nch * kSums);
  l.hyp = ws.take<double>(N * K * 8);
  l.cur = ws.take<double>(N * 8);
  l.hcount = ws.take<int>(N * K);
  l.bcount = ws.take<int>(N * nch);
  l.npts = ws.take<int>(N);
  l.status = ws.take<int>(N);
  return l;
}

// grid point g of pair n: matched when F(p) is finite and q = p + F(p), in fp64, lies in the frame
__device__ __forceinline__ bool grid_match(const View& flow, const FitDims& d, int n, int g, double& x, double& y,
                                           double& qx, double& qy) {
  if (g >= d.G) return false;
  const int i = g / d.gw, j = g - i * d.gw;
  const int px = d.stride / 2 + j * d.stride, py = d.stride / 2 + i * d.stride;
  const float ux = flow.at(n, 0, py, px), uy = flow.at(n, 1, py, px);
  x = px, y = py;
  qx = dadd(x, static_cast<double>(ux));
  qy = dadd(y, static_cast<double>(uy));
  return finite(ux) && finite(uy) && qx >= 0.0 && qx <= d.W - 1 && qy >= 0.0 && qy <= d.H - 1;
}

__global__ void __launch_bounds__(kPts) count_kernel(View flow, FitDims d, FitLayout l) {
  const int n = blockIdx.y, g = blockIdx.x * kPts + threadIdx.x;
  double x, y, qx, qy;
  const int c = __syncthreads_count(grid_match(flow, d, n, g, x, y, qx, qy));
  if (threadIdx.x == 0) l.bcount[static_cast<long long>(n) * d.nch + blockIdx.x] = c;
}

__global__ void scan_kernel(FitDims d, FitLayout l) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= d.N) return;
  int* b = l.bcount + static_cast<long long>(n) * d.nch;
  int s = 0;
  for (int k = 0; k < d.nch; ++k) {
    const int c = b[k];
    b[k] = s;
    s += c;
  }
  l.npts[n] = s;
}

__global__ void __launch_bounds__(kPts) write_kernel(View flow, FitDims d, FitLayout l) {
  __shared__ int warps[kPts / 32];
  const int n = blockIdx.y, g = blockIdx.x * kPts + threadIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double x, y, qx, qy;
  const bool m = grid_match(flow, d, n, g, x, y, qx, qy);
  const unsigned ballot = __ballot_sync(0xffffffffu, m);
  if (lane == 0) warps[wid] = __popc(ballot);
  __syncthreads();
  if (!m) return;
  int off = l.bcount[static_cast<long long>(n) * d.nch + blockIdx.x] + __popc(ballot & ((1u << lane) - 1u));
  for (int w = 0; w < wid; ++w) off += warps[w];
  double* p = l.L + (static_cast<long long>(n) * d.G + off) * 4;
  p[0] = ddiv(dsub(x, d.cx), d.nu);
  p[1] = ddiv(dsub(y, d.cy), d.nu);
  p[2] = ddiv(dsub(qx, d.cx), d.nu);
  p[3] = ddiv(dsub(qy, d.cy), d.nu);
}

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long seed, unsigned long long i) {
  unsigned long long z = seed + (i + 1ull) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// |(b - a) x (c - a)| >= kCollinear (false for NaN)
__device__ __forceinline__ bool spread(double ax, double ay, double bx, double by, double cx, double cy) {
  const double cr = dsub(dmul(dsub(bx, ax), dsub(cy, ay)), dmul(dsub(by, ay), dsub(cx, ax)));
  return fabs(cr) >= kCollinear;
}

// Gaussian elimination with partial pivoting of the 8x9 augmented matrix a[(r * 9 + c) * S] (column 8 the right-hand side),
// columns in order, the first largest |a| of rows k..7 the pivot, rows k + 1..7 eliminated in order, then back substitution
// from row 7; the solution is left in column 8.  False when a pivot is under kPivotMin (or NaN).
template <int S>
__device__ bool solve8(double* a) {
  for (int k = 0; k < 8; ++k) {
    int p = k;
    double best = fabs(a[(k * 9 + k) * S]);
    for (int i = k + 1; i < 8; ++i) {
      const double v = fabs(a[(i * 9 + k) * S]);
      if (v > best) best = v, p = i;
    }
    if (!(best >= kPivotMin)) return false;
    if (p != k)
      for (int j = k; j < 9; ++j) {
        const double t = a[(k * 9 + j) * S];
        a[(k * 9 + j) * S] = a[(p * 9 + j) * S];
        a[(p * 9 + j) * S] = t;
      }
    const double piv = a[(k * 9 + k) * S];
    for (int i = k + 1; i < 8; ++i) {
      const double f = ddiv(a[(i * 9 + k) * S], piv);
      for (int j = k + 1; j < 9; ++j) a[(i * 9 + j) * S] = dsub(a[(i * 9 + j) * S], dmul(f, a[(k * 9 + j) * S]));
    }
  }
  for (int k = 7; k >= 0; --k) {
    double s = a[(k * 9 + 8) * S];
    for (int j = k + 1; j < 8; ++j) s = dsub(s, dmul(a[(k * 9 + j) * S], a[(j * 9 + 8) * S]));
    a[(k * 9 + 8) * S] = ddiv(s, a[(k * 9 + k) * S]);
  }
  return true;
}

// p = (x^, y^, u^, v^) is an inlier of h when w > 0 and nu^2 |H p^ - q^|^2 < tau^2
__device__ __forceinline__ bool inlier(const double (&h)[8], const double* p, double nu2, double tau2) {
  const double x = p[0], y = p[1];
  const double w = dadd(dadd(dmul(h[6], x), dmul(h[7], y)), 1.0);
  if (!(w > 0.0)) return false;
  const double X = dadd(dadd(dmul(h[0], x), dmul(h[1], y)), h[2]);
  const double Y = dadd(dadd(dmul(h[3], x), dmul(h[4], y)), h[5]);
  const double ex = dsub(ddiv(X, w), p[2]), ey = dsub(ddiv(Y, w), p[3]);
  return dmul(nu2, dadd(dmul(ex, ex), dmul(ey, ey))) < tau2;
}

__global__ void __launch_bounds__(kHyp) hyp_kernel(FitDims d, unsigned long long seed, FitLayout l) {
  __shared__ double a[72 * kHyp];
  __shared__ double tile[kPts * 4];
  const int n = blockIdx.y, t = threadIdx.x, h = blockIdx.x * kHyp + t;
  const int np = l.npts[n];
  const double* L = l.L + static_cast<long long>(n) * d.G * 4;
  bool ok = h < d.K && np >= 4;
  double hh[8];
  if (ok) {
    unsigned long long idx[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) idx[j] = splitmix64(seed, 4ull * h + j) % static_cast<unsigned long long>(np);
    ok = idx[0] != idx[1] && idx[0] != idx[2] && idx[0] != idx[3] && idx[1] != idx[2] && idx[1] != idx[3] && idx[2] != idx[3];
    double P[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) P[j][k] = L[idx[j] * 4 + k];
#pragma unroll
    for (int o = 0; o < 4; o += 2)             // the source points, then the destination points
      ok = ok && spread(P[0][o], P[0][o + 1], P[1][o], P[1][o + 1], P[2][o], P[2][o + 1]) &&
           spread(P[0][o], P[0][o + 1], P[1][o], P[1][o + 1], P[3][o], P[3][o + 1]) &&
           spread(P[0][o], P[0][o + 1], P[2][o], P[2][o + 1], P[3][o], P[3][o + 1]) &&
           spread(P[1][o], P[1][o + 1], P[2][o], P[2][o + 1], P[3][o], P[3][o + 1]);
    if (ok) {
      double* m = a + t;
#pragma unroll
      for (int j = 0; j < 4; ++j) {            // rows 2j and 2j + 1: the u and v equations of point j
        const double x = P[j][0], y = P[j][1], u = P[j][2], v = P[j][3];
        const double ru[9] = {x, y, 1.0, 0.0, 0.0, 0.0, -dmul(u, x), -dmul(u, y), u};
        const double rv[9] = {0.0, 0.0, 0.0, x, y, 1.0, -dmul(v, x), -dmul(v, y), v};
#pragma unroll
        for (int c = 0; c < 9; ++c) {
          m[((2 * j) * 9 + c) * kHyp] = ru[c];
          m[((2 * j + 1) * 9 + c) * kHyp] = rv[c];
        }
      }
      ok = solve8<kHyp>(m);
#pragma unroll
      for (int k = 0; k < 8; ++k) hh[k] = m[(k * 9 + 8) * kHyp];
    }
  }
  int count = 0;
  if (np >= 4)                                 // uniform over the CTA
    for (int base = 0; base < np; base += kPts) {
      __syncthreads();
      for (int i = t; i < kPts * 4; i += kHyp) {
        const int pi = base + i / 4;
        tile[i] = pi < np ? L[static_cast<long long>(base) * 4 + i] : 0.0;
      }
      __syncthreads();
      const int m = min(kPts, np - base);
      if (ok)
        for (int i = 0; i < m; ++i) count += inlier(hh, tile + i * 4, d.nu2, d.tau2);
    }
  if (h >= d.K) return;
  const long long nh = static_cast<long long>(n) * d.K + h;
  l.hcount[nh] = ok ? count : -1;
  if (ok)
#pragma unroll
    for (int k = 0; k < 8; ++k) l.hyp[nh * 8 + k] = hh[k];
}

struct Best {
  int c, h;
};

__device__ __forceinline__ Best better(Best a, Best b) { return b.c > a.c || (b.c == a.c && b.h < a.h) ? b : a; }

__global__ void __launch_bounds__(256) argmax_kernel(FitDims d, FitLayout l) {
  __shared__ Best warps[8];
  const int n = blockIdx.x;
  Best b{-1, 0x7fffffff};
  for (int h = threadIdx.x; h < d.K; h += 256) b = better(b, Best{l.hcount[static_cast<long long>(n) * d.K + h], h});
  for (int o = 16; o > 0; o >>= 1) b = better(b, Best{__shfl_down_sync(0xffffffffu, b.c, o), __shfl_down_sync(0xffffffffu, b.h, o)});
  if ((threadIdx.x & 31) == 0) warps[threadIdx.x >> 5] = b;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < 8; ++w) b = better(b, warps[w]);
  const bool few = l.npts[n] < 4 || (d.K > 0 && b.c < 0);
  l.status[n] = few ? kFew : kOk;
  double* cur = l.cur + n * 8;
  for (int k = 0; k < 8; ++k)                  // the identity until round 0 refits when K = 0
    cur[k] = few || d.K == 0 ? (k == 0 || k == 4 ? 1.0 : 0.0) : l.hyp[(static_cast<long long>(n) * d.K + b.h) * 8 + k];
}

// entry e < 36 of the upper triangle, row-major: (i, j) with i <= j
__device__ __forceinline__ void tri(int e, int& i, int& j) {
  i = 0;
  while (e >= 8 - i) e -= 8 - i, ++i;
  j = i + e;
}

__global__ void __launch_bounds__(kPts) chunk_kernel(FitDims d, bool all, FitLayout l) {
  __shared__ double rows[18 * kPts];          // per point: the u row (8), the v row (8), u^, v^
  __shared__ unsigned char flag[kPts];
  const int n = blockIdx.y, base = blockIdx.x * kPts, t = threadIdx.x;
  const int np = l.npts[n];
  if (l.status[n] != kOk || base >= np) return;
  double h[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) h[k] = l.cur[n * 8 + k];
  const int i = base + t;
  bool in = false;
  if (i < np) {
    const double* p = l.L + (static_cast<long long>(n) * d.G + i) * 4;
    in = all || inlier(h, p, d.nu2, d.tau2);
    const double x = p[0], y = p[1], u = p[2], v = p[3];
    const double r[18] = {x,   y,   1.0, 0.0, 0.0, 0.0, -dmul(u, x), -dmul(u, y), 0.0, 0.0,
                          0.0, x,   y,   1.0, -dmul(v, x), -dmul(v, y), u,           v};
#pragma unroll
    for (int c = 0; c < 18; ++c) rows[c * kPts + t] = r[c];
  }
  flag[t] = in;
  __syncthreads();
  if (t >= kSums) return;
  const int m = min(kPts, np - base);
  double s = 0.0;
  if (t < 36) {
    int ei, ej;
    tri(t, ei, ej);
    for (int q = 0; q < m; ++q)
      if (flag[q])
        s = dadd(s, dadd(dmul(rows[ei * kPts + q], rows[ej * kPts + q]), dmul(rows[(8 + ei) * kPts + q], rows[(8 + ej) * kPts + q])));
  } else if (t < 44) {
    const int ei = t - 36;
    for (int q = 0; q < m; ++q)
      if (flag[q])
        s = dadd(s, dadd(dmul(rows[ei * kPts + q], rows[16 * kPts + q]), dmul(rows[(8 + ei) * kPts + q], rows[17 * kPts + q])));
  } else {
    int c = 0;
    for (int q = 0; q < m; ++q) c += flag[q];
    s = c;
  }
  l.chunk[(static_cast<long long>(n) * d.nch + blockIdx.x) * kSums + t] = s;
}

struct FitOut {
  double* A;                                  // [N][3][3]
  int *inliers, *matched, *status;
};

// H (normalized, h33 = 1) to pixels: G = H Tp, M = Tq^-1 G, A = M / m33; false when |m33| < kPivotMin (or NaN)
__device__ bool denormalize(const double (&h)[8], const FitDims& d, double* A) {
  const double hm[9] = {h[0], h[1], h[2], h[3], h[4], h[5], h[6], h[7], 1.0};
  double g[9];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    g[r * 3] = ddiv(hm[r * 3], d.nu);
    g[r * 3 + 1] = ddiv(hm[r * 3 + 1], d.nu);
    g[r * 3 + 2] = dsub(hm[r * 3 + 2], ddiv(dadd(dmul(hm[r * 3], d.cx), dmul(hm[r * 3 + 1], d.cy)), d.nu));
  }
  double m[9];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    m[c] = dadd(dmul(d.nu, g[c]), dmul(d.cx, g[6 + c]));
    m[3 + c] = dadd(dmul(d.nu, g[3 + c]), dmul(d.cy, g[6 + c]));
    m[6 + c] = g[6 + c];
  }
  if (!(fabs(m[8]) >= kPivotMin)) return false;
#pragma unroll
  for (int k = 0; k < 9; ++k) A[k] = ddiv(m[k], m[8]);
  return true;
}

__global__ void __launch_bounds__(32) solve_kernel(FitDims d, int round, int refine, FitLayout l, FitOut o) {
  __shared__ double a[72];
  const int n = blockIdx.x;
  if (threadIdx.x != 0) return;
  const int np = l.npts[n];
  double* A = o.A + n * 9;
  double* cur = l.cur + n * 8;
  int count = 0;
  if (l.status[n] == kOk) {
    const int nch = (np + kPts - 1) / kPts;
    const double* ch = l.chunk + static_cast<long long>(n) * d.nch * kSums;
    for (int e = 0; e < kSums; ++e) {
      double s = 0.0;
      for (int c = 0; c < nch; ++c) s = dadd(s, ch[c * kSums + e]);
      if (e < 36) {
        int i, j;
        tri(e, i, j);
        a[i * 9 + j] = s;
        a[j * 9 + i] = s;
      } else if (e < 44) {
        a[(e - 36) * 9 + 8] = s;
      } else {
        count = static_cast<int>(s);
      }
    }
    if (round < refine) {
      const bool ok = count >= 4 && solve8<1>(a);
      if (ok)
        for (int k = 0; k < 8; ++k) cur[k] = a[k * 9 + 8];
      else if (round == 0 && d.K == 0)         // no start to keep: a first refit over all points that fails is FEW
        l.status[n] = kFew;
    }
  }
  if (round < refine) return;
  double h[8];
  for (int k = 0; k < 8; ++k) h[k] = cur[k];
  bool ok = l.status[n] == kOk && denormalize(h, d, A);
  if (!ok)
    for (int k = 0; k < 9; ++k) A[k] = k % 4 == 0 ? 1.0 : 0.0;
  o.inliers[n] = ok ? count : 0;
  o.matched[n] = np;
  o.status[n] = ok ? kOk : kFew;
}

bool fit_args_ok(int N, int H, int W, int stride, int K, double tau, int refine) {
  return N > 0 && N <= 65535 && H > 0 && W > 0 && H <= kMaxSide && W <= kMaxSide && stride >= 1 && stride <= 256 &&
         K >= 0 && K <= 65536 && refine >= 0 && refine <= 64 && (K > 0 || refine > 0) && tau > 0.0 && tau <= 1e300;
}

// ------------------------------------------------------------------------------------------------------------ path

// (X Y) with each entry ((x_i0 y_0j) + (x_i1 y_1j)) + x_i2 y_2j, then every entry divided by the product's [2][2]
__device__ __forceinline__ M3 mul_norm(const M3& X, const M3& Y) {
  M3 P;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      P.m[i * 3 + j] = dadd(dadd(dmul(X.m[i * 3], Y.m[j]), dmul(X.m[i * 3 + 1], Y.m[3 + j])), dmul(X.m[i * 3 + 2], Y.m[6 + j]));
  const double z = P.m[8];
#pragma unroll
  for (int k = 0; k < 9; ++k) P.m[k] = ddiv(P.m[k], z);
  return P;
}

__device__ __forceinline__ M3 load3(const double* p) {
  M3 A;
#pragma unroll
  for (int k = 0; k < 9; ++k) A.m[k] = p[k];
  return A;
}

__device__ __forceinline__ void store3(double* p, const M3& A) {
#pragma unroll
  for (int k = 0; k < 9; ++k) p[k] = A.m[k];
}

__device__ __forceinline__ void accumulate(M3& num, double w, const M3& T) {
#pragma unroll
  for (int k = 0; k < 9; ++k) num.m[k] = dadd(num.m[k], dmul(w, T.m[k]));
}

// the largest alpha in [0, 1] with the four corners c +- alpha (cx, cy) of the centred rectangle mapped by P into the frame
// with w > 0: per corner and constraint f0 + alpha f1 >= 0, a bound f0 / -f1 where f1 < 0, and 0 where f0 < 0 (or NaN)
__device__ double crop_alpha(const M3& P, int H, int W) {
  const double cx = (W - 1) * 0.5, cy = (H - 1) * 0.5, wm = W - 1, hm = H - 1;
  const double* p = P.m;
  const double X0 = dadd(dadd(dmul(p[0], cx), dmul(p[1], cy)), p[2]);
  const double Y0 = dadd(dadd(dmul(p[3], cx), dmul(p[4], cy)), p[5]);
  const double W0 = dadd(dadd(dmul(p[6], cx), dmul(p[7], cy)), p[8]);
  double a = 1.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double dx = k & 1 ? cx : -cx, dy = k & 2 ? cy : -cy;
    const double X1 = dadd(dmul(p[0], dx), dmul(p[1], dy));
    const double Y1 = dadd(dmul(p[3], dx), dmul(p[4], dy));
    const double W1 = dadd(dmul(p[6], dx), dmul(p[7], dy));
    const double f0[5] = {W0, X0, dsub(dmul(wm, W0), X0), Y0, dsub(dmul(hm, W0), Y0)};
    const double f1[5] = {W1, X1, dsub(dmul(wm, W1), X1), Y1, dsub(dmul(hm, W1), Y1)};
#pragma unroll
    for (int c = 0; c < 5; ++c) {
      if (!(f0[c] >= 0.0)) a = 0.0;
      else if (f1[c] < 0.0) a = fmin(a, ddiv(f0[c], -f1[c]));
    }
  }
  return a;
}

struct PathArgs {
  const double* A;                            // [V][T-1][9]
  const double* taps;                         // [radius + 1]
  double* M;                                  // [V][T][9]
  double* Minv;                               // [V][T][9]
  double* alpha;                              // [V]
  int T, radius, H, W, crop;
  double crop_min;
};

__global__ void __launch_bounds__(kPathThreads) path_kernel(PathArgs p) {
  __shared__ double mins[kPathThreads / 32];
  const int v = blockIdx.x, T = p.T;
  const double* A = p.A + static_cast<long long>(v) * (T - 1) * 9;
  double* M = p.M + static_cast<long long>(v) * T * 9;
  double* Minv = p.Minv + static_cast<long long>(v) * T * 9;
  double amin = 1.0;
  for (int t = threadIdx.x; t < T; t += kPathThreads) {
    const double w0 = p.taps[0];
    M3 num, I;
#pragma unroll
    for (int k = 0; k < 9; ++k) num.m[k] = k % 4 == 0 ? w0 : 0.0, I.m[k] = k % 4 == 0 ? 1.0 : 0.0;
    const int jp = min(p.radius, T - 1 - t), jm = min(p.radius, t);
    M3 P = I;
    for (int j = 1; j <= jp; ++j) {           // T_t^{t+j} = A_{t+j-1} T_t^{t+j-1}
      P = mul_norm(load3(A + (t + j - 1) * 9), P);
      accumulate(num, p.taps[j], P);
    }
    P = I;
    for (int j = 1; j <= jm; ++j) {           // T_t^{t-j} = A_{t-j}^-1 T_t^{t-j+1}
      P = mul_norm(inv_norm(A + (t - j) * 9), P);
      accumulate(num, p.taps[j], P);
    }
    const double z = num.m[8];
#pragma unroll
    for (int k = 0; k < 9; ++k) num.m[k] = ddiv(num.m[k], z);
    store3(M + t * 9, num);
    amin = fmin(amin, crop_alpha(inv_norm(num.m), p.H, p.W));
  }
  for (int o = 16; o > 0; o >>= 1) amin = fmin(amin, __shfl_down_sync(0xffffffffu, amin, o));
  if ((threadIdx.x & 31) == 0) mins[threadIdx.x >> 5] = amin;
  __syncthreads();
  amin = mins[0];
  for (int w = 1; w < kPathThreads / 32; ++w) amin = fmin(amin, mins[w]);
  if (threadIdx.x == 0) p.alpha[v] = amin;
  const double a = dmul(amin < p.crop_min ? p.crop_min : amin, kShrink);
  const double z = ddiv(1.0, a), cx = (p.W - 1) * 0.5, cy = (p.H - 1) * 0.5;
  const M3 Z{{z, 0.0, dsub(cx, dmul(cx, z)), 0.0, z, dsub(cy, dmul(cy, z)), 0.0, 0.0, 1.0}};
  for (int t = threadIdx.x; t < T; t += kPathThreads) {
    M3 S = load3(M + t * 9);
    if (p.crop) S = mul_norm(Z, S);
    store3(M + t * 9, S);
    store3(Minv + t * 9, inv_norm(S.m));
  }
}

bool taps_radius_ok(int radius) { return radius >= 0 && radius <= 1024; }

// ------------------------------------------------------------------------------------------------------------ warp

__global__ void __launch_bounds__(kWarpThreads) warp_kernel(View frames, const double* __restrict__ maps, int C, int H, int W,
                                                           OutView out, OutMaskView valid) {
  const int n = blockIdx.y, hw = H * W;
  const int p = blockIdx.x * kWarpThreads + threadIdx.x;
  if (p >= hw) return;
  const int y = p / W, x = p - y * W;
  const double* m = maps + n * 9;
  double X, Y;
  const bool wq = project(m, x, y, X, Y);
  const float qx = __double2float_rn(X), qy = __double2float_rn(Y);
  const bool ok = wq && inside(qx, qy, H, W);
  for (int c = 0; c < C; ++c)
    out.p[n * out.b + c * out.c + y * out.y + x * out.x] = ok ? sample(frames, n, c, qx, qy, H, W) : 0.0f;
  valid.p[n * valid.b + y * valid.y + x * valid.x] = ok;
}

bool warp_shape_ok(int N, int C, int H, int W) {
  return N > 0 && N <= 65535 && C >= 1 && C <= 4 && H > 0 && W > 0 && H <= kMaxSide && W <= kMaxSide;
}

}  // namespace
}  // namespace rnc

using namespace rnc;

extern "C" {

size_t rnc_homography_fit_workspace_bytes(int N, int H, int W, int stride, int hypotheses) {
  if (!fit_args_ok(N, H, W, stride, hypotheses, 1.0, 1)) return 0;
  Carve ws{nullptr};
  fit_layout(ws, fit_dims(N, H, W, stride, hypotheses, 1.0));
  return ws.bytes;
}

int rnc_homography_fit(const float* flow, long long fn, long long fc, long long fy, long long fx, int N, int H, int W,
                       int stride, int hypotheses, double tau, int refine, unsigned long long seed, double* A, int* inliers,
                       int* matched, int* status, void* workspace, size_t workspace_bytes, void* stream) {
  if (!fit_args_ok(N, H, W, stride, hypotheses, tau, refine)) return RNC_ERR_BAD_SHAPE;
  if (!flow || !A || !inliers || !matched || !status || !workspace) return RNC_ERR_BAD_POINTER;
  if (!aligned(flow, 4) || !aligned(A, 8) || !aligned(inliers, 4) || !aligned(matched, 4) || !aligned(status, 4) ||
      !aligned(workspace, 16))
    return RNC_ERR_BAD_POINTER;
  const FitDims d = fit_dims(N, H, W, stride, hypotheses, tau);
  if (workspace_bytes < rnc_homography_fit_workspace_bytes(N, H, W, stride, hypotheses)) return RNC_ERR_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  Carve ws{static_cast<char*>(workspace)};
  const FitLayout l = fit_layout(ws, d);
  const View f{flow, fn, fc, fy, fx};
  const int nb = d.nch > 0 ? d.nch : 1;
  count_kernel<<<dim3(nb, N), kPts, 0, s>>>(f, d, l);
  if (int st = after_launch()) return st;
  scan_kernel<<<(N + 127) / 128, 128, 0, s>>>(d, l);
  if (int st = after_launch()) return st;
  write_kernel<<<dim3(nb, N), kPts, 0, s>>>(f, d, l);
  if (int st = after_launch()) return st;
  if (hypotheses > 0) {
    hyp_kernel<<<dim3((hypotheses + kHyp - 1) / kHyp, N), kHyp, 0, s>>>(d, seed, l);
    if (int st = after_launch()) return st;
  }
  argmax_kernel<<<N, 256, 0, s>>>(d, l);
  if (int st = after_launch()) return st;
  const FitOut o{A, inliers, matched, status};
  for (int r = 0; r <= refine; ++r) {
    chunk_kernel<<<dim3(nb, N), kPts, 0, s>>>(d, r == 0 && hypotheses == 0, l);
    if (int st = after_launch()) return st;
    solve_kernel<<<N, 32, 0, s>>>(d, r, refine, l, o);
    if (int st = after_launch()) return st;
  }
  return RNC_OK;
}

int rnc_stabilize_path(const double* A, int V, int T, const double* taps, int radius, int H, int W, int crop, double crop_min,
                       double* M, double* Minv, double* alpha, void* stream) {
  if (V <= 0 || V > 65535 || T < 2 || T > (1 << 24) || !taps_radius_ok(radius) || H <= 0 || W <= 0 || H > kMaxSide ||
      W > kMaxSide || !(crop_min > 0.0 && crop_min <= 1.0))
    return RNC_ERR_BAD_SHAPE;
  if (!A || !taps || !M || !Minv || !alpha) return RNC_ERR_BAD_POINTER;
  if (!aligned(A, 8) || !aligned(taps, 8) || !aligned(M, 8) || !aligned(Minv, 8) || !aligned(alpha, 8))
    return RNC_ERR_BAD_POINTER;
  path_kernel<<<V, kPathThreads, 0, as_stream(stream)>>>(PathArgs{A, taps, M, Minv, alpha, T, radius, H, W, crop != 0, crop_min});
  return after_launch();
}

int rnc_stabilize_warp(const float* frames, long long in, long long ic, long long iy, long long ix, const double* maps, int N,
                       int C, int H, int W, float* out, long long on, long long oc, long long oy, long long ox,
                       unsigned char* valid, long long vn, long long vy, long long vx, void* stream) {
  if (!warp_shape_ok(N, C, H, W)) return RNC_ERR_BAD_SHAPE;
  if (!frames || !maps || !out || !valid) return RNC_ERR_BAD_POINTER;
  if (!aligned(frames, 4) || !aligned(maps, 8) || !aligned(out, 4)) return RNC_ERR_BAD_POINTER;
  warp_kernel<<<dim3((H * W + kWarpThreads - 1) / kWarpThreads, N), kWarpThreads, 0, as_stream(stream)>>>(
      View{frames, in, ic, iy, ix}, maps, C, H, W, OutView{out, on, oc, oy, ox}, OutMaskView{valid, vn, 0, vy, vx});
  return after_launch();
}

}  // extern "C"
