"""Video stabilization from the forward flows: fit each pair's camera motion, smooth the camera path, warp and crop or fill the
uncovered borders from neighbouring frames, and score.

Inputs: one video of T >= 2 frames [C,H,W] and the forward flows F_k (frame k -> k+1, float32 [2,H,W], channel 0 = x) that
rnc.harness.run_sequences yields.  Every step below is fixed down to the order of its floating-point operations, each rounded
once (no FMA, no transcendental function on the device), so the kernels (csrc/stabilize.cu) and the host restatements here
(host_fit_homographies, host_smooth_path, host_warp_frames) give the same bits.

1. Motion of pair k: a homography A_k from frame k's pixel coordinates to frame k+1's (rnc_homography_fit).
   - Points: p = (s//2 + j s, s//2 + i s) on frame k, s = stride (default 8).  p is matched when both components of F_k(p)
     (the value at the pixel) are finite and q = p + F_k(p), added in fp64, lies in [0, W-1] x [0, H-1].  The matched points
     in raster order form the list L of n points.
   - Coordinates: fp64, normalized by the frame alone, x^ = (x - (W-1)/2) / nu and y^ = (y - (H-1)/2) / nu, nu = max(H, W) / 2,
     for p and q alike (subtraction, then division).
   - Hypotheses: hypothesis h of K (default 256) takes the points of L at splitmix64(seed, 4h + j) mod n, j = 0..3
     (splitmix64(seed, i): z = seed + (i + 1) 0x9E3779B97F4A7C15, z = (z ^ z >> 30) 0xBF58476D1CE4E5B9,
     z = (z ^ z >> 27) 0x94D049BB133111EB, z ^ z >> 31, all mod 2^64); so the draw does not depend on where the pair sits in a
     batch.  It is degenerate when two indices are equal; when three of its source or three of its destination points have
     |(b - a) x (c - a)| < 1e-9 (triples (0,1,2), (0,1,3), (0,2,3), (1,2,3), sources first; the cross product is
     (bx - ax)(cy - ay) - (by - ay)(cx - ax)); or when a pivot is under 1e-12.  Otherwise the DLT system with h33 = 1 is
     solved: rows 2j and 2j + 1 are [x, y, 1, 0, 0, 0, -(u x), -(u y) | u] and [0, 0, 0, x, y, 1, -(v x), -(v y) | v] for point
     j = (x, y) -> (u, v).  The solver (solve8) is Gaussian elimination over columns 0..7 in order: the pivot is the first row
     of k..7 with the largest |a| (a strict > scan from row k), which is swapped into row k; rows k+1..7 in order subtract
     f = a_ik / a_kk times row k (a_ij - f a_kj, columns k+1..8); then back substitution from row 7,
     x_k = (((b_k - a_k,k+1 x_k+1) - a_k,k+2 x_k+2) ...) / a_kk.
   - Scoring: with X = (h0 x + h1 y) + h2, Y = (h3 x + h4 y) + h5, w = (h6 x + h7 y) + 1, a point is an inlier when w > 0 and
     nu^2 ((X/w - u)^2 + (Y/w - v)^2) < tau^2 (tau in pixels, default 2; nu^2 and tau^2 rounded once).  The count is an
     integer; the most inliers wins, a tie goes to the smaller h.
   - Refinement: `refine` rounds (default 4).  Round r marks the inliers of the current H (every point of L in round 0 when
     K = 0, which makes K = 0 plain least squares over all points) and, with at least 4 of them, refits h33 = 1 by algebraic
     least squares: the normal matrix sum a a^T over the inliers' two rows, entry (i, j) of a point being
     (au_i au_j) + (av_i av_j) and right-hand side i (au_i u) + (av_i v), summed from 0.0 in point order within each chunk of
     256 consecutive points of L, then the chunk sums from 0.0 in chunk order; solved by solve8.  A singular refit keeps H.
     A last pass counts the final H's inliers.
   - Output: A_k = M / m33 with M = Tq^-1 H Tp the de-normalization (G = H Tp: g_r0 = h_r0 / nu, g_r1 = h_r1 / nu,
     g_r2 = h_r2 - ((h_r0 cx + h_r1 cy) / nu); then m_0c = nu g_0c + cx g_2c, m_1c = nu g_1c + cy g_2c, m_2c = g_2c), the final
     inlier count, n, and a status: OK, or FEW with A_k the identity and 0 inliers when n < 4, when no hypothesis is
     non-degenerate, when K = 0 and the first refit fails, or when |m33| < 1e-12 (H sends the frame centre to infinity).
2. Path (Matsushita et al., "Full-frame video stabilization with motion inpainting", PAMI 2006; rnc_stabilize_path).
   - T_t^{t+j} for j > 0 is A_{t+j-1} T_t^{t+j-1}, for j < 0 inv(A_{t+j}) T_t^{t+j+1}, from T_t^t = I.  A product's entries
     are ((x_i0 y_0j) + (x_i1 y_1j)) + x_i2 y_2j and every entry is then divided by its [2][2]; inv is the adjugate
     (entry k = a_p a_q - a_r a_s for (p, q, r, s) = _ADJ[k], row-major indices) divided by its [2][2].
   - S_t = sum_j w_|j| T_t^{t+j} / sum_j w_|j| over |j| <= radius (default 30), truncated at the video's ends: the weighted
     matrices are added entrywise from w_0 I, in the order j = 1, 2, ..., then j = -1, -2, ...; dividing by the [2][2] of
     the sum normalizes it to h33 = 1 and removes sum_j w_|j| with it.  The taps w_j = exp(-j^2 / (2 sigma^2)) (sigma default
     10 frames) are computed once on the host in fp64 (gaussian_taps) and passed in.
   - Output frame t shows I_t(S_t^-1 u).
3. Crop.  alpha is the largest scale in [0, 1] such that for every frame the four corners c +- alpha ((W-1)/2, (H-1)/2) of
   the centred rectangle map by inv(S_t) into the frame with w > 0.  With P = inv(S_t), a corner's X, Y and w are
   X0 + alpha X1 and so on, so each of the five constraints w >= 0, X >= 0, (W-1) w - X >= 0, Y >= 0, (H-1) w - Y >= 0
   (crop_alpha states the operations) is f0 + alpha f1 >= 0: f0 < 0 (the frame centre leaves the frame) gives alpha = 0,
   f1 < 0 bounds alpha by f0 / -f1, and alpha is the least bound; no bisection.  With crop=True the zoom by 1 / a about the
   centre, a = max(alpha, crop_min) (1 - 2^-36), is folded into the map, M_t = Z S_t, Z = [[z, 0, cx - cx z], [0, z,
   cy - cy z], [0, 0, 1]], z = 1 / a; with crop=False, M_t = S_t.  The factor 1 - 2^-36 moves the corners about 1e-8 px inside
   the frame, so rounding cannot push the binding corner out.  A video whose alpha falls below crop_min (default 0.5),
   including one whose frame centre leaves a frame, is zoomed by 1 / crop_min, and its uncovered pixels are 0 and flagged.
4. Warp (rnc_stabilize_warp): output pixel u = (x, y) of frame t takes q = inv(M_t) u, ((m0 x + m1 y) + m2) / ((m6 x + m7 y)
   + m8) and the same for y, in fp64, rounded once to float32.  It is valid when w > 0 and q lies in [0, W-1] x [0, H-1];
   its value is then csrc/bilinear.cuh's sample of each channel, otherwise 0 with valid = 0.
5. Fill (fill_uncovered, the motion inpainting of Matsushita et al.; csrc/stabilize_fill.cu): the pixels with valid = 0 are
   carried along the flows from the frames that see them, instead of being cropped.  Inputs, per video: the warped frames
   and valid masks of step 4, the maps M_t and M_t^-1 of step 2, the motions A_k of step 1, and the forward flows F_k (frame
   k -> k+1) and backward flows G_k (frame k+1 -> k) in input coordinates (run_sequences_bidirectional's flow_up and
   flow_up_bw).  pi(P p) is ((p0 x + p1 y) + p2) / ((p6 x + p7 y) + p8) and the same for y in fp64 (each product, sum and
   quotient rounded once), defined when the denominator is > 0; inv(A) is the adjugate divided by its [2][2] (as in step 2).
   a. Residual transfer (rnc_stabilize_flow_residual), forward, output pixel u of frame k: q = M_k^-1 u exactly as step 4
      computes it, with its validity; F = csrc/bilinear.cuh's sample of each channel of F_k at q; then
      R_k(u) = pi(M_{k+1} (q + F)) - pi(M_{k+1} pi(A_k q)), q + F added in fp64, the subtraction in fp64, rounded once to
      float32.  Backward, output pixel u of frame k+1: the same with M_{k+1}^-1, G_k, M_k and inv(A_k).  R is NaN where q is
      not valid, where F is not finite and where a projection is undefined.  So the camera's motion, known exactly, is taken
      out, and for a static scene R is 0 up to the flow's own error.
   b. Residual completion: R~ = rnc.inpaint.harmonic_fill(R, valid == 0, sweeps), the unknown set being output frame k's
      pixels with valid = 0 (frame k+1's for the backward residual) plus R's NaNs, which are exactly them when the flow is
      finite and every projection defined.
   c. Global re-add (rnc_stabilize_flow_readd): F~_k(u) = (pi(M_{k+1} pi(A_k q)) - u) + R~_k(u), q = M_k^-1 u rounded to
      float32 as in a (for every pixel, inside the frame or not), the subtraction and the addition in fp64, rounded once to
      float32; NaN where a projection is undefined; backward likewise.  The global term is exact for a homography across
      the whole border, where completing the full flow by a Laplace fill would bend it.
   d. Chains (rnc.inpaint's steps 3-4 on the output frames): occ, occ_bw = rnc.metrics.fb_consistency(F~, G~, alpha1,
      alpha2); rnc.inpaint.inpaint_propagate(warped frames, valid == 0, F~, G~, occ, occ_bw, max_distance); then
      harmonic_fill of the colours of the SOURCE_SPATIAL pixels.  The pixels with valid != 0 keep step 4's bits; source
      holds rnc.inpaint's SOURCE_* values, SOURCE_KNOWN for a pixel taken from its own frame.  In a stack of videos of
      different lengths, a shorter video's padding pairs are occluded in both directions, as rnc.harness.inpaint_videos
      pads them, so each video's result does not depend on the others.

Scores (stabilization_metrics, on the host in fp64, from the known maps rather than re-estimated features; Liu et al.,
"Bundled camera paths for video stabilization", SIGGRAPH 2013): cropping, the mean over frames of 1 / |det| of M_t's affine
part; distortion, the least over frames of that part's singular-value ratio; stability, from the output's inter-frame motion
B_t = M_{t+1} A_t M_t^-1 (the input's is A_t), whose translation (b02, b12) and rotation atan2(b10, b00) are accumulated into
paths: the energy of the five lowest non-zero frequencies of the paths' FFT over all non-zero ones (x and y added for the
translation; 1 for a path with no non-zero energy), reported for translation, rotation and their minimum.  The harness adds
ITF, the mean PSNR of consecutive frames (Matsushita et al.).
"""
import math

import numpy as np
import torch

from . import native
from .inpaint import _check_sweeps, _check_video, _complete, _max_distance, _propagate, psnr
from .restate import check_sides, inside, project, sample

DEFAULT_STRIDE, DEFAULT_HYPOTHESES, DEFAULT_TAU, DEFAULT_REFINE = 8, 256, 2.0, 4
DEFAULT_RADIUS, DEFAULT_SIGMA, DEFAULT_CROP_MIN = 30, 10.0, 0.5
OK, FEW = native.HOMOGRAPHY_OK, native.HOMOGRAPHY_FEW
PIVOT_MIN, COLLINEAR = 1e-12, 1e-9
CHUNK = 256
SHRINK = 1.0 - 2.0 ** -36
_M64 = (1 << 64) - 1


def _is_int(v):
    return isinstance(v, (int, np.integer)) and not isinstance(v, bool)


def _check_fit_params(stride, hypotheses, tau, refine, seed, what):
    if not _is_int(stride) or not 1 <= stride <= 256:
        raise ValueError(f"{what}: expected 1 <= stride <= 256, got {stride!r}")
    if not _is_int(hypotheses) or not 0 <= hypotheses <= 65536:
        raise ValueError(f"{what}: expected 0 <= hypotheses <= 65536, got {hypotheses!r}")
    if not _is_int(refine) or not 0 <= refine <= 64:
        raise ValueError(f"{what}: expected 0 <= refine <= 64, got {refine!r}")
    if hypotheses == 0 and refine == 0:
        raise ValueError(f"{what}: hypotheses = 0 needs refine >= 1 (the least-squares fit over all points)")
    if not isinstance(tau, (int, float)) or isinstance(tau, bool) or not 0 < tau <= 1e300:
        raise ValueError(f"{what}: expected a finite tau > 0, got {tau!r}")
    if not _is_int(seed) or not 0 <= seed <= _M64:
        raise ValueError(f"{what}: expected a seed in [0, 2^64), got {seed!r}")


def _check_path_params(radius, sigma, crop_min, what):
    if not _is_int(radius) or not 0 <= radius <= 1024:
        raise ValueError(f"{what}: expected 0 <= radius <= 1024, got {radius!r}")
    if not isinstance(sigma, (int, float)) or isinstance(sigma, bool) or not 0 < sigma <= 1e300:
        raise ValueError(f"{what}: expected a finite sigma > 0, got {sigma!r}")
    if not isinstance(crop_min, (int, float)) or isinstance(crop_min, bool) or not 0 < crop_min <= 1:
        raise ValueError(f"{what}: expected 0 < crop_min <= 1, got {crop_min!r}")


# ------------------------------------------------------------------------------------------------------------- the fit


def _check_flow(flow, what="fit_homographies"):
    if flow.dim() != 4 or flow.shape[1] != 2 or flow.shape[0] == 0:
        raise ValueError(f"{what}: expected flow [N,2,H,W], got {tuple(flow.shape)}")
    N, _, H, W = flow.shape
    if N > 65535:
        raise ValueError(f"{what}: at most 65535 pairs per call, got {N}")
    check_sides(H, W, what)
    return N, H, W


def fit_homographies(flow, stride=DEFAULT_STRIDE, hypotheses=DEFAULT_HYPOTHESES, tau=DEFAULT_TAU, refine=DEFAULT_REFINE, seed=0,
                     workspace=None):
    """The motion of N pairs: flow [N,2,H,W] (forward flows, any strides, float32 or converted to it).  Returns (A fp64
    [N,3,3], inliers int32 [N], matched int32 [N], status int32 [N], OK or FEW) on the flow's device.  CUDA tensors go through
    rnc_homography_fit (5 + 2 (refine + 1) launches on the current stream, no host synchronisation; `workspace`, a uint8 CUDA
    tensor of at least rnc_homography_fit_workspace_bytes, is used when given), CPU tensors through host_fit_homographies;
    they give the same bits, and a pair's result does not depend on N or its position.  ValueError before any launch for a
    bad shape, more than 65535 pairs, a side above 4096 or a bad stride, hypotheses, tau, refine or seed."""
    N, H, W = _check_flow(flow)
    _check_fit_params(stride, hypotheses, tau, refine, seed, "fit_homographies")
    if not flow.is_cuda:
        return _host_fit(flow, stride, hypotheses, tau, refine, seed)
    dev = flow.device
    f = flow.detach().float()
    A = torch.empty(N, 3, 3, dtype=torch.float64, device=dev)
    counts = torch.empty(3, N, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        nbytes = native.rnc.homography_fit_workspace_bytes(N, H, W, stride, hypotheses)
        if workspace is None or workspace.numel() < nbytes:
            workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        native.rnc.homography_fit(f, *f.stride(), N, H, W, stride, hypotheses, float(tau), refine, int(seed), A, counts[0],
                                  counts[1], counts[2], workspace, workspace.numel())
    return A, counts[0], counts[1], counts[2]


def splitmix64(seed, i):
    """splitmix64(seed, i) of numpy uint64 arrays i (the module docstring's draw), mod 2^64."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + (i.astype(np.uint64) + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def match_points(flow, stride):
    """(L fp64 [n,4] of x^, y^, u^, v^ in raster order, nu) of one pair's flow (numpy float32 [2,H,W]): the module docstring's
    points and normalization."""
    _, H, W = flow.shape
    ys, xs = np.arange(stride // 2, H, stride), np.arange(stride // 2, W, stride)
    y, x = (a.astype(np.float64).ravel() for a in np.meshgrid(ys, xs, indexing="ij"))
    ux = flow[0][np.ix_(ys, xs)].ravel().astype(np.float64)
    uy = flow[1][np.ix_(ys, xs)].ravel().astype(np.float64)
    qx, qy = x + ux, y + uy
    m = np.isfinite(ux) & np.isfinite(uy) & (qx >= 0) & (qx <= W - 1) & (qy >= 0) & (qy <= H - 1)
    cx, cy, nu = (W - 1) * 0.5, (H - 1) * 0.5, max(H, W) * 0.5
    L = np.stack([(x[m] - cx) / nu, (y[m] - cy) / nu, (qx[m] - cx) / nu, (qy[m] - cy) / nu], 1)
    return L, nu


def solve8(a):
    """solve8 of the module docstring on a batch of augmented systems a fp64 [B,8,9] (modified in place).  Returns (ok bool
    [B], x fp64 [B,8]); x is meaningless where ok is False."""
    B = a.shape[0]
    ok = np.ones(B, dtype=bool)
    r = np.arange(B)
    with np.errstate(all="ignore"):
        for k in range(8):
            best, p = np.abs(a[:, k, k]), np.full(B, k)
            for i in range(k + 1, 8):
                v = np.abs(a[:, i, k])
                up = v > best
                best, p = np.where(up, v, best), np.where(up, i, p)
            ok &= best >= PIVOT_MIN
            rows_k, rows_p = a[r, k].copy(), a[r, p].copy()
            a[r, p] = rows_k
            a[r, k] = rows_p
            for i in range(k + 1, 8):
                f = a[:, i, k] / a[:, k, k]
                a[:, i, k + 1:] = a[:, i, k + 1:] - f[:, None] * a[:, k, k + 1:]
        for k in range(7, -1, -1):
            s = a[:, k, 8].copy()
            for j in range(k + 1, 8):
                s = s - a[:, k, j] * a[:, j, 8]
            a[:, k, 8] = s / a[:, k, k]
    return ok, a[:, :, 8].copy()


def _rows(L):
    """The DLT rows of the points L [n,4]: au, av [n,8], and u, v."""
    x, y, u, v = L[:, 0], L[:, 1], L[:, 2], L[:, 3]
    z, o = np.zeros_like(x), np.ones_like(x)
    au = np.stack([x, y, o, z, z, z, -(u * x), -(u * y)], 1)
    av = np.stack([z, z, z, x, y, o, -(v * x), -(v * y)], 1)
    return au, av, u, v


def inliers_of(h, L, nu2, tau2):
    """The inlier test of hypotheses h fp64 [B,8] on the points L [n,4]: bool [B,n]."""
    x, y, u, v = (L[None, :, k] for k in range(4))
    h = h[:, :, None]
    with np.errstate(all="ignore"):
        w = (h[:, 6] * x + h[:, 7] * y) + 1.0
        X = (h[:, 0] * x + h[:, 1] * y) + h[:, 2]
        Y = (h[:, 3] * x + h[:, 4] * y) + h[:, 5]
        ex, ey = X / w - u, Y / w - v
        return (w > 0) & (nu2 * (ex * ex + ey * ey) < tau2)


def _cross_ok(P, o):
    ok = np.ones(P.shape[0], dtype=bool)
    for a, b, c in ((0, 1, 2), (0, 1, 3), (0, 2, 3), (1, 2, 3)):
        ax, ay, bx, by, cx, cy = P[:, a, o], P[:, a, o + 1], P[:, b, o], P[:, b, o + 1], P[:, c, o], P[:, c, o + 1]
        ok &= np.abs((bx - ax) * (cy - ay) - (by - ay) * (cx - ax)) >= COLLINEAR
    return ok


def _hypotheses(L, K, seed, nu2, tau2):
    """Every hypothesis's inlier count (-1 when degenerate) and H [K,8]."""
    n = L.shape[0]
    idx = (splitmix64(seed, np.arange(4 * K, dtype=np.uint64)) % np.uint64(n)).astype(np.int64).reshape(K, 4)
    ok = np.ones(K, dtype=bool)
    for a in range(4):
        for b in range(a + 1, 4):
            ok &= idx[:, a] != idx[:, b]
    P = L[idx]                                                        # [K,4,4]
    ok &= _cross_ok(P, 0) & _cross_ok(P, 2)
    sys_ = np.zeros((K, 8, 9))
    for j in range(4):
        x, y, u, v = P[:, j, 0], P[:, j, 1], P[:, j, 2], P[:, j, 3]
        sys_[:, 2 * j, :] = np.stack([x, y, np.ones(K), np.zeros(K), np.zeros(K), np.zeros(K), -(u * x), -(u * y), u], 1)
        sys_[:, 2 * j + 1, :] = np.stack([np.zeros(K), np.zeros(K), np.zeros(K), x, y, np.ones(K), -(v * x), -(v * y), v], 1)
    solved, h = solve8(sys_)
    ok &= solved
    counts = np.full(K, -1, dtype=np.int64)
    for s in range(0, K, 64):                                         # bounded memory: 64 hypotheses x n points at a time
        e = min(K, s + 64)
        counts[s:e] = np.where(ok[s:e], inliers_of(h[s:e], L, nu2, tau2).sum(1), -1)
    return counts, h


def _normal_sums(L, flags):
    """The refit's 36 upper-triangle entries, 8 right-hand sides and count: chunk sums in point order, then chunks in order."""
    au, av, u, v = _rows(L)
    iu, ju = np.triu_indices(8)
    terms = np.concatenate([au[:, iu] * au[:, ju] + av[:, iu] * av[:, ju], au * u[:, None] + av * v[:, None]], 1)
    total, count = np.zeros(44), 0
    for c in range(0, L.shape[0], CHUNK):
        sel = terms[c:c + CHUNK][flags[c:c + CHUNK]]
        part = np.add.accumulate(np.concatenate([np.zeros((1, 44)), sel]), 0)[-1]     # from 0.0, in point order
        total = total + part
        count += int(flags[c:c + CHUNK].sum())
    return total, count


def _refit(total):
    """The normal equations from _normal_sums' entries, solved by solve8: (ok, h [8])."""
    a = np.zeros((1, 8, 9))
    iu, ju = np.triu_indices(8)
    a[0, iu, ju] = total[:36]
    a[0, ju, iu] = total[:36]
    a[0, :, 8] = total[36:]
    ok, x = solve8(a)
    return bool(ok[0]), x[0]


def denormalize(h, H, W):
    """H (normalized, h33 = 1) to pixel coordinates, A = M / m33 as the module docstring writes it; None when |m33| < 1e-12."""
    cx, cy, nu = (W - 1) * 0.5, (H - 1) * 0.5, max(H, W) * 0.5
    hm = [float(v) for v in h] + [1.0]
    g = [0.0] * 9
    for r in range(3):
        g[3 * r] = hm[3 * r] / nu
        g[3 * r + 1] = hm[3 * r + 1] / nu
        g[3 * r + 2] = hm[3 * r + 2] - (hm[3 * r] * cx + hm[3 * r + 1] * cy) / nu
    m = [0.0] * 9
    for c in range(3):
        m[c] = nu * g[c] + cx * g[6 + c]
        m[3 + c] = nu * g[3 + c] + cy * g[6 + c]
        m[6 + c] = g[6 + c]
    if not abs(m[8]) >= PIVOT_MIN:
        return None
    return np.array([v / m[8] for v in m]).reshape(3, 3)


def host_fit_pair(flow, stride=DEFAULT_STRIDE, hypotheses=DEFAULT_HYPOTHESES, tau=DEFAULT_TAU, refine=DEFAULT_REFINE, seed=0):
    """One pair's fit on the host, flow numpy float32 [2,H,W].  Returns a dict: A fp64 [3,3], inliers, matched, status, and
    the trace: L, the winning hypothesis h_best (None under FEW or K = 0) and rounds, one (inlier flags, H after the round)
    per refine round."""
    _, H, W = flow.shape
    L, nu = match_points(flow, stride)
    n = L.shape[0]
    nu2, tau2 = nu * nu, float(tau) * float(tau)
    ident = np.array([1.0, 0, 0, 0, 1.0, 0, 0, 0])
    out = {"A": np.eye(3), "inliers": 0, "matched": n, "status": FEW, "L": L, "h_best": None, "rounds": []}
    if n < 4:
        return out
    cur = ident.copy()
    if hypotheses > 0:
        counts, hs = _hypotheses(L, hypotheses, seed, nu2, tau2)
        b = int(np.argmax(counts))                                    # the first of the largest: ties to the smaller h
        if counts[b] < 0:
            return out
        cur = hs[b].copy()
        out["h_best"] = cur.copy()
    count = 0
    for r in range(refine + 1):
        flags = np.ones(n, dtype=bool) if r == 0 and hypotheses == 0 else inliers_of(cur[None], L, nu2, tau2)[0]
        total, count = _normal_sums(L, flags)
        if r == refine:
            break
        solved, h = _refit(total) if count >= 4 else (False, None)
        if solved:
            cur = h
        elif r == 0 and hypotheses == 0:
            return out
        out["rounds"].append((flags, cur.copy()))
    A = denormalize(cur, H, W)
    if A is None:
        return out
    out.update(A=A, inliers=count, status=OK)
    return out


def _host_fit(flow, stride, hypotheses, tau, refine, seed):
    N = flow.shape[0]
    A = torch.empty(N, 3, 3, dtype=torch.float64)
    counts = torch.empty(3, N, dtype=torch.int32)
    for i in range(N):
        r = host_fit_pair(flow[i].detach().cpu().float().numpy(), stride, hypotheses, tau, refine, seed)
        A[i] = torch.from_numpy(r["A"])
        counts[:, i] = torch.tensor([r["inliers"], r["matched"], r["status"]], dtype=torch.int32)
    return A, counts[0], counts[1], counts[2]


def host_fit_homographies(flow, stride=DEFAULT_STRIDE, hypotheses=DEFAULT_HYPOTHESES, tau=DEFAULT_TAU, refine=DEFAULT_REFINE,
                          seed=0):
    """fit_homographies' rule in numpy fp64, all hypotheses of a pair at once (each elementwise operation is the kernel's,
    rounded once; the chunk sums by np.add.accumulate, which adds in order).  Serves CPU tensors and is the kernel's test
    reference.  Returns (A fp64 [N,3,3], inliers, matched, status int32 [N]) on the CPU."""
    _check_flow(flow)
    _check_fit_params(stride, hypotheses, tau, refine, seed, "fit_homographies")
    return _host_fit(flow, stride, hypotheses, tau, refine, seed)


# ------------------------------------------------------------------------------------------------------------ the path


def gaussian_taps(radius=DEFAULT_RADIUS, sigma=DEFAULT_SIGMA):
    """w_j = exp(-j^2 / (2 sigma^2)), j = 0..radius, fp64 [radius + 1] (a torch tensor on the CPU)."""
    _check_path_params(radius, sigma, 1.0, "gaussian_taps")
    return torch.tensor([math.exp(-(j * j) / (2.0 * sigma * sigma)) for j in range(radius + 1)], dtype=torch.float64)


def _mul_norm(X, Y):
    """Batched products [B,3,3] with the module docstring's order, each divided by its [2][2]."""
    P = np.empty(np.broadcast_shapes(X.shape, Y.shape))
    for i in range(3):
        for j in range(3):
            P[..., i, j] = (X[..., i, 0] * Y[..., 0, j] + X[..., i, 1] * Y[..., 1, j]) + X[..., i, 2] * Y[..., 2, j]
    return P / P[..., 2:3, 2:3]


_ADJ = ((4, 8, 5, 7), (2, 7, 1, 8), (1, 5, 2, 4), (5, 6, 3, 8), (0, 8, 2, 6), (2, 3, 0, 5), (3, 7, 4, 6), (1, 6, 0, 7),
        (0, 4, 1, 3))


def _inv(A):
    """The adjugate of [B,3,3], cofactor k = a_p a_q - a_r a_s for (p, q, r, s) = _ADJ[k], divided by its [2][2]."""
    a = A.reshape(*A.shape[:-2], 9)
    C = np.stack([a[..., p] * a[..., q] - a[..., r] * a[..., s] for p, q, r, s in _ADJ], -1).reshape(A.shape)
    return C / C[..., 2:3, 2:3]


def crop_alpha(S, H, W):
    """Per frame, the largest alpha in [0, 1] such that inv(S_t) maps the corners of the centred alpha (W-1) x alpha (H-1)
    rectangle into the frame with w > 0, by the closed form of the module docstring: S fp64 [T,3,3] (numpy).  Returns fp64
    [T]; the video's alpha is its minimum."""
    with np.errstate(all="ignore"):
        P = _inv(np.asarray(S, dtype=np.float64)).reshape(-1, 9)
        cx, cy, wm, hm = (W - 1) * 0.5, (H - 1) * 0.5, float(W - 1), float(H - 1)
        X0 = (P[:, 0] * cx + P[:, 1] * cy) + P[:, 2]
        Y0 = (P[:, 3] * cx + P[:, 4] * cy) + P[:, 5]
        W0 = (P[:, 6] * cx + P[:, 7] * cy) + P[:, 8]
        a = np.ones(P.shape[0])
        for k in range(4):
            dx, dy = (cx if k & 1 else -cx), (cy if k & 2 else -cy)
            X1 = P[:, 0] * dx + P[:, 1] * dy
            Y1 = P[:, 3] * dx + P[:, 4] * dy
            W1 = P[:, 6] * dx + P[:, 7] * dy
            for f0, f1 in ((W0, W1), (X0, X1), (wm * W0 - X0, wm * W1 - X1), (Y0, Y1), (hm * W0 - Y0, hm * W1 - Y1)):
                r = f0 / -f1
                a = np.where(~(f0 >= 0), 0.0, np.where((f1 < 0) & (r < a), r, a))
    return a


def _check_motion(motion, H, W, what):
    if motion.dim() != 4 or tuple(motion.shape[2:]) != (3, 3) or motion.shape[0] == 0 or motion.shape[1] == 0:
        raise ValueError(f"{what}: expected motion [V,T-1,3,3], got {tuple(motion.shape)}")
    if motion.shape[0] > 65535:
        raise ValueError(f"{what}: at most 65535 videos per call, got {motion.shape[0]}")
    check_sides(H, W, what)
    return motion.shape[0], motion.shape[1] + 1


def smooth_path(motion, H, W, radius=DEFAULT_RADIUS, sigma=DEFAULT_SIGMA, crop=True, crop_min=DEFAULT_CROP_MIN):
    """The smoothed path of V videos: motion fp64 [V,T-1,3,3] (the A_k of fit_homographies), frames of H x W.  Returns
    (M fp64 [V,T,3,3], Minv fp64 [V,T,3,3], alpha fp64 [V]) on motion's device: M_t maps frame t to the output (Z S_t with
    crop, S_t without), Minv_t is its adjugate inverse (the warp's input-from-output map), alpha the closed-form crop scale.
    CUDA tensors go through rnc_stabilize_path (one launch, a CTA per video), CPU tensors through host_smooth_path; they give
    the same bits.  ValueError before any launch for a bad shape, a side above 4096 or a bad radius, sigma or crop_min."""
    V, T = _check_motion(motion, H, W, "smooth_path")
    _check_path_params(radius, sigma, crop_min, "smooth_path")
    if not motion.is_cuda:
        return _host_path(motion, H, W, radius, sigma, crop, crop_min)
    dev = motion.device
    A = motion.detach().to(torch.float64).contiguous()
    taps = gaussian_taps(radius, sigma).to(dev)
    M = torch.empty(V, T, 3, 3, dtype=torch.float64, device=dev)
    Minv = torch.empty_like(M)
    alpha = torch.empty(V, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        native.rnc.stabilize_path(A, V, T, taps, radius, H, W, int(bool(crop)), float(crop_min), M, Minv, alpha)
    return M, Minv, alpha


def _host_path(motion, H, W, radius, sigma, crop, crop_min):
    V, T = motion.shape[0], motion.shape[1] + 1
    w = gaussian_taps(radius, sigma).numpy()
    M = np.empty((V, T, 3, 3))
    Minv = np.empty((V, T, 3, 3))
    alpha = np.empty(V)
    cx, cy = (W - 1) * 0.5, (H - 1) * 0.5
    eye = np.broadcast_to(np.eye(3), (T, 3, 3))
    t = np.arange(T)
    with np.errstate(all="ignore"):
        for v in range(V):
            A = motion[v].detach().cpu().to(torch.float64).numpy()
            num = np.where(np.eye(3, dtype=bool), w[0], 0.0) * np.ones((T, 1, 1))
            for sign in (1, -1):
                P = eye.copy()
                reach = np.minimum(radius, T - 1 - t) if sign > 0 else np.minimum(radius, t)
                for j in range(1, radius + 1):
                    live = j <= reach
                    if not live.any():
                        break
                    k = np.clip(t + j - 1 if sign > 0 else t - j, 0, T - 2)
                    step = A[k] if sign > 0 else _inv(A[k])
                    P = np.where(live[:, None, None], _mul_norm(step, P), P)
                    num = np.where(live[:, None, None], num + w[j] * P, num)
            S = num / num[:, 2:3, 2:3]
            alpha[v] = crop_alpha(S, H, W).min()
            a = (alpha[v] if not alpha[v] < crop_min else crop_min) * SHRINK
            z = 1.0 / a
            Z = np.array([[z, 0.0, cx - cx * z], [0.0, z, cy - cy * z], [0.0, 0.0, 1.0]])
            Mv = _mul_norm(Z[None], S) if crop else S
            M[v], Minv[v] = Mv, _inv(Mv)
    return torch.from_numpy(M), torch.from_numpy(Minv), torch.from_numpy(alpha)


def host_smooth_path(motion, H, W, radius=DEFAULT_RADIUS, sigma=DEFAULT_SIGMA, crop=True, crop_min=DEFAULT_CROP_MIN):
    """smooth_path's rule in numpy fp64, all frames of a video at once.  Returns (M, Minv, alpha) on the CPU."""
    _check_motion(motion, H, W, "smooth_path")
    _check_path_params(radius, sigma, crop_min, "smooth_path")
    return _host_path(motion, H, W, radius, sigma, crop, crop_min)


# ------------------------------------------------------------------------------------------------------------ the warp


def _check_warp(frames, maps):
    if frames.dim() != 4 or frames.shape[0] == 0:
        raise ValueError(f"warp_frames: expected frames [N,C,H,W], got {tuple(frames.shape)}")
    N, C, H, W = frames.shape
    if not 1 <= C <= 4:
        raise ValueError(f"warp_frames: expected 1 to 4 channels, got {C}")
    if tuple(maps.shape) != (N, 3, 3):
        raise ValueError(f"warp_frames: expected maps {[N, 3, 3]}, got {tuple(maps.shape)}")
    if frames.device != maps.device:
        raise ValueError(f"warp_frames: frames on {frames.device}, maps on {maps.device}; they must be on one device")
    if N > 65535:
        raise ValueError(f"warp_frames: at most 65535 frames per call, got {N}")
    check_sides(H, W, "warp_frames")
    return N, C, H, W


def warp_frames(frames, maps):
    """frames [N,C,H,W] (1 <= C <= 4, any strides, float32 or converted to it) warped by maps fp64 [N,3,3] (output ->
    input, smooth_path's Minv).  Returns (out float32 [N,C,H,W], valid uint8 [N,H,W]) on the frames' device.  CUDA tensors go
    through rnc_stabilize_warp (one launch), CPU tensors through host_warp_frames; they give the same bits.  ValueError
    before any launch for mismatched shapes or devices, a channel count outside 1..4 or a side above 4096."""
    N, C, H, W = _check_warp(frames, maps)
    if not frames.is_cuda:
        return host_warp_frames(frames, maps)
    dev = frames.device
    f = frames.detach().float()
    m = maps.detach().to(torch.float64).contiguous()
    out = torch.empty(N, C, H, W, dtype=torch.float32, device=dev)
    valid = torch.empty(N, H, W, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        native.rnc.stabilize_warp(f, *f.stride(), m, N, C, H, W, out, *out.stride(), valid, *valid.stride())
    return out, valid


def host_warp_frames(frames, maps):
    """warp_frames' rule on the host: q in numpy fp64, rounded to float32, and rnc.restate.sample.  Returns (out, valid) on
    the CPU."""
    N, C, H, W = _check_warp(frames, maps)
    out = torch.zeros(N, C, H, W, dtype=torch.float32)
    valid = torch.zeros(N, H, W, dtype=torch.uint8)
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    with np.errstate(all="ignore"):
        for n in range(N):
            m = maps[n].detach().cpu().to(torch.float64).numpy().ravel()
            X, Y, ok = project(m, x, y)
            qx, qy = X.astype(np.float32), Y.astype(np.float32)
            ok &= inside(qx, qy, H, W)
            px = torch.from_numpy(np.where(ok, qx, 0).astype(np.float64))
            py = torch.from_numpy(np.where(ok, qy, 0).astype(np.float64))
            s = sample(frames[n].detach().cpu().float().double(), px, py)
            okt = torch.from_numpy(ok)
            out[n] = torch.where(okt, s, 0.0).float()
            valid[n] = okt.to(torch.uint8)
    return out, valid


# ------------------------------------------------------------------------------------------------------------ the fill


def _check_flow_maps(flow, flow_bw, motion, maps, maps_inv, what):
    """(V, T, H, W) of stacked flows [V,T-1,2,H,W], motion [V,T-1,3,3] and maps [V,T,3,3] on one device."""
    if flow.dim() != 5 or flow.shape[2] != 2 or flow.shape[0] == 0 or flow.shape[1] == 0:
        raise ValueError(f"{what}: expected flow [V,T-1,2,H,W], got {tuple(flow.shape)}")
    V, T1, _, H, W = flow.shape
    T = T1 + 1
    for name, t, shape in (("flow_bw", flow_bw, (V, T1, 2, H, W)), ("motion", motion, (V, T1, 3, 3)),
                           ("maps", maps, (V, T, 3, 3)), ("maps_inv", maps_inv, (V, T, 3, 3))):
        if tuple(t.shape) != shape:
            raise ValueError(f"{what}: expected {name} {list(shape)}, got {tuple(t.shape)}")
    devs = {t.device for t in (flow, flow_bw, motion, maps, maps_inv)}
    if len(devs) != 1:
        raise ValueError(f"{what}: the flows, motion and maps must be on one device, got {sorted(map(str, devs))}")
    if V > 65535 or T > 65536:
        raise ValueError(f"{what}: at most 65535 videos of 65536 frames per call, got {V} of {T}")
    check_sides(H, W, what)
    return V, T, H, W


def _mats(*ts):
    return [t.detach().to(torch.float64).contiguous() for t in ts]


def flow_residual(flow, flow_bw, motion, maps, maps_inv):
    """Step 5a for V videos: flow, flow_bw [V,T-1,2,H,W] (forward and backward flows in input coordinates, any strides,
    float32 or converted to it), motion fp64 [V,T-1,3,3] (A_k), maps and maps_inv fp64 [V,T,3,3] (smooth_path's M and
    Minv).  Returns (res, res_bw) float32 [V,T-1,2,H,W], contiguous, on the flows' device: pair k's residual in output frame
    k's pixels and its backward residual in output frame k+1's, NaN where unknown.  CUDA tensors go through
    rnc_stabilize_flow_residual (one launch), CPU tensors through host_flow_residual; they give the same bits.  ValueError
    before any launch for mismatched shapes or devices, or a side above 4096."""
    V, T, H, W = _check_flow_maps(flow, flow_bw, motion, maps, maps_inv, "flow_residual")
    if not flow.is_cuda:
        return host_flow_residual(flow, flow_bw, motion, maps, maps_inv)
    f, b = flow.detach().float(), flow_bw.detach().float()
    A, M, Mi = _mats(motion, maps, maps_inv)
    res = torch.empty(2, V, T - 1, 2, H, W, dtype=torch.float32, device=flow.device)
    with torch.cuda.device(flow.device):
        native.rnc.stabilize_flow_residual(f, *f.stride(), b, *b.stride(), A, M, Mi, V, T, H, W, res[0], res[1])
    return res[0], res[1]


def _readd_(res, res_bw, motion, maps, maps_inv):
    """Step 5c in place on float32 contiguous res, res_bw [V,T-1,2,H,W]."""
    V, T1, _, H, W = res.shape
    if not res.is_cuda:
        r = _host_flows(res, res_bw, motion, maps, maps_inv, True)
        res.copy_(r[0])
        res_bw.copy_(r[1])
        return
    A, M, Mi = _mats(motion, maps, maps_inv)
    with torch.cuda.device(res.device):
        native.rnc.stabilize_flow_readd(A, M, Mi, V, T1 + 1, H, W, res, res_bw)


def add_global_motion(res, res_bw, motion, maps, maps_inv):
    """Step 5c for V videos: the completed residuals res, res_bw [V,T-1,2,H,W] (any strides, float32 or converted to it)
    with the camera's motion added back, as new float32 [V,T-1,2,H,W] tensors: the flows of the output frames, forward
    (frame k -> k+1, in frame k's pixels) and backward (frame k+1 -> k).  CUDA tensors go through rnc_stabilize_flow_readd
    (one launch), CPU tensors through host_add_global_motion; they give the same bits.  ValueError before any launch for
    mismatched shapes or devices, or a side above 4096."""
    _check_flow_maps(res, res_bw, motion, maps, maps_inv, "add_global_motion")
    if not res.is_cuda:
        return host_add_global_motion(res, res_bw, motion, maps, maps_inv)
    out = torch.stack([res.detach().float(), res_bw.detach().float()])
    _readd_(out[0], out[1], motion, maps, maps_inv)
    return out[0], out[1]


def _host_direction(src, dst, A, f, r):
    """One direction of step 5a (r None: f fp64 [2,H,W] holding the flow's float32 values) or 5c (r: the completed residual,
    fp64 [2,H,W] holding float32 values) over every output pixel: float32 [2,H,W]."""
    H, W = f.shape[-2:] if r is None else r.shape[-2:]
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    X, Y, ok = project(src, x, y)
    qx, qy = X.astype(np.float32).astype(np.float64), Y.astype(np.float32).astype(np.float64)
    bx, by, ok_b = project(A, qx, qy)
    gx, gy, ok_g = project(dst, bx, by)
    ok = ok & ok_b & ok_g
    if r is not None:
        out = np.stack([(gx - x) + r[0], (gy - y) + r[1]])
        return np.where(ok, out, np.nan).astype(np.float32)
    ok &= inside(qx, qy, H, W)
    px = torch.from_numpy(np.where(ok, qx, 0.0))
    py = torch.from_numpy(np.where(ok, qy, 0.0))
    u = sample(torch.from_numpy(f), px, py).numpy()
    ok &= np.isfinite(u).all(0)
    ax, ay, ok_a = project(dst, qx + u[0], qy + u[1])
    ok &= ok_a
    return np.where(ok, np.stack([ax - gx, ay - gy]), np.nan).astype(np.float32)


def _host_flows(a, b, motion, maps, maps_inv, readd):
    """Steps 5a (readd False: a, b the flows) and 5c (readd True: a, b the completed residuals), every video and pair."""
    V, T1, _, H, W = a.shape
    out = torch.empty(2, V, T1, 2, H, W, dtype=torch.float32)
    A, M, Mi = (t.detach().cpu().to(torch.float64).numpy().reshape(t.shape[0], t.shape[1], 9) for t in (motion, maps, maps_inv))
    with np.errstate(all="ignore"):
        for v in range(V):
            for k in range(T1):
                fa, fb = (t[v, k].detach().cpu().float().double().numpy() for t in (a, b))
                Ai = _inv(A[v, k].reshape(3, 3)).ravel()
                fw = _host_direction(Mi[v, k], M[v, k + 1], A[v, k], None if readd else fa, fa if readd else None)
                bw = _host_direction(Mi[v, k + 1], M[v, k], Ai, None if readd else fb, fb if readd else None)
                out[0, v, k], out[1, v, k] = torch.from_numpy(fw), torch.from_numpy(bw)
    return out[0], out[1]


def host_flow_residual(flow, flow_bw, motion, maps, maps_inv):
    """flow_residual's rule in numpy fp64, one output frame at a time and all its pixels at once; the flow sampled by
    rnc.restate.sample.  Serves CPU tensors and is the kernel's test reference.  Returns (res, res_bw) on the CPU."""
    _check_flow_maps(flow, flow_bw, motion, maps, maps_inv, "flow_residual")
    return _host_flows(flow, flow_bw, motion, maps, maps_inv, False)


def host_add_global_motion(res, res_bw, motion, maps, maps_inv):
    """add_global_motion's rule in numpy fp64, one output frame at a time.  Returns (flow, flow_bw) on the CPU."""
    _check_flow_maps(res, res_bw, motion, maps, maps_inv, "add_global_motion")
    return _host_flows(res, res_bw, motion, maps, maps_inv, True)


def _check_fill_params(sweeps, max_distance, alpha1, alpha2, what):
    _check_sweeps(sweeps, what)
    _max_distance(max_distance, what)
    for name, a in (("alpha1", alpha1), ("alpha2", alpha2)):
        if not isinstance(a, (int, float)) or isinstance(a, bool) or not 0 <= a <= 1e30:
            raise ValueError(f"{what}: expected a finite {name} >= 0, got {a!r}")


def _check_fill_uncovered(frames, valid, flow, flow_bw, motion, maps, maps_inv, sweeps, max_distance, alpha1, alpha2):
    V, T, H, W = _check_video(frames, valid, flow, flow_bw, "fill_uncovered")
    _check_flow_maps(flow, flow_bw, motion, maps, maps_inv, "fill_uncovered")
    if frames.device != flow.device or valid.device != flow.device:
        raise ValueError(f"fill_uncovered: the frames, valid masks, flows, motion and maps must be on one device, got "
                         f"{frames.device}, {valid.device} and {flow.device}")
    _check_fill_params(sweeps, max_distance, alpha1, alpha2, "fill_uncovered")
    return V, T, H, W


def _fill(frames, valid, flow, flow_bw, motion, maps, maps_inv, sweeps, max_distance, alpha1, alpha2, lengths=None):
    """Step 5 on the tensors' device: rnc.inpaint's two stages on the residuals, the motion re-added between them; lengths
    as rnc.inpaint._propagate's."""
    res, res_bw = flow_residual(flow, flow_bw, motion, maps, maps_inv)
    hole = (valid == 0).to(torch.uint8)
    _complete(res, res_bw, hole, sweeps)
    _readd_(res, res_bw, motion, maps, maps_inv)
    return _propagate(frames, hole, res, res_bw, sweeps, max_distance, alpha1, alpha2, lengths)


def fill_uncovered(frames, valid, flow, flow_bw, motion, maps, maps_inv, sweeps=512, max_distance=None, alpha1=0.01,
                   alpha2=0.5):
    """Step 5 for V videos stacked as rnc.inpaint stacks them: frames [V,T,3,H,W] and valid [V,T,H,W] (warp_frames' output,
    0..255), flow, flow_bw [V,T-1,2,H,W] (forward and backward flows in input coordinates), motion fp64 [V,T-1,3,3], maps
    and maps_inv fp64 [V,T,3,3] (smooth_path's M and Minv); any strides, the inputs are not modified.  sweeps is
    harmonic_fill's, for the residuals and the spatial fill; max_distance the longest chain in frames (None: T - 1);
    alpha1, alpha2 fb_consistency's.  Returns (frames float32 [V,T,3,H,W], source uint8 [V,T,H,W]): every pixel with
    valid != 0 keeps its bits and is SOURCE_KNOWN, every other one is filled.  CUDA tensors run on the kernels, CPU tensors
    through host_fill_uncovered; they give the same bits.  ValueError before any launch for mismatched shapes or devices,
    T < 2, a side above 4096, sweeps < 0, max_distance < 1 or a negative or non-finite alpha1 or alpha2."""
    _check_fill_uncovered(frames, valid, flow, flow_bw, motion, maps, maps_inv, sweeps, max_distance, alpha1, alpha2)
    if not frames.is_cuda:
        return host_fill_uncovered(frames, valid, flow, flow_bw, motion, maps, maps_inv, sweeps, max_distance, alpha1, alpha2)
    return _fill(frames, valid, flow, flow_bw, motion, maps, maps_inv, sweeps, max_distance, alpha1, alpha2)


def host_fill_uncovered(frames, valid, flow, flow_bw, motion, maps, maps_inv, sweeps=512, max_distance=None, alpha1=0.01,
                        alpha2=0.5):
    """fill_uncovered on CPU copies of the inputs, so through host_flow_residual, rnc.inpaint.host_harmonic_fill,
    host_add_global_motion, rnc.metrics.host_fb_consistency and rnc.inpaint.host_inpaint_propagate.  Returns CPU tensors."""
    _check_fill_uncovered(frames, valid, flow, flow_bw, motion, maps, maps_inv, sweeps, max_distance, alpha1, alpha2)
    return _fill(*(t.detach().cpu() for t in (frames, valid, flow, flow_bw, motion, maps, maps_inv)), sweeps, max_distance,
                 alpha1, alpha2)


# -------------------------------------------------------------------------------------------------------------- scores


def _energy_ratio(paths):
    """The energy of the five lowest non-zero frequencies over all non-zero ones, the paths' (a list of 1-D fp64 arrays)
    energies added; 1 when there is no non-zero energy."""
    low = total = 0.0
    for p in paths:
        e = np.abs(np.fft.rfft(p)) ** 2
        low += float(e[1:6].sum())
        total += float(e[1:].sum())
    return low / total if total > 0 else 1.0


def _stability(B):
    """(translation, rotation) stability of inter-frame motions B fp64 [K,3,3]."""
    tx, ty = np.cumsum(B[:, 0, 2]), np.cumsum(B[:, 1, 2])
    rot = np.cumsum(np.arctan2(B[:, 1, 0], B[:, 0, 0]))
    return _energy_ratio([tx, ty]), _energy_ratio([rot])


def stabilization_metrics(motion, transforms):
    """One video's scores on the host in fp64: motion [T-1,3,3] (A_t), transforms [T,3,3] (M_t).  Returns a dict: cropping
    (mean over frames of 1 / |det| of M_t's affine part), distortion (least singular-value ratio of that part),
    stability_translation, stability_rotation and stability (their minimum) of the output, whose inter-frame motion is
    B_t = M_{t+1} A_t M_t^-1, and input_stability_translation, input_stability_rotation and input_stability from A_t."""
    A = np.asarray(torch.as_tensor(motion).detach().cpu().to(torch.float64))
    M = np.asarray(torch.as_tensor(transforms).detach().cpu().to(torch.float64))
    if A.ndim != 3 or A.shape[1:] != (3, 3) or M.shape != (A.shape[0] + 1, 3, 3):
        raise ValueError(f"stabilization_metrics: expected motion [T-1,3,3] and transforms [T,3,3], got {A.shape} and "
                         f"{M.shape}")
    aff = M[:, :2, :2]
    cropping = float(np.mean(1.0 / np.abs(np.linalg.det(aff))))
    sv = np.linalg.svd(aff, compute_uv=False)
    distortion = float((sv[:, 1] / sv[:, 0]).min())
    B = M[1:] @ A @ np.linalg.inv(M[:-1])
    B = B / B[:, 2:3, 2:3]
    st, sr = _stability(B)
    it, ir = _stability(A)
    return {"cropping": cropping, "distortion": distortion, "stability_translation": st, "stability_rotation": sr,
            "stability": min(st, sr), "input_stability_translation": it, "input_stability_rotation": ir,
            "input_stability": min(it, ir)}


SCORES = ("cropping", "distortion", "stability_translation", "stability_rotation", "stability", "input_stability_translation",
          "input_stability_rotation", "input_stability")


def summarize_stabilization(videos):
    """The split's numbers from per-video records: a list of (stabilization_metrics dict, itf rows, input itf rows), a row
    being interpolation_error's (sq_sum, count) of frames (t + 1, t).  Each score is the mean over videos; itf and input_itf
    the mean over a video's pairs of rnc.inpaint.psnr (100 dB cap), then over videos; frames and videos, their numbers.  NaN
    without a video; in fp64."""
    out = {k: 0.0 for k in SCORES}
    itf = itf_in = 0.0
    frames = 0
    for scores, rows, rows_in in videos:
        for k in SCORES:
            out[k] += scores[k]
        itf += sum(psnr(s, c) for s, c in rows) / len(rows)
        itf_in += sum(psnr(s, c) for s, c in rows_in) / len(rows_in)
        frames += len(rows) + 1
    n = len(videos)
    res = {k: v / n if n else math.nan for k, v in out.items()}
    res.update(itf=itf / n if n else math.nan, input_itf=itf_in / n if n else math.nan, frames=frames, videos=n)
    return res
