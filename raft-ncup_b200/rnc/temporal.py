"""Blind video temporal consistency: remove the flicker of a video whose frames were processed one at a time, along the
backward flows, and score it by the warping error.

This is the screened Poisson formulation of Bonneel et al., "Blind Video Temporal Consistency" (SIGGRAPH Asia 2015): each
output frame keeps the gradients of its processed frame and is pulled toward the previous output, warped along the flow,
wherever the flow can be trusted.  Inputs, per video v of V: the original frames I_t, float32 [3,H,W] in 0..255; the processed
frames P_t, float32 [C,H,W] with 1 <= C <= 4 (stylised, colourised, tone-mapped or enhanced frames, per-frame depth or class
probabilities) in any range; for each pair k = 0..T-2 the backward flow G_k (frame k+1 -> frame k, float32 [2,H,W], channel
0 = x) and the mask occ_bw_k (uint8 [H,W] on frame k+1, occluded where non-zero), the flow_up_bw and occ_bw that
rnc.harness.run_sequences_bidirectional yields for pair k.  The output O starts with O_0 = P_0; step k -> k+1 covers every
pixel p = (x, y) of frame k+1:
1. Matched (rnc.segment's rule): u = G_k(p), p' = p + u with each component rounded once to float32; p is matched when both
   components of u are finite, occ_bw_k(p) == 0 and p' lies in [0, W-1] x [0, H-1].
2. Target and weight: a matched pixel has T_c = sample(O_k, c, p') and J_c = sample(I_k, c, p') (rnc.interp's clamped
   bilinear sample, csrc/bilinear.cuh), e_c = (I_{k+1,c}(p) - J_c) / 255, d2 = ((-0 + e_0^2) + e_1^2) + e_2^2 and
   w = lam / (1 + alpha d2), each operation rounded once in float32 in that order.  An unmatched pixel has w = 0.  The
   rational weight stands in for Lai et al.'s exp(-alpha d2): it needs no transcendental function, so the host restatement
   gives the kernel's bits.
3. Screened Poisson in correction form: D = O_{k+1} - P_{k+1} per channel solves (n + w_p) D_p - sum_q D_q = w_p (T_p - P_p),
   n the pixel's in-frame 4-neighbours.  From D = 0, `sweeps` red-black SOR sweeps run over every pixel, red ((x + y) even)
   before black: r = w (T - P) (0 where w is 0), den = n + w, s = the neighbours of D added up, left, right, down (starting
   from -0.0, so the first enters exactly), and D <- D + omega ((s + r) / den - D), each operation rounded once in float32
   with no FMA.  A pixel with den = 0 (an unmatched pixel of a 1x1 frame) keeps D = 0.  Finally O_{k+1} = P_{k+1} + D.  With
   w = 0 everywhere D stays 0, so lam = 0 and a frame without a matched pixel (a scene cut) return P's values.
4. omega per image: a pixel is weak when w < lam / 4 (unmatched pixels are weak when lam > 0).  D2 is the largest exact
   squared distance from a weak pixel to its nearest non-weak pixel (csrc/dist_transform.cuh, rnc.metrics.nearest_site), an
   integer maximum; L is the least integer with L^2 >= 4 D2; sigma = float32(sqrt(lam / 2)), computed on the host.  Then
   s = min(pi_f32 / (L + 1), sigma), or s = sigma when D2 = 0 (no weak pixel, or no other kind), and omega = 2 / (1 + s) in
   float32.  sigma is the rate at which the screening alone damps the error (a screened Laplacian's smallest eigenvalue over
   its largest is about lam / 8, and the optimal factor 2 / (1 + sqrt(1 - rho^2)) with rho = 1 - lam / 8 is about
   2 / (1 + sqrt(lam / 4))); inside a weak region of half-width D the screening is absent, and the region behaves as an
   unscreened square of side 2 D, hence pi / (L + 1).  L comes from the distance transform and not from a bounding box, so
   thin weak strips across the frame do not slow the solve down.
At the default 512 sweeps the solve converges for weak regions up to about 150 px across (tests/test_temporal.py reproduces
the measured table against scipy's direct solve); a wider weak region, or one that touches the border (whose half-width is
its full width), needs more sweeps.  A non-finite P or frame value at a matched pixel spreads through the solve.

Every floating-point operation of the step is rounded once in float32, so the kernels (csrc/temporal.cu) and the host
restatements (host_temporal_step, host_temporally_consistent) give the same bits.

Warping error (Lai et al., "Learning Blind Video Temporal Consistency", ECCV 2018), for any video V_t of C channels with the
flows and masks above: for frame k+1 and its matched pixels M, the fp64 sum over p in M and the channels of
((V_{k+1,c}(p) - sample(V_k, c, p')) / 255)^2 (the sample in float32, the difference, division, square and sums in fp64),
and the count |M|.  A frame's error is sum / count, over the frames with count > 0; a video's error the mean over its
frames; a split's the mean over its videos (summarize_temporal).  It is Lai et al.'s definition with images in [0, 1], with
the occlusion from rnc.metrics.fb_consistency instead of their flow network's; no value is comparable to their tables.
"""
import math

import numpy as np
import torch

from . import native
from .metrics import nearest_site
from .restate import PI_F32, check_sides, f32, follow, sample

DEFAULT_LAM = 0.1
DEFAULT_ALPHA = 50.0
DEFAULT_SWEEPS = 512


def sigma(lam):
    """float32(sqrt(float32(lam) / 2)), the screening's rate in omega's rule."""
    lam32 = float(np.float32(lam))
    return float(np.float32(math.sqrt(lam32 / 2)))


def omega(d2, lam):
    """The SOR factor of an image whose weak pixels lie at most sqrt(d2) from a non-weak one (d2 = 0: no weak pixel, or no
    other kind): 2 / (1 + s), s = min(pi_f32 / (L + 1), sigma(lam)) with L the least integer such that L^2 >= 4 d2, or
    sigma(lam) when d2 = 0; each float32 operation rounded once."""
    s = np.float32(sigma(lam))
    if d2 > 0:
        L = math.isqrt(4 * d2)
        L += L * L < 4 * d2
        s = min(np.float32(PI_F32) / np.float32(L + 1), s)
    return float(np.float32(2.0) / (np.float32(1.0) + np.float32(s)))


def _check_params(lam, alpha, sweeps, what):
    for name, v in (("lam", lam), ("alpha", alpha)):
        if not isinstance(v, (int, float)) or not 0 <= v <= float(np.finfo(np.float32).max):
            raise ValueError(f"{what}: expected a finite {name} >= 0, got {v!r}")
    if not isinstance(sweeps, int) or isinstance(sweeps, bool) or sweeps < 0:
        raise ValueError(f"{what}: expected sweeps >= 0, got {sweeps!r}")


def _check_step(out_prev, processed, frame_prev, frame, flow_bw, occ_bw, lam, alpha, sweeps):
    """(V, C, H, W) of temporal_step's arguments; ValueError for mismatched shapes, mixed devices, a channel count outside
    1..4, a side above 4096, more than 65535 videos or a bad parameter."""
    if processed.dim() != 4 or processed.shape[0] == 0:
        raise ValueError(f"temporal_step: expected processed [V,C,H,W], got {tuple(processed.shape)}")
    V, C, H, W = processed.shape
    for name, t, want in (("out_prev", out_prev, (V, C, H, W)), ("frame_prev", frame_prev, (V, 3, H, W)),
                          ("frame", frame, (V, 3, H, W)), ("flow_bw", flow_bw, (V, 2, H, W)), ("occ_bw", occ_bw, (V, H, W))):
        if tuple(t.shape) != want:
            raise ValueError(f"temporal_step: expected {name} {list(want)}, got {tuple(t.shape)}")
    devs = {t.device for t in (out_prev, processed, frame_prev, frame, flow_bw, occ_bw)}
    if len(devs) != 1:
        raise ValueError(f"temporal_step: the frames, flow and mask must be on one device, got {sorted(map(str, devs))}")
    if not 1 <= C <= native.HARMONIC_MAX_CHANNELS:
        raise ValueError(f"temporal_step: expected 1 to {native.HARMONIC_MAX_CHANNELS} processed channels, got {C}")
    if V > 65535:
        raise ValueError(f"temporal_step: at most 65535 videos per step, got {V}")
    check_sides(H, W, "temporal_step")
    _check_params(lam, alpha, sweeps, "temporal_step")
    return V, C, H, W


def temporal_step(out_prev, processed, frame_prev, frame, flow_bw, occ_bw, lam=DEFAULT_LAM, alpha=DEFAULT_ALPHA,
                  sweeps=DEFAULT_SWEEPS, out=None, workspace=None):
    """One step k -> k+1 of the rule for V videos: out_prev [V,C,H,W] (O_k), processed [V,C,H,W] (P_{k+1}), frame_prev and
    frame [V,3,H,W] (I_k, I_{k+1}, 0..255), flow_bw [V,2,H,W] (G_k), occ_bw [V,H,W] (occluded where non-zero); any strides,
    float32 or converted to it.  Returns float32 [V,C,H,W], O_{k+1}: `out` when given (it may be processed or out_prev
    itself, or a view of a stack), else a new tensor.  CUDA tensors go through rnc_temporal_step (5 + 2 sweeps launches on the
    current stream, no host synchronisation; the inputs are read through their strides, not copied; `workspace`, a uint8
    CUDA tensor of at least rnc_temporal_step_workspace_bytes, is used when given), CPU tensors through host_temporal_step;
    they give the same bits.  ValueError before any launch for mismatched shapes, mixed devices, a channel count outside
    1..4, a side above 4096, more than 65535 videos, lam or alpha negative or not finite, or sweeps < 0."""
    V, C, H, W = _check_step(out_prev, processed, frame_prev, frame, flow_bw, occ_bw, lam, alpha, sweeps)
    if out is not None and tuple(out.shape) != (V, C, H, W):
        raise ValueError(f"temporal_step: expected out {[V, C, H, W]}, got {tuple(out.shape)}")
    if not processed.is_cuda:
        res = _host_steps(out_prev, processed, frame_prev, frame, flow_bw, occ_bw, lam, alpha, sweeps)
        return res if out is None else out.copy_(res)
    dev = processed.device
    if out is None:
        out = torch.empty(V, C, H, W, dtype=torch.float32, device=dev)
    if out.dtype != torch.float32:
        raise ValueError(f"temporal_step: expected a float32 out, got {out.dtype}")
    o, p, i0, i1, g = (t.detach().float() for t in (out_prev, processed, frame_prev, frame, flow_bw))
    m = occ_bw.detach().to(torch.uint8)
    with torch.cuda.device(dev):
        nbytes = native.rnc.temporal_step_workspace_bytes(V, C, H, W)
        if workspace is None or workspace.numel() < nbytes:
            workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        native.rnc.temporal_step(o, *o.stride(), p, *p.stride(), i0, *i0.stride(), i1, *i1.stride(), g, *g.stride(), m,
                                 *m.stride(), V, C, H, W, float(lam), float(alpha), sigma(lam), sweeps, out, *out.stride(),
                                 workspace, workspace.numel())
    return out


def _host_step(O, P, I0, I1, G, occ, lam, alpha, sweeps):
    """One video's step on the host: O, P fp64 [C,H,W], I0, I1 fp64 [3,H,W], G fp64 [2,H,W] (float32 values), occ [H,W].
    Returns float32 [C,H,W]."""
    C, H, W = P.shape
    lam32, alpha32 = float(np.float32(lam)), float(np.float32(alpha))
    matched, cx, cy = follow(G, occ)
    e = f32(f32(I1 - sample(I0, cx, cy)) / 255.0)
    d2 = torch.full((H, W), -0.0, dtype=torch.float64)
    for c in range(3):
        d2 = f32(d2 + f32(e[c] * e[c]))
    w = torch.where(matched, f32(lam32 / f32(1.0 + f32(alpha32 * d2))), 0.0)
    r = torch.where(w > 0, f32(w * f32(sample(O, cx, cy) - P)), 0.0)
    n = torch.zeros(H, W, dtype=torch.float64)
    n[1:] += 1
    n[:, 1:] += 1
    n[:, :-1] += 1
    n[:-1] += 1
    den = f32(n + w)
    weak = (w < f32(torch.tensor(lam32 * 0.25, dtype=torch.float64))).numpy()
    site = nearest_site(~weak[None])[0]
    if site.min() < 0 or not weak.any():
        d2max = 0
    else:
        yy, xx = np.mgrid[:H, :W]
        d2max = int(((yy - site // W) ** 2 + (xx - site % W) ** 2).max())
    om = torch.tensor(omega(d2max, lam32), dtype=torch.float32)
    # the sweeps in float32: torch's CPU + - * / on float32 are IEEE-rounded, as the kernel's __*_rn.  Missing neighbours
    # are padded with -0.0, which adds exactly (x + -0.0 == x for every x), so the sum is the kernel's over the in-frame ones
    Dp = torch.full((C, H + 2, W + 2), -0.0, dtype=torch.float32)
    D = Dp[:, 1:-1, 1:-1]
    D.zero_()
    r32, den32 = r.float(), den.float()
    live = den32 != 0
    parity = (torch.arange(H).view(H, 1) + torch.arange(W).view(1, W)) % 2
    colours = (live & (parity == 0), live & (parity == 1))
    for _ in range(sweeps):
        for m in colours:
            s = Dp[:, :-2, 1:-1] + Dp[:, 1:-1, :-2]
            s += Dp[:, 1:-1, 2:]
            s += Dp[:, 2:, 1:-1]
            new = D + om * ((s + r32) / den32 - D)
            D.copy_(torch.where(m, new, D))
    return P.float() + D


def _host_steps(out_prev, processed, frame_prev, frame, flow_bw, occ_bw, lam, alpha, sweeps):
    V, C, H, W = processed.shape
    out = torch.empty(V, C, H, W, dtype=torch.float32)
    for v in range(V):
        O, P, I0, I1, G = (t[v].detach().cpu().float().double() for t in (out_prev, processed, frame_prev, frame, flow_bw))
        out[v] = _host_step(O, P, I0, I1, G, occ_bw[v].detach().cpu(), lam, alpha, sweeps)
    return out


def host_temporal_step(out_prev, processed, frame_prev, frame, flow_bw, occ_bw, lam=DEFAULT_LAM, alpha=DEFAULT_ALPHA,
                       sweeps=DEFAULT_SWEEPS):
    """temporal_step's rule in torch, one video at a time and all its pixels at once (a colour's pixels only read the other
    colour, so updating them together is the sequential sweep): the target and weight in fp64 on float32 operands, each
    operation rounded once to float32; the sweeps in float32; omega's distance by rnc.metrics.nearest_site.  Serves CPU
    tensors and is the kernel's test reference.  Returns float32 [V,C,H,W] on the CPU."""
    _check_step(out_prev, processed, frame_prev, frame, flow_bw, occ_bw, lam, alpha, sweeps)
    return _host_steps(out_prev, processed, frame_prev, frame, flow_bw, occ_bw, lam, alpha, sweeps)


# ------------------------------------------------------------------------------------------------------- whole videos


def _check_video(processed, frames, flow_bw, occ_bw, what):
    """(V, T, C, H, W) of a stacked video; ValueError for mismatched shapes, T < 2, mixed devices, a channel count outside
    1..4 or a side above 4096."""
    if processed.dim() != 5 or processed.shape[0] == 0:
        raise ValueError(f"{what}: expected processed [V,T,C,H,W], got {tuple(processed.shape)}")
    V, T, C, H, W = processed.shape
    if T < 2:
        raise ValueError(f"{what}: a video needs T >= 2 frames, got {T}")
    for name, t, want in (("frames", frames, (V, T, 3, H, W)), ("flow_bw", flow_bw, (V, T - 1, 2, H, W)),
                          ("occ_bw", occ_bw, (V, T - 1, H, W))):
        if tuple(t.shape) != want:
            raise ValueError(f"{what}: expected {name} {list(want)}, got {tuple(t.shape)}")
    devs = {t.device for t in (processed, frames, flow_bw, occ_bw)}
    if len(devs) != 1:
        raise ValueError(f"{what}: the frames, flows and masks must be on one device, got {sorted(map(str, devs))}")
    if not 1 <= C <= native.HARMONIC_MAX_CHANNELS:
        raise ValueError(f"{what}: expected 1 to {native.HARMONIC_MAX_CHANNELS} processed channels, got {C}")
    if V > 65535:
        raise ValueError(f"{what}: at most 65535 videos, got {V}")
    check_sides(H, W, what)
    return V, T, C, H, W


def temporally_consistent(processed, frames, flow_bw, occ_bw, lam=DEFAULT_LAM, alpha=DEFAULT_ALPHA, sweeps=DEFAULT_SWEEPS):
    """The rule over whole videos: processed [V,T,C,H,W] (P_t), frames [V,T,3,H,W] (I_t, 0..255), flow_bw [V,T-1,2,H,W]
    (G_k), occ_bw [V,T-1,H,W]; any strides (the stacked pair results are read through views, not copied).  Returns float32
    [V,T,C,H,W], O, frame 0 being P_0.  T-1 steps of temporal_step, each written straight into its frame of the result; CUDA
    tensors take T-1 calls of rnc_temporal_step on the current stream, CPU tensors run host_temporal_step's rule; they give
    the same bits.  ValueError before any launch for mismatched shapes, mixed devices, T < 2, a channel count outside 1..4,
    a side above 4096, more than 65535 videos or a bad lam, alpha or sweeps."""
    V, T, C, H, W = _check_video(processed, frames, flow_bw, occ_bw, "temporally_consistent")
    _check_params(lam, alpha, sweeps, "temporally_consistent")
    out = torch.empty(V, T, C, H, W, dtype=torch.float32, device=processed.device)
    out[:, 0] = processed[:, 0]
    ws = None
    if out.is_cuda:
        ws = torch.empty(native.rnc.temporal_step_workspace_bytes(V, C, H, W), dtype=torch.uint8, device=out.device)
    for k in range(T - 1):
        temporal_step(out[:, k], processed[:, k + 1], frames[:, k], frames[:, k + 1], flow_bw[:, k], occ_bw[:, k], lam, alpha,
                      sweeps, out=out[:, k + 1], workspace=ws)
    return out


def host_temporally_consistent(processed, frames, flow_bw, occ_bw, lam=DEFAULT_LAM, alpha=DEFAULT_ALPHA,
                               sweeps=DEFAULT_SWEEPS):
    """temporally_consistent through host_temporal_step's restatement.  Returns float32 [V,T,C,H,W] on the CPU."""
    V, T, C, H, W = _check_video(processed, frames, flow_bw, occ_bw, "temporally_consistent")
    _check_params(lam, alpha, sweeps, "temporally_consistent")
    out = torch.empty(V, T, C, H, W, dtype=torch.float32)
    out[:, 0] = processed[:, 0].cpu()
    for k in range(T - 1):
        out[:, k + 1] = _host_steps(out[:, k], processed[:, k + 1], frames[:, k], frames[:, k + 1], flow_bw[:, k], occ_bw[:, k],
                                    lam, alpha, sweeps)
    return out


# ------------------------------------------------------------------------------------------------------- warping error


def _check_warp(video, flow_bw, occ_bw):
    if video.dim() != 5 or video.shape[0] == 0 or video.shape[2] == 0:
        raise ValueError(f"warping_error: expected video [V,T,C,H,W], got {tuple(video.shape)}")
    V, T, C, H, W = video.shape
    if T < 2:
        raise ValueError(f"warping_error: a video needs T >= 2 frames, got {T}")
    if tuple(flow_bw.shape) != (V, T - 1, 2, H, W):
        raise ValueError(f"warping_error: expected flow_bw {[V, T - 1, 2, H, W]}, got {tuple(flow_bw.shape)}")
    if tuple(occ_bw.shape) != (V, T - 1, H, W):
        raise ValueError(f"warping_error: expected occ_bw {[V, T - 1, H, W]}, got {tuple(occ_bw.shape)}")
    devs = {t.device for t in (video, flow_bw, occ_bw)}
    if len(devs) != 1:
        raise ValueError(f"warping_error: the video, flows and masks must be on one device, got {sorted(map(str, devs))}")
    if V * (T - 1) > 65535 or H * W >= 1 << 30:
        raise ValueError(f"warping_error: {V} videos of {T} frames of {H}x{W} exceed the kernel's limits (V (T - 1) <= 65535, "
                         f"H*W < 2^30)")
    return V, T, C, H, W


def warping_error(video, flow_bw, occ_bw):
    """The warping error's per-frame partials of V videos: video [V,T,C,H,W] (any C, 0..255 scale), flow_bw [V,T-1,2,H,W],
    occ_bw [V,T-1,H,W]; any strides.  Returns (sum fp64 [V,T-1], count int64 [V,T-1]) on the tensors' device, entry [v, k]
    for frame k+1: the sum over its matched pixels and channels of ((V_{k+1}(p) - V_k(p')) / 255)^2 and their number.  CUDA
    tensors go through rnc_warping_error_partials (two launches on the current stream; a frame's sum does not depend on V, its
    position or the GPU), CPU tensors through host_warping_error; the counts are equal and the sums agree to their last bits.
    ValueError for mismatched shapes, mixed devices, T < 2 or more than 65535 pairs."""
    V, T, C, H, W = _check_warp(video, flow_bw, occ_bw)
    if not video.is_cuda:
        return host_warping_error(video, flow_bw, occ_bw)
    dev = video.device
    v, g = video.detach().float(), flow_bw.detach().float()
    m = occ_bw.detach().to(torch.uint8)
    s = torch.empty(V, T - 1, dtype=torch.float64, device=dev)
    count = torch.empty(V, T - 1, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        ws = torch.empty(native.rnc.warping_error_partials_workspace_bytes(V, T, C, H, W), dtype=torch.uint8, device=dev)
        native.rnc.warping_error_partials(v, *v.stride(), g, *g.stride(), m, *m.stride(), V, T, C, H, W, s, count, ws,
                                          ws.numel())
    return s, count


def host_warping_error(video, flow_bw, occ_bw):
    """warping_error on the host: the matching and the sample as temporal_step's, the rest in numpy fp64, per pixel the
    channels added in order and the pixels summed by numpy.  Returns (sum fp64 [V,T-1], count int64 [V,T-1]) on the CPU."""
    V, T, C, H, W = _check_warp(video, flow_bw, occ_bw)
    s = torch.zeros(V, T - 1, dtype=torch.float64)
    count = torch.zeros(V, T - 1, dtype=torch.int64)
    for v in range(V):
        vid = video[v].detach().cpu().float().double()
        for k in range(T - 1):
            G = flow_bw[v, k].detach().cpu().float().double()
            occ = occ_bw[v, k].detach().cpu()
            matched, cx, cy = follow(G, occ)
            e = ((vid[k + 1] - sample(vid[k], cx, cy)) / 255.0).numpy()
            t = np.zeros((H, W))
            for c in range(C):
                t = t + e[c] * e[c]
            mk = matched.numpy()
            s[v, k] = float(t[mk].sum())
            count[v, k] = int(mk.sum())
    return s, count


def summarize_temporal(videos):
    """The split's numbers from per-video records: a list of one list per video of (wp_sum, wo_sum, count, sq_sum, sq_count,
    ssim_sum, ssim_count) per frame t = 1..T-1: the warping-error partials of frame t of the processed video and of the output
    (one matched set, so one count), then rnc.interp.interpolation_error's and rnc.inpaint.ssim's partials of O_t against
    P_t (NaN where not computed).  warping_error_processed and warping_error: each the mean of sum / count over a video's
    frames with count > 0, then over the videos with such a frame; psnr (rnc.inpaint.psnr, 100 dB cap) and ssim: each the
    mean over a video's frames, then over the videos; frames and videos, their numbers.  NaN without a frame; in fp64."""
    from .inpaint import psnr
    wp, wo, p, s, frames, n, nw = 0.0, 0.0, 0.0, 0.0, 0, 0, 0
    for rows in videos:
        if not rows:
            continue
        warped = [(a / c, b / c) for a, b, c, *_ in rows if c > 0]
        if warped:
            wp += sum(a for a, _ in warped) / len(warped)
            wo += sum(b for _, b in warped) / len(warped)
            nw += 1
        p += sum(psnr(sq, c) for _, _, _, sq, c, _, _ in rows) / len(rows)
        s += sum(ss / sc for *_, ss, sc in rows) / len(rows)
        frames += len(rows)
        n += 1
    return {"warping_error_processed": wp / nw if nw else math.nan, "warping_error": wo / nw if nw else math.nan,
            "psnr": p / n if n else math.nan, "ssim": s / n if n else math.nan, "frames": frames, "videos": n}
