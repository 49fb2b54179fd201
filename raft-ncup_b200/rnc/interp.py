"""Frame interpolation from both flows and the occlusion masks, and the interpolation error of a predicted frame.

`interpolate(frame0, frame1, flow, flow_bw, occ, occ_bw, times)` synthesises the frames between frame0 and frame1 at times t in
(0, 1), from the forward flow F (0 -> 1), the backward flow G (1 -> 0) and the occlusion masks rnc.metrics.fb_consistency gives
for them (rnc.harness.bidirectional_flow returns all four).  This is the interpolation algorithm of the Middlebury benchmark
(Baker, Scharstein, Lewis, Roth, Black and Szeliski, "A Database and Evaluation Methodology for Optical Flow", IJCV 2011,
§3.3) with two changes: the occlusion masks are fb_consistency's, and holes take the motion of the nearest filled pixel instead
of Middlebury's outside-in fill.  Per image and per t:

1. Splat the flow to time t.  A frame-0 pixel x is a source when occ0(x) == 0, F(x) is finite and q = rint(x + t F(x)) (round
   half to even) lies in the frame; it proposes the motion u = F(x) at q, keyed by its photometric error
   e = sum_c |I1^_c(x + F(x)) - I0_c(x)| (channels added in order 0, 1, 2).  A frame-1 pixel y likewise, with occ1, the target
   rint(y + (1 - t) G(y)), u = -G(y) and e = sum_c |I0^_c(y + G(y)) - I1_c(y)|.  I^ is a bilinear sample with the coordinates
   clamped to [0, W-1] x [0, H-1].  Each target keeps the proposal of smallest (e, source index), frame 0's sources having
   indices 0..HW-1 and frame 1's HW..2HW-1.
2. Fill the holes.  A pixel without a proposal takes u from the nearest pixel with one, in exact squared Euclidean distance,
   ties to the smallest column and then the smallest row (a feature transform).  In an image without a proposal, u = 0.
3. Composite.  With x0 = x - t u and x1 = x + (1 - t) u, v0 is true when x0 lies in the frame and occ0(rint(x0)) == 0, v1
   likewise with occ1; the output is (1 - t) I0^(x0) + t I1^(x1) when v0 == v1, I0^(x0) when only v0, I1^(x1) when only v1.

Every floating-point operation is rounded once in float32 (bilinear weights bx*by, ax*by, bx*ay, ax*ay and taps added in that
order), so `host_interpolate` (CPU tensors, and the kernels' test reference) and rnc_interpolate (csrc/interp.cu, CUDA tensors)
give the same bits.  The splat keeps its minimum with an integer atomicMin on (float bits of e) << 32 | index, so the winner does
not depend on the order in which threads run, and no step has a floating-point atomic: each output depends only on its own image
and time, whatever the batch.

A known limit, shared with Middlebury's algorithm: the masks belong to the frames, not to time t, so where the fill gives a hole
at a motion boundary the motion of the wrong side, the visible sample it picks can be the other layer's.

`interpolation_error(pred, gt)` gives per frame the fp64 sum over pixels of sum_c (pred - gt)^2 and the pixel count, through
rnc_interp_error on CUDA (a fixed summation order, so an image's sum does not depend on the batch or the GPU) and
`host_interpolation_error` on the CPU.  `summarize_interpolation` turns the partials of a split into Middlebury's interpolation
error (IE) and the PSNR.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import native
from .metrics import InterpPartials, nearest_site
from .restate import f32, inside, sample

NO_PROPOSAL = np.uint64(0xFFFFFFFFFFFFFFFF)


def _times(times):
    """times as float32 values; ValueError unless 1 <= len <= INTERP_MAX_TIMES and each is in (0, 1) after rounding."""
    try:
        ts = [float(torch.tensor(float(t), dtype=torch.float32)) for t in times]
    except TypeError as e:
        raise ValueError(f"interpolate: times must be a sequence of numbers, got {times!r}") from e
    if not 1 <= len(ts) <= native.INTERP_MAX_TIMES:
        raise ValueError(f"interpolate: expected 1 to {native.INTERP_MAX_TIMES} times, got {len(ts)}")
    bad = [t for t in ts if not 0.0 < t < 1.0]
    if bad:
        raise ValueError(f"interpolate: every time must lie in (0, 1) (as float32), got {bad}")
    return ts


def _check(frame0, frame1, flow, flow_bw, occ, occ_bw):
    if frame0.dim() != 4 or frame0.shape[1] != 3 or frame1.shape != frame0.shape:
        raise ValueError(f"interpolate: expected two [B,3,H,W] frames of one shape, got {tuple(frame0.shape)} and "
                         f"{tuple(frame1.shape)}")
    B, _, H, W = frame0.shape
    if B == 0 or H == 0 or W == 0:
        raise ValueError(f"interpolate: empty frames {tuple(frame0.shape)}")
    for name, t, want in (("flow", flow, (B, 2, H, W)), ("flow_bw", flow_bw, (B, 2, H, W)), ("occ", occ, (B, H, W)),
                          ("occ_bw", occ_bw, (B, H, W))):
        if tuple(t.shape) != want:
            raise ValueError(f"interpolate: expected {name} {list(want)}, got {tuple(t.shape)}")
    devs = {t.device for t in (frame0, frame1, flow, flow_bw, occ, occ_bw)}
    if len(devs) != 1:
        raise ValueError(f"interpolate: the frames, flows and masks must be on one device, got {sorted(map(str, devs))}")


def interpolate(frame0, frame1, flow, flow_bw, occ, occ_bw, times=(0.5,)):
    """The frames between frame0 and frame1 at each of `times` (the algorithm above).  frame0, frame1: [B,3,H,W] in 0..255;
    flow (frame 0 -> 1), flow_bw (1 -> 0): [B,2,H,W]; occ, occ_bw: [B,H,W], fb_consistency's masks of flow and flow_bw,
    visible where 0 (any strides; float32 and uint8, or converted to them); times: 1 to 64 numbers in (0, 1).  Returns float32
    [B,T,3,H,W], not rounded.  CUDA tensors go through rnc_interpolate (enqueued on the current stream, no host
    synchronisation; H, W <= 4096 and B*T <= 65535), CPU tensors through host_interpolate; they give the same bits.
    ValueError before any launch for mismatched shapes, mixed devices or a time outside (0, 1)."""
    _check(frame0, frame1, flow, flow_bw, occ, occ_bw)
    ts = _times(times)
    if not frame0.is_cuda:
        return host_interpolate(frame0, frame1, flow, flow_bw, occ, occ_bw, ts)
    f0, f1, fw, bw = (t.detach().float() for t in (frame0, frame1, flow, flow_bw))
    o0, o1 = (o.detach().to(torch.uint8).contiguous() for o in (occ, occ_bw))
    B, _, H, W = f0.shape
    T = len(ts)
    dev = f0.device
    out = torch.empty(B, T, 3, H, W, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        nbytes = native.rnc.interpolate_workspace_bytes(B, T, H, W)
        if nbytes == 0:
            raise ValueError(f"interpolate: {B} pairs of {H}x{W} at {T} times exceed the kernels' limits (H, W <= 4096, "
                             f"B*T <= 65535)")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        native.rnc.interpolate(f0, *f0.stride(), f1, *f1.stride(), fw, *fw.stride(), bw, *bw.stride(), o0, o1,
                               (C.c_float * T)(*ts), T, B, H, W, out, ws, ws.numel())
    return out


def host_interpolate(frame0, frame1, flow, flow_bw, occ, occ_bw, times=(0.5,)):
    """interpolate's definition in torch and numpy, one image at a time: each floating-point operation evaluated in fp64 on
    float32 operands and rounded once to float32 (the IEEE float32 result, as rnc.metrics.host_fb_consistency does), in the
    kernels' order; the splat's minimum with numpy.minimum.at on the uint64 keys; the fill by nearest_site.  Serves CPU
    tensors and is the kernels' test reference."""
    _check(frame0, frame1, flow, flow_bw, occ, occ_bw)
    ts = _times(times)
    frames = [f.detach().cpu().float().double() for f in (frame0, frame1)]
    flows = [f.detach().cpu().float().double() for f in (flow, flow_bw)]
    occs = [o.detach().cpu().to(torch.uint8) for o in (occ, occ_bw)]
    B, _, H, W = frames[0].shape
    T, hw = len(ts), H * W
    xs = torch.arange(W, dtype=torch.float64).view(1, W).expand(H, W)
    ys = torch.arange(H, dtype=torch.float64).view(H, 1).expand(H, W)
    index = np.arange(hw, dtype=np.uint64)
    out = torch.empty(B, T, 3, H, W, dtype=torch.float32)
    for b in range(B):
        keys = np.full((T, hw), NO_PROPOSAL, dtype=np.uint64)
        for s in (0, 1):
            f = flows[s][b]
            ok = (occs[s][b] == 0) & torch.isfinite(f[0]) & torch.isfinite(f[1])
            f = torch.where(ok, f, 0.0)
            smp = sample(frames[1 - s][b], f32(xs + f[0]), f32(ys + f[1]))
            d = f32(smp - frames[s][b]).abs()
            e = f32(f32(d[0] + d[1]) + d[2])
            bits = e.float().numpy().reshape(-1).view(np.uint32).astype(np.uint64)
            key = (bits << np.uint64(32)) | (index + np.uint64(s * hw))
            for k, t in enumerate(ts):
                tt = t if s == 0 else float(f32(torch.tensor(1.0 - t, dtype=torch.float64)))
                qx = torch.round(f32(xs + f32(tt * f[0])))
                qy = torch.round(f32(ys + f32(tt * f[1])))
                go = (ok & inside(qx, qy, H, W)).reshape(-1).numpy()
                target = (qy * W + qx).reshape(-1).numpy()[go].astype(np.int64)
                np.minimum.at(keys[k], target, key[go])
        site = nearest_site((keys != NO_PROPOSAL).reshape(T, H, W)).reshape(T, hw)
        for k, t in enumerate(ts):
            has = site[k] >= 0
            src = np.where(has, keys[k][np.maximum(site[k], 0)] & np.uint64(0xFFFFFFFF), 0).astype(np.int64)
            back = torch.from_numpy(src >= hw)
            q = torch.from_numpy(np.where(src >= hw, src - hw, src))
            u = [torch.where(torch.from_numpy(has), torch.where(back, -flows[1][b, c].reshape(-1)[q],
                                                                flows[0][b, c].reshape(-1)[q]), 0.0).view(H, W)
                 for c in (0, 1)]
            omt = float(f32(torch.tensor(1.0 - t, dtype=torch.float64)))
            x0, y0 = f32(xs - f32(t * u[0])), f32(ys - f32(t * u[1]))
            x1, y1 = f32(xs + f32(omt * u[0])), f32(ys + f32(omt * u[1]))
            vis = []
            for o, px, py in ((occs[0][b], x0, y0), (occs[1][b], x1, y1)):
                ix = torch.round(px).clamp(0, W - 1).long()
                iy = torch.round(py).clamp(0, H - 1).long()
                vis.append(inside(px, py, H, W) & (o[iy, ix] == 0))
            s0, s1 = sample(frames[0][b], x0, y0), sample(frames[1][b], x1, y1)
            blend = f32(f32(omt * s0) + f32(t * s1))
            out[b, k] = torch.where(vis[0] == vis[1], blend, torch.where(vis[0], s0, s1)).float()
    return out


def _check_error(pred, gt):
    if pred.dim() != 4 or pred.shape[1] != 3 or gt.shape != pred.shape:
        raise ValueError(f"interpolation_error: expected pred and gt of one [N,3,H,W] shape, got {tuple(pred.shape)} and "
                         f"{tuple(gt.shape)}")
    if pred.device != gt.device:
        raise ValueError(f"interpolation_error: pred is on {pred.device}, gt on {gt.device}; they must be on one device")
    if pred.numel() == 0:
        raise ValueError(f"interpolation_error: empty frames {tuple(pred.shape)}")


def interpolation_error(pred, gt):
    """pred, gt: [N,3,H,W] (any strides; float32, or converted to it).  Returns InterpPartials of N frames on their device:
    per frame the fp64 sum over pixels of sum_c (pred - gt)^2 (each difference and square in fp64) and the pixel count H*W.
    CUDA tensors go through rnc_interp_error (enqueued on the current stream), CPU tensors through host_interpolation_error;
    they agree to the last few bits (the summation orders differ).  On CUDA a frame's sum does not depend on N, on its position
    in the batch or on the GPU."""
    _check_error(pred, gt)
    if not pred.is_cuda:
        return host_interpolation_error(pred, gt)
    p, g = pred.detach().float(), gt.detach().float()
    N, _, H, W = p.shape
    dev = p.device
    sq = torch.empty(N, dtype=torch.float64, device=dev)
    count = torch.empty(N, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        nbytes = native.rnc.interp_error_workspace_bytes(N, H, W)
        if nbytes == 0:
            raise ValueError(f"interpolation_error: {N} frames of {H}x{W} exceed the kernel's limits (N <= 65535, "
                             f"H*W < 2^30)")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        native.rnc.interp_error(p, *p.stride(), g, *g.stride(), N, H, W, sq, count, ws, ws.numel())
    return InterpPartials(sq, count)


def host_interpolation_error(pred, gt):
    """interpolation_error in numpy fp64: per pixel ((p0 - g0)^2 + (p1 - g1)^2) + (p2 - g2)^2, summed over the frame."""
    _check_error(pred, gt)
    d = pred.detach().cpu().float().double().numpy() - gt.detach().cpu().float().double().numpy()
    d2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]
    N, _, H, W = pred.shape
    return InterpPartials(torch.from_numpy(d2.reshape(N, -1).sum(1)), torch.full((N,), H * W, dtype=torch.int64))


def summarize_interpolation(partials):
    """The split's numbers from per-frame InterpPartials, combined in frame order in fp64: ie, Middlebury's interpolation error,
    the mean over frames of sqrt(sq_sum / count); psnr, the mean over frames of 10 log10(255^2 / MSE) with MSE = sq_sum /
    (3 count) over pixels and channels (+inf for a frame predicted exactly); frames, their number.  NaN without a frame."""
    sq = partials.sq_sum.cpu().tolist()
    count = partials.count.cpu().tolist()
    ie = psnr = 0.0
    for s, c in zip(sq, count):
        ie += math.sqrt(s / c)
        mse = s / (3 * c)
        psnr += 10 * math.log10(255.0 ** 2 / mse) if mse > 0 else math.inf
    n = len(sq)
    return {"ie": ie / n if n else math.nan, "psnr": psnr / n if n else math.nan, "frames": n}
