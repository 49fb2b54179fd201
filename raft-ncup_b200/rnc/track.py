"""Point tracking through video by chaining the bidirectional flows, and the TAP-Vid metrics of the tracks.

Inputs, per video v of V: T >= 2 frames of one size H x W; the forward flows F_k (frame k -> k+1) and backward flows G_k (frame
k+1 -> k) for k = 0..T-2, each float32 [2,H,W] with channel 0 = x; the occlusion masks occ_k (uint8 [H,W], on frame k, of F_k)
and occ_bw_k (on frame k+1, of G_k), visible where 0.  These are the flow_up, flow_up_bw, occ and occ_bw that
rnc.harness.run_sequences_bidirectional yields for pair k, stacked to [V,T-1,...].  Queries: float32 [V,N,3], each (t, x, y)
with t an integer in [0, T-1] and (x, y) pixel coordinates in [0, W-1] x [0, H-1], pixel centres at integers (the flows'
convention).  The order is (t, x, y), as the flow's channels; TAP-Vid's files store (t, y, x).

Outputs: tracks float32 [V,N,T,2] (x, y) and visible uint8 [V,N,T].  The rule, for each query:
1. At frame t_q the position is the query and the point is visible.
2. Forward, for k = t_q .. T-2, with position p at frame k: u = F_k^(p), a bilinear sample with the coordinates clamped to
   the frame (rnc.interp's sample: taps (y0,x0), (y0,x1), (y1,x0), (y1,x1) weighted bx*by, ax*by, bx*ay, ax*ay, added in that
   order).  If both components of u are finite, p' = p + u; otherwise p' = p.  The point is lost at frame k+1, and for the
   rest of this direction, when it was lost at frame k, u is not finite, occ_k(rint(p)) != 0 (round half to even) or p' lies
   outside [0, W-1] x [0, H-1].  visible = not lost.  Positions keep advancing while lost, so a lost point's track is the
   flow's extrapolation.
3. Backward, for k = t_q-1 .. 0, the same rule with G_k and occ_bw_k, stepping from frame k+1 to frame k.
A lost point is not re-acquired.  Every floating-point operation is rounded once in float32, with no FMA, so `host_track` (CPU
tensors, and the kernel's test reference) and rnc_track (csrc/track.cu, CUDA tensors) give the same bits.  The kernel keeps a
point in registers over all T frames, in one launch for all V videos; a point's outputs depend only on its own video.

Metrics (Doersch et al., "TAP-Vid: A Benchmark for Tracking Any Point in a Video", NeurIPS 2022 Datasets and Benchmarks): per
video, over its (point, frame) pairs except each point's query frame, positions scaled to 256x256 (x * 256 / W and y * 256 / H
in float32, rounded once), within_d = dx^2 + dy^2 < d^2 in float32 for d in THRESHOLDS.  `track_metrics` gives the integer
counts the metrics are ratios of (the COUNT_* layout below), so they are exact and do not depend on the batch, the order or
the number of GPUs; `summarize_tracking` turns them into occlusion accuracy, < delta^x_avg and Average Jaccard, each per video
and then averaged over videos, as TAP-Vid does.
"""
import math

import torch

from . import native
from .interp import _sample
from .metrics import _f32

THRESHOLDS = (1, 2, 4, 8, 16)
# the columns of a video's counts (RNC_TRACK_COUNTS): pairs evaluated, occlusion agreements, gt visible, then per threshold
# within & gt visible, true positives (within & gt visible & pred visible) and false positives (pred visible & (not gt
# visible or not within))
COUNT_EVALUATED, COUNT_OCC_AGREE, COUNT_GT_VISIBLE, COUNT_WITHIN, COUNT_TP, COUNT_FP = 0, 1, 2, 3, 8, 13
assert len(THRESHOLDS) == native.TRACK_THRESHOLDS and COUNT_FP + len(THRESHOLDS) == native.TRACK_COUNTS


def grid_queries(H, W, t, stride=1):
    """Queries at every stride-th pixel of frame t, in row-major order: float32 [N,3] of (t, x, y), N = ceil(H / stride) *
    ceil(W / stride).  Dense tracking is these queries through `track` or rnc.harness.track_points."""
    if stride < 1 or H < 1 or W < 1:
        raise ValueError(f"grid_queries: expected H, W, stride >= 1, got {H}, {W}, {stride}")
    ys, xs = torch.meshgrid(torch.arange(0, H, stride, dtype=torch.float32), torch.arange(0, W, stride, dtype=torch.float32),
                            indexing="ij")
    return torch.stack([torch.full_like(xs, float(t)), xs, ys], -1).reshape(-1, 3)


def check_queries(queries, T, H, W, what="track"):
    """ValueError unless queries is [..., 3] with every t an integer in [0, T-1] and every (x, y) in [0, W-1] x [0, H-1] (as
    float32).  The test runs on the queries' device; the host waits for its two flags only."""
    if queries.dim() < 1 or queries.shape[-1] != 3:
        raise ValueError(f"{what}: expected queries [..., 3] of (t, x, y), got {tuple(queries.shape)}")
    if T < 2:
        raise ValueError(f"{what}: a video needs T >= 2 frames, got {T}")
    q = queries.detach().float().reshape(-1, 3)
    t, x, y = q.unbind(1)
    bad_t = ~((t >= 0) & (t <= T - 1) & (t == torch.floor(t)))
    bad_xy = ~((x >= 0) & (x <= W - 1) & (y >= 0) & (y <= H - 1))
    any_t, any_xy = torch.stack([bad_t.any(), bad_xy.any()]).tolist()
    if any_t:
        raise ValueError(f"{what}: every query t must be an integer in [0, {T - 1}], got {t[bad_t][:4].tolist()}")
    if any_xy:
        raise ValueError(f"{what}: every query (x, y) must lie in [0, {W - 1}] x [0, {H - 1}], got "
                         f"{q[bad_xy][:4, 1:].tolist()}")


def _check(flow, flow_bw, occ, occ_bw, queries):
    """(V, N, T, H, W) of track's arguments; ValueError for mismatched shapes, T < 2, mixed devices or a bad query."""
    if flow.dim() != 5 or flow.shape[2] != 2 or tuple(flow_bw.shape) != tuple(flow.shape):
        raise ValueError(f"track: expected flow and flow_bw of one [V,T-1,2,H,W] shape, got {tuple(flow.shape)} and "
                         f"{tuple(flow_bw.shape)}")
    V, T1, _, H, W = flow.shape
    if V == 0 or H == 0 or W == 0:
        raise ValueError(f"track: empty flows {tuple(flow.shape)}")
    for name, t in (("occ", occ), ("occ_bw", occ_bw)):
        if tuple(t.shape) != (V, T1, H, W):
            raise ValueError(f"track: expected {name} {[V, T1, H, W]}, got {tuple(t.shape)}")
    if queries.dim() != 3 or queries.shape[0] != V or queries.shape[2] != 3:
        raise ValueError(f"track: expected queries [{V},N,3], got {tuple(queries.shape)}")
    devs = {t.device for t in (flow, flow_bw, occ, occ_bw, queries)}
    if len(devs) != 1:
        raise ValueError(f"track: the flows, masks and queries must be on one device, got {sorted(map(str, devs))}")
    check_queries(queries, T1 + 1, H, W)
    return V, queries.shape[1], T1 + 1, H, W


def track(flow, flow_bw, occ, occ_bw, queries):
    """Tracks of the queries (the rule above).  flow, flow_bw: [V,T-1,2,H,W]; occ, occ_bw: [V,T-1,H,W], visible where 0 (any
    strides; float32 and uint8, or converted to them); queries: [V,N,3] of (t, x, y).  Returns (tracks float32 [V,N,T,2],
    visible uint8 [V,N,T]).  CUDA tensors go through rnc_track (one launch, enqueued on the current stream after the
    queries' check, whose two flags the host waits for), CPU tensors through host_track; they give the same bits.
    ValueError before any launch for mismatched shapes, T < 2, mixed devices, or a query whose t is not an integer in
    [0, T-1] or whose (x, y) is outside the frame."""
    V, N, T, H, W = _check(flow, flow_bw, occ, occ_bw, queries)
    if not flow.is_cuda:
        return host_track(flow, flow_bw, occ, occ_bw, queries)
    dev = flow.device
    tracks = torch.empty(V, N, T, 2, dtype=torch.float32, device=dev)
    visible = torch.empty(V, N, T, dtype=torch.uint8, device=dev)
    if N == 0:
        return tracks, visible
    fw, bw = (f.detach().float() for f in (flow, flow_bw))
    o, ob = (m.detach().to(torch.uint8) for m in (occ, occ_bw))
    q = queries.detach().float().contiguous()
    with torch.cuda.device(dev):
        native.rnc.track(fw, *fw.stride(), bw, *bw.stride(), o, *o.stride(), ob, *ob.stride(), q, V, N, T, H, W, tracks,
                         visible)
    return tracks, visible


def _chain(f, o, q, T, forward):
    """One direction of the rule for every query of a video: f [T-1,2,H,W] fp64 holding float32 values, o [T-1,H,W] uint8,
    q [N,3].  Returns the (x, y) positions [N,T,2] and visible flags [N,T] of the frames this direction writes, and the mask
    of those (point, frame) entries."""
    H, W = f.shape[-2:]
    N = q.shape[0]
    tq = q[:, 0].long()
    x, y = q[:, 1].clone(), q[:, 2].clone()
    lost = torch.zeros(N, dtype=torch.bool)
    pos = torch.zeros(N, T, 2, dtype=torch.float64)
    vis = torch.zeros(N, T, dtype=torch.bool)
    wrote = torch.zeros(N, T, dtype=torch.bool)
    for k in (range(T - 1) if forward else range(T - 2, -1, -1)):
        act = tq <= k if forward else tq >= k + 1
        if not act.any():
            continue
        u = _sample(f[k], x, y)
        fin = torch.isfinite(u[0]) & torch.isfinite(u[1])
        # a point not yet lost lies in the frame, so the clamp only keeps a lost point's index in range
        ix, iy = torch.round(x).clamp(0, W - 1).long(), torch.round(y).clamp(0, H - 1).long()
        now = lost | ~fin | (o[k][iy, ix] != 0)
        nx, ny = torch.where(fin, _f32(x + u[0]), x), torch.where(fin, _f32(y + u[1]), y)
        now = now | ~((nx >= 0) & (nx <= W - 1) & (ny >= 0) & (ny <= H - 1))
        x, y, lost = torch.where(act, nx, x), torch.where(act, ny, y), torch.where(act, now, lost)
        t = k + 1 if forward else k
        pos[act, t, 0], pos[act, t, 1] = x[act], y[act]
        vis[act, t] = ~lost[act]
        wrote[act, t] = True
    return pos, vis, wrote


def host_track(flow, flow_bw, occ, occ_bw, queries):
    """track's rule in torch, one video at a time and all its points at once: each floating-point operation evaluated in fp64
    on float32 operands and rounded once to float32 (the IEEE float32 result, as rnc.interp.host_interpolate), in the kernel's
    order.  Serves CPU tensors and is the kernel's test reference."""
    V, N, T, H, W = _check(flow, flow_bw, occ, occ_bw, queries)
    tracks = torch.empty(V, N, T, 2, dtype=torch.float32)
    visible = torch.empty(V, N, T, dtype=torch.uint8)
    for v in range(V):
        q = queries[v].detach().cpu().float().double()
        pos = torch.zeros(N, T, 2, dtype=torch.float64)
        vis = torch.zeros(N, T, dtype=torch.bool)
        tq = q[:, 0].long()
        pos[torch.arange(N), tq] = q[:, 1:]
        vis[torch.arange(N), tq] = True
        for f, o, forward in ((flow, occ, True), (flow_bw, occ_bw, False)):
            p, s, wrote = _chain(f[v].detach().cpu().float().double(), o[v].detach().cpu().to(torch.uint8), q, T, forward)
            pos = torch.where(wrote[..., None], p, pos)
            vis = torch.where(wrote, s, vis)
        tracks[v] = pos.float()
        visible[v] = vis.to(torch.uint8)
    return tracks, visible


def _check_metrics(tracks, visible, gt_tracks, gt_visible, queries, H, W):
    if tracks.dim() != 4 or tracks.shape[3] != 2 or tuple(gt_tracks.shape) != tuple(tracks.shape):
        raise ValueError(f"track_metrics: expected tracks and gt_tracks of one [V,N,T,2] shape, got {tuple(tracks.shape)} and "
                         f"{tuple(gt_tracks.shape)}")
    V, N, T, _ = tracks.shape
    for name, t in (("visible", visible), ("gt_visible", gt_visible)):
        if tuple(t.shape) != (V, N, T):
            raise ValueError(f"track_metrics: expected {name} {[V, N, T]}, got {tuple(t.shape)}")
    if tuple(queries.shape) != (V, N, 3):
        raise ValueError(f"track_metrics: expected queries {[V, N, 3]}, got {tuple(queries.shape)}")
    if V == 0 or H < 1 or W < 1:
        raise ValueError(f"track_metrics: expected V >= 1 videos of H, W >= 1, got V = {V}, {H}x{W}")
    devs = {t.device for t in (tracks, visible, gt_tracks, gt_visible, queries)}
    if len(devs) != 1:
        raise ValueError(f"track_metrics: the tracks and queries must be on one device, got {sorted(map(str, devs))}")
    check_queries(queries, T, H, W, "track_metrics")
    return V, N, T


def track_metrics(tracks, visible, gt_tracks, gt_visible, queries, H, W):
    """Per-video TAP-Vid counts of predicted tracks against the ground truth.  tracks, gt_tracks: [V,N,T,2] (x, y) in the
    pixels of H x W frames; visible, gt_visible: [V,N,T] (non-zero is visible; TAP-Vid's `occluded` is its negation);
    queries: [V,N,3] (t, x, y), whose t frames are not evaluated.  Returns int64 [V, native.TRACK_COUNTS] on the tensors'
    device (the COUNT_* columns).  CUDA tensors go through rnc_track_metrics (enqueued on the current stream after the
    queries' check, whose two flags the host waits for), CPU tensors through host_track_metrics; the counts are equal."""
    V, N, T = _check_metrics(tracks, visible, gt_tracks, gt_visible, queries, H, W)
    if not tracks.is_cuda:
        return host_track_metrics(tracks, visible, gt_tracks, gt_visible, queries, H, W)
    dev = tracks.device
    counts = torch.zeros(V, native.TRACK_COUNTS, dtype=torch.int64, device=dev)
    if N == 0:
        return counts
    tr, gt = (t.detach().float().contiguous() for t in (tracks, gt_tracks))
    vis, gvis = ((t.detach() != 0).to(torch.uint8).contiguous() for t in (visible, gt_visible))
    q = queries.detach().float().contiguous()
    with torch.cuda.device(dev):
        nbytes = native.rnc.track_metrics_workspace_bytes(V, N, T)
        if nbytes == 0:
            raise ValueError(f"track_metrics: {V} videos of {N} points over {T} frames exceed the kernel's limits "
                             f"(V <= 65535, N*T < 2^30)")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        native.rnc.track_metrics(tr, vis, gt, gvis, q, V, N, T, H, W, counts, ws, ws.numel())
    return counts


def host_track_metrics(tracks, visible, gt_tracks, gt_visible, queries, H, W):
    """track_metrics in torch: the scaled coordinates, differences, squares and their sum each rounded once to float32."""
    V, N, T = _check_metrics(tracks, visible, gt_tracks, gt_visible, queries, H, W)
    p, g = (t.detach().cpu().float().double() for t in (tracks, gt_tracks))
    pv, gv = (t.detach().cpu() != 0 for t in (visible, gt_visible))
    scale = torch.tensor([W, H], dtype=torch.float64)
    d = _f32(_f32(_f32(p * 256) / scale) - _f32(_f32(g * 256) / scale))
    d2 = _f32(_f32(d[..., 0] * d[..., 0]) + _f32(d[..., 1] * d[..., 1]))
    tq = queries.detach().cpu().float()[..., 0].long()
    ev = torch.ones(V, N, T, dtype=torch.bool)
    ev.scatter_(2, tq[..., None], False)

    def count(m):
        return (m & ev).sum((1, 2))
    cols = [count(ev), count(pv == gv), count(gv)]
    within = [d2 < float(delta * delta) for delta in THRESHOLDS]
    cols += [count(w & gv) for w in within]
    cols += [count(w & gv & pv) for w in within]
    cols += [count(pv & (~gv | ~w)) for w in within]
    return torch.stack(cols, 1).to(torch.int64)


def _ratio(a, b):
    return a / b if b else math.nan


def summarize_tracking(counts):
    """TAP-Vid's numbers from per-video counts ([V, TRACK_COUNTS] int64, or a list of V count lists), each per video and then
    averaged over videos in fp64: occlusion_accuracy (agreements / evaluated pairs), pts_within_<d> (within & gt visible /
    gt visible) and their mean over d, average_pts_within_thresh (< delta^x_avg), jaccard_<d> (true positives / (gt visible +
    false positives)) and their mean over d, average_jaccard; videos, their number.  A ratio with a zero denominator is NaN
    (a video without a visible ground-truth point has no position accuracy), and NaN without a video."""
    rows = counts.tolist() if isinstance(counts, torch.Tensor) else [list(c) for c in counts]
    n = len(rows)
    keys = ["occlusion_accuracy", "average_pts_within_thresh", "average_jaccard"]
    keys += [f"pts_within_{d}" for d in THRESHOLDS] + [f"jaccard_{d}" for d in THRESHOLDS]
    out = dict.fromkeys(keys, 0.0)
    for c in rows:
        per = {"occlusion_accuracy": _ratio(c[COUNT_OCC_AGREE], c[COUNT_EVALUATED])}
        for j, d in enumerate(THRESHOLDS):
            per[f"pts_within_{d}"] = _ratio(c[COUNT_WITHIN + j], c[COUNT_GT_VISIBLE])
            per[f"jaccard_{d}"] = _ratio(c[COUNT_TP + j], c[COUNT_GT_VISIBLE] + c[COUNT_FP + j])
        per["average_pts_within_thresh"] = sum(per[f"pts_within_{d}"] for d in THRESHOLDS) / len(THRESHOLDS)
        per["average_jaccard"] = sum(per[f"jaccard_{d}"] for d in THRESHOLDS) / len(THRESHOLDS)
        for k in keys:
            out[k] += per[k]
    out = {k: (v / n if n else math.nan) for k, v in out.items()}
    out["videos"] = n
    return out
