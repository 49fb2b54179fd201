"""Video object segmentation by label propagation along the backward flows, and the DAVIS semi-supervised metrics J and F.

Propagation.  Inputs, per video v of V: the labels of frame 0, L_0 uint8 [H,W] (0 background, 1..254 objects; 255 is not a
label); for each pair k = 0..T-2 the backward flow G_k (frame k+1 -> frame k, float32 [2,H,W], channel 0 = x) and the mask
occ_bw_k (uint8 [H,W] on frame k+1, occluded where non-zero).  These are the flow_up_bw and occ_bw that
rnc.harness.run_sequences_bidirectional yields for pair k.  Frame 0's output is L_0; step k -> k+1, for every pixel p = (x, y)
of frame k+1:
1. u = G_k(p), read at the pixel itself, and p' = p + u, each component rounded once to float32.
2. p is matched when both components of u are finite, occ_bw_k(p) == 0 and p' lies in [0, W-1] x [0, H-1].
3. A matched pixel takes the bilinear vote of L_k at p': the taps (y0,x0), (y0,x1), (y1,x0), (y1,x1), with x1 = min(x0+1, W-1)
   and y1 = min(y0+1, H-1), weigh bx*by, ax*by, bx*ay, ax*ay (each rounded once; rnc.interp's sample); for each distinct label
   among the taps its weights are added in tap order, each addition rounded once; the largest sum wins, a tie the smaller
   label.
4. An unmatched pixel takes the label of the nearest matched pixel of frame k+1: least exact squared Euclidean distance, ties
   to the smallest column, then the smallest row (rnc.metrics.nearest_site, the feature transform of rnc.interp's hole
   fill).  In a frame without a matched pixel every pixel is 0.
Only hard labels are carried from frame to frame, so bilinear blur does not build up over a video, and the fill keeps false
occlusions at object edges from eroding an object frame after frame.  `propagate_step` and `propagate` run CUDA tensors
through rnc_propagate_labels (csrc/segment.cu) and CPU tensors through `host_propagate_step`, which holds float32 values in
fp64 and rounds each operation once, so both give the same labels.

Metrics (Perazzi et al., "A Benchmark Dataset and Evaluation Methodology for Video Object Segmentation", CVPR 2016; Pont-Tuset
et al., "The 2017 DAVIS Challenge on Video Object Segmentation", 2017), restated from the definitions of the public DAVIS
2017 toolkit's semi-supervised evaluation:
- Objects are 1..K, K the largest non-void label of the ground truth's frame 0; the scored frames are 1..T-2 (the first and
  last are dropped).  A ground-truth value of 255 is void.  For object o the predicted mask is M = (pred == o) & non-void and
  the ground-truth mask G = (gt == o).
- J = |M & G| / |M | G|, and 1 when the union is empty.
- The boundary map of a mask s (the toolkit's seg2bmap at full resolution): with e[:, :-1] = s[:, 1:], so[:-1, :] = s[1:, :]
  and se[:-1, :-1] = s[1:, 1:] (zero elsewhere), b = (s ^ e) | (s ^ so) | (s ^ se); then b[-1, :] = s[-1, :] ^ e[-1, :],
  b[:, -1] = s[:, -1] ^ so[:, -1] and b[-1, -1] = 0.
- F: with r = ceil(0.008 * sqrt(H^2 + W^2)) in fp64 (8 at 480x854, 18 at 1080x1920), a boundary pixel of one mask matches
  when a boundary pixel of the other lies at squared distance <= r^2 (the toolkit's dilation by disk(r)).  With n_fg, n_gt
  the boundary sizes of M and G and fg_match, gt_match their matched pixels: P, R = 1, 0 for (n_fg, n_gt) = (0, > 0); 0, 1
  for (> 0, 0); 1, 1 for (0, 0); else fg_match / n_fg and gt_match / n_gt.  F = 2PR / (P + R), and 0 when P + R = 0.
- Per object over its scored frames: the mean M, the recall O (the fraction of frames with a value > 0.5) and the decay D =
  mean(bin 0) - mean(bin 3), bin i = v[ids[i] : ids[i+1] + 1] with ids = round(linspace(1, n, 5) + 1e-10) - 1 (the bins
  overlap, as in the toolkit).
- J-Mean, J-Recall, J-Decay, F-Mean, F-Recall and F-Decay are each the mean of the per-object values over all objects of all
  videos, and J&F-Mean = (J-Mean + F-Mean) / 2.
`segmentation_counts` gives the integer counts J and F are ratios of (the COUNT_* columns), through rnc_segmentation_counts
for CUDA tensors and `host_segmentation_counts` for CPU tensors; they are exact, so the metrics do not depend on the batch,
the order or the number of GPUs.  `summarize_segmentation` forms the statistics from them in fp64.
"""
import math

import numpy as np
import torch

from . import native
from .metrics import _f32, nearest_site

MAX_SIDE = 4096                             # csrc/dist_transform.cuh's kSiteMaxSide
VOID = 255
# the columns of a (frame, object)'s counts (RNC_SEGMENT_COUNTS)
COUNT_INTER, COUNT_UNION, COUNT_N_FG, COUNT_N_GT, COUNT_FG_MATCH, COUNT_GT_MATCH = range(6)
assert COUNT_GT_MATCH + 1 == native.SEGMENT_COUNTS
_COUNTS_WORKSPACE_CAP = 1 << 30             # segmentation_counts runs as many frames per launch as fit in this


def check_labels(labels, what="propagate"):
    """ValueError unless labels is an integer tensor with every value in 0..254.  The test runs on the labels' device; the
    host waits for its flag only."""
    if labels.dtype.is_floating_point or labels.dtype.is_complex:
        raise ValueError(f"{what}: expected integer labels, got {labels.dtype}")
    if labels.numel() and bool(((labels < 0) | (labels > 254)).any()):
        bad = labels[(labels < 0) | (labels > 254)][:4].tolist()
        raise ValueError(f"{what}: labels must lie in 0..254 (255 is void, not a label), got {bad}")


def _check_sides(H, W, what):
    if not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE):
        raise ValueError(f"{what}: frames of {H}x{W}; the kernels take 1 <= H, W <= {MAX_SIDE}")


def _check_step(labels, flow_bw, occ_bw):
    """(V, H, W) of propagate_step's arguments; ValueError for mismatched shapes, mixed devices or a frame side above 4096."""
    if labels.dim() != 3 or labels.shape[0] == 0:
        raise ValueError(f"propagate_step: expected labels [V,H,W], got {tuple(labels.shape)}")
    V, H, W = labels.shape
    if tuple(flow_bw.shape) != (V, 2, H, W):
        raise ValueError(f"propagate_step: expected flow_bw {[V, 2, H, W]}, got {tuple(flow_bw.shape)}")
    if tuple(occ_bw.shape) != (V, H, W):
        raise ValueError(f"propagate_step: expected occ_bw {[V, H, W]}, got {tuple(occ_bw.shape)}")
    devs = {t.device for t in (labels, flow_bw, occ_bw)}
    if len(devs) != 1:
        raise ValueError(f"propagate_step: the labels, flow and mask must be on one device, got {sorted(map(str, devs))}")
    _check_sides(H, W, "propagate_step")
    return V, H, W


def propagate_step(labels, flow_bw, occ_bw):
    """One step of the rule for V videos: labels [V,H,W] (L_k, integer values 0..254), flow_bw [V,2,H,W] (G_k, float32 or
    converted to it), occ_bw [V,H,W] (occluded where non-zero), any strides.  Returns uint8 [V,H,W], L_{k+1}.  CUDA tensors
    go through rnc_propagate_labels (enqueued on the current stream after the labels' check, whose flag the host waits
    for), CPU tensors through host_propagate_step; the labels are equal.  ValueError before any launch for mismatched shapes,
    mixed devices, a label outside 0..254 or a side above 4096."""
    _check_step(labels, flow_bw, occ_bw)
    check_labels(labels, "propagate_step")
    return _step(labels, flow_bw, occ_bw)


def _step(labels, flow_bw, occ_bw, out=None, ws=None):
    """propagate_step without its checks, into out (uint8 [V,H,W], any strides, not overlapping labels) when given."""
    if not labels.is_cuda:
        res = _host_steps(labels, flow_bw, occ_bw)
        return res if out is None else out.copy_(res)
    V, H, W = labels.shape
    dev = labels.device
    lab = labels.detach().to(torch.uint8)
    g = flow_bw.detach().float()
    o = occ_bw.detach().to(torch.uint8)
    if out is None:
        out = torch.empty(V, H, W, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        nbytes = native.rnc.propagate_labels_workspace_bytes(V, H, W)
        if ws is None or ws.numel() < nbytes:
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        native.rnc.propagate_labels(lab, *lab.stride(), g, *g.stride(), o, *o.stride(), V, H, W, out, *out.stride(), ws,
                                    ws.numel())
    return out


def _check_video(first_labels, flow_bw, occ_bw):
    if first_labels.dim() != 3 or first_labels.shape[0] == 0:
        raise ValueError(f"propagate: expected first_labels [V,H,W], got {tuple(first_labels.shape)}")
    V, H, W = first_labels.shape
    if flow_bw.dim() != 5 or flow_bw.shape[0] != V or tuple(flow_bw.shape[2:]) != (2, H, W):
        raise ValueError(f"propagate: expected flow_bw [{V},T-1,2,{H},{W}], got {tuple(flow_bw.shape)}")
    T1 = flow_bw.shape[1]
    if T1 < 1:
        raise ValueError(f"propagate: a video needs T >= 2 frames, got {T1 + 1}")
    if tuple(occ_bw.shape) != (V, T1, H, W):
        raise ValueError(f"propagate: expected occ_bw {[V, T1, H, W]}, got {tuple(occ_bw.shape)}")
    devs = {t.device for t in (first_labels, flow_bw, occ_bw)}
    if len(devs) != 1:
        raise ValueError(f"propagate: the labels, flows and masks must be on one device, got {sorted(map(str, devs))}")
    _check_sides(H, W, "propagate")
    check_labels(first_labels, "propagate")
    return V, T1 + 1, H, W


def propagate(first_labels, flow_bw, occ_bw):
    """The labels of every frame of V videos from those of frame 0: first_labels [V,H,W], flow_bw [V,T-1,2,H,W], occ_bw
    [V,T-1,H,W], any strides (the stacked pair results are read through views, not copied).  Returns uint8 [V,T,H,W], frame 0
    being first_labels.  T-1 steps of propagate_step's rule, each written straight into its frame of the result; CUDA tensors
    take T-1 launches of rnc_propagate_labels on the current stream after the labels' check.  ValueError before any launch
    for mismatched shapes, mixed devices, T < 2, a label outside 0..254 or a side above 4096."""
    V, T, H, W = _check_video(first_labels, flow_bw, occ_bw)
    out = torch.empty(V, T, H, W, dtype=torch.uint8, device=first_labels.device)
    out[:, 0] = first_labels
    ws = None
    if out.is_cuda:
        ws = torch.empty(native.rnc.propagate_labels_workspace_bytes(V, H, W), dtype=torch.uint8, device=out.device)
    for k in range(T - 1):
        _step(out[:, k], flow_bw[:, k], occ_bw[:, k], out[:, k + 1], ws)
    return out


def _host_vote(L, G, occ):
    """One frame of the rule on the host: L uint8 [H,W], G fp64 [2,H,W] holding float32 values, occ [H,W].  Returns the
    int64 labels [H,W]."""
    H, W = L.shape
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    ux, uy = G[0], G[1]
    px, py = _f32(xs + ux), _f32(ys + uy)
    matched = (torch.isfinite(ux) & torch.isfinite(uy) & (occ == 0) & (px >= 0) & (px <= W - 1) & (py >= 0)
               & (py <= H - 1))
    cx, cy = torch.where(matched, px, 0.0), torch.where(matched, py, 0.0)      # an unmatched pixel's vote is discarded
    x0, y0 = torch.floor(cx), torch.floor(cy)
    ax, ay = _f32(cx - x0), _f32(cy - y0)
    bx, by = _f32(1 - ax), _f32(1 - ay)
    ix, iy = x0.long(), y0.long()
    ix1, iy1 = (ix + 1).clamp(max=W - 1), (iy + 1).clamp(max=H - 1)
    lab = L.long()
    taps = [lab[iy, ix], lab[iy, ix1], lab[iy1, ix], lab[iy1, ix1]]
    w = [_f32(bx * by), _f32(ax * by), _f32(bx * ay), _f32(ax * ay)]
    best = torch.full((H, W), -1.0, dtype=torch.float64)
    vote = torch.full((H, W), VOID, dtype=torch.int64)
    for i in range(4):
        first = torch.ones(H, W, dtype=torch.bool)
        for j in range(i):
            first &= taps[j] != taps[i]
        s = w[i]
        for j in range(i + 1, 4):
            s = torch.where(taps[j] == taps[i], _f32(s + w[j]), s)
        take = first & ((s > best) | ((s == best) & (taps[i] < vote)))
        best, vote = torch.where(take, s, best), torch.where(take, taps[i], vote)
    site = torch.from_numpy(nearest_site(matched.numpy()[None])[0])
    fill = torch.where(site >= 0, vote.reshape(-1)[site.clamp(min=0)], 0)
    return torch.where(matched, vote, fill)


def _host_steps(labels, flow_bw, occ_bw):
    V, H, W = labels.shape
    out = torch.empty(V, H, W, dtype=torch.uint8)
    for v in range(V):
        out[v] = _host_vote(labels[v].detach().cpu().to(torch.uint8), flow_bw[v].detach().cpu().float().double(),
                            occ_bw[v].detach().cpu()).to(torch.uint8)
    return out


def host_propagate_step(labels, flow_bw, occ_bw):
    """propagate_step's rule in torch, one video at a time and all its pixels at once: each floating-point operation evaluated
    in fp64 on float32 operands and rounded once to float32 (the IEEE float32 result, as rnc.track.host_track), the fill by
    rnc.metrics.nearest_site.  Serves CPU tensors and is the kernel's test reference.  Returns uint8 [V,H,W] on the CPU."""
    _check_step(labels, flow_bw, occ_bw)
    check_labels(labels, "propagate_step")
    return _host_steps(labels, flow_bw, occ_bw)


def host_propagate(first_labels, flow_bw, occ_bw):
    """propagate through host_propagate_step's restatement.  Returns uint8 [V,T,H,W] on the CPU."""
    V, T, H, W = _check_video(first_labels, flow_bw, occ_bw)
    out = torch.empty(V, T, H, W, dtype=torch.uint8)
    out[:, 0] = first_labels.cpu()
    for k in range(T - 1):
        out[:, k + 1] = _host_steps(out[:, k], flow_bw[:, k], occ_bw[:, k])
    return out


# ------------------------------------------------------------------------------------------------------------ J and F


def tolerance(H, W):
    """DAVIS's boundary tolerance r in pixels: ceil(0.008 * sqrt(H^2 + W^2)), in fp64."""
    return math.ceil(0.008 * math.sqrt(H * H + W * W))


def seg2bmap(s):
    """The boundary map of a bool numpy mask [..., H, W] at full resolution, as the DAVIS toolkit defines it (above)."""
    s = np.asarray(s, dtype=bool)
    e, so, se = np.zeros_like(s), np.zeros_like(s), np.zeros_like(s)
    e[..., :, :-1] = s[..., :, 1:]
    so[..., :-1, :] = s[..., 1:, :]
    se[..., :-1, :-1] = s[..., 1:, 1:]
    b = (s ^ e) | (s ^ so) | (s ^ se)
    b[..., -1, :] = s[..., -1, :] ^ e[..., -1, :]
    b[..., :, -1] = s[..., :, -1] ^ so[..., :, -1]
    b[..., -1, -1] = False
    return b


def _check_counts(pred, gt, K):
    if pred.dim() != 3 or tuple(gt.shape) != tuple(pred.shape):
        raise ValueError(f"segmentation_counts: expected pred and gt of one [N,H,W] shape, got {tuple(pred.shape)} and "
                         f"{tuple(gt.shape)}")
    if pred.device != gt.device:
        raise ValueError(f"segmentation_counts: pred and gt must be on one device, got {pred.device} and {gt.device}")
    if not (isinstance(K, int) and 0 <= K <= 254):
        raise ValueError(f"segmentation_counts: expected an object count K in 0..254, got {K!r}")
    for name, t in (("pred", pred), ("gt", gt)):
        if t.dtype.is_floating_point or t.dtype.is_complex:
            raise ValueError(f"segmentation_counts: expected integer {name} labels, got {t.dtype}")
    _check_sides(pred.shape[1], pred.shape[2], "segmentation_counts")
    return pred.shape


def segmentation_counts(pred, gt, K):
    """Per (frame, object) DAVIS counts of predicted labels against the ground truth: pred, gt [N,H,W] integer labels with
    values 0..255 (gt 255 is void; any strides), K the number of objects (1..K are scored).  Returns int64
    [N,K,SEGMENT_COUNTS] on the tensors' device (the COUNT_* columns).  CUDA tensors go through rnc_segmentation_counts (on
    the current stream, as many frames per launch as a 1 GiB workspace holds), CPU tensors through host_segmentation_counts;
    the counts are equal."""
    N, H, W = _check_counts(pred, gt, K)
    if not pred.is_cuda:
        return host_segmentation_counts(pred, gt, K)
    dev = pred.device
    counts = torch.empty(N, K, native.SEGMENT_COUNTS, dtype=torch.int64, device=dev)
    if N == 0 or K == 0:
        return counts
    p, g = (t.detach().to(torch.uint8) for t in (pred, gt))
    step = max(1, min(N, 32767 // K, _COUNTS_WORKSPACE_CAP // (8 * K * H * W)))
    with torch.cuda.device(dev):
        ws = torch.empty(native.rnc.segmentation_counts_workspace_bytes(min(step, N), K, H, W), dtype=torch.uint8, device=dev)
        for lo in range(0, N, step):
            n = min(step, N - lo)
            pn, gn = p[lo:lo + n], g[lo:lo + n]
            native.rnc.segmentation_counts(pn, *pn.stride(), gn, *gn.stride(), n, K, H, W, counts[lo:lo + n], ws, ws.numel())
    return counts


def host_segmentation_counts(pred, gt, K):
    """segmentation_counts' definition in numpy int64: seg2bmap's boundaries, each pixel's exact squared distance to the
    other mask's boundary by rnc.metrics.nearest_site, and the counts.  Returns int64 [N,K,SEGMENT_COUNTS] on the CPU."""
    N, H, W = _check_counts(pred, gt, K)
    out = torch.zeros(N, K, native.SEGMENT_COUNTS, dtype=torch.int64)
    if N == 0 or K == 0:
        return out
    p = pred.detach().cpu().long().numpy()[:, None]
    g = gt.detach().cpu().long().numpy()[:, None]
    o = np.arange(1, K + 1).reshape(1, K, 1, 1)
    M = (p == o) & (g != VOID)                                          # [N,K,H,W]
    G = g == o
    bM, bG = seg2bmap(M), seg2bmap(G)
    site = nearest_site(np.concatenate([bM, bG]).reshape(2 * N * K, H, W)).reshape(2, N, K, H, W)
    y = np.arange(H).reshape(H, 1)
    x = np.arange(W).reshape(1, W)
    d2 = np.where(site >= 0, (y - site // W) ** 2 + (x - site % W) ** 2, np.iinfo(np.int64).max)
    r2 = tolerance(H, W) ** 2
    cols = [M & G, M | G, bM, bG, bM & (d2[1] <= r2), bG & (d2[0] <= r2)]
    return torch.from_numpy(np.stack([c.sum((2, 3)) for c in cols], -1).astype(np.int64))


def region_similarity(c):
    """J of one (frame, object)'s counts."""
    return 1.0 if c[COUNT_UNION] == 0 else c[COUNT_INTER] / c[COUNT_UNION]


def contour_accuracy(c):
    """F of one (frame, object)'s counts."""
    n_fg, n_gt = c[COUNT_N_FG], c[COUNT_N_GT]
    if n_fg == 0 and n_gt == 0:
        P, R = 1.0, 1.0
    elif n_fg == 0:
        P, R = 1.0, 0.0
    elif n_gt == 0:
        P, R = 0.0, 1.0
    else:
        P, R = c[COUNT_FG_MATCH] / n_fg, c[COUNT_GT_MATCH] / n_gt
    return 0.0 if P + R == 0 else 2 * P * R / (P + R)


def decay_bins(n):
    """The toolkit's four decay bins of n per-frame values, as (start, stop) slices: ids = round(linspace(1, n, 5) + 1e-10)
    - 1 and bin i = [ids[i], ids[i+1] + 1)."""
    ids = (np.round(np.linspace(1, n, 5) + 1e-10) - 1).astype(np.int64)
    return [(int(ids[i]), int(ids[i + 1]) + 1) for i in range(4)]


def statistics(values):
    """(mean, recall, decay) of one object's per-frame values, in fp64."""
    v = np.asarray(values, dtype=np.float64)
    bins = [v[a:b] for a, b in decay_bins(len(v))]
    return float(v.mean()), float((v > 0.5).mean()), float(bins[0].mean() - bins[3].mean())


KEYS = ("J&F-Mean", "J-Mean", "J-Recall", "J-Decay", "F-Mean", "F-Recall", "F-Decay")


def summarize_segmentation(counts):
    """DAVIS's numbers from per-video counts: a list of one [F_v, K_v, SEGMENT_COUNTS] tensor or nested list per video, over
    its scored frames.  Each object's J and F statistics over its frames, then J-Mean, J-Recall, J-Decay, F-Mean, F-Recall
    and F-Decay as means over all objects of all videos, and J&F-Mean; objects and videos, their numbers.  NaN without an
    object."""
    per = {k: [] for k in KEYS[1:]}
    for c in counts:
        rows = c.tolist() if isinstance(c, torch.Tensor) else c
        K = len(rows[0]) if rows else 0
        for o in range(K):
            for m, fn in (("J", region_similarity), ("F", contour_accuracy)):
                mean, recall, decay = statistics([fn(frame[o]) for frame in rows])
                per[f"{m}-Mean"].append(mean)
                per[f"{m}-Recall"].append(recall)
                per[f"{m}-Decay"].append(decay)
    out = {k: (float(np.mean(v)) if v else math.nan) for k, v in per.items()}
    out = {"J&F-Mean": (out["J-Mean"] + out["F-Mean"]) / 2, **out}
    out["objects"] = len(per["J-Mean"])
    out["videos"] = len(counts)
    return out
