"""Validation metrics (evaluate.py:88-182) as per-image partials that any number of batches, or of GPUs, combine exactly.

`flow_metrics(flow, gt, valid)` gives per image the int64 counts of valid pixels, of EPE < 1, < 3 and < 5 and of KITTI
outliers, and the fp64 sum of the valid pixels' EPE.  CUDA tensors go through rnc_flow_metrics (csrc/flow_metrics.cu), CPU
tensors through `host_partials`, the same float32 formulas in torch; the kernel's counts equal the host's and its sums agree
to the last few bits.  `summarize(partials, mode)` turns the partials of a whole split, in image order, into the numbers the
reference prints.  Both paths give an image's partials independently of the batch it came in, so a split's result does not
depend on the batch size or on how the images were spread over ranks.

`sparsification(flow, gt, valid, score)` evaluates a per-pixel confidence score the same way: per image, the sparsification
curve (the mean EPE of the valid pixels left once the lowest-scored fraction f_k = k/100 is removed) and its ideal (the
largest errors removed instead) as partial sums; `summarize_sparsification` gives the split's curves and their AUSE.  CUDA
tensors go through rnc_sparsification (csrc/sparsification.cu), CPU tensors through `host_sparsification`.
"""
from collections import namedtuple

import numpy as np
import torch

from . import native

# counts: int64 [N, 5] (valid, epe < 1, < 3, < 5, outliers); epe_sum: float64 [N]
Partials = namedtuple("Partials", "counts epe_sum")
# count: int64 [N, 100] (valid pixels kept at f_k); kept_epe, ideal_epe: float64 [N, 100] (their EPE sum, score / ideal order)
SparsPartials = namedtuple("SparsPartials", "count kept_epe ideal_epe")
FRACTIONS = 100


def _check(flow, gt, valid):
    if flow.dim() != 4 or flow.shape[1] != 2 or gt.shape != flow.shape:
        raise ValueError(f"flow_metrics: expected flow and gt of one [B,2,H,W] shape, got {tuple(flow.shape)} and "
                         f"{tuple(gt.shape)}")
    if valid is not None and tuple(valid.shape) != (flow.shape[0],) + tuple(flow.shape[2:]):
        raise ValueError(f"flow_metrics: expected valid [B,H,W] = {(flow.shape[0],) + tuple(flow.shape[2:])}, got "
                         f"{tuple(valid.shape)}")
    if len({t.device for t in (flow, gt, valid) if t is not None}) != 1:
        raise ValueError("flow_metrics: flow, gt and valid must be on one device")


def flow_metrics(flow, gt, valid=None):
    """flow, gt: [B,2,H,W] (any strides; float32, or converted to it); valid: [B,H,W] or None (every pixel valid).
    Returns Partials of B images on the tensors' device; on CUDA it is enqueued on the current stream."""
    _check(flow, gt, valid)
    if not flow.is_cuda:
        return host_partials(flow, gt, valid)
    flow, gt = flow.float(), gt.float()
    valid = None if valid is None else valid.float()
    B, _, H, W = flow.shape
    dev = flow.device
    counts = torch.empty(B, 5, dtype=torch.int64, device=dev)
    epe_sum = torch.empty(B, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        ws = torch.empty(native.rnc.flow_metrics_workspace_bytes(B, H, W), dtype=torch.uint8, device=dev)
        vs = (0, 0, 0) if valid is None else valid.stride()
        native.rnc.flow_metrics(flow, *flow.stride(), gt, *gt.stride(), valid, *vs, B, H, W, counts, epe_sum, ws, ws.numel())
    return Partials(counts, epe_sum)


def _f32(x):
    """x (fp64) rounded to float32, kept in fp64.  Each of + - * / sqrt evaluated in fp64 on float32 operands and rounded once
    to float32 is the IEEE float32 result (53 >= 2 * 24 + 2 bits), whatever the CPU's vector library rounds."""
    return x.float().double()


def _norm(v):
    return _f32(_f32(_f32(v[0] * v[0]) + _f32(v[1] * v[1])).sqrt())


def host_partials(flow, gt, valid=None):
    """The partials of the reference's float32 formulas (evaluate.py:163-171), one image at a time, summed in fp64.  Every
    operation is rounded as IEEE float32 rounds it, as numpy, CUDA and torch on the GPU do; torch's CPU float32 sqrt is not
    correctly rounded on every CPU (AVX-512: one ulp off for a fraction of a percent of inputs)."""
    _check(flow, gt, valid)
    counts, sums = [], []
    for b in range(flow.shape[0]):
        f, g = flow[b].float().double(), gt[b].float().double()
        epe = _norm(_f32(f - g))
        mag = _norm(g)
        val = torch.ones_like(epe, dtype=torch.bool) if valid is None else valid[b] >= 0.5
        out = (epe > 3.0) & (_f32(epe / mag).float() > 0.05)     # compared in float32: 0.05 is rounded to 0.05f
        counts.append(torch.stack([val.sum(), (val & (epe < 1)).sum(), (val & (epe < 3)).sum(), (val & (epe < 5)).sum(),
                                   (val & out).sum()]))
        sums.append(torch.where(val, epe, 0.0).double().sum())
    if not counts:
        return Partials(torch.zeros(0, 5, dtype=torch.int64), torch.zeros(0, dtype=torch.float64))
    return Partials(torch.stack(counts).to(torch.int64), torch.stack(sums))


def cat(parts):
    """One Partials of a list of them, in order."""
    if not parts:
        return Partials(torch.zeros(0, 5, dtype=torch.int64), torch.zeros(0, dtype=torch.float64))
    return Partials(torch.cat([p.counts for p in parts]), torch.cat([p.epe_sum for p in parts]))


def _ratio(a, b):
    return a / b if b else float("nan")


def summarize(partials, mode):
    """The metrics of a split from its per-image partials, combined in image order in fp64.
    mode "sintel" or "chairs" (evaluate.py:95-137): EPE, 1px, 3px, 5px pooled over every pixel.
    mode "kitti" (evaluate.py:163-179): EPE is the mean over images of each image's mean EPE over its valid pixels (NaN for an
    image without one, as in the reference); 1px/3px/5px and F1 (in percent) are pooled over all valid pixels."""
    if mode not in ("sintel", "chairs", "kitti"):
        raise ValueError(f"summarize: mode must be 'sintel', 'chairs' or 'kitti', got {mode!r}")
    counts = partials.counts.cpu().tolist()
    sums = partials.epe_sum.cpu().tolist()
    tot = [sum(c[k] for c in counts) for k in range(5)]
    res = {"1px": _ratio(tot[1], tot[0]), "3px": _ratio(tot[2], tot[0]), "5px": _ratio(tot[3], tot[0])}
    if mode == "kitti":
        epe = 0.0
        for s, c in zip(sums, counts):
            epe += s / c[0] if c[0] else float("nan")
        res["epe"] = _ratio(epe, len(counts))
        res["f1"] = 100 * _ratio(tot[4], tot[0])
    else:
        epe = 0.0
        for s in sums:
            epe += s
        res["epe"] = _ratio(epe, tot[0])
    return {k: res[k] for k in ("epe", "1px", "3px", "5px", "f1") if k in res}


def _check_score(flow, score):
    want = (flow.shape[0],) + tuple(flow.shape[2:])
    if score is None or tuple(score.shape) != want:
        raise ValueError(f"sparsification: expected score [B,H,W] = {want}, got "
                         f"{None if score is None else tuple(score.shape)}")
    if score.device != flow.device:
        raise ValueError("sparsification: flow, gt, valid and score must be on one device")


def sparsification(flow, gt, valid, score):
    """flow, gt: [B,2,H,W]; valid: [B,H,W] or None (every pixel valid); score: [B,H,W], higher is more confident (any
    strides; float32, or converted to it).  Returns SparsPartials of B images on the tensors' device: for k = 0..99, with N
    valid pixels and m_k = floor(k*N/100) of them removed, count[:, k] = N - m_k and the fp64 EPE sums of the pixels kept in
    score order (kept_epe) and in ideal order (ideal_epe); see host_sparsification.  On CUDA it is enqueued on the current
    stream."""
    _check(flow, gt, valid)
    _check_score(flow, score)
    if not flow.is_cuda:
        return host_sparsification(flow, gt, valid, score)
    flow, gt, score = flow.float(), gt.float(), score.float()
    valid = None if valid is None else valid.float()
    B, _, H, W = flow.shape
    dev = flow.device
    count = torch.empty(B, FRACTIONS, dtype=torch.int64, device=dev)
    kept = torch.empty(B, FRACTIONS, dtype=torch.float64, device=dev)
    ideal = torch.empty(B, FRACTIONS, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        nbytes = native.rnc.sparsification_workspace_bytes(B, H, W)
        if nbytes == 0:
            raise ValueError(f"sparsification: {B} images of {H}x{W} exceed the sort's 2^31 pixels")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        vs = (0, 0, 0) if valid is None else valid.stride()
        native.rnc.sparsification(flow, *flow.stride(), gt, *gt.stride(), valid, *vs, score, *score.stride(), B, H, W, count,
                                  kept, ideal, ws, ws.numel())
    return SparsPartials(count, kept, ideal)


def _nan_first_order(v):
    """Stable ascending order of v with every NaN first (ties keep their index order)."""
    nan = torch.isnan(v)
    o = torch.argsort(torch.where(nan, float("-inf"), v), stable=True)
    return o[torch.argsort((~nan[o]).to(torch.int8), stable=True)]


def host_sparsification(flow, gt, valid, score):
    """sparsification's definition, one image at a time in fp64 on float32 values.  EPE as host_partials rounds it; valid
    where valid >= 0.5.  Score order: the valid pixels by score ascending, a NaN score below -inf, ties by row-major index.
    Ideal order: by EPE descending, a NaN EPE largest.  Removing the first m_k = floor(k*N/100) (k = 0..99) of each order
    leaves count = N - m_k pixels; kept_epe / ideal_epe are the fp64 sums of their EPE.  An image with N = 0 gives zeros."""
    _check(flow, gt, valid)
    _check_score(flow, score)
    B = flow.shape[0]
    count = torch.zeros(B, FRACTIONS, dtype=torch.int64)
    kept = torch.zeros(B, FRACTIONS, dtype=torch.float64)
    ideal = torch.zeros(B, FRACTIONS, dtype=torch.float64)
    for b in range(B):
        f, g = flow[b].float().double(), gt[b].float().double()
        epe = _norm(_f32(f - g)).reshape(-1)
        val = torch.ones_like(epe, dtype=torch.bool) if valid is None else (valid[b] >= 0.5).reshape(-1)
        e, s = epe[val], score[b].float().reshape(-1)[val]
        n = e.numel()
        if n == 0:
            continue
        m = torch.tensor([k * n // FRACTIONS for k in range(FRACTIONS)])
        count[b] = n - m
        for out, order in ((kept, _nan_first_order(s)), (ideal, _nan_first_order(-e))):
            tail = e[order].flip(0).cumsum(0).flip(0)            # tail[j]: the sum of the pixels from j on
            out[b] = tail[m]
    return SparsPartials(count, kept, ideal)


def summarize_sparsification(partials):
    """The split's curves from per-image SparsPartials, in image order in fp64 over the images with a valid pixel:
    sparsification[k] (and ideal[k]) is the mean over those images of kept_epe[k] / count[k] (ideal_epe[k] / count[k]), and
    ause = numpy.trapezoid(sparsification - ideal, x=f_k) over f_k = k/100.  NaN everywhere when no image has a valid pixel."""
    count = partials.count.cpu().tolist()
    kept = partials.kept_epe.cpu().tolist()
    orc = partials.ideal_epe.cpu().tolist()
    sp, orr, n = [0.0] * FRACTIONS, [0.0] * FRACTIONS, 0
    for c, ke, oe in zip(count, kept, orc):
        if c[0] == 0:
            continue
        n += 1
        for k in range(FRACTIONS):
            sp[k] += ke[k] / c[k]
            orr[k] += oe[k] / c[k]
    if n == 0:
        nan = float("nan")
        return {"sparsification": [nan] * FRACTIONS, "ideal": [nan] * FRACTIONS, "ause": nan}
    sp = [v / n for v in sp]
    orr = [v / n for v in orr]
    x = np.arange(FRACTIONS) / FRACTIONS
    ause = float(np.trapezoid(np.array(sp) - np.array(orr), x=x))
    return {"sparsification": sp, "ideal": orr, "ause": ause}


def confidence_score(conf):
    """The score validate ranks pixels by: the harmonic mean of the NCUP output confidence's two planes, [B,2,H,W] ->
    [B,H,W] float32, 2*c_u*c_v / (c_u + c_v) and 0 where c_u + c_v == 0, each operation rounded once.  With a per-component
    variance proportional to 1/c, the EPE's variance goes as 1/c_u + 1/c_v, whose order is the harmonic mean's reversed."""
    if conf.dim() != 4 or conf.shape[1] != 2:
        raise ValueError(f"confidence_score: expected a [B,2,H,W] confidence, got {tuple(conf.shape)}")
    cu, cv = conf[:, 0].float(), conf[:, 1].float()
    den = cu + cv
    return torch.where(den == 0, torch.zeros_like(den), (2 * cu * cv) / den)


OCC_INCONSISTENT, OCC_OUTSIDE = 1, 2          # bits of fb_consistency's occ


def _check_fb(flow_fw, flow_bw):
    if flow_fw.dim() != 4 or flow_fw.shape[1] != 2 or flow_bw.shape != flow_fw.shape:
        raise ValueError(f"fb_consistency: expected forward and backward flows of one [B,2,H,W] shape, got "
                         f"{tuple(flow_fw.shape)} and {tuple(flow_bw.shape)}")
    if flow_fw.device != flow_bw.device:
        raise ValueError(f"fb_consistency: the flows are on {flow_fw.device} and {flow_bw.device}; they must be on one device")
    if flow_fw.numel() == 0:
        raise ValueError(f"fb_consistency: empty flows {tuple(flow_fw.shape)}")


def fb_consistency(flow_fw, flow_bw, alpha1=0.01, alpha2=0.5):
    """Forward-backward consistency (UnFlow, Meister et al. 2018) of B flow pairs at full resolution.  flow_fw: [B,2,H,W]
    from frame 1 to frame 2, flow_bw: from frame 2 to frame 1 (any strides; float32, or converted to it).

    Per pixel x of direction F -> G (and G -> F): the target p = x + F(x), G^(p) sampled bilinearly with zero padding on
    align_corners=True pixel coordinates (utils.utils.bilinear_sampler), err = |F(x) + G^(p)|, and occ with bit 0
    (OCC_INCONSISTENT) where |F + G^|^2 > alpha1 (|F|^2 + |G^|^2) + alpha2 or that sum is not finite, and bit 1 (OCC_OUTSIDE)
    where p lies outside [0, W-1] x [0, H-1].  A pixel whose target is outside, or whose inputs hold a NaN, gets err = +inf
    and the bits that apply.  Returns (occ_fw, occ_bw) uint8 [B,H,W] and (err_fw, err_bw) float32 [B,H,W]: CUDA tensors
    through rnc_fb_consistency (one launch, enqueued on the current stream), CPU tensors through host_fb_consistency; both
    round every operation once in float32, in the same order, so they give the same bits."""
    _check_fb(flow_fw, flow_bw)
    if not flow_fw.is_cuda:
        return host_fb_consistency(flow_fw, flow_bw, alpha1, alpha2)
    fw, bw = flow_fw.float(), flow_bw.float()
    B, _, H, W = fw.shape
    dev = fw.device
    occ = torch.empty(2, B, H, W, dtype=torch.uint8, device=dev)
    err = torch.empty(2, B, H, W, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        native.rnc.fb_consistency(fw, *fw.stride(), bw, *bw.stride(), B, H, W, float(alpha1), float(alpha2), occ[0], occ[1],
                                  err[0], err[1])
    return occ[0], occ[1], err[0], err[1]


def _fb_direction(f, g, a1, a2):
    """One direction of host_fb_consistency: f, g fp64 [B,2,H,W] holding float32 values; a1, a2 float32 values."""
    B, _, H, W = f.shape
    u = torch.arange(W, dtype=torch.float64).view(1, 1, W)
    v = torch.arange(H, dtype=torch.float64).view(1, H, 1)
    fu, fv = f[:, 0], f[:, 1]
    px, py = _f32(u + fu), _f32(v + fv)
    inside = (px >= 0) & (px <= W - 1) & (py >= 0) & (py <= H - 1)
    x0, y0 = torch.floor(px), torch.floor(py)
    ax, ay = _f32(px - x0), _f32(py - y0)
    bx, by = _f32(1 - ax), _f32(1 - ay)
    ix = torch.where(inside, x0, 0).long()
    iy = torch.where(inside, y0, 0).long()
    bi = torch.arange(B).view(B, 1, 1).expand_as(ix)

    def tap(dx, dy, c):
        x, y = ix + dx, iy + dy
        ok = (x < W) & (y < H)
        return torch.where(ok, g[bi, c, y.clamp(max=H - 1), x.clamp(max=W - 1)], 0.0)

    w00, w01, w10, w11 = _f32(bx * by), _f32(ax * by), _f32(bx * ay), _f32(ax * ay)
    gs = []
    for c in range(2):
        s = _f32(tap(0, 0, c) * w00)
        s = _f32(s + _f32(tap(1, 0, c) * w01))
        s = _f32(s + _f32(tap(0, 1, c) * w10))
        gs.append(_f32(s + _f32(tap(1, 1, c) * w11)))
    su, sv = _f32(fu + gs[0]), _f32(fv + gs[1])
    lhs = _f32(_f32(su * su) + _f32(sv * sv))
    mf = _f32(_f32(fu * fu) + _f32(fv * fv))
    mg = _f32(_f32(gs[0] * gs[0]) + _f32(gs[1] * gs[1]))
    rhs = _f32(_f32(a1 * _f32(mf + mg)) + a2)
    finite = torch.isfinite(lhs)
    inf = torch.full_like(lhs, float("inf"))
    err = torch.where(inside & finite, _f32(torch.where(finite, lhs, 0.0).sqrt()), inf)
    occ = torch.where(inside, (~finite | (lhs > rhs)).to(torch.uint8), torch.full_like(lhs, 3, dtype=torch.uint8))
    return occ, err.float()


def host_fb_consistency(flow_fw, flow_bw, alpha1=0.01, alpha2=0.5):
    """fb_consistency's definition in torch: each operation evaluated in fp64 on float32 operands and rounded once to float32
    (the IEEE float32 result, as in host_partials), in the kernel's order.  Serves CPU tensors and is the kernel's test
    reference."""
    _check_fb(flow_fw, flow_bw)
    f, g = flow_fw.detach().cpu().float().double(), flow_bw.detach().cpu().float().double()
    a1, a2 = float(torch.tensor(alpha1, dtype=torch.float32)), float(torch.tensor(alpha2, dtype=torch.float32))
    occ_fw, err_fw = _fb_direction(f, g, a1, a2)
    occ_bw, err_bw = _fb_direction(g, f, a1, a2)
    return occ_fw, occ_bw, err_fw, err_bw
