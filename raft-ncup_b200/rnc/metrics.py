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

`region_partials(flow, gt, valid, occ=..., noc=..., fg=...)` splits the flow metrics' partials by region (Sintel's matched /
unmatched, occlusion-boundary distance and speed bins; KITTI's background / foreground over all and non-occluded pixels; the
definitions are below), and `summarize_regions` gives the split's per-region EPE or Fl.  `boundary_dist2(occ)` is the exact
distance transform they use.  CUDA tensors go through rnc_boundary_dist2 and rnc_region_metrics (csrc/region_metrics.cu),
CPU tensors through `host_boundary_dist2` and `host_region_partials`.
"""
from collections import namedtuple

import numpy as np
import torch

from . import native
from .restate import f32

# counts: int64 [N, 5] (valid, epe < 1, < 3, < 5, outliers); epe_sum: float64 [N]
Partials = namedtuple("Partials", "counts epe_sum")
# count: int64 [N, 100] (valid pixels kept at f_k); kept_epe, ideal_epe: float64 [N, 100] (their EPE sum, score / ideal order)
SparsPartials = namedtuple("SparsPartials", "count kept_epe ideal_epe")
FRACTIONS = 100
# counts: int64 [N, cells, 5] (as Partials.counts, per cell); epe_sum: float64 [N, cells]; fg: bool [N] (KITTI: the image
# came with a foreground mask)
RegionPartials = namedtuple("RegionPartials", "counts epe_sum fg")
# sq_sum: float64 [N], per frame the sum over pixels of sum_c (pred - gt)^2; count: int64 [N], its pixels (rnc.interp)
InterpPartials = namedtuple("InterpPartials", "sq_sum count")

# the partials of no image, per type (RegionPartials with 0 cells)
_EMPTY = {Partials: Partials(torch.zeros(0, 5, dtype=torch.int64), torch.zeros(0, dtype=torch.float64)),
          SparsPartials: SparsPartials(torch.zeros(0, FRACTIONS, dtype=torch.int64),
                                       *(torch.zeros(0, FRACTIONS, dtype=torch.float64) for _ in range(2))),
          RegionPartials: RegionPartials(torch.zeros(0, 0, 5, dtype=torch.int64), torch.zeros(0, 0, dtype=torch.float64),
                                         torch.zeros(0, dtype=torch.bool)),
          InterpPartials: InterpPartials(torch.zeros(0, dtype=torch.float64), torch.zeros(0, dtype=torch.int64))}


def cat(kind, parts):
    """One `kind` partials (Partials, SparsPartials, RegionPartials or InterpPartials) of a list of them, in image order."""
    if not parts:
        return _EMPTY[kind]
    return kind(*(torch.cat(f) for f in zip(*parts)))


def images(partials):
    """Per-image records of partials: one tuple per image of its fields' values as Python numbers and lists (what
    validate gathers over ranks)."""
    return list(zip(*(f.cpu().tolist() for f in partials)))


def from_images(kind, records):
    """The `kind` partials of per-image records, on the CPU: the inverse of images."""
    if not records:
        return _EMPTY[kind]
    return kind(*(torch.tensor(col, dtype=e.dtype) for col, e in zip(zip(*records), _EMPTY[kind])))


def _strides(t):
    """The element strides of an optional [B,H,W] mask; zeros for None, which the kernels do not read."""
    return (0, 0, 0) if t is None else t.stride()


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
        native.rnc.flow_metrics(flow, *flow.stride(), gt, *gt.stride(), valid, *_strides(valid), B, H, W, counts, epe_sum, ws,
                                ws.numel())
    return Partials(counts, epe_sum)


def _norm(v):
    return f32(f32(f32(v[0] * v[0]) + f32(v[1] * v[1])).sqrt())


def host_partials(flow, gt, valid=None):
    """The partials of the reference's float32 formulas (evaluate.py:163-171), one image at a time, summed in fp64.  Every
    operation is rounded as IEEE float32 rounds it, as numpy, CUDA and torch on the GPU do; torch's CPU float32 sqrt is not
    correctly rounded on every CPU (AVX-512: one ulp off for a fraction of a percent of inputs)."""
    _check(flow, gt, valid)
    counts, sums = [], []
    for b in range(flow.shape[0]):
        f, g = flow[b].float().double(), gt[b].float().double()
        epe = _norm(f32(f - g))
        mag = _norm(g)
        val = torch.ones_like(epe, dtype=torch.bool) if valid is None else valid[b] >= 0.5
        out = (epe > 3.0) & (f32(epe / mag).float() > 0.05)     # compared in float32: 0.05 is rounded to 0.05f
        counts.append(torch.stack([val.sum(), (val & (epe < 1)).sum(), (val & (epe < 3)).sum(), (val & (epe < 5)).sum(),
                                   (val & out).sum()]))
        sums.append(torch.where(val, epe, 0.0).double().sum())
    if not counts:
        return Partials(torch.zeros(0, 5, dtype=torch.int64), torch.zeros(0, dtype=torch.float64))
    return Partials(torch.stack(counts).to(torch.int64), torch.stack(sums))


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
        native.rnc.sparsification(flow, *flow.stride(), gt, *gt.stride(), valid, *_strides(valid), score, *score.stride(), B, H,
                                  W, count, kept, ideal, ws, ws.numel())
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
        epe = _norm(f32(f - g)).reshape(-1)
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
    px, py = f32(u + fu), f32(v + fv)
    inside = (px >= 0) & (px <= W - 1) & (py >= 0) & (py <= H - 1)
    x0, y0 = torch.floor(px), torch.floor(py)
    ax, ay = f32(px - x0), f32(py - y0)
    bx, by = f32(1 - ax), f32(1 - ay)
    ix = torch.where(inside, x0, 0).long()
    iy = torch.where(inside, y0, 0).long()
    bi = torch.arange(B).view(B, 1, 1).expand_as(ix)

    def tap(dx, dy, c):
        x, y = ix + dx, iy + dy
        ok = (x < W) & (y < H)
        return torch.where(ok, g[bi, c, y.clamp(max=H - 1), x.clamp(max=W - 1)], 0.0)

    w00, w01, w10, w11 = f32(bx * by), f32(ax * by), f32(bx * ay), f32(ax * ay)
    gs = []
    for c in range(2):
        s = f32(tap(0, 0, c) * w00)
        s = f32(s + f32(tap(1, 0, c) * w01))
        s = f32(s + f32(tap(0, 1, c) * w10))
        gs.append(f32(s + f32(tap(1, 1, c) * w11)))
    su, sv = f32(fu + gs[0]), f32(fv + gs[1])
    lhs = f32(f32(su * su) + f32(sv * sv))
    mf = f32(f32(fu * fu) + f32(fv * fv))
    mg = f32(f32(gs[0] * gs[0]) + f32(gs[1] * gs[1]))
    rhs = f32(f32(a1 * f32(mf + mg)) + a2)
    finite = torch.isfinite(lhs)
    inf = torch.full_like(lhs, float("inf"))
    err = torch.where(inside & finite, f32(torch.where(finite, lhs, 0.0).sqrt()), inf)
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


# ----------------------------------------------------------------------------------------------------------- region metrics
#
# The per-region errors the Sintel and KITTI 2015 benchmarks publish, as this project defines them (the Sintel server does not
# publish its pixel conventions, so these are not claimed to reproduce its values to the last pixel).  Per pixel: epe, mag =
# |gt| and the outlier test epe > 3 & epe / mag > 0.05 in rnc_flow_metrics' float32 arithmetic.  A region counts only the
# pixels with valid >= 0.5 (every pixel when valid is None), and every region metric is pooled over the pixels of the whole
# split.
#
# Sintel-style (occ: [H,W] per image, occluded where >= 0.5):
#   matched = not occluded, unmatched = occluded.
#   A boundary pixel has a 4-neighbour inside the image whose occlusion label differs from its own (pixels on both sides of
#   the boundary count).  d2(p) is the exact squared Euclidean distance, in pixels, from p to the nearest boundary pixel of
#   its image, over the whole image whatever valid says (DIST2_NONE in an image without a boundary).
#   d0-10: d2 < 100; d10-60: 100 <= d2 < 3600; d60-140: 3600 <= d2 < 19600; farther, or no boundary: no d-bin.
#   s0-10: mag < 10; s10-40: 10 <= mag < 40; s40+: mag >= 40; a NaN mag: no s-bin.
# KITTI-style (noc: [H,W], the validity of the non-occluded ground truth, where >= 0.5; fg: [H,W] or None, foreground where
#   >= 0.5, from the object map): Fl (the outlier rate, in percent) over all, background and foreground pixels, each over all
#   valid pixels and over the valid pixels inside noc.
#
# A cell is one joint label of a pixel; region_partials gives per image and per cell the five counts and the fp64 EPE sum of
# flow_metrics, and a region is a sum of cells.  Sintel: cell = 16*occluded + 4*d + s (d, s: the bin's index, 3 for none),
# 32 cells.  KITTI: cell = 2*(not noc) + fg, 4 cells.

DIST2_NONE = native.DIST2_NONE
SINTEL_CELLS, KITTI_CELLS = native.REGION_CELLS[native.REGIONS_SINTEL], native.REGION_CELLS[native.REGIONS_KITTI]
# region -> its cells, in increasing order
SINTEL_REGIONS = {"matched": list(range(16)), "unmatched": list(range(16, 32)),
                  **{k: [c for c in range(32) if (c >> 2) & 3 == i] for i, k in enumerate(("d0-10", "d10-60", "d60-140"))},
                  **{k: [c for c in range(32) if c & 3 == i] for i, k in enumerate(("s0-10", "s10-40", "s40+"))}}
KITTI_REGIONS = {"all": [0, 1, 2, 3], "bg": [0, 2], "fg": [1, 3], "all_noc": [0, 1], "bg_noc": [0], "fg_noc": [1]}


def _check_mask(name, m, flow):
    want = (flow.shape[0],) + tuple(flow.shape[2:])
    if tuple(m.shape) != want:
        raise ValueError(f"region_partials: expected {name} [B,H,W] = {want}, got {tuple(m.shape)}")
    if m.device != flow.device:
        raise ValueError(f"region_partials: {name} is on {m.device}, the flow on {flow.device}; they must be on one device")


def _check_regions(flow, gt, valid, occ, noc, fg):
    _check(flow, gt, valid)
    if (occ is None) == (noc is None):
        raise ValueError("region_partials: give occ (Sintel-style) or noc (KITTI-style), not both or neither")
    if occ is not None and fg is not None:
        raise ValueError("region_partials: fg goes with noc (KITTI-style), not with occ")
    for name, m in (("occ", occ), ("noc", noc), ("fg", fg)):
        if m is not None:
            _check_mask(name, m, flow)


def boundary_dist2(occ):
    """occ: [B,H,W] (any strides; float32, or converted to it), occluded where >= 0.5.  Returns int32 [B,H,W]: per pixel the
    exact squared Euclidean distance to the nearest occlusion-boundary pixel of its image, DIST2_NONE in an image without
    one.  CUDA tensors go through rnc_boundary_dist2 (enqueued on the current stream; 1 <= H, W <= 4096), CPU tensors through
    host_boundary_dist2; both are exact integers, so they are equal."""
    if occ.dim() != 3 or occ.numel() == 0:
        raise ValueError(f"boundary_dist2: expected a non-empty [B,H,W] mask, got {tuple(occ.shape)}")
    if not occ.is_cuda:
        return host_boundary_dist2(occ)
    occ = occ.float()
    B, H, W = occ.shape
    d2 = torch.empty(B, H, W, dtype=torch.int32, device=occ.device)
    with torch.cuda.device(occ.device):
        native.rnc.boundary_dist2(occ, *occ.stride(), B, H, W, d2)
    return d2


def _boundary(lab):
    """Boundary pixels of a bool [B,H,W] label map: a 4-neighbour inside the image holds the other label."""
    bnd = np.zeros_like(lab)
    dy = lab[:, 1:] != lab[:, :-1]
    bnd[:, 1:] |= dy
    bnd[:, :-1] |= dy
    dx = lab[:, :, 1:] != lab[:, :, :-1]
    bnd[:, :, 1:] |= dx
    bnd[:, :, :-1] |= dx
    return bnd


def nearest_site(sites):
    """An exact feature transform: sites, bool numpy [N,H,W] -> int64 [N,H,W], per pixel the row-major index of its
    nearest site in exact squared Euclidean distance, ties to the smallest column and then the smallest row; -1 in an image
    without a site.  host_boundary_dist2 and rnc.interp's hole fill use it.  The kernels' algorithm (csrc/dist_transform.cuh)
    in numpy, every row of the batch at once: the nearest site in each column (the upper one on a tie), then along each row
    the lower envelope of the parabolas q -> g(q)^2 + (x - q)^2 (Felzenszwalb and Huttenlocher), intersections compared by
    cross-multiplying, and per pixel the leftmost parabola of least value."""
    N, H, W = sites.shape
    rows = np.empty((N, H, W), dtype=np.int64)
    last = np.full((N, W), -1, dtype=np.int64)
    for y in range(H):
        last = np.where(sites[:, y], y, last)
        rows[:, y] = last
    nxt = np.full((N, W), -1, dtype=np.int64)
    for y in range(H - 1, -1, -1):
        nxt = np.where(sites[:, y], y, nxt)
        r = rows[:, y]
        rows[:, y] = np.where((nxt >= 0) & ((r < 0) | (nxt - y < y - r)), nxt, r)
    R = N * H
    rows = rows.reshape(R, W)
    y_of = np.tile(np.arange(H, dtype=np.int64), N)[:, None]
    q_all = np.arange(W, dtype=np.int64)
    F = np.where(rows >= 0, (y_of - rows) ** 2 + q_all * q_all, -1)
    v = np.zeros((R, W), dtype=np.int64)
    n = np.zeros(R, dtype=np.int64)
    idx_all = np.arange(R)
    for q in range(W):
        fq = F[:, q]
        popping = fq >= 0
        while True:
            idx = idx_all[popping & (n > 1)]
            if idx.size == 0:
                break
            p, r = v[idx, n[idx] - 1], v[idx, n[idx] - 2]
            fp, fr = F[idx, p], F[idx, r]
            pop = (fq[idx] - fp) * (p - r) <= (fp - fr) * (q - p)
            n[idx[pop]] -= 1
            popping[idx[~pop]] = False
        push = idx_all[fq >= 0]
        v[push, n[push]] = q
        n[push] += 1
    out = np.full((R, W), -1, dtype=np.int64)
    k = np.zeros(R, dtype=np.int64)
    some = idx_all[n > 0]
    for x in range(W):
        while True:                 # move on to the next parabola while it is strictly below the current one at x
            idx = some[k[some] + 1 < n[some]]
            a, c = v[idx, k[idx]], v[idx, k[idx] + 1]
            step = 2 * x * (c - a) > F[idx, c] - F[idx, a]
            if not step.any():
                break
            k[idx[step]] += 1
        q = v[some, k[some]]
        out[some, x] = rows[some, q] * W + q
    return out.reshape(N, H, W)


def host_boundary_dist2(occ):
    """boundary_dist2 in numpy int64, exact: the squared distance from each pixel to its nearest boundary pixel (nearest_site,
    the kernels' separable transform)."""
    lab = (occ.detach().cpu().float() >= 0.5).numpy()
    B, H, W = lab.shape
    site = nearest_site(_boundary(lab))
    y = np.arange(H, dtype=np.int64).reshape(1, H, 1)
    x = np.arange(W, dtype=np.int64).reshape(1, 1, W)
    d2 = (y - site // W) ** 2 + (x - site % W) ** 2
    return torch.from_numpy(np.where(site >= 0, d2, DIST2_NONE).astype(np.int32))


def region_partials(flow, gt, valid=None, occ=None, noc=None, fg=None):
    """flow, gt: [B,2,H,W]; valid: [B,H,W] or None (every pixel valid); then either occ (Sintel-style) or noc and optionally
    fg (KITTI-style), each [B,H,W] (any strides; float32, or converted to it).  Returns RegionPartials of B images on the
    tensors' device (the region definitions above).  CUDA tensors go through rnc_boundary_dist2 and rnc_region_metrics
    (enqueued on the current stream), CPU tensors through host_region_partials; the counts are equal and the sums agree to
    the last few bits.  An image's partials do not depend on the batch it came in."""
    _check_regions(flow, gt, valid, occ, noc, fg)
    if not flow.is_cuda:
        return host_region_partials(flow, gt, valid, occ, noc, fg)
    flow, gt = flow.float(), gt.float()
    valid = None if valid is None else valid.float()
    B, _, H, W = flow.shape
    dev = flow.device
    kind = native.REGIONS_SINTEL if occ is not None else native.REGIONS_KITTI
    cells = native.REGION_CELLS[kind]
    mask = (occ if occ is not None else noc).float()
    fg = None if fg is None else fg.float()
    counts = torch.empty(B, cells, 5, dtype=torch.int64, device=dev)
    epe_sum = torch.empty(B, cells, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        d2 = boundary_dist2(mask) if occ is not None else None
        ws = torch.empty(native.rnc.region_metrics_workspace_bytes(kind, B, H, W), dtype=torch.uint8, device=dev)
        native.rnc.region_metrics(kind, flow, *flow.stride(), gt, *gt.stride(), valid, *_strides(valid), mask, *mask.stride(),
                                  d2, fg, *_strides(fg), B, H, W, counts, epe_sum, ws, ws.numel())
    return RegionPartials(counts, epe_sum, torch.full((B,), fg is not None, dtype=torch.bool))


def host_region_partials(flow, gt, valid=None, occ=None, noc=None, fg=None):
    """region_partials' definition, one image at a time: the pixel values as host_partials rounds them, the cell of each valid
    pixel, and per cell the counts and the fp64 sum of its EPEs (numpy.bincount)."""
    _check_regions(flow, gt, valid, occ, noc, fg)
    B = flow.shape[0]
    cells = SINTEL_CELLS if occ is not None else KITTI_CELLS
    d2 = host_boundary_dist2(occ).to(torch.int64) if occ is not None else None
    counts = torch.zeros(B, cells, 5, dtype=torch.int64)
    sums = torch.zeros(B, cells, dtype=torch.float64)
    for b in range(B):
        f, g = flow[b].detach().cpu().float().double(), gt[b].detach().cpu().float().double()
        epe = _norm(f32(f - g))
        mag = _norm(g)
        val = torch.ones_like(epe, dtype=torch.bool) if valid is None else valid[b].cpu() >= 0.5
        out = (epe > 3.0) & (f32(epe / mag).float() > 0.05)
        if occ is not None:
            d = (d2[b] >= 100).long() + (d2[b] >= 3600).long() + (d2[b] >= 19600).long()    # DIST2_NONE: 3
            s = torch.where(torch.isnan(mag), 3, (mag >= 10).long() + (mag >= 40).long())
            cell = 16 * (occ[b].cpu().float() >= 0.5).long() + 4 * d + s
        else:
            cell = 2 * (~(noc[b].cpu().float() >= 0.5)).long()
            if fg is not None:
                cell = cell + (fg[b].cpu().float() >= 0.5).long()
        c, e = cell[val].numpy(), epe[val].numpy()
        o = out[val].numpy()
        counts[b] = torch.from_numpy(np.stack([np.bincount(c[m], minlength=cells)
                                               for m in (np.ones_like(o), e < 1, e < 3, e < 5, o)], 1))
        sums[b] = torch.from_numpy(np.bincount(c, weights=e, minlength=cells).astype(np.float64))
    return RegionPartials(counts, sums, torch.full((B,), fg is not None, dtype=torch.bool))


def cat_regions(parts):
    """One RegionPartials of a list of them (of one style), in order: cat(RegionPartials, parts), under its public name."""
    return cat(RegionPartials, parts)


def summarize_regions(partials):
    """The split's region metrics from its per-image RegionPartials, pooled over pixels.  Each region's counts are exact
    integer sums; its EPE sum adds, image by image in order, the image's cells of the region in increasing order (fp64).
    Sintel-style (32 cells): epe_matched, epe_unmatched, epe_d0-10, epe_d10-60, epe_d60-140, epe_s0-10, epe_s10-40, epe_s40+.
    KITTI-style (4 cells): fl_all and fl_all_noc, and when every image came with fg also fl_bg, fl_fg, fl_bg_noc and
    fl_fg_noc, in percent as summarize's f1 (fl_all counts f1's pixels, so it equals f1 bit for bit).  region_pixels: each
    returned region's valid-pixel count.  A region without a pixel gives NaN."""
    counts = partials.counts.cpu().tolist()
    sums = partials.epe_sum.cpu().tolist()
    cells = partials.counts.shape[1]
    if cells not in (SINTEL_CELLS, KITTI_CELLS):
        raise ValueError(f"summarize_regions: expected {SINTEL_CELLS} (Sintel) or {KITTI_CELLS} (KITTI) cells, got {cells}")
    res, pixels = {}, {}
    if cells == SINTEL_CELLS:
        for name, cs in SINTEL_REGIONS.items():
            n = sum(c[k][0] for c in counts for k in cs)
            epe = 0.0
            for s in sums:
                si = 0.0
                for k in cs:
                    si += s[k]
                epe += si
            res["epe_" + name] = _ratio(epe, n)
            pixels[name] = n
    else:
        names = list(KITTI_REGIONS) if bool(partials.fg.all()) else ["all", "all_noc"]
        for name in names:
            cs = KITTI_REGIONS[name]
            n = sum(c[k][0] for c in counts for k in cs)
            res["fl_" + name] = 100 * _ratio(sum(c[k][4] for c in counts for k in cs), n)
            pixels[name] = n
    res["region_pixels"] = pixels
    return res


def occlusion_counts(pred, occ, valid=None):
    """Scores a predicted occlusion mask against the ground truth: pred [B,H,W], occluded where non-zero (fb_consistency's
    occ: inconsistent or leaving the frame); occ [B,H,W], occluded where >= 0.5; valid [B,H,W] or None.  Returns int64 [B,3]
    on their device: per image the valid pixels predicted and truly occluded, predicted occluded, and truly occluded (integer
    sums, so the same on any device and in any order)."""
    p, t = pred != 0, occ >= 0.5
    v = torch.ones_like(p) if valid is None else valid >= 0.5
    return torch.stack([(p & t & v).sum((1, 2)), (p & v).sum((1, 2)), (t & v).sum((1, 2))], 1).to(torch.int64)


def summarize_occlusion(counts):
    """occ_precision, occ_recall and occ_f1 of the split from occlusion_counts' rows, pooled over pixels; NaN when a
    denominator is 0."""
    tp, pp, ap = (sum(r[k] for r in counts.cpu().tolist()) for k in range(3))
    return {"occ_precision": _ratio(tp, pp), "occ_recall": _ratio(tp, ap), "occ_f1": _ratio(2 * tp, pp + ap)}
