"""What the host restatements of the video kernels share, each written once in the order its kernel computes it, and the
frame-size check of the modules that call those kernels.

The restatements hold float32 values in fp64 tensors and round every operation once with f32, so that they give the
kernels' bits: csrc/bilinear.cuh's sample, taps, in-frame test and flow-follow rule, and csrc/homography.cuh's projection.
"""
import math

import numpy as np
import torch

MAX_SIDE = 4096                             # csrc/dist_transform.cuh's kSiteMaxSide
PI_F32 = float(np.float32(math.pi))


def f32(x):
    """x (fp64) rounded to float32, kept in fp64.  Each of + - * / sqrt evaluated in fp64 on float32 operands and rounded once
    to float32 is the IEEE float32 result (53 >= 2 * 24 + 2 bits), whatever the CPU's vector library rounds."""
    return x.float().double()


def check_sides(H, W, what):
    if not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE):
        raise ValueError(f"{what}: frames of {H}x{W}; the kernels take 1 <= H, W <= {MAX_SIDE}")


def inside(x, y, H, W):
    """(x, y) lies in [0, W-1] x [0, H-1]: torch or numpy, elementwise; false for NaN."""
    return (x >= 0) & (x <= W - 1) & (y >= 0) & (y <= H - 1)


def follow(G, occ):
    """Every pixel p of a frame follows its flow u = G(p) (fp64 [2,H,W] holding float32 values) to p' = p + u when u is
    finite, occ(p) == 0 and p' lies in the frame.  Returns (matched bool [H,W], px, py fp64 [H,W]): p' where matched and 0
    elsewhere, so that a sample there stays in the frame and is discarded."""
    H, W = occ.shape
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    px, py = f32(xs + G[0]), f32(ys + G[1])
    matched = torch.isfinite(G[0]) & torch.isfinite(G[1]) & (occ == 0) & inside(px, py, H, W)
    return matched, torch.where(matched, px, 0.0), torch.where(matched, py, 0.0)


def bilinear_taps(px, py, H, W):
    """The four bilinear taps at (px, py) (fp64, float32 values) with the coordinates clamped to the frame: a list of
    (iy, ix, weight) in tap order (y0, x0), (y0, x1), (y1, x0), (y1, x1), weighted bx*by, ax*by, bx*ay, ax*ay."""
    px, py = px.clamp(0, W - 1), py.clamp(0, H - 1)
    x0, y0 = torch.floor(px), torch.floor(py)
    ax, ay = f32(px - x0), f32(py - y0)
    bx, by = f32(1 - ax), f32(1 - ay)
    ix, iy = x0.long(), y0.long()
    ix1, iy1 = (ix + 1).clamp(max=W - 1), (iy + 1).clamp(max=H - 1)
    return [(iy, ix, f32(bx * by)), (iy, ix1, f32(ax * by)), (iy1, ix, f32(bx * ay)), (iy1, ix1, f32(ax * ay))]


def sample(img, px, py, k=None):
    """Bilinear samples of img (fp64 holding float32 values) at (px, py): the taps weighted and added in tap order.  img is
    [C,H,W], or [K,C,H,W] with k the per-element frame index.  Returns [C, ...]."""
    s = None
    for ty, tx, w in bilinear_taps(px, py, *img.shape[-2:]):
        t = f32((img[:, ty, tx] if k is None else img[k, :, ty, tx].T) * w)
        s = t if s is None else f32(s + t)
    return s


def project(m, x, y):
    """pi(m (x, y, 1)) in numpy fp64, each operation rounded once: (X / w, Y / w, w > 0)."""
    X = (m[0] * x + m[1] * y) + m[2]
    Y = (m[3] * x + m[4] * y) + m[5]
    w = (m[6] * x + m[7] * y) + m[8]
    return X / w, Y / w, w > 0
