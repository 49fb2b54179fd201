"""An fp64 model of the unsupervised losses' arithmetic (csrc/photometric.cu, rnc/unsupervised.py, DESIGN §3.16) with
per-pixel error bounds, the stimuli that reach the regimes the kernels were designed around, and the model's self-checks.
tests/test_gpu_photometric_error_model.py holds the kernels to these bounds.

The model takes the fp64 restatement's values (g(I1), W^ and dW^/dp from rnc.unsupervised._warp on the kernel's float32 sample
positions, see snapped()) and follows each kernel's operations, adding at every float32 operation the error that operation
may make:
  - every rounding to float32: at most U = 2^-24 of the value;
  - rsqrtf 2 ulp, powf 4 ulp, expf 2 ulp (the CUDA Programming Guide's single-precision table; one ulp of x is at most
    2^-23 |x|), sqrtf and the division IEEE-rounded (the build passes neither -use_fast_math nor -prec-div=false);
  - the float32 constants 0.81f, 0.1f, 0.01f, 0.4f, 0.2f, 1e-6f against their decimal values;
  - an input error e propagated through a function f by sup |f'| over [x - e, x + e] (each f's sup is closed-form below);
  - a float32 sum of terms t_1..t_n in a fixed order: u sum_j |t_1 + ... + t_j| (the partial sums, first order).
Contracting a product and a sum into one fma rounds once where the bound allows two, so the bounds hold with or without
contraction (the build does not pass -fmad=false).  Second-order terms (products of two relative errors, each below 1e-4) are
covered by SLACK.  The kernel's own fp64 state (g(I1), W^) may differ from the restatement's by FMA contraction: E_STATE.

Census forward, per pixel (census_fwd_kernel, offsets dy-major): delta = A(p+d) - A(p) rounded once from fp64 to fp32;
c = delta rsqrtf(0.81f + delta^2); e = c1 - c2; phi = e^2 / (0.1f + e^2); h = the 49-term float32 sum; t = h + 0.01f;
l = powf(t, 0.4f); k = v 0.4f l / t.
Census backward, per pixel (census_bwd_kernel): kw = k(q) + k(q+d), A = 0.2f e / den^2 (den = 0.1f + e^2), B = 0.81f r2^3
(r2 = rsqrtf(0.81f + delta2^2)), G = the 49-term float32 sum of kw A B, times scale, times dW^/dpx and dW^/dpy (fp64 rounded to
fp32).  The fp64 value of G follows the gather identity of photometric.cu; test_model_matches_the_host_restatement holds it to
autograd of host_census_loss.
Smoothness (SmoothPixel, smoothness_bwd_kernel): w = expf(-kappa (s / 765)), s = the float32 sum of |dI_c|; d = the float32
second difference; each term sqrtf(d^2 + 1e-6f) w, summed in fp64; the gradient gathers coef d rsqrtf(d^2 + 1e-6f) w over the
three terms of each axis that hold the pixel, times the axis's scale.
"""
import math
from typing import NamedTuple

import pytest
import torch
import torch.nn.functional as F

from rnc.unsupervised import EDGE_CONSTANT, _warp, host_census_hamming, host_census_loss, host_smoothness_loss

U = 2.0 ** -24
RSQRT_ULP, POW_ULP, EXP_ULP = 2, 4, 2
SLACK = 1.01
E_STATE = 2.0 ** -40           # |kernel fp64 state - restatement|: a few 2^-53 * 255, with room
TINY = 2.0 ** -126             # expf results below the normal range carry an absolute error, not a relative one
R = 3                          # census radius
TILE_X, TILE_Y = 32, 8         # census tile


def f32err(c):
    return abs(float(torch.tensor(c, dtype=torch.float32).double()) - c)


def f32(c):
    return torch.tensor(c, dtype=torch.float32)


E081, E001, E04, E1M6 = (f32err(c) for c in (0.81, 0.01, 0.4, 1e-6))      # 0.1f and 0.2f: within the constants below


# -------------------------------------------------------------------------------------------------------- fp64 restatement
def snapped(flow):
    """flow in fp64 with x + F and y + F rounded to float32 as the kernels round them, so that the fp64 restatement takes its
    bilinear taps at the same floor (elsewhere the derivative of the sample jumps).  Non-finite values stay non-finite."""
    h, w = flow.shape[-2:]
    xs = torch.arange(w, device=flow.device, dtype=torch.float32).view(1, w)
    ys = torch.arange(h, device=flow.device, dtype=torch.float32).view(h, 1)
    return torch.stack([(xs + flow[:, 0].float()).double() - xs.double(), (ys + flow[:, 1].float()).double() - ys.double()], 1)


def gray(im):
    return 0.2989 * im[:, 0] + 0.5870 * im[:, 1] + 0.1140 * im[:, 2]


def warp_state(image1, image2, flow):
    """The census state of the fp64 restatement: g(I1), W^, dW^/dpx, dW^/dpy [N,H,W] (fp64) at the kernel's sample positions,
    computed on the CPU and returned on flow's device."""
    f = snapped(flow.cpu()).requires_grad_()
    wh = _warp(gray(image2.cpu().double()), f)
    (dw,) = torch.autograd.grad(wh.sum(), f)
    return tuple(t.to(flow.device) for t in (gray(image1.cpu().double()), wh.detach(), dw[:, 0], dw[:, 1]))


def weights(mask, N, H, W, device):
    v = torch.zeros(N, H, W, dtype=torch.float64, device=device)
    v[:, R:H - R, R:W - R] = 1
    return v if mask is None else v * (mask.to(device) != 0).double()


def offsets():
    return [(dy, dx) for dy in range(2 * R + 1) for dx in range(2 * R + 1)]      # the kernels' dy-major order


def shifted(p, dy, dx, H, W):
    return p[:, dy:dy + H, dx:dx + W]


def psi(x):
    return x / torch.sqrt(0.81 + x * x)


def dpsi(x):
    return 0.81 / (0.81 + x * x) ** 1.5


def sup_dphi(e, err):
    """sup |phi'| on [|e| - err, |e| + err]: phi'(x) = 0.2 x / (0.1 + x^2)^2 rises to its maximum at x^2 = 1/30, then falls."""
    def dphi(x):
        return 0.2 * x / (0.1 + x * x) ** 2
    lo, hi = (e.abs() - err).clamp_min(0), e.abs() + err
    peak = math.sqrt(1 / 30)
    return torch.where((lo <= peak) & (hi >= peak), dphi(torch.tensor(peak, dtype=e.dtype)),
                       torch.maximum(dphi(lo), dphi(hi)))


def sup_d2phi(e, err):
    """sup |phi''| on that interval: |phi''(x)| <= 0.2 (0.1 + 3 x^2) / (0.1 + x^2)^3, which falls in |x| (20 at 0)."""
    m = (e.abs() - err).clamp_min(0)
    return 0.2 * (0.1 + 3 * m * m) / (0.1 + m * m) ** 3


SUP_D2PSI = 1.07               # sup |psi''| = 2.43 x / (0.81 + x^2)^2.5 at x = 0.45: 1.0601


class CensusModel(NamedTuple):
    h: torch.Tensor            # [N,H,W], every pixel
    l: torch.Tensor            # v l
    k: torch.Tensor            # v 0.4 l / (h + 0.01)
    v: torch.Tensor
    err_l: torch.Tensor
    err_k: torch.Tensor


def census_forward_model(g1, wh, v):
    """h, v l, k and their bounds from the fp64 state (g1, wh [N,H,W]) and the weights v."""
    N, H, W = g1.shape
    p1, pw = F.pad(g1, (R, R, R, R)), F.pad(wh, (R, R, R, R))
    h = torch.zeros_like(g1)
    err_phi = torch.zeros_like(g1)
    partial = torch.zeros_like(g1)
    for dy, dx in offsets():
        d1, d2 = shifted(p1, dy, dx, H, W) - g1, shifted(pw, dy, dx, H, W) - wh
        e, ee = census_e(d1, d2)
        phi = e * e / (0.1 + e * e)
        err_phi += sup_dphi(e, ee) * ee + 3.3 * U * phi
        h += phi
        partial += h
    err_h = err_phi + U * partial
    t = h + 0.01
    err_t = err_h + U * t + E001
    tm = (t - err_t).clamp_min(0.005)
    lt = t.log().abs()
    ell = t ** 0.4
    kk = 0.4 * t ** -0.6
    err_l = 0.4 * tm ** -0.6 * err_t + (2 * POW_ULP * U + lt * E04) * ell
    err_k = 0.24 * tm ** -1.6 * err_t + ((2 * POW_ULP + 0.25 + 2) * U + lt * E04) * kk
    return CensusModel(h, v * ell, v * kk, v, SLACK * v * err_l, SLACK * v * err_k)


def census_e(d1, d2):
    """e = c(delta1) - c(delta2) and its bound: each delta rounded to fp32 (plus the state's error), c = delta rsqrtf(s),
    s = 0.81f + delta^2 (rounded, 2 u), rsqrtf 2 ulp, the product rounded: 6.03 u of |c|."""
    c_round = (0.5 * (2 * U + E081 / 0.81) + 2 * RSQRT_ULP * U + U)
    e1 = U * d1.abs() + 2 * E_STATE
    e2 = U * d2.abs() + 2 * E_STATE
    c1, c2 = psi(d1), psi(d2)
    ec = (dpsi((d1.abs() - e1).clamp_min(0)) * e1 + c_round * c1.abs() +
          dpsi((d2.abs() - e2).clamp_min(0)) * e2 + c_round * c2.abs())
    e = c1 - c2
    return e, ec + U * (e.abs() + ec)


def census_backward_model(g1, wh, dwx, dwy, cm, scale, scale_rel):
    """The census gradient [N,2,H,W] in fp64 (the gather identity) and its bound.  scale: the fp64 scale the restatement
    applies, scale_rel: the relative error of the float32 scale the kernel receives."""
    N, H, W = g1.shape
    p1, pw = F.pad(g1, (R, R, R, R)), F.pad(wh, (R, R, R, R))
    pk, pek = F.pad(cm.k, (R, R, R, R)), F.pad(cm.err_k, (R, R, R, R))
    G = torch.zeros_like(g1)
    err = torch.zeros_like(g1)
    partial = torch.zeros_like(g1)
    for dy, dx in offsets():
        d1, d2 = shifted(p1, dy, dx, H, W) - g1, shifted(pw, dy, dx, H, W) - wh
        e, ee = census_e(d1, d2)
        kw = cm.k + shifted(pk, dy, dx, H, W)
        ekw = cm.err_k + shifted(pek, dy, dx, H, W) + U * kw
        den = 0.1 + e * e
        A = 0.2 * e / (den * den)
        eA = sup_d2phi(e, ee) * ee + 7.8 * U * A.abs()
        B = dpsi(d2)
        eB = SUP_D2PSI * (U * d2.abs() + 2 * E_STATE) + (3 * (0.5 * (2 * U + E081 / 0.81) + 2 * RSQRT_ULP * U) + 3.1 * U) * B
        P = kw * A * B
        err += ekw * A.abs() * B + kw * eA * B + kw * A.abs() * eB + 2 * U * P.abs()
        G += P
        partial += G.abs()
    err_G = scale * (err + U * partial) + (scale_rel + U) * scale * G.abs()
    Gs = scale * G
    grad = torch.stack([Gs * dwx, Gs * dwy], 1)
    bound = torch.stack([err_G * dwx.abs() + Gs.abs() * (U * dwx.abs() + E_STATE) + U * (Gs * dwx).abs(),
                         err_G * dwy.abs() + Gs.abs() * (U * dwy.abs() + E_STATE) + U * (Gs * dwy).abs()], 1)
    return grad, SLACK * bound


# smoothness ---------------------------------------------------------------------------------------------------------------
def edge_weights(image, kappa=EDGE_CONSTANT):
    """w and its bound at the centres of the x-terms ([N,1,H,W-2], x = 1..W-2) and of the y-terms ([N,1,H-2,W]), from the
    float32 image: s = |dI_0| + |dI_1| + |dI_2| (three differences and two sums, 3 u s), s / 765 and the product by -kappa
    (u each), then expf."""
    im = image.double()
    out = []
    for diff in (im[..., 1:-1] - im[..., :-2], im[..., 1:-1, :] - im[..., :-2, :]):
        a = -kappa * diff.abs().sum(1, keepdim=True) / 765.0
        w = torch.exp(a)
        out.append((w, w * torch.expm1(5 * U * a.abs()) + 2 * EXP_ULP * U * w + TINY))
    return out


def second_diffs(flow):
    """d and its bound at the centres of the x-terms ([N,2,H,W-2]) and of the y-terms, from the float32 flow: (a - 2b) + c,
    two roundings (or one, contracted)."""
    f = flow.double()
    out = []
    for a, b, c in ((f[..., 2:], f[..., 1:-1], f[..., :-2]), (f[..., 2:, :], f[..., 1:-1, :], f[..., :-2, :])):
        d = a - 2 * b + c
        out.append((d, U * ((a - 2 * b).abs() + d.abs()) + 2.0 ** -52 * (a.abs() + 2 * b.abs() + c.abs())))
    return out


class SmoothModel(NamedTuple):
    sx: torch.Tensor           # [N] row sums of the x- and y-terms
    sy: torch.Tensor
    err_sx: torch.Tensor
    err_sy: torch.Tensor


def smoothness_forward_model(image, flow, kappa=EDGE_CONSTANT):
    """The rows' fp64 sums of the x- and y-terms and their bounds: each term sqrtf(d^2 + 1e-6f) w (the sum rounded, sqrtf
    IEEE, the product rounded), summed in fp64."""
    res = []
    for (w, ew), (d, ed) in zip(edge_weights(image, kappa), second_diffs(flow)):
        s = d * d + 1e-6
        rho = torch.sqrt(s)
        erho = ed + rho * (0.5 * (2 * U + E1M6 / s) + U)
        term = rho * w
        eterm = erho * w + rho * ew + U * term
        S = term.flatten(1).sum(1)
        res += [S, SLACK * eterm.flatten(1).sum(1) + 2.0 ** -52 * term[0].numel() * S.abs()]
    return SmoothModel(res[0], res[2], res[1], res[3])


def sup_dsign(d, err):
    """sup |d/dx (x / sqrt(x^2 + 1e-6))| = 1e-6 / (m^2 + 1e-6)^1.5 on [|d| - err, |d| + err], m the lower end."""
    m = (d.abs() - err).clamp_min(0)
    return 1e-6 / (m * m + 1e-6) ** 1.5


def smoothness_backward_model(image, flow, scale, scale_rel, kappa=EDGE_CONSTANT):
    """The smoothness gradient [N,2,H,W] in fp64 with the axes' scales (sx, sy) and its bound."""
    N, _, H, W = flow.shape
    grad = torch.zeros(N, 2, H, W, dtype=torch.float64, device=flow.device)
    bound = torch.zeros_like(grad)
    for axis, ((w, ew), (d, ed)) in enumerate(zip(edge_weights(image, kappa), second_diffs(flow))):
        s = d * d + 1e-6
        sg = d / torch.sqrt(s)
        esg = torch.clamp(sup_dsign(d, ed) * ed, max=2.0) + (0.5 * (2 * U + E1M6 / s) + 2 * RSQRT_ULP * U + U) * sg.abs()
        t = sg * w
        et = esg * w + sg.abs() * ew + U * t.abs()
        # the terms centred at pos - 1, pos, pos + 1 hold the pixel at pos with weights 1, -2, 1, in the kernel's order
        ga, ega, partial = torch.zeros_like(grad), torch.zeros_like(grad), torch.zeros_like(grad)
        for o, coef in ((-1, 1.0), (0, -2.0), (1, 1.0)):
            ga = ga + coef * term_at(t, o, axis)
            ega = ega + abs(coef) * term_at(et, o, axis)
            partial = partial + ga.abs()
        grad += scale[axis] * ga
        bound += scale[axis] * (ega + U * partial + (scale_rel + U) * ga.abs())
    bound += U * grad.abs()
    return grad, SLACK * bound


def term_at(t, o, axis):
    """t holds the terms by centre along the axis (centre c at index c - 1, c = 1..len-2); at each pixel pos, the term
    centred at pos + o, 0 where there is none."""
    N, C, H, W = t.shape
    H, W = (H, W + 2) if axis == 0 else (H + 2, W)
    out = torch.zeros(N, C, H, W, dtype=t.dtype, device=t.device)
    n = (W if axis == 0 else H) - 2
    lo, hi = max(0, 1 - o), n + 1 - o
    if axis == 0:
        out[..., lo:hi] = t[..., lo + o - 1:hi + o - 1]
    else:
        out[..., lo:hi, :] = t[..., lo + o - 1:hi + o - 1, :]
    return out


# -------------------------------------------------------------------------------------------------------------- stimuli
DX, DY = 2, 1                  # each pair's frame 2 is frame 1 translated by (DX, DY): the true flow
FRAMES = ("smooth", "quantised", "flat", "saturated", "constant", "noise")
FLOWS = ("true", "integer", "random", "edges", "leaving", "huge", "nonfinite", "piecewise")
# shapes: narrow single tiles, and a full 32x8 tile whose halo reaches into a partial right or bottom tile
SMALL_SHAPES = [(1, 8, 8), (2, 9, 8), (3, 8, 33), (5, 13, 37), (8, 47, 65)]
# the reference's training crops (Things 400x720, Sintel 368x768, KITTI 288x960) and the full Sintel and KITTI frames
LARGE_SHAPES = [(2, 400, 720), (2, 368, 768), (2, 288, 960), (1, 436, 1024), (1, 375, 1242)]


def stimulus_frames(kind, N, H, W, g):
    """Two float32 [N,3,H,W] frames in 0..255, frame 2 = frame 1 translated by (DX, DY) (crops of one canvas), except for
    "noise" (independent uniform frames)."""
    if kind == "noise":
        return torch.rand(N, 3, H, W, generator=g) * 255, torch.rand(N, 3, H, W, generator=g) * 255
    h, w = H + DY, W + DX
    smooth = F.interpolate(torch.rand(N, 3, 20, 36, generator=g), size=(h, w), mode="bicubic",
                           align_corners=False).clamp(0, 1) * 255
    if kind == "smooth":
        big = smooth
    elif kind == "quantised":
        big = smooth.round()
    elif kind == "flat":                 # 8x8 patches of one integer intensity each
        low = torch.randint(0, 256, (N, 3, (h + 7) // 8, (w + 7) // 8), generator=g).float()
        big = low.repeat_interleave(8, 2).repeat_interleave(8, 3)[..., :h, :w]
    elif kind == "saturated":            # high contrast, clipped, with 12x12 blocks of 0 and of 255
        ys, xs = torch.arange(h).view(h, 1), torch.arange(w).view(1, w)
        block = (ys // 12 + xs // 12) % 3
        big = (smooth * 1.5 - 64).clamp(0, 255)
        big = torch.where(block == 0, 0.0, torch.where(block == 1, 255.0, big))
    elif kind == "constant":
        big = torch.full((N, 3, h, w), 200.0)
    else:
        raise ValueError(kind)
    return big[:, :, DY:, DX:].contiguous(), big[:, :, :H, :W].contiguous()


def stimulus_flow(kind, N, H, W, g):
    """A float32 flow [N,2,H,W] of the family `kind`."""
    f = torch.empty(N, 2, H, W)
    f[:, 0], f[:, 1] = DX, DY
    ys, xs = torch.arange(H).view(1, H, 1).float(), torch.arange(W).view(1, 1, W).float()
    if kind == "true":
        pass
    elif kind == "integer":
        f = torch.randint(-3, 4, (N, 2, H, W), generator=g).float()
    elif kind == "random":
        f = torch.randn(N, 2, H, W, generator=g) * 4
    elif kind == "edges":                # targets at exactly W-1 or H-1, or in (-1, 0)
        pick = torch.randint(0, 5, (N, H, W), generator=g)
        frac = 0.01 + 0.98 * torch.rand(N, H, W, generator=g)        # float32 fractions: px + 1 is not exact in float32
        f[:, 0] = torch.where(pick == 0, W - 1 - xs, torch.where(pick == 1, -xs - frac, f[:, 0]))
        f[:, 1] = torch.where(pick == 2, H - 1 - ys, torch.where(pick == 3, -ys - frac, f[:, 1]))
    elif kind == "leaving":              # 16x16 blocks whose targets all leave the frame
        block = (ys // 16 + xs // 16).long() % 3
        f[:, 0] = torch.where(block == 0, f[:, 0] + 2 * W, f[:, 0])
        f[:, 1] = torch.where(block == 1, f[:, 1] - 2 * H, f[:, 1])
    elif kind == "huge":                 # +-1e12 in 8x8 blocks and scattered pixels
        block = ((ys // 8 + xs // 8).long() % 4 == 0) | (torch.rand(N, H, W, generator=g) < 0.05)
        sign = torch.where(torch.rand(N, 2, H, W, generator=g) < 0.5, -1e12, 1e12)
        f = torch.where(block[:, None], sign, f)
    elif kind == "nonfinite":            # NaN in 8x8 blocks; NaN, +inf, -inf in one channel of scattered pixels
        block = (ys // 8 + xs // 8).long() % 5 == 0
        f = torch.where(block[:, None].expand_as(f), math.nan, f)
        val = torch.tensor([math.nan, math.inf, -math.inf])[torch.randint(0, 3, (N, H, W), generator=g)]
        hit = torch.rand(N, H, W, generator=g) < 0.05
        ch = torch.randint(0, 2, (N, H, W), generator=g)
        for c in range(2):
            f[:, c] = torch.where(hit & (ch == c), val, f[:, c])
    elif kind == "piecewise":            # affine in bands of 24 columns, dyadic coefficients: second differences exactly 0
        band = (xs // 24).long().expand(N, H, W)
        nb = int(band.max()) + 1
        coef = torch.randint(-2, 3, (N, 2, 3, nb), generator=g) / 4.0
        coef[:, :, 0] *= 8
        for c in range(2):
            a, b, e = (coef[:, c, j].gather(1, band.flatten(1)).view(N, H, W) for j in range(3))
            f[:, c] = a + b * xs + e * ys
    else:
        raise ValueError(kind)
    return f


def stimulus(frames, flow, N, H, W, seed=0):
    """(image1, image2, flow): float32 CPU tensors, from a seed alone."""
    g = torch.Generator().manual_seed(seed)
    i1, i2 = stimulus_frames(frames, N, H, W, g)
    return i1, i2, stimulus_flow(flow, N, H, W, g)


def cases(shapes, rotate=False):
    """(frames, flow, N, H, W, seed) for every family pair at each shape, or with rotate, each frame family once per shape with
    the flow families taking turns (every flow family still meets several shapes)."""
    out = []
    for s, (N, H, W) in enumerate(shapes):
        for i, fr in enumerate(FRAMES):
            fls = [FLOWS[(i + s * len(FRAMES) + j) % len(FLOWS)] for j in range(2)] if rotate else FLOWS
            for fl in fls:
                out.append((fr, fl, N, H, W, 1000 * s + 10 * i + FLOWS.index(fl)))
    return out


# ---------------------------------------------------------------------------------------------- bounds of a whole case
class Bounds(NamedTuple):
    state: tuple               # g1, wh, dwx, dwy (fp64)
    cm: CensusModel
    S: torch.Tensor            # [N] fp64 row sums of v l
    err_S: torch.Tensor
    M: torch.Tensor            # [N] int64
    census_grad: torch.Tensor  # at census_scale
    census_bound: torch.Tensor
    census_scale: float
    sm: SmoothModel
    smooth_grad: torch.Tensor  # at smooth_scale
    smooth_bound: torch.Tensor
    smooth_scale: tuple


def model(i1, i2, flow, mask, census_scale, smooth_scale, census_rel=U, smooth_rel=U):
    """Every value the kernels compute for one case, in fp64, and its bound.  census_scale and smooth_scale are the fp64 scales
    of the gradients; the kernels receive them rounded to float32 (relative error census_rel, smooth_rel)."""
    N, _, H, W = flow.shape
    state = warp_state(i1, i2, flow)
    v = weights(mask, N, H, W, flow.device)
    cm = census_forward_model(state[0], state[1], v)
    gc, bc = census_backward_model(*state, cm, census_scale, census_rel)
    sm = smoothness_forward_model(i1, flow)
    gs, bs = smoothness_backward_model(i1, flow, smooth_scale, smooth_rel)
    S = cm.l.flatten(1).sum(1)
    err_S = cm.err_l.flatten(1).sum(1) + 2.0 ** -52 * H * W * S
    return Bounds(state, cm, S, err_S, v.flatten(1).sum(1).long(), gc, bc, census_scale, sm, gs, bs, smooth_scale)


def ratio(got, ref, bound):
    """max |got - ref| / bound over the elements where ref is finite (0 where got equals ref, inf where a nonzero difference
    meets a zero bound or got is NaN); where ref is not finite, got must be the same non-finite value class."""
    got, ref, bound = got.double(), ref.double().to(got.device), bound.double().to(got.device)
    fin = torch.isfinite(ref)
    if not torch.equal(torch.isfinite(got), fin) or not torch.equal(torch.isnan(got), torch.isnan(ref)):
        return math.inf
    diff = (got - ref).abs()[fin]
    r = torch.where(diff == 0, torch.zeros_like(diff), diff / bound[fin])
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------ fp32 emulations of the kernels
F081, F01, F001, F04, F02, F1M6, F765, FKAPPA = (f32(c) for c in (0.81, 0.1, 0.01, 0.4, 0.2, 1e-6, 765.0, EDGE_CONSTANT))


def fmul_add(a, b, c, fma):
    """a b + c in float32: one rounding when contracted to an fma, two otherwise."""
    return (a.double() * b.double() + c.double()).float() if fma else a * b + c


def emulate_census(g1, wh, dwx, dwy, v, scale, fma):
    """census_fwd_kernel's v l and k, then census_bwd_kernel's gradient at the float32 scale: float32, the kernels' order."""
    N, H, W = g1.shape
    p1, pw = F.pad(g1, (R, R, R, R)), F.pad(wh, (R, R, R, R))

    def e_of(dy, dx):
        d1 = (shifted(p1, dy, dx, H, W) - g1).float()
        d2 = (shifted(pw, dy, dx, H, W) - wh).float()
        r1, r2 = torch.rsqrt(fmul_add(d1, d1, F081, fma)), torch.rsqrt(fmul_add(d2, d2, F081, fma))
        return fmul_add(d1, r1, -(d2 * r2), fma), r2

    h = torch.zeros(N, H, W)
    for dy, dx in offsets():
        e, _ = e_of(dy, dx)
        e2 = e * e
        h = h + e2 / (F01 + e2)
    on = v > 0
    t = h + F001
    ell = torch.pow(t, F04)
    k = torch.where(on, (F04 * ell) / t, 0.0)
    ell = torch.where(on, ell, 0.0)
    pk = F.pad(k, (R, R, R, R))
    G = torch.zeros(N, H, W)
    for dy, dx in offsets():
        e, r2 = e_of(dy, dx)
        kw = k + shifted(pk, dy, dx, H, W)
        den = fmul_add(e, e, F01, fma)
        G = fmul_add(kw * ((F02 * e) / (den * den)), F081 * r2 * r2 * r2, G, fma)
    G = G * f32(scale)
    return ell, k, torch.stack([G * dwx.float(), G * dwy.float()], 1)


def emulate_smoothness(image, flow, scale, fma):
    """SmoothPixel's row sums (float32 terms, fp64 sums) and smoothness_bwd_kernel's gradient, in float32."""
    N, _, H, W = flow.shape
    ws = []
    for p, q in ((image[..., 1:-1], image[..., :-2]), (image[..., 1:-1, :], image[..., :-2, :])):
        s = (p[:, 0] - q[:, 0]).abs() + (p[:, 1] - q[:, 1]).abs() + (p[:, 2] - q[:, 2]).abs()
        ws.append(torch.exp(-FKAPPA * (s / F765))[:, None])
    sums, grad = [], torch.zeros(N, 2, H, W)
    for axis, (w, (a, b, c)) in enumerate(zip(ws, ((flow[..., 2:], flow[..., 1:-1], flow[..., :-2]),
                                                   (flow[..., 2:, :], flow[..., 1:-1, :], flow[..., :-2, :])))):
        d = fmul_add(f32(-2.0), b, a, fma) + c
        sums.append((torch.sqrt(fmul_add(d, d, F1M6, fma)) * w).double().flatten(1).sum(1))
        sw = d * torch.rsqrt(fmul_add(d, d, F1M6, fma))
        ga = torch.zeros(N, 2, H, W)
        for o, coef in ((-1, 1.0), (0, -2.0), (1, 1.0)):
            ga = fmul_add(f32(coef) * term_at(sw, o, axis), term_at(w.expand_as(sw), o, axis), ga, fma)
        grad = fmul_add(f32(scale[axis]), ga, grad, fma)
    return sums[0], sums[1], grad


# ----------------------------------------------------------------------------------------------------------------- tests
def smooth_scales(N, H, W):
    return (0.5 / (N * 2 * H * (W - 2)), 0.5 / (N * 2 * (H - 2) * W))


def case_mask(N, H, W, seed):
    g = torch.Generator().manual_seed(seed + 7)
    m = torch.rand(N, H, W, generator=g) < 0.8
    if N > 1:
        m[N - 1] = False
    return m


SELF_CHECK = [(2, 13, 37), (1, 47, 65)]


@pytest.mark.parametrize("fma", [False, True])
def test_fp32_emulation_lies_within_the_bounds(fma):
    """The float32 emulations of the kernels' operation order, with and without fma contraction, against the fp64 model:
    every element within its bound (the bounds are not violated by the order they claim), and the worst ratio well above 0
    (the bounds are not vacuous)."""
    worst = {}
    for fr, fl, N, H, W, seed in cases(SELF_CHECK):
        i1, i2, flow = stimulus(fr, fl, N, H, W, seed)
        mask = case_mask(N, H, W, seed)
        b = model(i1, i2, flow, mask, 1.0 / (float(mask[:, R:H - R, R:W - R].sum()) + 1e-6), smooth_scales(N, H, W))
        ell, k, gc = emulate_census(*b.state, b.cm.v, b.census_scale, fma)
        sx, sy, gs = emulate_smoothness(i1, flow, b.smooth_scale, fma)
        r = {"l": ratio(ell, b.cm.l, b.cm.err_l), "k": ratio(k, b.cm.k, b.cm.err_k),
             "census grad": ratio(gc, b.census_grad, b.census_bound),
             "smooth sums": max(ratio(sx, b.sm.sx, b.sm.err_sx), ratio(sy, b.sm.sy, b.sm.err_sy)),
             "smooth grad": ratio(gs, b.smooth_grad, b.smooth_bound)}
        for what, v in r.items():
            for key in (fr, fl, what):
                worst[key] = max(worst.get(key, 0.0), v)
    print(f"fma={fma}: worst emulation error / bound", {k: f"{v:.3g}" for k, v in worst.items()})
    assert all(v <= 1 for v in worst.values()), worst
    for what in ("l", "k", "census grad", "smooth sums", "smooth grad"):
        assert worst[what] > 1e-3, (what, worst[what])


def test_model_matches_the_host_restatement():
    """The model's fp64 values are rnc.unsupervised's: h, the census term and its autograd gradient (which checks the gather
    identity the backward kernel and the model use), the smoothness term and its gradient."""
    for fr, fl in (("smooth", "random"), ("flat", "edges"), ("noise", "nonfinite"), ("saturated", "leaving")):
        N, H, W = 2, 13, 37
        i1, i2, flow = stimulus(fr, fl, N, H, W, seed=3)
        mask = case_mask(N, H, W, 3)
        f = snapped(flow).requires_grad_()
        loss = host_census_loss(i1.double(), i2.double(), f, mask)
        loss.backward()
        M = float(weights(mask, N, H, W, "cpu").sum())
        b = model(i1, i2, flow, mask, 1.0 / (M + 1e-6), smooth_scales(N, H, W))
        h = host_census_hamming(i1.double(), i2.double(), f.detach())
        assert torch.allclose(b.cm.h, h, rtol=0, atol=1e-12)
        assert float(b.S.sum() / (M + 1e-6)) == pytest.approx(loss.item(), rel=1e-12)
        assert torch.allclose(b.census_grad, f.grad, rtol=0, atol=1e-12 * float(f.grad.abs().max()))
        if fl == "nonfinite":
            continue
        fs = flow.double().requires_grad_()
        sm = host_smoothness_loss(i1.double(), fs)
        sm.backward()
        sx, sy = smooth_scales(N, H, W)
        assert float(sx * b.sm.sx.sum() + sy * b.sm.sy.sum()) == pytest.approx(sm.item(), rel=1e-12)
        assert torch.allclose(b.smooth_grad, fs.grad, rtol=0, atol=1e-12 * float(fs.grad.abs().max()))


def test_stimuli_reach_the_regimes_they_claim():
    """Coverage: near-zero and exactly-zero deltas, pixels in partial tiles, targets in (-1, 0) and at exactly W-1 / H-1, W^ = 0
    blocks, non-finite and +-1e12 flows, and edge weights spread over (1e-6, 1]."""
    N, H, W = 2, 47, 65
    counts = dict(small_delta=0, zero_delta=0, neg_frac_x=0, last_x=0, neg_frac_y=0, last_y=0, wh0=0, nonfinite=0, huge=0,
                  flat_second_diff=0)
    wdec = torch.zeros(7, dtype=torch.long)             # edge weights by decade: (1e-6, 1e-5], ..., (0.1, 1), exactly 1
    for fr, fl, n, h, w, seed in cases([(N, H, W)]):
        i1, i2, flow = stimulus(fr, fl, n, h, w, seed)
        g1, wh, _, _ = warp_state(i1, i2, flow)
        if fr != "noise":
            for dy, dx in offsets():
                if (dy, dx) == (R, R):
                    continue
                d = shifted(F.pad(g1, (R,) * 4), dy, dx, h, w) - g1
                d = d[:, R:h - R, R:w - R]
                counts["small_delta"] += int(((d.abs() < 1) & (d != 0)).sum())
                counts["zero_delta"] += int((d == 0).sum())
        px = torch.arange(w).view(1, 1, w) + snapped(flow)[:, 0]
        py = torch.arange(h).view(1, h, 1) + snapped(flow)[:, 1]
        counts["neg_frac_x"] += int(((px > -1) & (px < 0)).sum())
        counts["neg_frac_y"] += int(((py > -1) & (py < 0)).sum())
        counts["last_x"] += int((px == w - 1).sum())
        counts["last_y"] += int((py == h - 1).sum())
        counts["wh0"] += int((wh[:, R:h - R, R:w - R] == 0).sum())
        counts["nonfinite"] += int((~torch.isfinite(flow)).sum())
        counts["huge"] += int((flow.abs() == 1e12).sum())
        counts["flat_second_diff"] += int((second_diffs(flow)[0][0] == 0).sum())
        for wt, _ in edge_weights(i1):
            idx = torch.where(wt == 1, 6, (wt.log10().floor() + 6).clamp(-1, 5).long())
            wdec += torch.bincount(idx[idx >= 0], minlength=7)
    print("coverage", counts, "edge weights per decade from 1e-6", wdec.tolist())
    assert all(v >= 100 for v in counts.values()), counts
    assert all(int(c) >= 100 for c in wdec), wdec
    # a full tile followed by a partial one along x and along y, in the shapes the GPU tests run
    shapes = SMALL_SHAPES + LARGE_SHAPES
    assert any(W > TILE_X and W % TILE_X and H > TILE_Y and H % TILE_Y for _, H, W in shapes)
    assert any(H % TILE_Y for _, H, _ in LARGE_SHAPES) and any(W % TILE_X for _, _, W in LARGE_SHAPES)
    assert sorted(N for N, _, _ in SMALL_SHAPES + LARGE_SHAPES)[-1] == 8 and min(N for N, _, _ in SMALL_SHAPES) == 1
