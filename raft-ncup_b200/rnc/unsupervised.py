"""Unsupervised losses: train the flow on video without ground-truth flow (UnFlow, Meister et al. 2018; UFlow, Jonschkowski et
al. 2020; SMURF, Stone et al. 2021, which fine-tunes RAFT this way).  DESIGN §3.16.

The losses work on N rows; row r has a source image I1 and a target image I2 ([3,H,W] in 0..255), a full-resolution flow F
([2,H,W]) and optionally a mask m in {0, 1} ([H,W]).  Images and masks are constants: no gradient reaches them.

Census term.  g(I) = 0.2989 R + 0.5870 G + 0.1140 B.  W^(x, y) is the bilinear sample of g(I2) at (x + F0, y + F1): align_corners
pixel coordinates, x0 = floor(px), taps outside the frame = 0 (the sampling of rnc_fb_consistency and bilinear_sampler); its
derivative with respect to F is that formula's, with the floor convention at integer positions.  The census of an intensity
image A at p: for each of the 49 offsets d in {-3..3}^2, c_d(p) = delta / sqrt(0.81 + delta^2), delta = A(p+d) - A(p), A = 0
outside the frame.  h(p) = sum_d e^2 / (0.1 + e^2) with e = c_d^{g(I1)}(p) - c_d^{W^}(p) (the soft Hamming distance),
l(p) = (h(p) + 0.01)^0.4, v(p) = m(p) [3 <= x <= W-4 and 3 <= y <= H-4], and

    C = sum_r S_r / (sum_r M_r + 1e-6),   S_r = sum_p v l (fp64),   M_r = sum_p v,

the sums over rows in row order.

Smoothness term (second order, edge-aware), on each flow channel k: the x-terms rho(F_k(x+1,y) - 2 F_k(x,y) + F_k(x-1,y))
exp(-kappa mean_c |I1_c(x,y) - I1_c(x-1,y)| / 255) for 1 <= x <= W-2, the y-terms the same along y, rho(d) = sqrt(d^2 + 1e-6),
kappa = 150, and Sm = (sum x-terms / (N 2 H (W-2)) + sum y-terms / (N 2 (H-2) W)) / 2.

Sequence loss over the n predictions of a bidirectional forward (2B rows; row j < B has I1 = image1[j], I2 = image2[j], row B + j
the reverse pair): L = sum_i gamma^(n-1-i) (C_i + lambda Sm_i), i = 0..n-1 (sequence_loss's weighting), the masks computed once
from the last prediction, detached: m = (occ == 0) of rnc.metrics.fb_consistency(pred[:B], pred[B:], alpha1, alpha2) for each
direction (its bit 1 masks the pixels whose target leaves the frame).  The defaults (gamma 0.85, lambda 2, alpha1 0.01, alpha2
0.5) are untuned.

`census_loss` and `smoothness_loss` are autograd Functions over csrc/photometric.cu's kernels (CUDA only; differentiable in the
flow); `host_census_loss` and `host_smoothness_loss` restate them in plain torch for any device and dtype (the fp64 test reference,
and the fp32 comparison of tools/unsupervised_bench.py).  The kernels keep 28 bytes per pixel for the census backward and sum in
a fixed order: the loss and its gradient are bit-identical from run to run, and a row's do not depend on the batch around it.
"""
import torch
import torch.nn.functional as F

from .engine import _require_cuda
from .metrics import fb_consistency
from .native import rnc

EDGE_CONSTANT = 150.0
CENSUS_RADIUS = 3
STATE_BYTES = 28                     # per pixel, rnc_census_loss_fwd's state: fp64 g(I1), W^; fp32 dW^/dpx, dW^/dpy, v dl/dh


def _check(what, flow, images, mask=None):
    """ValueError unless flow is a floating [N,2,H,W] with H, W >= 8, every image a floating [N,3,H,W] of that size that does
    not require grad, and mask None or a bool / uint8 [N,H,W]."""
    if not isinstance(flow, torch.Tensor) or flow.dim() != 4 or flow.shape[1] != 2:
        raise ValueError(f"{what}: expected flow [N,2,H,W], got {getattr(flow, 'shape', type(flow))}")
    if not flow.is_floating_point():
        raise ValueError(f"{what}: flow must be floating point, got {flow.dtype}")
    N, _, H, W = flow.shape
    if N < 1 or H < 8 or W < 8:
        raise ValueError(f"{what}: expected N >= 1 rows of at least 8x8 pixels, got flow {tuple(flow.shape)}")
    for name, im in images:
        if not isinstance(im, torch.Tensor) or tuple(im.shape) != (N, 3, H, W):
            raise ValueError(f"{what}: expected {name} [{N},3,{H},{W}], got {tuple(getattr(im, 'shape', ()))}")
        if not im.is_floating_point():
            raise ValueError(f"{what}: {name} must be floating point (0..255), got {im.dtype}")
        if im.requires_grad:
            raise ValueError(f"{what}: {name} requires grad; the images are constants of the loss (pass {name}.detach())")
    if mask is not None:
        if not isinstance(mask, torch.Tensor) or tuple(mask.shape) != (N, H, W):
            raise ValueError(f"{what}: expected mask [{N},{H},{W}], got {tuple(getattr(mask, 'shape', ()))}")
        if mask.dtype not in (torch.bool, torch.uint8):
            raise ValueError(f"{what}: mask must be bool or uint8, got {mask.dtype}")


def _census_fwd(image1, image2, flow, mask):
    """rnc_census_loss_fwd on CUDA tensors: (S [N] fp64, M [N] int64, total [2] fp64 = (sum S, sum M), state: the 28 N H W
    bytes rnc_census_loss_bwd reads)."""
    dev = _require_cuda(flow, image1, image2, mask)
    i1, i2, f = image1.detach().float(), image2.detach().float(), flow.detach().float()
    m = None if mask is None else mask.detach().to(torch.uint8).contiguous()
    N, _, H, W = f.shape
    S = torch.empty(N, dtype=torch.float64, device=dev)
    M = torch.empty(N, dtype=torch.int64, device=dev)
    total = torch.empty(2, dtype=torch.float64, device=dev)
    state = torch.empty((N * H * W * STATE_BYTES + 7) // 8, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        nbytes = rnc.census_loss_workspace_bytes(N, H, W)
        if nbytes == 0:
            raise ValueError(f"census_loss: {N} rows of {H}x{W} exceed the kernel's limits (N <= 65535, H*W < 2^30)")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        rnc.census_loss_fwd(i1, *i1.stride(), i2, *i2.stride(), f, *f.stride(), m, N, H, W, S, M, total, state, ws, nbytes)
    return S, M, total, state


class CensusLossFn(torch.autograd.Function):
    """(flow, image1, image2, mask) -> the census term C (a float32 scalar); differentiable in flow."""

    @staticmethod
    def forward(ctx, flow, image1, image2, mask):
        _, _, total, state = _census_fwd(image1, image2, flow, mask)
        ctx.save_for_backward(state, total)
        ctx.dims = tuple(flow.shape[:1] + flow.shape[2:])
        return (total[0] / (total[1] + 1e-6)).float()

    @staticmethod
    def backward(ctx, g):
        state, total = ctx.saved_tensors
        N, H, W = ctx.dims
        grad = torch.empty(N, 2, H, W, dtype=torch.float32, device=state.device)
        with torch.cuda.device(state.device):
            scale = (g.double() / (total[1] + 1e-6)).float().reshape(1)      # a device scalar: no host synchronisation
            rnc.census_loss_bwd(state, N, H, W, scale, grad)
        return grad, None, None, None


def census_loss(image1, image2, flow, mask=None):
    """The census term C of N rows (module docstring) on CUDA tensors: image1, image2 [N,3,H,W] in 0..255 (any strides,
    floating, converted to float32), flow [N,2,H,W] (any strides), mask None (all ones) or bool / uint8 [N,H,W].  Returns a
    float32 scalar, differentiable in flow only; enqueued on the current stream with no host synchronisation, forward or
    backward.  ValueError for bad shapes or dtypes and for an image that requires grad; CPU tensors raise RncUnavailable."""
    _check("census_loss", flow, (("image1", image1), ("image2", image2)), mask)
    _require_cuda(flow, image1, image2, mask)
    return CensusLossFn.apply(flow, image1, image2, mask)


def _smoothness_counts(N, H, W):
    return N * 2 * H * (W - 2), N * 2 * (H - 2) * W


class SmoothnessLossFn(torch.autograd.Function):
    """(flow, image, edge_constant) -> the smoothness term Sm (a float32 scalar); differentiable in flow."""

    @staticmethod
    def forward(ctx, flow, image, edge_constant):
        dev = _require_cuda(flow, image)
        f, im = flow.detach().float(), image.detach().float()
        N, _, H, W = f.shape
        sx = torch.empty(N, dtype=torch.float64, device=dev)
        sy = torch.empty(N, dtype=torch.float64, device=dev)
        total = torch.empty(2, dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            nbytes = rnc.smoothness_workspace_bytes(N, H, W)
            if nbytes == 0:
                raise ValueError(f"smoothness_loss: {N} rows of {H}x{W} exceed the kernel's limits (N <= 65535, H*W < 2^30)")
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            rnc.smoothness_fwd(im, *im.stride(), f, *f.stride(), N, H, W, float(edge_constant), sx, sy, total, ws, nbytes)
        cx, cy = _smoothness_counts(N, H, W)
        ctx.save_for_backward(f, im)
        ctx.edge_constant = float(edge_constant)
        return (0.5 * (total[0] / cx + total[1] / cy)).float()

    @staticmethod
    def backward(ctx, g):
        f, im = ctx.saved_tensors
        N, _, H, W = f.shape
        cx, cy = _smoothness_counts(N, H, W)
        grad = torch.empty(N, 2, H, W, dtype=torch.float32, device=f.device)
        with torch.cuda.device(f.device):
            scale = (g.double() * torch.tensor([0.5 / cx, 0.5 / cy], dtype=torch.float64, device=f.device)).float()
            rnc.smoothness_bwd(im, *im.stride(), f, *f.stride(), N, H, W, ctx.edge_constant, scale, grad)
        return grad, None, None


def smoothness_loss(image, flow, edge_constant=EDGE_CONSTANT):
    """The smoothness term Sm of N rows (module docstring) on CUDA tensors: image [N,3,H,W] in 0..255 (I1 of each row; any
    strides), flow [N,2,H,W].  Returns a float32 scalar, differentiable in flow only, with no host synchronisation.  Errors as
    census_loss."""
    _check("smoothness_loss", flow, (("image", image),))
    _require_cuda(flow, image)
    return SmoothnessLossFn.apply(flow, image, edge_constant)


# ------------------------------------------------------------------------------------------------ host restatements


def _gray(im):
    return 0.2989 * im[:, 0] + 0.5870 * im[:, 1] + 0.1140 * im[:, 2]


def _warp(img, flow):
    """img [N,H,W] sampled bilinearly at (x + flow0, y + flow1): taps outside the frame 0, x0 = floor(px) (so the derivative
    at an integer position is the right one), written out tap by tap."""
    N, H, W = img.shape
    xs = torch.arange(W, dtype=flow.dtype, device=flow.device).view(1, 1, W)
    ys = torch.arange(H, dtype=flow.dtype, device=flow.device).view(1, H, 1)
    px, py = xs + flow[:, 0], ys + flow[:, 1]
    x0, y0 = torch.floor(px.detach()), torch.floor(py.detach())
    ax, ay = px - x0, py - y0
    n = torch.arange(N, device=flow.device).view(N, 1, 1)

    def tap(tx, ty):
        inside = (tx >= 0) & (tx <= W - 1) & (ty >= 0) & (ty <= H - 1)
        v = img[n, ty.clamp(0, H - 1).long(), tx.clamp(0, W - 1).long()]
        return torch.where(inside, v, torch.zeros_like(v))

    return ((1 - ay) * ((1 - ax) * tap(x0, y0) + ax * tap(x0 + 1, y0)) +
            ay * ((1 - ax) * tap(x0, y0 + 1) + ax * tap(x0 + 1, y0 + 1)))


def _census(a):
    """[N,H,W] -> [N,49,H,W]: c_d for the offsets d = (dx, dy), dy-major, each in -3..3; 0 outside the frame."""
    H, W = a.shape[-2:]
    r = CENSUS_RADIUS
    p = F.pad(a, (r, r, r, r))
    d = torch.stack([p[:, dy:dy + H, dx:dx + W] for dy in range(2 * r + 1) for dx in range(2 * r + 1)], 1) - a[:, None]
    return d / torch.sqrt(0.81 + d * d)


def host_census_hamming(image1, image2, flow):
    """h [N,H,W] of every pixel (the soft Hamming distance of the module docstring), in flow's dtype and on its device."""
    g1 = _gray(image1.detach().to(flow.dtype))
    w = _warp(_gray(image2.detach().to(flow.dtype)), flow)
    e = _census(g1) - _census(w)
    return (e * e / (0.1 + e * e)).sum(1)


def host_census_loss(image1, image2, flow, mask=None):
    """census_loss in plain torch, on flow's device and in its dtype, differentiable in flow by autograd.  Per-row sums, then
    the rows in row order."""
    _check("host_census_loss", flow, (("image1", image1), ("image2", image2)), mask)
    N, _, H, W = flow.shape
    r = CENSUS_RADIUS
    v = torch.zeros(N, H, W, dtype=flow.dtype, device=flow.device)
    v[:, r:H - r, r:W - r] = 1
    if mask is not None:
        v = v * (mask.to(flow.device) != 0).to(flow.dtype)
    ell = (host_census_hamming(image1, image2, flow) + 0.01) ** 0.4
    S, M = (v * ell).flatten(1).sum(1), v.flatten(1).sum(1)
    total, count = S[0], M[0]
    for i in range(1, N):
        total, count = total + S[i], count + M[i]
    return total / (count + 1e-6)


def host_smoothness_loss(image, flow, edge_constant=EDGE_CONSTANT):
    """smoothness_loss in plain torch, on flow's device and in its dtype, differentiable in flow by autograd."""
    _check("host_smoothness_loss", flow, (("image", image),))
    N, _, H, W = flow.shape
    im = image.detach().to(flow.dtype)
    wx = torch.exp(-edge_constant * (im[..., 1:] - im[..., :-1]).abs().mean(1) / 255)[..., :W - 2]     # at x = 1..W-2
    wy = torch.exp(-edge_constant * (im[..., 1:, :] - im[..., :-1, :]).abs().mean(1) / 255)[..., :H - 2, :]
    dx = flow[..., 2:] - 2 * flow[..., 1:-1] + flow[..., :-2]
    dy = flow[..., 2:, :] - 2 * flow[..., 1:-1, :] + flow[..., :-2, :]
    tx = (torch.sqrt(dx * dx + 1e-6) * wx[:, None]).sum()
    ty = (torch.sqrt(dy * dy + 1e-6) * wy[:, None]).sum()
    cx, cy = _smoothness_counts(N, H, W)
    return 0.5 * (tx / cx + ty / cy)


# ------------------------------------------------------------------------------------------------ sequence loss


def _sequence_loss(census, smooth, flow_preds, image1, image2, gamma, smooth_weight, alpha1, alpha2):
    if len(flow_preds) == 0:
        raise ValueError("unsupervised_loss: expected at least one prediction")
    if image1.dim() != 4 or image1.shape != image2.shape:
        raise ValueError(f"unsupervised_loss: expected two [B,3,H,W] images of one shape, got {tuple(image1.shape)} and "
                         f"{tuple(image2.shape)}")
    B, _, H, W = image1.shape
    for p in flow_preds:
        if tuple(p.shape) != (2 * B, 2, H, W):
            raise ValueError(f"unsupervised_loss: expected predictions [2B,2,H,W] = {[2 * B, 2, H, W]} (forward(..., "
                             f"bidirectional=True)), got {tuple(p.shape)}")
    last = flow_preds[-1].detach()
    occ_fw, occ_bw, _, _ = fb_consistency(last[:B], last[B:], alpha1, alpha2)
    mask = torch.cat([occ_fw, occ_bw]) == 0
    src, tgt = torch.cat([image1, image2]).detach(), torch.cat([image2, image1]).detach()
    n = len(flow_preds)
    loss = 0.0
    for i, pred in enumerate(flow_preds):
        c, s = census(src, tgt, pred, mask), smooth(src, pred)
        loss = loss + gamma ** (n - i - 1) * (c + smooth_weight * s)
    vals = torch.stack([c.detach().double(), s.detach().double(), (occ_fw != 0).double().mean(),
                        (occ_bw != 0).double().mean()]).tolist()
    return loss, dict(zip(("census", "smoothness", "occluded_fw", "occluded_bw"), vals))


def unsupervised_loss(flow_preds, image1, image2, gamma=0.85, smooth_weight=2.0, alpha1=0.01, alpha2=0.5):
    """The sequence loss of the module docstring over flow_preds, a list of [2B,2,H,W] predictions of
    model(image1, image2, bidirectional=True) (row j: image1[j] -> image2[j], row B + j the reverse), on census_loss and
    smoothness_loss.  image1, image2: [B,3,H,W] in 0..255.  Returns (loss, metrics) like rnc.train.sequence_loss: metrics
    holds the last prediction's census and smoothness terms and the occluded fractions of each direction (occluded_fw,
    occluded_bw)."""
    return _sequence_loss(census_loss, smoothness_loss, flow_preds, image1, image2, gamma, smooth_weight, alpha1, alpha2)


def host_unsupervised_loss(flow_preds, image1, image2, gamma=0.85, smooth_weight=2.0, alpha1=0.01, alpha2=0.5):
    """unsupervised_loss on host_census_loss and host_smoothness_loss (the same masks), on any device and dtype."""
    return _sequence_loss(host_census_loss, host_smoothness_loss, flow_preds, image1, image2, gamma, smooth_weight, alpha1,
                          alpha2)
