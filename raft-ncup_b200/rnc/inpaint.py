"""Flow-guided video inpainting: fill masked regions of a video along the completed bidirectional flows, and score the result
by PSNR and SSIM.

This is the propagation core of DFVI (Xu et al., "Deep Flow-Guided Video Inpainting", CVPR 2019) and FGVC (Gao et al.,
"Flow-edge Guided Video Completion", ECCV 2020), with the flow completion done by a harmonic (Laplace) fill instead of a
learned or edge-guided one.  Inputs, per video v of V: T >= 2 frames I_t, float32 [3,H,W] in 0..255; hole masks M_t, uint8
[H,W], non-zero where a pixel is to be filled; the forward flows F_k (frame k -> k+1) and backward flows G_k (frame k+1 -> k),
float32 [2,H,W], for k = 0..T-2 (rnc.harness.run_sequences_bidirectional's flow_up and flow_up_bw, stacked to [V,T-1,...]).
Every floating-point operation is rounded once in float32, with no FMA, so the host restatements (host_harmonic_fill,
host_inpaint_propagate, host_inpaint) and the kernels (csrc/inpaint.cu) give the same bits.

1. Harmonic fill (`harmonic_fill`, for flows and colours alike): values [N,C,H,W], unknown uint8 [N,H,W], sweeps.  A pixel is
   known when unknown is 0 there and all C of its values are finite; a known pixel is copied through unchanged.  Each other
   pixel starts from the values of its nearest known pixel (rnc.metrics.nearest_site: exact squared distance, ties to the
   smallest column, then the smallest row), or 0 in an image without a known pixel.  Then `sweeps` red-black SOR sweeps run
   over the unknown pixels, red ((x + y) even) before black: per pixel and channel s = the sum of its in-frame 4-neighbours,
   added in the order up, left, right, down (starting from -0.0, so the first neighbour enters exactly), avg = s / n with n
   the number of in-frame neighbours, and u <- u + omega (avg - u).  omega = 2 / (1 + pi_f32 / (L + 1)) per image, L the
   larger side of the bounding box of its unknown pixels, in float32 arithmetic: the optimal SOR factor of a square of side
   L + 1 with sin(pi / (L + 1)) ~ pi / (L + 1), bit-exact on host and device without a sin.  A pixel without an in-frame
   neighbour (a 1x1 image) keeps its start.  The values the input holds at unknown pixels are never read.
2. Flow completion: F~_k = harmonic_fill(F_k, M_k), G~_k = harmonic_fill(G_k, M_{k+1}); occ~_k, occ~_bw_k =
   rnc.metrics.fb_consistency(F~, G~, alpha1, alpha2).
3. Temporal propagation (`inpaint_propagate`): each hole pixel p of frame t runs one chain per direction.  Forward, from x = p
   at frame k = t and distance d = 0: the chain stops without a candidate when k = T-1, d = max_distance or
   occ~_k(rint(x)) != 0 (round half to even); otherwise u = F~_k^(x) (rnc.interp's clamped bilinear sample) and x' = x + u,
   and the chain stops without a candidate when x' leaves [0, W-1] x [0, H-1]; otherwise k, d, x <- k + 1, d + 1, x'.  When
   M_k(rint(x)) = 0 the chain ends with a candidate: the bilinear taps of I_k at x whose mask is 0 (the tap at rint(x) is
   one, of weight >= 0.25), c = (sum w_i I_i) / (sum w_i), weights and weighted colours each added in tap order, so no hole
   colour is read; its distance is d.  Backward likewise with G~_{k-1} and occ~_bw_{k-1}, from frame k to k-1.  With both
   candidates c = (d_b c_f + d_f c_b) / (d_f + d_b), the nearer frame weighing more; with one, its colour.  The source map,
   uint8 [T,H,W], says which: SOURCE_KNOWN (0, not a hole), SOURCE_FORWARD (1), SOURCE_BACKWARD (2), SOURCE_BOTH (3),
   SOURCE_SPATIAL (4, no candidate; the colour is written as 0 here).
4. Spatial fill: harmonic_fill of the three colour channels with the SOURCE_SPATIAL pixels as the unknown set.
Pixels outside the holes are the input's bits; only the masks and the known pixels determine the output.

Scoring (`validate_inpainting` in rnc.harness): only frames with a hole pixel are scored.  PSNR per frame from
rnc.interp.interpolation_error's fp64 squared-error sum, MSE over pixels and channels, data range 255, 100 dB for a frame
without error.  SSIM per frame (Wang, Bovik, Sheikh and Simoncelli, "Image Quality Assessment: From Error Visibility to
Structural Similarity", IEEE TIP 2004): an 11-tap Gaussian of sigma 1.5 (normalised in fp64, float32 taps) applied
separably, rows then columns, taps in order; C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2; the mean of the map over the pixels
whose 11x11 window lies inside the frame and over the 3 channels.  Each metric is averaged over a video's scored frames,
then over videos (`summarize_inpainting`).
"""
import math

import numpy as np
import torch

from . import native
from .metrics import fb_consistency, nearest_site
from .restate import PI_F32, bilinear_taps, check_sides, f32, inside, sample

DEFAULT_SWEEPS = 512
SOURCE_KNOWN, SOURCE_FORWARD, SOURCE_BACKWARD, SOURCE_BOTH, SOURCE_SPATIAL = (
    native.INPAINT_KNOWN, native.INPAINT_FORWARD, native.INPAINT_BACKWARD, native.INPAINT_BOTH, native.INPAINT_SPATIAL)
SSIM_RADIUS = 5
_g = np.exp(-(np.arange(-SSIM_RADIUS, SSIM_RADIUS + 1, dtype=np.float64) ** 2) / (2 * 1.5 ** 2))
SSIM_TAPS = (_g / _g.sum()).astype(np.float32)          # csrc/inpaint.cu's kGauss
SSIM_C1, SSIM_C2 = float(np.float32((0.01 * 255) ** 2)), float(np.float32((0.03 * 255) ** 2))
PSNR_CAP = 100.0
_FILL_WORKSPACE_CAP = 1 << 30               # harmonic_fill runs as many images per call as fit in this


def omega(L):
    """The SOR factor of an image whose unknown pixels' bounding box has the larger side L: 2 / (1 + pi_f32 / (L + 1)), each
    operation rounded once to float32."""
    t = torch.tensor(float(L + 1), dtype=torch.float64)
    return float(f32(2.0 / f32(1.0 + f32(PI_F32 / t))))


def _check_sweeps(sweeps, what):
    if not isinstance(sweeps, int) or sweeps < 0:
        raise ValueError(f"{what}: expected sweeps >= 0, got {sweeps!r}")


def _check_fill(values, unknown, sweeps):
    if values.dim() not in (4, 5):
        raise ValueError(f"harmonic_fill: expected values [N,C,H,W] or [V,T,C,H,W], got {tuple(values.shape)}")
    lead, (C, H, W) = tuple(values.shape[:-3]), tuple(values.shape[-3:])
    if tuple(unknown.shape) != (*lead, H, W):
        raise ValueError(f"harmonic_fill: expected unknown {[*lead, H, W]}, got {tuple(unknown.shape)}")
    if values.device != unknown.device:
        raise ValueError(f"harmonic_fill: values and unknown must be on one device, got {values.device} and {unknown.device}")
    if not 1 <= C <= native.HARMONIC_MAX_CHANNELS:
        raise ValueError(f"harmonic_fill: expected 1 to {native.HARMONIC_MAX_CHANNELS} channels, got {C}")
    check_sides(H, W, "harmonic_fill")
    _check_sweeps(sweeps, "harmonic_fill")


def harmonic_fill(values, unknown, sweeps=DEFAULT_SWEEPS, out=None):
    """Step 1 of the rule: values [N,C,H,W] or [V,T,C,H,W] (any strides; float32, or converted to it), unknown [N,H,W] or
    [V,T,H,W] (non-zero where a pixel is to be filled), 1 <= C <= 4.  Returns float32 of values' shape: `out` when given (it
    may be values itself, for a fill in place), else a new tensor.  CUDA tensors go through rnc_harmonic_fill (enqueued on the
    current stream, no host synchronisation; as many images per call as a 1 GiB workspace holds), CPU tensors through
    host_harmonic_fill; they give the same bits.  ValueError before any launch for mismatched shapes, mixed devices, a
    channel count outside 1..4, a side above 4096 or sweeps < 0."""
    _check_fill(values, unknown, sweeps)
    if out is not None and tuple(out.shape) != tuple(values.shape):
        raise ValueError(f"harmonic_fill: expected out {list(values.shape)}, got {tuple(out.shape)}")
    if not values.is_cuda:
        res = host_harmonic_fill(values, unknown, sweeps)
        return res if out is None else out.copy_(res)
    v = values.detach().float()
    if out is None:
        out = torch.empty(values.shape, dtype=torch.float32, device=values.device)
    if out.dtype != torch.float32:
        raise ValueError(f"harmonic_fill: expected a float32 out, got {out.dtype}")
    u = unknown.detach().to(torch.uint8)
    five = v.dim() == 5
    if not five:                                        # [N,...] as [N,1,...]
        v, u, o = v[:, None], u[:, None], out[:, None]
    else:
        o = out
    A, B, C, H, W = v.shape
    if A == 0 or B == 0:
        return out
    per = max(1, min(A, 65535 // B, _FILL_WORKSPACE_CAP // max(1, 5 * B * H * W)))
    with torch.cuda.device(v.device):
        ws = torch.empty(native.rnc.harmonic_fill_workspace_bytes(min(per, A), B, C, H, W), dtype=torch.uint8,
                         device=v.device)
        for lo in range(0, A, per):
            n = min(per, A - lo)
            vc, uc, oc = v[lo:lo + n], u[lo:lo + n], o[lo:lo + n]
            native.rnc.harmonic_fill(vc, *vc.stride(), uc, *uc.stride(), n, B, C, H, W, sweeps, oc, *oc.stride(), ws,
                                     ws.numel())
    return out


def _neighbour_sum(u):
    """Per pixel of u (fp64 [C,H,W] holding float32 values): the in-frame 4-neighbours added up, left, right, down from
    -0.0, each addition rounded once, and their count [H,W]."""
    C, H, W = u.shape
    s = torch.full_like(u, -0.0)
    n = torch.zeros(H, W, dtype=torch.float64)
    for dy, dx in ((-1, 0), (0, -1), (0, 1), (1, 0)):
        nb = torch.zeros_like(u)
        has = torch.zeros(H, W, dtype=torch.bool)
        ys, yd = (slice(0, H + dy), slice(-dy, H)) if dy < 0 else (slice(dy, H), slice(0, H - dy))
        xs, xd = (slice(0, W + dx), slice(-dx, W)) if dx < 0 else (slice(dx, W), slice(0, W - dx))
        nb[:, yd, xd] = u[:, ys, xs]
        has[yd, xd] = True
        s = torch.where(has, f32(s + nb), s)
        n = n + has
    return s, n


def _host_fill_image(v, unk, sweeps):
    """One image of the rule: v fp64 [C,H,W] holding float32 values, unk bool [H,W].  Returns fp64 [C,H,W]."""
    C, H, W = v.shape
    known = ~unk & torch.isfinite(v).all(0)
    site = torch.from_numpy(nearest_site(known.numpy()[None])[0])
    near = v.reshape(C, -1)[:, site.clamp(min=0).reshape(-1)].view(C, H, W)
    u = torch.where(known, v, torch.where(site >= 0, near, 0.0))
    todo = ~known
    if sweeps == 0 or not todo.any():
        return u
    ys, xs = torch.nonzero(todo, as_tuple=True)
    w = omega(max(int(xs.max() - xs.min()) + 1, int(ys.max() - ys.min()) + 1))
    parity = (torch.arange(H).view(H, 1) + torch.arange(W).view(1, W)) % 2
    _, n = _neighbour_sum(u)
    todo = todo & (n > 0)
    colours = (todo & (parity == 0), todo & (parity == 1))
    for _ in range(sweeps):
        for m in colours:
            s, _ = _neighbour_sum(u)
            u = torch.where(m, f32(u + f32(w * f32(f32(s / n.clamp(min=1)) - u))), u)
    return u


def host_harmonic_fill(values, unknown, sweeps=DEFAULT_SWEEPS):
    """harmonic_fill's rule in torch, one image at a time and all its pixels at once (a colour's pixels only read the other
    colour, so updating them together is the sequential sweep): each floating-point operation evaluated in fp64 on float32
    operands and rounded once to float32, the start by rnc.metrics.nearest_site.  Serves CPU tensors and is the kernel's
    test reference.  Returns float32 of values' shape on the CPU."""
    _check_fill(values, unknown, sweeps)
    C, H, W = values.shape[-3:]
    v = values.detach().cpu().float().double().reshape(-1, C, H, W)
    u = unknown.detach().cpu().reshape(-1, H, W) != 0
    out = torch.empty(v.shape, dtype=torch.float32)
    for i in range(v.shape[0]):
        out[i] = _host_fill_image(v[i], u[i], sweeps).float()
    return out.view(values.shape)


# ------------------------------------------------------------------------------------------------------- propagation


def _max_distance(max_distance, what, T=2):
    """max_distance, or max(T - 1, 1) for None (so only a caller that uses the value needs T); else ValueError unless >= 1."""
    if max_distance is None:
        return max(T - 1, 1)
    if not isinstance(max_distance, int) or max_distance < 1:
        raise ValueError(f"{what}: expected max_distance >= 1 or None, got {max_distance!r}")
    return max_distance


def _check_video(frames, masks, flow, flow_bw, what):
    """(V, T, H, W) of a stacked video; ValueError for mismatched shapes, T < 2, mixed devices or a side above 4096."""
    if frames.dim() != 5 or frames.shape[2] != 3:
        raise ValueError(f"{what}: expected frames [V,T,3,H,W], got {tuple(frames.shape)}")
    V, T, _, H, W = frames.shape
    if V == 0:
        raise ValueError(f"{what}: expected at least one video, got {tuple(frames.shape)}")
    if T < 2:
        raise ValueError(f"{what}: a video needs T >= 2 frames, got {T}")
    if tuple(masks.shape) != (V, T, H, W):
        raise ValueError(f"{what}: expected masks {[V, T, H, W]}, got {tuple(masks.shape)}")
    for name, t in (("flow", flow), ("flow_bw", flow_bw)):
        if tuple(t.shape) != (V, T - 1, 2, H, W):
            raise ValueError(f"{what}: expected {name} {[V, T - 1, 2, H, W]}, got {tuple(t.shape)}")
    check_sides(H, W, what)
    return V, T, H, W


def _check_propagate(frames, masks, flow, flow_bw, occ, occ_bw):
    V, T, H, W = _check_video(frames, masks, flow, flow_bw, "inpaint_propagate")
    for name, t in (("occ", occ), ("occ_bw", occ_bw)):
        if tuple(t.shape) != (V, T - 1, H, W):
            raise ValueError(f"inpaint_propagate: expected {name} {[V, T - 1, H, W]}, got {tuple(t.shape)}")
    devs = {t.device for t in (frames, masks, flow, flow_bw, occ, occ_bw)}
    if len(devs) != 1:
        raise ValueError(f"inpaint_propagate: the frames, masks, flows and occlusion masks must be on one device, got "
                         f"{sorted(map(str, devs))}")
    return V, T, H, W


def inpaint_propagate(frames, masks, flow, flow_bw, occ, occ_bw, max_distance=None):
    """Step 3 of the rule for V videos: frames [V,T,3,H,W], masks [V,T,H,W] (holes where non-zero), the completed flows
    flow, flow_bw [V,T-1,2,H,W] and their masks occ, occ_bw [V,T-1,H,W] (occluded where non-zero), any strides; max_distance
    the longest chain in frames (None: T - 1).  Returns (frames float32 [V,T,3,H,W], source uint8 [V,T,H,W]); a
    SOURCE_SPATIAL pixel's colour is 0, for step 4 to fill.  CUDA tensors go through rnc_inpaint_propagate (one launch on the
    current stream; the inputs are read through their strides, not copied), CPU tensors through host_inpaint_propagate; they
    give the same bits.  ValueError before any launch for mismatched shapes, mixed devices, T < 2, a side above 4096 or
    max_distance < 1."""
    V, T, H, W = _check_propagate(frames, masks, flow, flow_bw, occ, occ_bw)
    maxd = _max_distance(max_distance, "inpaint_propagate", T)
    if not frames.is_cuda:
        return host_inpaint_propagate(frames, masks, flow, flow_bw, occ, occ_bw, max_distance)
    dev = frames.device
    im, fw, bw = (t.detach().float() for t in (frames, flow, flow_bw))
    m, o, ob = (t.detach().to(torch.uint8) for t in (masks, occ, occ_bw))
    out = torch.empty(V, T, 3, H, W, dtype=torch.float32, device=dev)
    source = torch.empty(V, T, H, W, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        native.rnc.inpaint_propagate(im, *im.stride(), m, *m.stride(), fw, *fw.stride(), bw, *bw.stride(), o, *o.stride(), ob,
                                     *ob.stride(), V, T, H, W, maxd, out, source)
    return out, source


def _host_chain(I, M, f, o, t, x, y, maxd, forward):
    """One direction of the chains of a video's hole pixels: I fp64 [T,3,H,W], M bool [T,H,W] (hole), f fp64 [T-1,2,H,W],
    o bool [T-1,H,W], start frames t [n] and positions x, y [n] (fp64).  Returns (found bool [n], colour fp64 [3,n],
    distance long [n])."""
    T, _, H, W = I.shape
    n = t.shape[0]
    k, d = t.clone(), torch.zeros(n, dtype=torch.long)
    live = torch.ones(n, dtype=torch.bool)
    found = torch.zeros(n, dtype=torch.bool)
    step = 1 if forward else -1
    for _ in range(T - 1):
        live &= ~((k == (T - 1 if forward else 0)) | (d == maxd))
        if not live.any():
            break
        pair = (k if forward else k - 1).clamp(0, T - 2)
        ix, iy = torch.round(x).long(), torch.round(y).long()
        live &= ~o[pair, iy, ix]
        u = sample(f, x, y, pair)
        nx, ny = f32(x + u[0]), f32(y + u[1])
        live &= inside(nx, ny, H, W)
        x, y = torch.where(live, nx, x), torch.where(live, ny, y)
        k, d = torch.where(live, k + step, k), torch.where(live, d + 1, d)
        hit = live & ~M[k, torch.round(y).long(), torch.round(x).long()]
        found |= hit
        live &= ~hit
    # the masked bilinear colour at each candidate's end (every element computes one; only found ones are kept)
    ws = torch.full((n,), -0.0, dtype=torch.float64)
    s = torch.full((3, n), -0.0, dtype=torch.float64)
    for ty, tx, w in bilinear_taps(x, y, H, W):
        ok = ~M[k, ty, tx]
        ws = torch.where(ok, f32(ws + w), ws)
        s = torch.where(ok, f32(s + f32(w * I[k, :, ty, tx].T)), s)
    return found, f32(s / ws), d



def host_inpaint_propagate(frames, masks, flow, flow_bw, occ, occ_bw, max_distance=None):
    """inpaint_propagate's rule in torch, one video at a time and all its hole pixels at once: each floating-point operation
    evaluated in fp64 on float32 operands and rounded once to float32, in the kernel's order.  Serves CPU tensors and is the
    kernel's test reference.  Returns (frames float32 [V,T,3,H,W], source uint8 [V,T,H,W]) on the CPU."""
    V, T, H, W = _check_propagate(frames, masks, flow, flow_bw, occ, occ_bw)
    maxd = _max_distance(max_distance, "inpaint_propagate", T)
    out = torch.empty(V, T, 3, H, W, dtype=torch.float32)
    source = torch.zeros(V, T, H, W, dtype=torch.uint8)
    for v in range(V):
        I = frames[v].detach().cpu().float().double()
        M = masks[v].detach().cpu() != 0
        t, y, x = torch.nonzero(M, as_tuple=True)
        xf, yf = x.double(), y.double()
        fw = _host_chain(I, M, flow[v].detach().cpu().float().double(), occ[v].detach().cpu() != 0, t, xf, yf, maxd, True)
        bw = _host_chain(I, M, flow_bw[v].detach().cpu().float().double(), occ_bw[v].detach().cpu() != 0, t, xf, yf, maxd,
                         False)
        (hf, cf, df), (hb, cb, db) = fw, bw
        both = f32(f32(f32(db.double() * cf) + f32(df.double() * cb)) / (df + db).double().clamp(min=1))
        c = torch.where(hf & hb, both, torch.where(hf, cf, torch.where(hb, cb, 0.0)))
        o = torch.where(M[:, None], 0.0, I)
        o[t, :, y, x] = c.T
        out[v] = o.float()
        src = torch.full_like(t, SOURCE_SPATIAL)
        src = torch.where(hf & hb, SOURCE_BOTH, torch.where(hf, SOURCE_FORWARD, torch.where(hb, SOURCE_BACKWARD, src)))
        source[v, t, y, x] = src.to(torch.uint8)
    return out, source


# ------------------------------------------------------------------------------------------------------- all four steps


def _check_inpaint(frames, masks, flow, flow_bw, sweeps, max_distance):
    V, T, H, W = _check_video(frames, masks, flow, flow_bw, "inpaint")
    devs = {t.device for t in (frames, masks, flow, flow_bw)}
    if len(devs) != 1:
        raise ValueError(f"inpaint: the frames, masks and flows must be on one device, got {sorted(map(str, devs))}")
    _check_sweeps(sweeps, "inpaint")
    _max_distance(max_distance, "inpaint", T)
    return V, T, H, W


def _complete(flow, flow_bw, hole, sweeps):
    """Step 2's completion in place: forward flows under their pair's first frame's holes, backward under the second's."""
    harmonic_fill(flow, hole[:, :-1], sweeps, out=flow)
    harmonic_fill(flow_bw, hole[:, 1:], sweeps, out=flow_bw)


def _propagate(frames, hole, flow, flow_bw, sweeps, max_distance, alpha1, alpha2, lengths=None):
    """Step 2's consistency check and steps 3-4 on the completed flows, on the tensors' device.  With lengths, video v's
    pairs from lengths[v] - 1 on are padding: occluded in both directions, so no chain enters them."""
    V, T1, _, H, W = flow.shape
    occ, occ_bw, _, _ = fb_consistency(flow.reshape(V * T1, 2, H, W), flow_bw.reshape(V * T1, 2, H, W), alpha1, alpha2)
    occ, occ_bw = occ.reshape(V, T1, H, W), occ_bw.reshape(V, T1, H, W)
    for v, n in enumerate(lengths or ()):
        occ[v, n - 1:] = 1
        occ_bw[v, n - 1:] = 1
    out, source = inpaint_propagate(frames, hole, flow, flow_bw, occ, occ_bw, max_distance)
    harmonic_fill(out, source == SOURCE_SPATIAL, sweeps, out=out)
    return out, source


def _run(frames, masks, flow, flow_bw, sweeps, max_distance, alpha1, alpha2, lengths=None):
    """Steps 2-4 with the flows (float32) completed in place, on the tensors' device; lengths as _propagate's."""
    m = masks.detach().to(torch.uint8)
    _complete(flow, flow_bw, m, sweeps)
    return _propagate(frames, m, flow, flow_bw, sweeps, max_distance, alpha1, alpha2, lengths)


def inpaint(frames, masks, flow, flow_bw, sweeps=DEFAULT_SWEEPS, max_distance=None, alpha1=0.01, alpha2=0.5):
    """Steps 2-4 of the rule for V videos: frames [V,T,3,H,W] (0..255), masks [V,T,H,W] (holes where non-zero), flow,
    flow_bw [V,T-1,2,H,W] (run_sequences_bidirectional's flow_up and flow_up_bw, stacked), any strides; the inputs are not
    modified.  Returns (frames float32 [V,T,3,H,W], source uint8 [V,T,H,W]).  CUDA tensors run on the kernels, CPU tensors
    through the host restatements (host_inpaint); they give the same bits.  ValueError before any launch for mismatched
    shapes, mixed devices, T < 2, a side above 4096, sweeps < 0 or max_distance < 1."""
    _check_inpaint(frames, masks, flow, flow_bw, sweeps, max_distance)
    fw, bw = (f.detach().float().clone() for f in (flow, flow_bw))
    return _run(frames, masks, fw, bw, sweeps, max_distance, alpha1, alpha2)


def host_inpaint(frames, masks, flow, flow_bw, sweeps=DEFAULT_SWEEPS, max_distance=None, alpha1=0.01, alpha2=0.5):
    """inpaint on CPU copies of the inputs, so through host_harmonic_fill, rnc.metrics.host_fb_consistency and
    host_inpaint_propagate.  Returns CPU tensors."""
    _check_inpaint(frames, masks, flow, flow_bw, sweeps, max_distance)
    fw, bw = (f.detach().cpu().float().clone() for f in (flow, flow_bw))
    return _run(frames.cpu(), masks.cpu(), fw, bw, sweeps, max_distance, alpha1, alpha2)


# ------------------------------------------------------------------------------------------------------- scoring


def _check_ssim(pred, gt):
    if pred.dim() != 4 or pred.shape[1] != 3 or tuple(gt.shape) != tuple(pred.shape):
        raise ValueError(f"ssim: expected pred and gt of one [N,3,H,W] shape, got {tuple(pred.shape)} and {tuple(gt.shape)}")
    if pred.device != gt.device:
        raise ValueError(f"ssim: pred and gt must be on one device, got {pred.device} and {gt.device}")
    N, _, H, W = pred.shape
    side = 2 * SSIM_RADIUS + 1
    if N == 0 or H < side or W < side:
        raise ValueError(f"ssim: expected at least one frame of at least {side}x{side}, got {tuple(pred.shape)}")
    return N, H, W


def ssim(pred, gt):
    """SSIM's per-frame partials of pred against gt ([N,3,H,W], 0..255, any strides; float32 or converted to it): (sum fp64
    [N], the SSIM map summed over the 3 channels and the pixels whose 11x11 window lies inside the frame; count int64 [N],
    its number of terms) on the tensors' device.  A frame's SSIM is sum / count.  CUDA tensors go through rnc_ssim_partials
    (on the current stream; a frame's sum does not depend on N, its position or the GPU), CPU tensors through host_ssim;
    the maps are the same bits and the sums agree to their last bits.  ValueError for mismatched shapes, mixed devices or a
    frame smaller than 11x11."""
    N, H, W = _check_ssim(pred, gt)
    if not pred.is_cuda:
        return host_ssim(pred, gt)
    p, g = pred.detach().float(), gt.detach().float()
    dev = p.device
    s = torch.empty(N, dtype=torch.float64, device=dev)
    count = torch.empty(N, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        nbytes = native.rnc.ssim_partials_workspace_bytes(N, H, W)
        if nbytes == 0:
            raise ValueError(f"ssim: {N} frames of {H}x{W} exceed the kernel's limits (N <= 65535, H*W < 2^30)")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        native.rnc.ssim_partials(p, *p.stride(), g, *g.stride(), N, H, W, s, count, ws, ws.numel())
    return s, count


def _separable(q):
    """The Gaussian of q (fp64 [..., H, W] holding float32 values) over the windows inside the frame, rows then columns, taps
    in order, each operation rounded once: [..., H-10, W-10]."""
    H, W = q.shape[-2:]
    n = 2 * SSIM_RADIUS + 1
    g = [float(t) for t in SSIM_TAPS]
    h = f32(g[0] * q[..., :, 0:W - n + 1])
    for j in range(1, n):
        h = f32(h + f32(g[j] * q[..., :, j:j + W - n + 1]))
    m = f32(g[0] * h[..., 0:H - n + 1, :])
    for i in range(1, n):
        m = f32(m + f32(g[i] * h[..., i:i + H - n + 1, :]))
    return m


def host_ssim_map(pred, gt):
    """The float32 SSIM map of each frame and channel, [N,3,H-10,W-10] as float32: the kernel's operations in its order."""
    _check_ssim(pred, gt)
    a, b = (t.detach().cpu().float().double() for t in (pred, gt))
    mx, my, sxx, syy, sxy = (_separable(q) for q in (a, b, f32(a * a), f32(b * b), f32(a * b)))
    mx2, my2, mxy = f32(mx * mx), f32(my * my), f32(mx * my)
    sx, sy, sxy = f32(sxx - mx2), f32(syy - my2), f32(sxy - mxy)
    num = f32(f32(f32(2 * mxy) + SSIM_C1) * f32(f32(2 * sxy) + SSIM_C2))
    den = f32(f32(f32(mx2 + my2) + SSIM_C1) * f32(f32(sx + sy) + SSIM_C2))
    return f32(num / den).float()


def host_ssim(pred, gt):
    """ssim on the host: host_ssim_map summed per frame in numpy fp64.  Returns (sum fp64 [N], count int64 [N]) on the CPU."""
    N, H, W = _check_ssim(pred, gt)
    m = host_ssim_map(pred, gt).double().numpy().reshape(N, -1)
    return torch.from_numpy(m.sum(1)), torch.full((N,), m.shape[1], dtype=torch.int64)


def psnr(sq_sum, count):
    """The PSNR of one frame from interpolation_error's partials: 10 log10(255^2 / MSE), MSE = sq_sum / (3 count) over pixels
    and channels; PSNR_CAP (100 dB) for a frame without error."""
    mse = sq_sum / (3 * count)
    return PSNR_CAP if mse == 0 else 10 * math.log10(255.0 ** 2 / mse)


def summarize_inpainting(videos):
    """The split's numbers from per-video records: a list of one list per video of (sq_sum, count, ssim_sum, ssim_count) per
    scored frame (interpolation_error's and ssim's partials).  psnr and ssim are each the mean over a video's scored frames,
    then over the videos with a scored frame, in fp64; frames and videos, their numbers.  NaN without a scored frame."""
    p, s, frames, n = 0.0, 0.0, 0, 0
    for rows in videos:
        if not rows:
            continue
        p += sum(psnr(sq, c) for sq, c, _, _ in rows) / len(rows)
        s += sum(ss / sc for _, _, ss, sc in rows) / len(rows)
        frames += len(rows)
        n += 1
    return {"psnr": p / n if n else math.nan, "ssim": s / n if n else math.nan, "frames": frames, "videos": n}
