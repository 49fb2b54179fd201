"""The census and smoothness kernels (csrc/photometric.cu) held to the fp64 model of tests/test_photometric_error_model.py,
pixel by pixel and row by row: natural, quantised, flat, saturated and constant frames besides noise; true, integer, edge,
leaving, +-1e12, non-finite and piecewise-linear flows; narrow and partial tiles, the reference's training crops and the full
Sintel and KITTI frames.  The entry points are called directly, with test-owned state and workspace, and every output buffer
is filled with NaN first, so an element the kernels leave unwritten fails."""
import math

import pytest
import torch

from rnc.metrics import fb_consistency
from rnc.native import rnc
from rnc.unsupervised import census_loss, host_unsupervised_loss, smoothness_loss, unsupervised_loss
from test_photometric_error_model import (DX, DY, E_STATE, LARGE_SHAPES, SMALL_SHAPES, U, case_mask, cases, model, ratio,
                                          smooth_scales, stimulus, weights)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STATE_BYTES = 28


def layout(i1, i2, flow, mask):
    """On the GPU: channel-last images, the flow the second half of a 2N-row channel-last tensor, the mask as given."""
    N = flow.shape[0]

    def cl(t):
        return t.permute(0, 2, 3, 1).contiguous().to(DEV).permute(0, 3, 1, 2)

    big = cl(torch.cat([torch.zeros_like(flow), flow]))
    return cl(i1), cl(i2), big[N:], None if mask is None else mask.to(DEV)


def run_kernels(i1, i2, flow, mask, census_scale, smooth_scale):
    """Every output of rnc_census_loss_fwd / _bwd and rnc_smoothness_fwd / _bwd, from NaN-filled buffers."""
    N, _, H, W = flow.shape
    n = N * H * W
    state = torch.full((n * STATE_BYTES,), 255, dtype=torch.uint8, device=DEV)      # all-ones bits: NaN in fp64 and fp32
    nbytes = rnc.census_loss_workspace_bytes(N, H, W)
    ws = torch.full((nbytes,), 255, dtype=torch.uint8, device=DEV)
    S, total = (torch.full((k,), math.nan, dtype=torch.float64, device=DEV) for k in (N, 2))
    M = torch.full((N,), -1, dtype=torch.int64, device=DEV)
    m = None if mask is None else mask.to(torch.uint8).contiguous()
    rnc.census_loss_fwd(i1, *i1.stride(), i2, *i2.stride(), flow, *flow.stride(), m, N, H, W, S, M, total, state, ws, nbytes)
    gc = torch.full((N, 2, H, W), math.nan, device=DEV)
    rnc.census_loss_bwd(state, N, H, W, torch.tensor([census_scale], dtype=torch.float32, device=DEV), gc)
    sx, sy, stotal = (torch.full((k,), math.nan, dtype=torch.float64, device=DEV) for k in (N, N, 2))
    sws = torch.full((rnc.smoothness_workspace_bytes(N, H, W),), 255, dtype=torch.uint8, device=DEV)
    rnc.smoothness_fwd(i1, *i1.stride(), flow, *flow.stride(), N, H, W, 150.0, sx, sy, stotal, sws, sws.numel())
    gs = torch.full((N, 2, H, W), math.nan, device=DEV)
    rnc.smoothness_bwd(i1, *i1.stride(), flow, *flow.stride(), N, H, W, 150.0,
                       torch.tensor(smooth_scale, dtype=torch.float32, device=DEV), gs)
    torch.cuda.synchronize()

    def plane(buf, at, dtype):
        size = torch.finfo(dtype).bits // 8
        return buf[at:at + size * n].view(dtype).view(N, H, W)

    return dict(g1=plane(state, 0, torch.float64), wh=plane(state, 8 * n, torch.float64),
                dwx=plane(state, 16 * n, torch.float32), dwy=plane(state, 20 * n, torch.float32),
                k=plane(state, 24 * n, torch.float32), l=plane(ws, 0, torch.float32),
                S=S, M=M, total=total, gc=gc, sx=sx, sy=sy, stotal=stotal, gs=gs)


def census_scale_of(mask, N, H, W):
    return 1.0 / (float(weights(mask, N, H, W, DEV).sum()) + 1e-6)


def check_case(fr, fl, N, H, W, seed, mask="random"):
    """{quantity: worst error / bound} of one case; 0 bounds allow no error at all."""
    i1, i2, flow = stimulus(fr, fl, N, H, W, seed)
    mask = case_mask(N, H, W, seed) if mask == "random" else mask
    cs, ss = census_scale_of(mask, N, H, W), smooth_scales(N, H, W)
    got = run_kernels(*layout(i1, i2, flow, mask), cs, ss)
    b = model(i1.to(DEV), i2.to(DEV), flow.to(DEV), mask, cs, ss)
    g1, wh, dwx, dwy = b.state
    r = {}
    r["state g1, W^"] = max(ratio(got["g1"], g1, torch.full_like(g1, E_STATE)),
                            ratio(got["wh"], wh, torch.full_like(wh, E_STATE)))
    if r["state g1, W^"] > 1:
        d = (got["wh"] - wh).abs().nan_to_num(math.inf)
        at = [int(i) for i in torch.unravel_index(d.argmax(), d.shape)]
        n, y, x = at
        print(f"  {fr}/{fl} {N}x{H}x{W}: W^ at {at}: kernel {float(got['wh'][n, y, x])!r} fp64 {float(wh[n, y, x])!r}, flow "
              f"{flow[n, :, y, x].tolist()}, g1 kernel {float(got['g1'][n, y, x])!r} fp64 {float(g1[n, y, x])!r}")
    r["state dW^/dp"] = max(ratio(got["dwx"], dwx, U * dwx.abs() + E_STATE), ratio(got["dwy"], dwy, U * dwy.abs() + E_STATE))
    r["v l"] = ratio(got["l"], b.cm.l, b.cm.err_l)
    r["k"] = ratio(got["k"], b.cm.k, b.cm.err_k)
    assert torch.equal(got["M"].cpu(), b.M.cpu()) and int(got["total"][1]) == int(b.M.sum()), (got["M"], b.M)
    r["S_r, total"] = max(ratio(got["S"], b.S, b.err_S), ratio(got["total"][:1], b.S.sum()[None], b.err_S.sum()[None]))
    r["census grad"] = ratio(got["gc"], b.census_grad, b.census_bound)
    r["smooth sums"] = max(ratio(got["sx"], b.sm.sx, b.sm.err_sx), ratio(got["sy"], b.sm.sy, b.sm.err_sy),
                           ratio(got["stotal"], torch.stack([b.sm.sx.sum(), b.sm.sy.sum()]),
                                 torch.stack([b.sm.err_sx.sum(), b.sm.err_sy.sum()])))
    r["smooth grad"] = ratio(got["gs"], b.smooth_grad, b.smooth_bound)
    return r


def run_cases(todo):
    worst, failed = {}, []
    for fr, fl, N, H, W, seed in todo:
        r = check_case(fr, fl, N, H, W, seed)
        for what, v in r.items():
            for key in (f"frames {fr}", f"flow {fl}", what):
                worst[key] = max(worst.get(key, 0.0), v)
            if not v <= 1:
                failed.append((fr, fl, N, H, W, what, v))
    for key, v in worst.items():
        print(f"  {key:24s} worst error / bound {v:.3g}")
    assert not failed, failed[:10]
    return worst


@pytest.mark.parametrize("N,H,W", SMALL_SHAPES)
def test_small_and_partial_tiles_within_the_bounds(N, H, W):
    print(f"\n{N}x{H}x{W}, every frame and flow family")
    worst = run_cases(cases([(N, H, W)]))
    # every family reaches a nonzero error somewhere: the comparison is not trivially exact
    assert worst["census grad"] > 0 and worst["smooth grad"] > 0 and worst["v l"] > 0


@pytest.mark.parametrize("N,H,W", LARGE_SHAPES)
def test_training_crops_and_full_frames_within_the_bounds(N, H, W):
    print(f"\n{N}x{H}x{W}, the frame families with the flow families in turn")
    worst = run_cases(cases([(N, H, W)], rotate=True))
    assert worst["census grad"] > 0 and worst["smooth grad"] > 0 and worst["v l"] > 0


def test_no_mask_equals_an_all_ones_mask_and_rows_are_independent_of_the_batch():
    N, H, W = 3, 375, 1242
    i1, i2, flow = stimulus("quantised", "edges", N, H, W, seed=11)
    ones = torch.ones(N, H, W, dtype=torch.bool)
    cs, ss = census_scale_of(ones, N, H, W), smooth_scales(N, H, W)
    a = run_kernels(*layout(i1, i2, flow, None), cs, ss)
    b = run_kernels(*layout(i1, i2, flow, ones), cs, ss)
    assert all(torch.equal(a[k], b[k]) for k in a), [k for k in a if not torch.equal(a[k], b[k])]
    mask = case_mask(N, H, W, 11)
    full = run_kernels(*layout(i1, i2, flow, mask), cs, ss)
    per_row = ("g1", "wh", "dwx", "dwy", "k", "l", "S", "M", "gc", "sx", "sy", "gs")
    for r in range(N):
        one = run_kernels(*layout(i1[r:r + 1], i2[r:r + 1], flow[r:r + 1], mask[r:r + 1]), cs, ss)
        assert all(torch.equal(full[k][r:r + 1], one[k]) for k in per_row), (r, [k for k in per_row
                                                                                 if not torch.equal(full[k][r:r + 1], one[k])])


def test_mask_dtypes_and_strides_give_the_same_bits():
    """census_loss with a bool, a uint8 and a transposed (non-contiguous) mask, and with contiguous inputs: the same loss and
    gradient bits."""
    N, H, W = 4, 47, 65
    i1, i2, flow = stimulus("smooth", "random", N, H, W, seed=5)
    mask = case_mask(N, H, W, 5)
    ci1, ci2, cflow, cmask = i1.to(DEV), i2.to(DEV), flow.to(DEV), mask.to(DEV)
    masks = [cmask, cmask.to(torch.uint8), cmask.transpose(1, 2).contiguous().transpose(1, 2)]
    assert not masks[2].is_contiguous()
    out = []
    for (a, b, f), m in [(layout(i1, i2, flow, None)[:3], mk) for mk in masks] + [((ci1, ci2, cflow), cmask)]:
        f = f.detach().clone().requires_grad_()
        loss = census_loss(a, b, f, m) + 2 * smoothness_loss(a, f)
        loss.backward()
        out.append((loss.detach(), f.grad))
    for l, g in out[1:]:
        assert torch.equal(l, out[0][0]) and torch.equal(g, out[0][1])


def test_sequence_loss_within_the_summed_bound():
    """unsupervised_loss on 12 fixed predictions of [2,2,400,720] against host_unsupervised_loss in fp64: the loss within the
    sum of the per-prediction bounds, each prediction's gradient within its per-pixel bound times gamma^(n-1-i)."""
    B, H, W, n, gamma, lam = 1, 400, 720, 12, 0.85, 2.0
    im1, im2, _ = stimulus("smooth", "true", B, H, W, seed=21)
    g = torch.Generator().manual_seed(21)
    true = torch.tensor([DX, DY], dtype=torch.float32).view(1, 2, 1, 1).expand(B, 2, H, W)
    preds = []
    for i in range(n):
        noise = torch.randn(2 * B, 2, H, W, generator=g) * (n - i) / n
        p = torch.cat([true, -true]) + noise
        preds.append((p * 4096).round() / 4096)         # x + F exact in float32: the restatement samples where the kernel does
    im1, im2 = im1.to(DEV), im2.to(DEV)
    p32 = [p.to(DEV).requires_grad_() for p in preds]
    loss, _ = unsupervised_loss(p32, im1, im2, gamma=gamma, smooth_weight=lam)
    loss.backward()
    p64 = [p.to(DEV).double().requires_grad_() for p in preds]
    ref, _ = host_unsupervised_loss(p64, im1.double(), im2.double(), gamma=gamma, smooth_weight=lam)
    ref.backward()
    last = p32[-1].detach()
    occ_fw, occ_bw, _, _ = fb_consistency(last[:B], last[B:])
    mask = torch.cat([occ_fw, occ_bw]) == 0
    src, tgt = torch.cat([im1, im2]), torch.cat([im2, im1])
    N = 2 * B
    Mtot = float(weights(mask, N, H, W, DEV).sum())
    cx, cy = smooth_scales(N, H, W)
    err_loss, terms, worst = 0.0, [], 0.0
    for i in range(n):
        w = gamma ** (n - 1 - i)
        b = model(src, tgt, p32[i].detach(), mask, w / (Mtot + 1e-6), (w * lam * cx, w * lam * cy), 2 * U, 2 * U)
        C = float(b.S.sum()) / (Mtot + 1e-6)
        Sm = cx * float(b.sm.sx.sum()) + cy * float(b.sm.sy.sum())
        eC = float(b.err_S.sum()) / (Mtot + 1e-6) + U * C
        eSm = cx * float(b.sm.err_sx.sum()) + cy * float(b.sm.err_sy.sum()) + U * Sm
        terms.append(w * (C + lam * Sm))
        err_loss += w * (eC + lam * eSm) + 3 * U * w * (C + lam * Sm)
        gref = b.census_grad + b.smooth_grad
        bound = b.census_bound + b.smooth_bound + U * gref.abs()
        r = ratio(p32[i].grad, p64[i].grad, bound)
        assert torch.allclose(gref, p64[i].grad, rtol=0, atol=1e-9 * float(gref.abs().max()))
        print(f"  prediction {i}: gradient worst error / bound {r:.3g}")
        worst = max(worst, r)
    err_loss += U * sum(abs(sum(terms[:j + 1])) for j in range(n))
    r_loss = abs(float(loss) - float(ref)) / err_loss
    print(f"sequence loss {float(loss):.8f} (fp64 {float(ref):.10f}): error / bound {r_loss:.3g}; gradients {worst:.3g}")
    assert r_loss <= 1 and worst <= 1 and worst > 0
