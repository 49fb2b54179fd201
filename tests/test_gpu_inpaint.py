"""Video inpainting on the GPU (rnc_harmonic_fill, rnc_inpaint_propagate, rnc_ssim_partials): the kernels against the host
restatements bit for bit on awkward inputs and strided views, batch independence, inpaint_videos cold and warm at several
batch sizes and with NaN in its holes, and validate_inpainting end to end."""
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import build_model
from rnc.harness import inpaint_videos, run_sequences_bidirectional, validate_inpainting
from rnc.inpaint import (SOURCE_SPATIAL, harmonic_fill, host_harmonic_fill, host_inpaint_propagate, host_ssim, inpaint,
                         inpaint_propagate, ssim)
from rnc.synth import shift_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def smooth(shape, g, scale):
    """A smooth random field of shape [..., H, W]."""
    *lead, H, W = shape
    n = math.prod(lead)
    low = torch.randn(n, 1, max(H // 8, 2), max(W // 8, 2), generator=g) * scale
    return F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False).view(*lead, H, W)


def holes(shape, g):
    """Hole masks [..., H, W]: random blocks, one touching the top-left border, one the bottom-right, and sparse pixels."""
    *lead, H, W = shape
    m = (torch.rand(*lead, H, W, generator=g) < 0.02).to(torch.uint8)
    m[..., H // 4:H // 4 + max(H // 5, 2), W // 3:W // 3 + max(W // 4, 2)] = 1
    m[..., :max(H // 6, 1), :max(W // 7, 1)] = 1
    m[..., H - max(H // 8, 1):, W - max(W // 5, 1):] = 1
    return m


def fill_inputs(N, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    v = smooth((N, C, H, W), g, 20.0)
    unk = holes((N, H, W), g)
    v[0, 0, 1, 1] = float("nan")                                        # known pixels with non-finite values
    v[-1, C - 1, H - 2, W // 2] = float("inf")
    v[unk[:, None].expand_as(v) != 0] = float("nan")                    # never read
    unk[N // 2] = 1                                                     # an all-hole image
    return v, unk


@pytest.mark.parametrize("N,C,H,W,sweeps", [(6, 2, 37, 23, 512), (4, 3, 23, 37, 7), (2, 2, 480, 854, 6), (1, 3, 480, 854, 3)])
def test_harmonic_fill_equals_the_host_restatement(N, C, H, W, sweeps):
    v, unk = fill_inputs(N, C, H, W, seed=N * 10 + H)
    got = harmonic_fill(v.to(DEV), unk.to(DEV), sweeps)
    want = host_harmonic_fill(v, unk, sweeps)
    assert torch.equal(got.cpu(), want)
    assert torch.equal(want[N // 2], torch.zeros(C, H, W)) and torch.isfinite(want).all()


def test_harmonic_fill_reads_strided_inputs_and_fills_in_place():
    V, T, C, H, W = 2, 3, 2, 30, 44
    v, unk = fill_inputs(V * T, C, H, W, seed=5)
    want = host_harmonic_fill(v, unk, 40).view(V, T, C, H, W)
    big = torch.zeros(V, T, C + 1, H + 3, W + 5, device=DEV)
    big[:, :, 1:, 2:H + 2, 3:W + 3] = v.view(V, T, C, H, W).to(DEV)
    vv = big[:, :, 1:, 2:H + 2, 3:W + 3]                                # strided in every dimension but x
    uu = unk.view(V, T, H, W).to(DEV).transpose(-1, -2).contiguous().transpose(-1, -2)   # x-major masks
    assert not vv.is_contiguous() and not uu.is_contiguous()
    assert torch.equal(harmonic_fill(vv, uu, 40).cpu(), want)
    out = harmonic_fill(vv, uu, 40, out=vv)                             # in place, through the same strides
    assert out is vv and torch.equal(vv.cpu(), want)
    assert big[:, :, 0].eq(0).all()                                     # nothing written outside the view


def video(V, T, H, W, seed, scale=3.0):
    """Frames in 0..255 with NaN in the holes, hole masks (border blocks, an all-hole frame), fractional flows with NaN and
    +-inf entries and random occlusions."""
    g = torch.Generator().manual_seed(seed)
    frames = torch.rand(V, T, 3, H, W, generator=g) * 255
    masks = holes((V, T, H, W), g)
    masks[0, T // 2] = 1
    frames[masks[:, :, None].expand_as(frames) != 0] = float("nan")
    flow, flow_bw = (smooth((V, T - 1, 2, H, W), g, scale) for _ in range(2))
    flow[0, 0, 0, 2:5, 3:7] = float("nan")
    flow_bw[-1, -1, 1, H // 2, :] = float("inf")
    flow[-1, 0, 1, :, W // 3] = -float("inf")
    occ, occ_bw = ((torch.rand(V, T - 1, H, W, generator=g) < 0.05).to(torch.uint8) for _ in range(2))
    return frames, masks, flow, flow_bw, occ, occ_bw


@pytest.mark.parametrize("V,T,H,W", [(1, 6, 37, 23), (4, 5, 37, 23), (1, 4, 480, 854), (3, 3, 480, 854)])
def test_inpaint_propagate_equals_the_host_restatement(V, T, H, W):
    args = video(V, T, H, W, seed=V * 100 + H)
    for maxd in (None, 2):
        got = inpaint_propagate(*(a.to(DEV) for a in args), max_distance=maxd)
        want = host_inpaint_propagate(*args, max_distance=maxd)
        assert torch.equal(got[1].cpu(), want[1])
        assert torch.equal(got[0].cpu(), want[0])
        assert all((want[1] == s).any() for s in range(5))


def test_inpaint_propagate_reads_strided_inputs():
    V, T, H, W = 2, 4, 30, 44
    frames, masks, flow, flow_bw, occ, occ_bw = video(V, T, H, W, seed=7)
    want = host_inpaint_propagate(frames, masks, flow, flow_bw, occ, occ_bw)
    big = torch.zeros(V, T - 1, 3, H + 3, W + 5)
    big[:, :, 1:, 2:H + 2, 3:W + 3] = flow
    fv = big.to(DEV)[:, :, 1:, 2:H + 2, 3:W + 3]
    im = frames.to(DEV).permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)     # channel-last frames
    xm = [t.to(DEV).transpose(-1, -2).contiguous().transpose(-1, -2) for t in (masks, occ, occ_bw)]
    assert not fv.is_contiguous() and not im.is_contiguous() and not xm[0].is_contiguous()
    got = inpaint_propagate(im, xm[0], fv, flow_bw.to(DEV), xm[1], xm[2])
    assert torch.equal(got[0].cpu(), want[0]) and torch.equal(got[1].cpu(), want[1])


def test_ssim_kernel_matches_the_host():
    g = torch.Generator().manual_seed(3)
    a = torch.rand(5, 3, 480, 854, generator=g) * 255
    b = (a + torch.randn(5, 3, 480, 854, generator=g) * 10).clamp(0, 255)
    b[1] = a[1]
    s, c = ssim(a.to(DEV), b.to(DEV))
    hs, hc = host_ssim(a, b)
    assert torch.equal(c.cpu(), hc)
    assert torch.allclose(s.cpu(), hs, rtol=1e-12, atol=0)
    assert float(s[1] / c[1]) == 1.0
    small = ssim(a[:, :, :37, :23].to(DEV), b[:, :, :37, :23].to(DEV))
    hsmall = host_ssim(a[:, :, :37, :23], b[:, :, :37, :23])
    assert torch.equal(small[1].cpu(), hsmall[1]) and torch.allclose(small[0].cpu(), hsmall[0], rtol=1e-12, atol=0)


def test_a_video_is_the_same_alone_or_in_a_batch_and_from_call_to_call():
    frames, masks, flow, flow_bw, occ, occ_bw = (t.to(DEV) for t in video(4, 5, 40, 64, seed=8))
    batched = inpaint_propagate(frames, masks, flow, flow_bw, occ, occ_bw)
    again = inpaint_propagate(frames, masks, flow, flow_bw, occ, occ_bw)
    assert all(torch.equal(x, y) for x, y in zip(batched, again))
    for v in range(4):
        alone = inpaint_propagate(frames[v:v + 1], masks[v:v + 1], flow[v:v + 1], flow_bw[v:v + 1], occ[v:v + 1],
                                  occ_bw[v:v + 1])
        assert torch.equal(alone[0][0], batched[0][v]) and torch.equal(alone[1][0], batched[1][v])
    v5, u5 = (t.to(DEV) for t in fill_inputs(5, 2, 40, 64, seed=9))
    filled = harmonic_fill(v5, u5, 50)
    for i in range(5):
        assert torch.equal(harmonic_fill(v5[i:i + 1], u5[i:i + 1], 50)[0], filled[i])
    a = frames[:, 0].nan_to_num(0.0)
    s, c = ssim(a, a.flip(-1))
    for i in range(4):
        si, ci = ssim(a[i:i + 1], a[i:i + 1].flip(-1))
        assert torch.equal(si[0], s[i]) and torch.equal(ci[0], c[i])
    full = inpaint(frames, masks, flow, flow_bw, sweeps=30)
    assert torch.isfinite(full[0]).all() and (full[1] == SOURCE_SPATIAL).any()
    assert all(torch.equal(x, y) for x, y in zip(full, inpaint(frames, masks, flow, flow_bw, sweeps=30)))


# ----------------------------------------------------------------------------------------------------------- harness


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


H, W, ITERS, SWEEPS = 64, 128, 6, 64


def videos():
    seqs = [[f.to(DEV) for f in shift_sequence(n, H, W, seed=s, dy=1, dx=2)] for s, n in enumerate((5, 3, 4))]
    masks = []
    for k, n in enumerate((5, 3, 4)):
        m = torch.zeros(n, H, W, dtype=torch.uint8)
        for t in range(n):
            m[t, 12 + t:30 + t, 40 + 3 * t:64 + 3 * t] = 1
            m[t, 40:50, 90 + k:100 + k] = 1
        masks.append(m)
    return seqs, masks


def stacked_inpaint(m, seqs, masks, warm_start, batch_size):
    """run_sequences_bidirectional on the masked videos, then rnc.inpaint.inpaint of each video alone."""
    seen = [[torch.where(h.to(DEV) != 0, 0.0, f) for f, h in zip(seq, mk)] for seq, mk in zip(seqs, masks)]
    got = {}
    for s, k, r in run_sequences_bidirectional(m, seen, ITERS, warm_start=warm_start, batch_size=batch_size, device=DEV):
        got[s, k] = (r["flow_up"].clone(), r["flow_up_bw"].clone())
    out = []
    for s, (seq, mk) in enumerate(zip(seqs, masks)):
        fw, bw = (torch.stack([got[s, k][j] for k in range(len(seq) - 1)])[None] for j in (0, 1))
        res = inpaint(torch.stack(seq)[None], mk[None].to(DEV), fw, bw, sweeps=SWEEPS)
        out.append((res[0][0], res[1][0]))
    return out


@pytest.mark.parametrize("warm_start", [False, True])
def test_inpaint_videos_is_the_sequence_pass_then_inpaint_at_any_batch_size(warm_start, monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft_nc_dbl").to(DEV)
    seqs, masks = videos()
    with torch.no_grad():
        want = stacked_inpaint(m, seqs, masks, warm_start, 3)
        for bs in (1, 3, 8):
            got = inpaint_videos(m, seqs, masks, ITERS, warm_start=warm_start, batch_size=bs, device=DEV, sweeps=SWEEPS)
            assert len(got) == 3
            for (o, s), (wo, ws), seq in zip(got, want, seqs):
                assert o.shape == (len(seq), 3, H, W) and s.shape == (len(seq), H, W) and o.is_cuda
                assert torch.equal(s, ws), bs
                assert torch.equal(o, wo), bs
        poisoned = [[torch.where(h.to(DEV)[None] != 0, float("nan"), f) for f, h in zip(seq, mk)]
                    for seq, mk in zip(seqs, masks)]
        got = inpaint_videos(m, poisoned, masks, ITERS, warm_start=warm_start, batch_size=3, device=DEV, sweeps=SWEEPS)
        for (o, s), (wo, ws) in zip(got, want):
            assert torch.equal(o, wo) and torch.equal(s, ws)
    for (_, s), mk in zip(want, masks):                                  # random weights occlude nearly every chain
        assert torch.equal(s == 0, mk.to(DEV) == 0)


def test_validate_inpainting_runs_end_to_end(monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft").to(DEV)
    seqs, masks = videos()
    masks[1][1] = 0                                                     # an unscored frame
    res = validate_inpainting(m, seqs, masks, ITERS, batch_size=2, device=DEV, sweeps=SWEEPS)
    assert res["videos"] == 3 and res["frames"] == 11
    assert 10 < res["psnr"] < 100 and 0 < res["ssim"] < 1
    print(res)
