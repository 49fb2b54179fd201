"""Temporal consistency on the GPU (rnc_temporal_step, rnc_warping_error_partials): the kernels against the host
restatements bit for bit at small, odd and full frame sizes with C = 1..4, on strided slices of stacks with non-finite flows
and targets on the last row and column; batch independence and run-to-run determinism; make_temporally_consistent against
the host pipeline fed the same flows; validate_temporal_consistency end to end."""
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import build_model
from rnc.harness import make_temporally_consistent, run_sequences_bidirectional, validate_temporal_consistency
from rnc.temporal import (host_temporal_step, host_temporally_consistent, host_warping_error, temporal_step,
                          temporally_consistent, warping_error)
from rnc.synth import shift_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def smooth(shape, g, scale):
    """A smooth random field of shape [..., H, W]."""
    *lead, H, W = shape
    n = math.prod(lead)
    low = torch.randn(n, 1, max(H // 8, 2), max(W // 8, 2), generator=g) * scale
    return F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False).view(*lead, H, W)


def videos(V, T, C, H, W, seed):
    """Frames in 0..255 that partly agree along the flow, smooth fractional backward flows with NaN and +-inf entries and
    targets exactly on x = W-1 and y = H-1, random occlusions with an occluded block, and flickering processed frames."""
    g = torch.Generator().manual_seed(seed)
    I = torch.rand(V, T, 3, H, W, generator=g) * 255
    I[:, 1:] = 0.6 * I[:, 1:] + 0.4 * I[:, :-1]
    G = smooth((V, T - 1, 2, H, W), g, 4.0)
    G[0, 0, 0, 2:5, 3:7] = float("nan")
    G[-1, -1, 1, H // 2, :] = float("inf")
    G[-1, 0, 0, :, W // 3] = -float("inf")
    G[0, -1, 0, H // 3, 0], G[0, -1, 1, H // 3, 0] = W - 1.0, 0.0
    G[0, -1, 0, 0, W // 2], G[0, -1, 1, 0, W // 2] = 0.0, H - 1.0
    occ = (torch.rand(V, T - 1, H, W, generator=g) < 0.05).to(torch.uint8)
    occ[:, :, H // 4:H // 4 + max(H // 3, 1), W // 5:W // 5 + max(W // 4, 1)] = 1
    occ[-1, -1] = 1                                                     # a scene cut
    P = smooth((V, T, C, H, W), g, 40.0) + torch.randn(V, T, 1, 1, 1, generator=g) * 10
    return P, I, G, occ


@pytest.mark.parametrize("V,C,H,W,sweeps", [(1, 1, 8, 8, 512), (3, 2, 13, 37, 512), (2, 4, 13, 37, 40), (1, 3, 436, 1024, 64),
                                            (2, 4, 375, 1242, 24), (2, 1, 375, 1242, 16)])
def test_the_step_equals_the_host_restatement(V, C, H, W, sweeps):
    P, I, G, occ = videos(V, 3, C, H, W, seed=V * 100 + C * 10 + H)
    for k, lam, alpha in ((0, 0.1, 50.0), (1, 0.7, 5.0)):
        O = P[:, k] + 3.0
        args = (O, P[:, k + 1], I[:, k], I[:, k + 1], G[:, k], occ[:, k])
        got = temporal_step(*(a.to(DEV) for a in args), lam, alpha, sweeps)
        want = host_temporal_step(*args, lam, alpha, sweeps)
        assert torch.equal(got.cpu(), want), k
    lam0 = temporal_step(*(a.to(DEV) for a in args), 0.0, 50.0, sweeps)
    assert torch.equal(lam0.cpu(), P[:, 2])


def test_strided_slices_of_stacks_give_the_host_bits_and_each_video_is_itself_alone():
    V, T, C, H, W = 3, 5, 3, 40, 64
    P, I, G, occ = videos(V, T, C, H, W, seed=7)
    want = host_temporally_consistent(P, I, G, occ, sweeps=60)
    big = torch.zeros(V, T, C + 1, H + 3, W + 5, device=DEV)
    big[:, :, 1:, 2:H + 2, 3:W + 3] = P.to(DEV)
    pv = big[:, :, 1:, 2:H + 2, 3:W + 3]                                # strided in every dimension but x
    iv = I.to(DEV).permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)       # channel-last frames
    gv = torch.zeros(V, T - 1, 3, H, W, device=DEV)
    gv[:, :, 1:] = G.to(DEV)
    gv = gv[:, :, 1:]
    ov = occ.to(DEV).transpose(-1, -2).contiguous().transpose(-1, -2)   # x-major masks
    assert not any(t.is_contiguous() for t in (pv, iv, gv, ov))
    got = temporally_consistent(pv, iv, gv, ov, sweeps=60)
    assert torch.equal(got.cpu(), want)
    assert torch.equal(temporally_consistent(pv, iv, gv, ov, sweeps=60), got)      # run to run
    for v in range(V):
        alone = temporally_consistent(pv[v:v + 1], iv[v:v + 1], gv[v:v + 1], ov[v:v + 1], sweeps=60)
        assert torch.equal(alone[0], got[v]), v
    assert torch.equal(got[-1, -1].cpu(), P[-1, -1])                    # the scene cut keeps P
    out = pv[:, 1].clone()
    inplace = temporal_step(got[:, 0], out, iv[:, 0], iv[:, 1], gv[:, 0], ov[:, 0], sweeps=60, out=out)
    assert inplace is out and torch.equal(out, got[:, 1])               # out may be processed itself


def test_the_warping_error_partials_equal_the_host():
    for V, T, C, H, W in ((2, 4, 3, 37, 23), (1, 3, 1, 436, 1024), (3, 2, 4, 375, 1242)):
        P, I, G, occ = videos(V, T, C, H, W, seed=T * 10 + C)
        pv = P.to(DEV).permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)
        s, c = warping_error(pv, G.to(DEV), occ.to(DEV))
        hs, hc = host_warping_error(P, G, occ)
        assert torch.equal(c.cpu(), hc) and (hc[-1, -1] == 0).all() and (hc > 0).sum() >= V * (T - 1) - 1
        assert torch.allclose(s.cpu(), hs, rtol=1e-12, atol=0)
        for v in range(V):                                              # a video's partials do not depend on the batch
            sv, cv = warping_error(pv[v:v + 1], G[v:v + 1].to(DEV), occ[v:v + 1].to(DEV))
            assert torch.equal(sv[0], s[v]) and torch.equal(cv[0], c[v])


# ----------------------------------------------------------------------------------------------------------- harness


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


H, W, ITERS, SWEEPS = 64, 128, 6, 64


def split():
    seqs = [[f.to(DEV) for f in shift_sequence(n, H, W, seed=s, dy=1, dx=2)] for s, n in enumerate((5, 3, 4))]
    procs = []
    for k, seq in enumerate(seqs):
        g = torch.Generator().manual_seed(k)
        C = (3, 1, 4)[k]
        gain = 1 + 0.1 * torch.randn(len(seq), 1, 1, 1, generator=g)
        procs.append(torch.stack([torch.cat([f, f[:1]])[:C].cpu() for f in seq]) * gain + 5 * torch.randn(len(seq), 1, 1, 1,
                                                                                                            generator=g))
    return seqs, procs


@pytest.mark.parametrize("warm_start", [False, True])
def test_make_temporally_consistent_is_the_sequence_pass_then_the_host_rule(warm_start, monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft_nc_dbl").to(DEV)
    seqs, procs = split()
    with torch.no_grad():
        got = {}
        for s, k, r in run_sequences_bidirectional(m, seqs, ITERS, warm_start=warm_start, batch_size=3, device=DEV):
            got[s, k] = (r["flow_up_bw"].cpu(), r["occ_bw"].cpu())
        for bs in (1, 3):
            outs = make_temporally_consistent(m, seqs, procs, ITERS, warm_start=warm_start, batch_size=bs, device=DEV,
                                              sweeps=SWEEPS)
            assert len(outs) == 3
            for s, (seq, p, o) in enumerate(zip(seqs, procs, outs)):
                G, occ = (torch.stack([got[s, k][j] for k in range(len(seq) - 1)])[None] for j in (0, 1))
                want = host_temporally_consistent(p[None], torch.stack(seq).cpu()[None], G, occ, sweeps=SWEEPS)[0]
                assert o.is_cuda and torch.equal(o.cpu(), want), (bs, s)


def test_validate_temporal_consistency_runs_end_to_end(monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft").to(DEV)
    seqs, procs = split()
    res = validate_temporal_consistency(m, seqs, procs, ITERS, batch_size=2, device=DEV, sweeps=SWEEPS)
    assert res["videos"] == 3 and res["frames"] == 4 + 2 + 3
    # random weights occlude nearly every pixel, so a frame may have no matched pixel: both errors are NaN or neither
    assert math.isnan(res["warping_error"]) == math.isnan(res["warping_error_processed"])
    assert math.isnan(res["psnr"]) and math.isnan(res["ssim"])          # videos 2 and 3 are not colour
    colour = validate_temporal_consistency(m, seqs[:1], procs[:1], ITERS, batch_size=2, device=DEV, sweeps=SWEEPS)
    assert colour["videos"] == 1 and 10 < colour["psnr"] <= 100 and 0 < colour["ssim"] <= 1
    print(res, colour)
