"""Video object segmentation on the GPU (rnc_propagate_labels, rnc_segmentation_counts): the kernels against the host
restatements bit for bit, batch independence and repeatability, and propagate_masks and validate_segmentation against
run_sequences_bidirectional's outputs propagated and scored on the host."""
import pytest
import torch
import torch.nn.functional as F

from conftest import build_model
from rnc.harness import propagate_masks, run_sequences_bidirectional, validate_segmentation
from rnc.segment import (host_propagate, host_propagate_step, host_segmentation_counts, propagate, propagate_step,
                         segmentation_counts, summarize_segmentation)
from rnc.synth import shift_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def random_video(V, T, H, W, seed, labels=254, scale=4.0):
    """Blocky labels 0..labels on frame 0, smooth fractional backward flows (some leaving the frame) with NaN and +-inf
    entries, random occluded pixels and occluded blocks."""
    g = torch.Generator().manual_seed(seed)
    low = torch.randint(0, labels + 1, (V, 1, max(H // 6, 2), max(W // 6, 2)), generator=g).float()
    first = F.interpolate(low, size=(H, W), mode="nearest")[:, 0].to(torch.uint8)
    flow = torch.randn(V * (T - 1), 2, max(H // 8, 2), max(W // 8, 2), generator=g) * scale
    flow = F.interpolate(flow, size=(H, W), mode="bilinear", align_corners=False).view(V, T - 1, 2, H, W)
    flow[0, 0, 0, 2:5, 3:7] = float("nan")
    flow[-1, -1, 1, H // 2, :] = float("inf")
    flow[0, -1, 0, :, W // 3] = -float("inf")
    flow[-1, 0, :, 1, 1] = float("nan")
    occ = (torch.rand(V, T - 1, H, W, generator=g) < 0.05).to(torch.uint8)
    occ[:, :, H // 3:H // 3 + max(H // 8, 2), W // 4:W // 4 + max(W // 8, 2)] = 1
    return first, flow, occ


@pytest.mark.parametrize("V,T,H,W", [(1, 6, 37, 23), (5, 5, 37, 23), (1, 3, 480, 854), (5, 3, 480, 854)])
def test_propagate_equals_the_host_restatement(V, T, H, W):
    first, flow, occ = random_video(V, T, H, W, seed=V * 100 + H)
    got = propagate(first.to(DEV), flow.to(DEV), occ.to(DEV))
    want = host_propagate(first, flow, occ)
    assert torch.equal(got.cpu(), want)
    assert len(torch.unique(want[:, -1])) > (100 if H > 100 else 10)
    step = propagate_step(first.to(DEV), flow[:, 0].to(DEV), occ[:, 0].to(DEV))
    assert torch.equal(step.cpu(), host_propagate_step(first, flow[:, 0], occ[:, 0]))


def test_propagate_reads_strided_inputs():
    V, T, H, W = 3, 4, 30, 44
    first, flow, occ = random_video(V, T, H, W, seed=7)
    big = torch.zeros(V, T - 1, 3, H + 3, W + 5)
    big[:, :, 1:, 2:H + 2, 3:W + 3] = flow
    fv = big.to(DEV)[:, :, 1:, 2:H + 2, 3:W + 3]                        # strided in every dimension but x
    ov = occ.to(DEV).transpose(-1, -2).contiguous().transpose(-1, -2)   # x-major masks
    lv = first.to(DEV).transpose(-1, -2).contiguous().transpose(-1, -2)
    assert not fv.is_contiguous() and not ov.is_contiguous() and not lv.is_contiguous()
    got = propagate(lv, fv, ov)
    assert torch.equal(got.cpu(), host_propagate(first, flow, occ))


def test_a_video_is_the_same_alone_or_in_a_batch_and_from_call_to_call():
    first, flow, occ = (t.to(DEV) for t in random_video(5, 5, 40, 64, seed=8))
    full = propagate(first, flow, occ)
    assert torch.equal(full, propagate(first, flow, occ))
    assert torch.equal(propagate(first[3:4], flow[3:4], occ[3:4])[0], full[3])


def scored(V, N, H, W, K, seed):
    """Predictions near a blocky ground truth of objects 1..K, with void pixels."""
    g = torch.Generator().manual_seed(seed)
    low = torch.randint(0, K + 1, (N, 1, H // 16, W // 16), generator=g).float()
    gt = F.interpolate(low, size=(H, W), mode="nearest")[:, 0].to(torch.uint8)
    pred = torch.roll(gt, shifts=(3, -5), dims=(1, 2))
    noise = torch.rand(N, H, W, generator=g) < 0.02
    pred[noise] = torch.randint(0, K + 1, (int(noise.sum()),), generator=g, dtype=torch.uint8)
    gt[:, H // 2:H // 2 + 12, :W // 3] = 255
    gt[0, -1, :] = 255
    return pred, gt


@pytest.mark.parametrize("N,H,W,K", [(6, 37, 23, 3), (2, 480, 854, 10)])
def test_segmentation_counts_equal_the_host(N, H, W, K):
    pred, gt = scored(1, N, max(H, 32), max(W, 32), K, seed=N)
    pred, gt = pred[:, :H, :W], gt[:, :H, :W]
    want = host_segmentation_counts(pred, gt, K)
    got = segmentation_counts(pred.to(DEV), gt.to(DEV), K)
    assert torch.equal(got.cpu(), want)
    assert want[..., 2].sum() > 0 and (want[..., 4] < want[..., 2]).any()
    one = segmentation_counts(pred[1:2].to(DEV), gt[1:2].to(DEV), K)    # a frame alone
    assert torch.equal(one[0], got[1])
    big = torch.zeros(N, H + 2, W + 3, dtype=torch.uint8, device=DEV)  # strided
    big[:, 1:H + 1, 2:W + 2] = pred.to(DEV)
    assert torch.equal(segmentation_counts(big[:, 1:H + 1, 2:W + 2], gt.to(DEV), K), got)


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


H, W, ITERS = 64, 128, 6


def videos():
    seqs = [[f.to(DEV) for f in shift_sequence(n, H, W, seed=s, dy=1, dx=2)] for s, n in enumerate((5, 3, 4))]
    gts = []
    for n in (5, 3, 4):
        gt = torch.zeros(n, H, W, dtype=torch.uint8)
        for t in range(n):
            gt[t, 10 + t:30 + t, 20 + 2 * t:50 + 2 * t] = 1
            gt[t, 35 + t:55 + t, 70 + 2 * t:100 + 2 * t] = 2
            gt[t, :2, :8] = 255
        gts.append(gt)
    return seqs, gts


def host_masks(m, seqs, firsts, warm_start, batch_size=2):
    """run_sequences_bidirectional's outputs collected per video, then host_propagate of each video alone."""
    got = {}
    for s, k, r in run_sequences_bidirectional(m, seqs, ITERS, warm_start=warm_start, batch_size=batch_size, device=DEV):
        got[s, k] = {name: r[name].cpu() for name in ("flow_up_bw", "occ_bw")}
    out = []
    for s, first in enumerate(firsts):
        flow = torch.stack([got[s, k]["flow_up_bw"] for k in range(len(seqs[s]) - 1)])[None]
        occ = torch.stack([got[s, k]["occ_bw"] for k in range(len(seqs[s]) - 1)])[None]
        out.append(host_propagate(first[None].cpu(), flow, occ)[0])
    return out


@pytest.mark.parametrize("warm_start,batch_size", [(False, 2), (True, 2), (False, 1), (True, 3)])
def test_propagate_masks_is_the_sequence_pass_then_host_propagate(warm_start, batch_size, monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft_nc_dbl").to(DEV)
    seqs, gts = videos()
    firsts = [torch.where(gt[0] == 255, 0, gt[0]) for gt in gts]
    with torch.no_grad():
        got = propagate_masks(m, seqs, firsts, ITERS, warm_start=warm_start, batch_size=batch_size, device=DEV)
        want = host_masks(m, seqs, firsts, warm_start, batch_size)
    assert len(got) == 3
    for lab, w, seq in zip(got, want, seqs):
        assert lab.shape == (len(seq), H, W) and lab.dtype == torch.uint8 and lab.is_cuda
        assert torch.equal(lab.cpu(), w)


def test_validate_segmentation_equals_the_host_counts(monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft").to(DEV)
    seqs, gts = videos()
    res = validate_segmentation(m, seqs, gts, ITERS, batch_size=2, device=DEV)
    firsts = [torch.where(gt[0] == 255, 0, gt[0]) for gt in gts]
    with torch.no_grad():
        mine = host_masks(m, seqs, firsts, False)
    counts = [host_segmentation_counts(p[1:-1], gt[1:-1], 2) for p, gt in zip(mine, gts)]
    assert res == summarize_segmentation(counts) and res["videos"] == 3 and res["objects"] == 6
    print(res)
