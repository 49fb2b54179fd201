"""Confidence evaluation on the GPU: rnc_sparsification's counts equal host_sparsification's exactly and its sums agree within
an fp64 reordering bound at the Sintel, KITTI and Chairs shapes, odd shapes and heavily tied scores; its results repeat bit for
bit and do not depend on the batch; validate(confidence=True) on raft_nc_dbl keeps the flow metrics bit for bit and equals the
host definition on a direct forward's flows and confidences; and two NCCL ranks give the single-process dict when two GPUs are
visible."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import build_model, frames
from test_sparsification import K, assert_sums_close

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def check(flow, gt, valid, score):
    """The kernel against the host path.  Both sum the same count[b, k] fp64 numbers in different orders, so each is within
    (count - 1) * u * sum|x| of the exact sum and they are within twice that of each other; every kept EPE is >= 0, so
    sum|x| <= the image's total EPE, kept_epe[b, 0]."""
    from rnc.metrics import host_sparsification, sparsification
    p = sparsification(flow, gt, valid, score)
    h = host_sparsification(flow.cpu(), gt.cpu(), None if valid is None else valid.cpu(), score.cpu())
    assert p.count.is_cuda and p.count.shape == (flow.shape[0], K)
    assert torch.equal(p.count.cpu(), h.count)
    tot = h.kept_epe[:, :1]
    mags = torch.where(torch.isfinite(tot), tot, torch.zeros_like(tot)).expand(-1, K)
    assert_sums_close(p.kept_epe.cpu(), h.kept_epe, h.count, mags)
    assert_sums_close(p.ideal_epe.cpu(), h.ideal_epe, h.count, mags)
    return p


def sintel_batch(B=8, seed=0):
    """Flows and scores read through the unpadded views of padded 440-row batches, as validate hands them over."""
    from utils.utils import InputPadder
    g = torch.Generator(device=DEV).manual_seed(seed)
    flow_up = torch.randn(B, 2, 440, 1024, device=DEV, generator=g) * 6
    conf_up = torch.rand(B, 2, 440, 1024, device=DEV, generator=g)
    padder = InputPadder((3, 436, 1024))
    view = padder.unpad(flow_up)
    gt = view.detach().clone() + torch.randn(B, 2, 436, 1024, device=DEV, generator=g) * 3
    score = padder.unpad(conf_up)[:, 0]
    assert not view.is_contiguous() and not score.is_contiguous() and score.shape == (B, 436, 1024)
    return view, gt, score


def test_sintel_views_equal_host():
    flow, gt, score = sintel_batch()
    check(flow, gt, None, score)
    valid = (torch.rand(8, 436, 1024, device=DEV) > 0.1).float()
    check(flow, gt, valid, score)


def test_kitti_sparse_valid_equals_host():
    g = torch.Generator(device=DEV).manual_seed(1)
    gt = torch.randn(3, 2, 375, 1242, device=DEV, generator=g) * 20
    flow = gt + torch.randn(3, 2, 375, 1242, device=DEV, generator=g) * 4
    valid = (torch.rand(3, 375, 1242, device=DEV, generator=g) > 0.8).float()   # sparse, as KITTI's lidar ground truth
    valid[2] = 0                                                                # an image without a valid pixel
    score = torch.rand(3, 375, 1242, device=DEV, generator=g)
    p = check(flow, gt, valid, score)
    assert p.count[2].tolist() == [0] * K and p.kept_epe[2].tolist() == [0.0] * K and p.ideal_epe[2].tolist() == [0.0] * K


@pytest.mark.parametrize("B,H,W", [(1, 384, 512), (64, 384, 512), (3, 37, 53), (2, 1, 2049)])
def test_chairs_and_odd_sizes_equal_host(B, H, W):
    g = torch.Generator(device=DEV).manual_seed(B * H + W)
    gt = torch.randn(B, 2, H, W, device=DEV, generator=g) * 5
    flow = gt + torch.randn(B, 2, H, W, device=DEV, generator=g) * 2
    check(flow, gt, None, torch.randn(B, H, W, device=DEV, generator=g))


def test_tied_and_special_scores_equal_host():
    g = torch.Generator(device=DEV).manual_seed(4)
    flow = torch.randn(4, 2, 96, 160, device=DEV, generator=g) * 4
    gt = torch.randn(4, 2, 96, 160, device=DEV, generator=g) * 4
    score = torch.floor(torch.rand(4, 96, 160, device=DEV, generator=g) * 4) / 4        # 4 levels: heavy ties
    score[0, 0, :50] = float("nan")
    score[0, 1, :20] = float("inf")
    score[0, 2, :20] = -float("inf")
    score[1, 3, ::2] = -0.0                                                       # -0 ties with +0: index order
    score[1, 3, 1::2] = 0.0
    score[2] = 0.5                                                                # one level: index order only
    flow[0, 0, 4, 4] = float("nan")
    flow[1, 1, 7, 8] = float("inf")
    valid = (torch.rand(4, 96, 160, device=DEV, generator=g) > 0.2).float()
    valid[0, 4, 4] = 1
    valid[1, 7, 8] = 1
    check(flow, gt, valid, score)
    check(flow, gt, None, score)


def test_repeats_and_does_not_depend_on_the_batch():
    from rnc.metrics import sparsification
    flow, gt, score = sintel_batch(seed=2)
    valid = (torch.rand(8, 436, 1024, device=DEV) > 0.3).float()
    a, b = sparsification(flow, gt, valid, score), sparsification(flow, gt, valid, score)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    for k in range(8):
        one = sparsification(flow[k:k + 1], gt[k:k + 1], valid[k:k + 1], score[k:k + 1])
        assert all(torch.equal(x[0], y[k]) for x, y in zip(one, a)), k
    rev = sparsification(flow.flip(0), gt.flip(0), valid.flip(0), score.flip(0))
    assert all(torch.equal(x.flip(0), y) for x, y in zip(rev, a))


@pytest.fixture
def det(monkeypatch):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


@pytest.mark.parametrize("sparse", [False, True])
def test_validate_confidence_equals_host_definition_of_the_same_forward(sparse, det):
    from rnc.harness import validate
    from rnc.metrics import (confidence_score, flow_metrics, host_sparsification, summarize_sparsification)
    from utils.utils import InputPadder
    m = build_model("raft_nc_dbl").to(DEV)
    im1, im2 = frames(3, 436, 1024, seed=5)
    g = torch.Generator().manual_seed(6)
    gt = torch.randn(3, 2, 436, 1024, generator=g) * 2
    valid = (torch.rand(3, 436, 1024, generator=g) > 0.5).float() if sparse else None
    samples = [(im1[i], im2[i], gt[i]) + ((valid[i],) if sparse else ()) for i in range(3)]
    mode = "kitti" if sparse else "sintel"
    plain = validate(m, samples, iters=2, mode=mode, batch_size=8)
    res = validate(m, samples, iters=2, mode=mode, batch_size=8, confidence=True)
    assert {k: res[k] for k in plain} == plain                                   # the flow metrics, bit for bit
    with torch.no_grad():
        padder = InputPadder(im1.shape, mode=mode)
        p1, p2 = padder.pad(im1.to(DEV), im2.to(DEV))
        _, flow_pr, conf = m(p1, p2, iters=2, test_mode=True, return_confidence=True)
        flow, conf = padder.unpad(flow_pr), padder.unpad(conf)
        fm = flow_metrics(flow, gt.to(DEV), None if valid is None else valid.to(DEV))
    want = summarize_sparsification(host_sparsification(flow.cpu(), gt, valid, confidence_score(conf).cpu()))
    assert res["sparsification"] == pytest.approx(want["sparsification"], rel=1e-12, abs=0)
    assert res["ideal"] == pytest.approx(want["ideal"], rel=1e-12, abs=0)
    # the AUSE is a trapezoid sum of curve differences: its error is that of the curves (relative 1e-12), times their size
    assert res["ause"] == pytest.approx(want["ause"], rel=0, abs=1e-12 * max(want["sparsification"]))
    assert all(o <= s * (1 + 1e-12) for o, s in zip(res["ideal"], res["sparsification"]))
    assert res["ause"] >= 0
    mean_epe = sum((fm.epe_sum.cpu() / fm.counts[:, 0].cpu()).tolist()) / 3
    assert res["sparsification"][0] == pytest.approx(mean_epe, rel=1e-12)
    assert res["ideal"][0] == pytest.approx(mean_epe, rel=1e-12)


def test_validate_confidence_of_the_convex_model_raises():
    from rnc.harness import validate
    im1, im2 = frames(1, 64, 96, seed=3)
    with pytest.raises(ValueError):
        validate(build_model("raft").to(DEV), [(im1[0], im2[0], torch.zeros(2, 64, 96))], iters=1, confidence=True)


def nccl_samples():
    im1, im2 = frames(5, 96, 160, seed=8)
    g = torch.Generator().manual_seed(9)
    return [(im1[i], im2[i], torch.randn(2, 96, 160, generator=g), (torch.rand(96, 160, generator=g) > 0.4).float())
            for i in range(5)]


def _nccl_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RNC_LOOKUP="ffma")
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from rnc.harness import validate
        torch.use_deterministic_algorithms(True)
        res = validate(build_model("raft_nc_dbl").cuda(), nccl_samples(), iters=2, batch_size=1, confidence=True)
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
def test_nccl_two_ranks_equal_world_1(monkeypatch):
    from rnc.harness import validate
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        want = validate(build_model("raft_nc_dbl").to(DEV), nccl_samples(), iters=2, batch_size=1, confidence=True)
    finally:
        torch.use_deterministic_algorithms(prev)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        got = [r for _, r in sorted(q.get(timeout=600) for _ in range(2))]
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.terminate()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    assert got == [want, want]
