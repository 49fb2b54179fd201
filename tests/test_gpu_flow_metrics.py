"""Validation metrics on the GPU: rnc_flow_metrics' counts equal the host partials exactly and its sums agree to 1e-12 at the
Sintel, KITTI and Chairs shapes, through strided views, at the edges (zero-magnitude ground truth, NaN, inf); its results
repeat bit for bit and do not depend on the batch; validate on raft_nc_dbl equals the host metrics of the same flows; and two
NCCL ranks give the single-process dict when two GPUs are visible."""
import math
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import build_model, frames
from test_flow_metrics import edge_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def check(flow, gt, valid=None):
    from rnc.metrics import flow_metrics, host_partials
    p = flow_metrics(flow, gt, valid)
    h = host_partials(flow.cpu(), gt.cpu(), None if valid is None else valid.cpu())
    assert p.counts.is_cuda and p.counts.shape == (flow.shape[0], 5)
    assert torch.equal(p.counts.cpu(), h.counts)
    torch.testing.assert_close(p.epe_sum.cpu(), h.epe_sum, rtol=1e-12, atol=0, equal_nan=True)
    return p


def sintel_batch(B=8, seed=0):
    """Flows read through the unpadded view of a padded 440-row batch, as validate hands them over."""
    from utils.utils import InputPadder
    g = torch.Generator(device=DEV).manual_seed(seed)
    flow_up = torch.randn(B, 2, 440, 1024, device=DEV, generator=g) * 6
    view = InputPadder((3, 436, 1024)).unpad(flow_up)
    gt = view.detach().clone() + torch.randn(B, 2, 436, 1024, device=DEV, generator=g) * 3
    assert not view.is_contiguous() and view.shape == (B, 2, 436, 1024)
    return view, gt


def test_sintel_view_equals_host():
    flow, gt = sintel_batch()
    check(flow, gt)
    valid = (torch.rand(8, 436, 1024, device=DEV) > 0.1).float()
    check(flow, gt, valid)


def test_kitti_sparse_valid_equals_host():
    g = torch.Generator(device=DEV).manual_seed(1)
    gt = torch.randn(3, 2, 375, 1242, device=DEV, generator=g) * 20
    flow = gt + torch.randn(3, 2, 375, 1242, device=DEV, generator=g) * 4
    valid = (torch.rand(3, 375, 1242, device=DEV, generator=g) > 0.8).float()   # sparse, as KITTI's lidar ground truth
    valid[2] = 0                                                                # an image without a valid pixel
    p = check(flow, gt, valid)
    assert p.counts[2].tolist() == [0, 0, 0, 0, 0]
    # channel-last storage of the flow, read as [B,2,H,W]
    check(flow.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2), gt, valid)


@pytest.mark.parametrize("B,H,W", [(1, 384, 512), (64, 384, 512), (3, 37, 53), (2, 1, 2049)])
def test_chairs_and_odd_sizes_equal_host(B, H, W):
    g = torch.Generator(device=DEV).manual_seed(B * H + W)
    gt = torch.randn(B, 2, H, W, device=DEV, generator=g) * 5
    flow = gt + torch.randn(B, 2, H, W, device=DEV, generator=g) * 2
    check(flow, gt)


def test_edge_values_equal_host():
    flow, gt, valid = (t.to(DEV) for t in edge_case())
    check(flow, gt, valid)
    check(flow, gt)
    g = torch.Generator(device=DEV).manual_seed(4)
    flow = torch.randn(4, 2, 33, 47, device=DEV, generator=g) * 4
    gt = torch.randn(4, 2, 33, 47, device=DEV, generator=g) * 4
    gt[1, :, :5] = 0                                    # zero-magnitude ground truth
    flow[0, 0, 3, 4] = float("nan")
    flow[1, 1, 7, 8] = float("inf")
    flow[2, 0, 9, 9] = -float("inf")
    gt[2, :, 9, 9] = 0
    flow[3, :, 1, 1] = float("nan")
    valid = torch.ones(4, 33, 47, device=DEV)
    valid[3, 1, 1] = 0                                  # an invalid NaN does not count
    p = check(flow, gt, valid)
    s = p.epe_sum.cpu()
    assert math.isnan(s[0]) and math.isinf(s[1]) and math.isinf(s[2]) and math.isfinite(s[3])


def test_repeats_and_does_not_depend_on_the_batch():
    from rnc.metrics import flow_metrics
    flow, gt = sintel_batch(seed=2)
    valid = (torch.rand(8, 436, 1024, device=DEV) > 0.3).float()
    a, b = flow_metrics(flow, gt, valid), flow_metrics(flow, gt, valid)
    assert torch.equal(a.counts, b.counts) and torch.equal(a.epe_sum, b.epe_sum)
    for k in range(8):
        one = flow_metrics(flow[k:k + 1], gt[k:k + 1], valid[k:k + 1])
        assert torch.equal(one.counts[0], a.counts[k]) and torch.equal(one.epe_sum[0], a.epe_sum[k]), k
    rev = flow_metrics(flow.flip(0), gt.flip(0), valid.flip(0))
    assert torch.equal(rev.counts.flip(0), a.counts) and torch.equal(rev.epe_sum.flip(0), a.epe_sum)


@pytest.fixture
def det(monkeypatch):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


@pytest.mark.parametrize("sparse", [False, True])
def test_validate_equals_host_metrics_of_the_same_flows(sparse, det):
    from rnc.harness import validate
    from rnc.metrics import host_partials, summarize
    from utils.utils import InputPadder
    m = build_model("raft_nc_dbl").to(DEV)
    im1, im2 = frames(3, 436, 1024, seed=5)
    g = torch.Generator().manual_seed(6)
    gt = torch.randn(3, 2, 436, 1024, generator=g) * 2
    valid = (torch.rand(3, 436, 1024, generator=g) > 0.5).float() if sparse else None
    samples = [(im1[i], im2[i], gt[i]) + ((valid[i],) if sparse else ()) for i in range(3)]
    mode = "kitti" if sparse else "sintel"
    res = validate(m, samples, iters=2, mode=mode, batch_size=8)
    with torch.no_grad():
        padder = InputPadder(im1.shape, mode=mode)
        p1, p2 = padder.pad(im1.to(DEV), im2.to(DEV))
        _, flow_pr = m(p1, p2, iters=2, test_mode=True)
        flow = padder.unpad(flow_pr).cpu()
    want = summarize(host_partials(flow, gt, valid), mode)
    assert res.keys() == want.keys()
    for k in res:
        if k == "epe":
            assert res[k] == pytest.approx(want[k], rel=1e-12, abs=0)
        else:
            assert res[k] == want[k], k


def _nccl_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from rnc.harness import validate
        torch.use_deterministic_algorithms(True)
        res = validate(build_model("raft_nc_dbl").cuda(), nccl_samples(), iters=2, batch_size=1)
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def nccl_samples():
    im1, im2 = frames(5, 96, 160, seed=8)
    g = torch.Generator().manual_seed(9)
    return [(im1[i], im2[i], torch.randn(2, 96, 160, generator=g), (torch.rand(96, 160, generator=g) > 0.4).float())
            for i in range(5)]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
def test_nccl_two_ranks_equal_world_1(monkeypatch):
    from rnc.harness import validate
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        want = validate(build_model("raft_nc_dbl").to(DEV), nccl_samples(), iters=2, batch_size=1)
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
