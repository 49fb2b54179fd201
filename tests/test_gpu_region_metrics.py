"""Per-region validation metrics on the GPU: rnc_boundary_dist2 equals the exact host transform integer for integer, and
rnc_region_metrics' partials equal the host's (counts exactly, sums to 1e-12) at the Chairs, Sintel and KITTI shapes, through
strided views and at the edges of test_flow_metrics.edge_case; both repeat bit for bit and do not depend on the batch;
validate(regions=True) on raft_nc_dbl equals the host region metrics of the same flows and keeps its other keys; and two
NCCL ranks give the single-process dict when two GPUs are visible."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import build_model, frames
from test_flow_metrics import edge_case
from test_region_metrics import same

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def occ_masks(B, H, W, seed):
    """Occluded discs of different sizes (the boundary distances reach past the last bin) plus speckle, and one image
    without a boundary when B > 2."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H, device=DEV), torch.arange(W, device=DEV), indexing="ij")
    occ = torch.stack([((yy - H / 2) ** 2 + (xx - W * (b + 1) / (B + 1)) ** 2 < (H / (3 + b)) ** 2).float() for b in range(B)])
    occ = torch.maximum(occ, (torch.rand(B, H, W, device=DEV, generator=g) > 0.9995).float())
    if B > 2:
        occ[2] = 0
    return occ


def check_dist2(occ):
    from rnc.metrics import boundary_dist2, host_boundary_dist2
    d = boundary_dist2(occ)
    assert d.is_cuda and d.dtype == torch.int32
    assert torch.equal(d.cpu(), host_boundary_dist2(occ.cpu()))
    return d


def check(flow, gt, valid=None, **masks):
    from rnc.metrics import host_region_partials, region_partials
    p = region_partials(flow, gt, valid, **masks)
    h = host_region_partials(flow.cpu(), gt.cpu(), None if valid is None else valid.cpu(),
                             **{k: v.cpu() for k, v in masks.items()})
    assert p.counts.is_cuda and p.counts.shape == h.counts.shape
    assert torch.equal(p.counts.cpu(), h.counts)
    torch.testing.assert_close(p.epe_sum.cpu(), h.epe_sum, rtol=1e-12, atol=0, equal_nan=True)
    assert torch.equal(p.fg, h.fg)
    return p


@pytest.mark.parametrize("B,H,W", [(2, 384, 512), (3, 436, 1024), (2, 376, 1242), (3, 1, 1), (2, 1, 700), (2, 700, 1),
                                   (1, 4096, 37)])
def test_dist2_equals_host(B, H, W):
    d = check_dist2(occ_masks(B, H, W, seed=H + W))
    if B > 2:
        assert (d[2] == 2 ** 31 - 1).all()                 # the image without a boundary


def test_dist2_through_strided_views_and_repeats():
    occ = occ_masks(4, 436, 1024, seed=1)
    a = check_dist2(occ)
    assert torch.equal(check_dist2(occ.transpose(1, 2).contiguous().transpose(1, 2)), a)     # column-major storage
    padded = torch.zeros(4, 440, 1030, device=DEV)
    padded[:, 2:438, 3:1027] = occ
    assert torch.equal(check_dist2(padded[:, 2:438, 3:1027]), a)
    from rnc.metrics import boundary_dist2
    assert torch.equal(boundary_dist2(occ), a) and torch.equal(boundary_dist2(occ[1:2]), a[1:2])


def sintel_batch(B=4, seed=0):
    """Flows read through the unpadded view of a padded 440-row batch, as validate hands them over."""
    from utils.utils import InputPadder
    g = torch.Generator(device=DEV).manual_seed(seed)
    flow_up = torch.randn(B, 2, 440, 1024, device=DEV, generator=g) * 15
    view = InputPadder((3, 436, 1024)).unpad(flow_up)
    gt = view.detach().clone() + torch.randn(B, 2, 436, 1024, device=DEV, generator=g) * 3
    return view, gt


def test_sintel_regions_equal_host():
    flow, gt = sintel_batch()
    occ = occ_masks(4, 436, 1024, seed=2)
    check(flow, gt, occ=occ)
    valid = (torch.rand(4, 436, 1024, device=DEV) > 0.1).float()
    p = check(flow, gt, valid, occ=occ)
    from rnc.metrics import flow_metrics
    assert torch.equal(p.counts.sum(1), flow_metrics(flow, gt, valid).counts)


def test_kitti_regions_equal_host():
    g = torch.Generator(device=DEV).manual_seed(3)
    gt = torch.randn(3, 2, 376, 1242, device=DEV, generator=g) * 20
    flow = gt + torch.randn(3, 2, 376, 1242, device=DEV, generator=g) * 4
    valid = (torch.rand(3, 376, 1242, device=DEV, generator=g) > 0.8).float()
    noc = valid * (torch.rand(3, 376, 1242, device=DEV, generator=g) > 0.2).float()
    fg = occ_masks(3, 376, 1242, seed=4)
    check(flow, gt, valid, noc=noc, fg=fg)
    check(flow, gt, valid, noc=noc)
    # channel-last flow storage, a transposed fg
    check(flow.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2), gt, valid, noc=noc,
          fg=fg.transpose(1, 2).contiguous().transpose(1, 2))


@pytest.mark.parametrize("B,H,W", [(1, 384, 512), (8, 384, 512), (3, 37, 53), (2, 1, 2049)])
def test_chairs_and_odd_sizes_equal_host(B, H, W):
    g = torch.Generator(device=DEV).manual_seed(B * H + W)
    gt = torch.randn(B, 2, H, W, device=DEV, generator=g) * 25
    flow = gt + torch.randn(B, 2, H, W, device=DEV, generator=g) * 2
    check(flow, gt, occ=occ_masks(B, H, W, seed=5))


def test_edge_values_equal_host():
    flow, gt, valid = (t.to(DEV) for t in edge_case())
    flow[0, 0, 2, 5] = float("nan")
    gt[0, 1, 3, 0] = float("nan")
    flow[0, 1, 3, 1] = float("inf")
    occ = torch.zeros(2, 4, 6, device=DEV)
    occ[0, :, 3:] = 1
    check(flow, gt, valid, occ=occ)
    check(flow, gt, occ=occ)
    check(flow, gt, valid, noc=1 - occ, fg=occ)


def test_repeats_and_does_not_depend_on_the_batch():
    from rnc.metrics import region_partials
    flow, gt = sintel_batch(seed=6)
    occ = occ_masks(4, 436, 1024, seed=7)
    valid = (torch.rand(4, 436, 1024, device=DEV) > 0.3).float()
    a, b = region_partials(flow, gt, valid, occ=occ), region_partials(flow, gt, valid, occ=occ)
    assert torch.equal(a.counts, b.counts) and torch.equal(a.epe_sum, b.epe_sum)
    for k in range(4):
        one = region_partials(flow[k:k + 1], gt[k:k + 1], valid[k:k + 1], occ=occ[k:k + 1])
        assert torch.equal(one.counts[0], a.counts[k]) and torch.equal(one.epe_sum[0], a.epe_sum[k]), k
    rev = region_partials(flow.flip(0), gt.flip(0), valid.flip(0), occ=occ.flip(0))
    assert torch.equal(rev.counts.flip(0), a.counts) and torch.equal(rev.epe_sum.flip(0), a.epe_sum)


@pytest.fixture
def det(monkeypatch):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def model_samples(sparse, n=3, H=436, W=1024, seed=5):
    im1, im2 = frames(n, H, W, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    gt = torch.randn(n, 2, H, W, generator=g) * 2
    occ = occ_masks(n, H, W, seed=seed).cpu()
    out = []
    for i in range(n):
        if sparse:
            valid = (torch.rand(H, W, generator=g) > 0.5).float()
            out.append((im1[i], im2[i], gt[i], valid, {"noc": valid * (torch.rand(H, W, generator=g) > 0.2), "fg": occ[i]}))
        else:
            out.append((im1[i], im2[i], gt[i], None, {"occ": occ[i]}))
    return out


@pytest.mark.parametrize("sparse", [False, True])
def test_validate_regions_equals_host_of_the_same_flows(sparse, det):
    from rnc.harness import validate
    from rnc.metrics import host_region_partials, summarize_regions
    from utils.utils import InputPadder
    m = build_model("raft_nc_dbl").to(DEV)
    samples = model_samples(sparse)
    mode = "kitti" if sparse else "sintel"
    plain = validate(m, [s[:4] for s in samples], iters=2, mode=mode, batch_size=8)
    res = validate(m, samples, iters=2, mode=mode, batch_size=8, regions=True)
    assert {k: res[k] for k in plain} == plain                              # the old keys, bit for bit
    im1, im2 = torch.stack([s[0] for s in samples]), torch.stack([s[1] for s in samples])
    with torch.no_grad():
        padder = InputPadder(im1.shape, mode=mode)
        p1, p2 = padder.pad(im1.to(DEV), im2.to(DEV))
        flow = padder.unpad(m(p1, p2, iters=2, test_mode=True)[1]).cpu()
    masks = {k: torch.stack([s[4][k] for s in samples]) for k in samples[0][4]}
    valid = torch.stack([s[3] for s in samples]) if sparse else None
    want = summarize_regions(host_region_partials(flow, torch.stack([s[2] for s in samples]), valid, **masks))
    got = {k: res[k] for k in res if k not in plain}
    assert got.keys() == want.keys() and got["region_pixels"] == want["region_pixels"]
    for k in want:
        if k.startswith("fl_"):
            assert got[k] == want[k], k
        elif k != "region_pixels":
            assert got[k] == pytest.approx(want[k], rel=1e-12, abs=0, nan_ok=True), k
    if sparse:
        assert res["fl_all"] == res["f1"]


def test_validate_regions_with_consistency_scores_the_occlusions(det):
    from rnc.harness import validate
    from rnc.metrics import host_fb_consistency, summarize_occlusion
    from utils.utils import InputPadder
    m = build_model("raft_nc_dbl").to(DEV)
    samples = model_samples(False, n=2, H=96, W=160, seed=9)
    plain = validate(m, [s[:4] for s in samples], iters=2, batch_size=8, consistency=True)
    res = validate(m, samples, iters=2, batch_size=8, consistency=True, regions=True)
    assert {k: res[k] for k in plain} == plain
    im1, im2 = torch.stack([s[0] for s in samples]), torch.stack([s[1] for s in samples])
    with torch.no_grad():
        padder = InputPadder(im1.shape)
        p1, p2 = padder.pad(im1.to(DEV), im2.to(DEV))
        fw = padder.unpad(m(p1, p2, iters=2, test_mode=True)[1]).cpu()
        bw = padder.unpad(m(p2, p1, iters=2, test_mode=True)[1]).cpu()
    pred = host_fb_consistency(fw, bw)[0] != 0
    occ = torch.stack([s[4]["occ"] for s in samples]) >= 0.5
    rows = torch.stack([(pred & occ).sum((1, 2)), pred.sum((1, 2)), occ.sum((1, 2))], 1)
    assert {k: res[k] for k in ("occ_precision", "occ_recall", "occ_f1")} == summarize_occlusion(rows)


def _nccl_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RNC_LOOKUP="ffma")
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from rnc.harness import validate
        torch.use_deterministic_algorithms(True)
        res = validate(build_model("raft_nc_dbl").cuda(), nccl_samples(), iters=2, batch_size=1, regions=True)
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def nccl_samples():
    return model_samples(False, n=5, H=96, W=160, seed=8)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
def test_nccl_two_ranks_equal_world_1(monkeypatch):
    from rnc.harness import validate
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        want = validate(build_model("raft_nc_dbl").to(DEV), nccl_samples(), iters=2, batch_size=1, regions=True)
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
    assert same(got[0], want) and same(got[1], want)
