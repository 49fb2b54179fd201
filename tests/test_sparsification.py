"""Confidence evaluation on the host: host_sparsification against an independent numpy restatement of the definition (ties,
invalid pixels, empty images, N around 100, NaN and inf scores and flows, strided views), summarize_sparsification on
hand-built partials, confidence_score, validate(confidence=True) with a stub model at several batch sizes and under gloo at
world sizes 2 and 3, and the argument checks of the Python functions and of rnc_sparsification."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from test_flow_metrics import CSRC, ROOT, run_ranks

K = 100
U = 2.0 ** -53


def numpy_sparsification(flow, gt, valid, score):
    """The definition in numpy: float32 EPE, valid pixels ranked by np.lexsort on (index, score) with NaN first (by score
    ascending, and by EPE descending for the ideal), sums of what is kept in exact arithmetic (math.fsum)."""
    flow, gt, score = (np.asarray(t, dtype=np.float32) for t in (flow, gt, score))
    B = flow.shape[0]
    count = np.zeros((B, K), np.int64)
    kept = np.zeros((B, K))
    ideal = np.zeros((B, K))
    for b in range(B):
        d = flow[b] - gt[b]
        epe = np.sqrt(d[0] * d[0] + d[1] * d[1]).ravel()
        val = np.ones(epe.shape, bool) if valid is None else (np.asarray(valid[b], np.float32) >= 0.5).ravel()
        idx = np.flatnonzero(val)
        n = idx.size
        if n == 0:
            continue
        e = epe[idx].astype(np.float64)
        s = score[b].ravel()[idx].astype(np.float64)
        m = np.arange(K) * n // K
        count[b] = n - m
        for out, key in ((kept, s), (ideal, -e)):
            nan = np.isnan(key)
            order = np.lexsort((idx, np.where(nan, 0.0, key), ~nan))    # last key first: NaN, then the value, then the index
            ranked = e[order]
            out[b] = [math.fsum(ranked[mk:]) if np.isfinite(ranked[mk:]).all() else float(np.sum(ranked[mk:])) for mk in m]
    return count, kept, ideal


def assert_sums_close(got, want, terms, magnitudes):
    """got and want are fp64 sums of the same `terms` numbers: each differs from the exact sum by at most (terms - 1) * u *
    sum|x| (Higham, any order of a recursive sum), so they differ from each other by at most twice that.  Non-finite sums
    must be the same non-finite value."""
    got, want = torch.as_tensor(got, dtype=torch.float64), torch.as_tensor(want, dtype=torch.float64)
    finite = torch.isfinite(want)
    assert torch.equal(torch.isfinite(got), finite)
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    assert torch.equal(got[torch.isinf(want)], want[torch.isinf(want)])
    bound = 2 * (torch.as_tensor(terms, dtype=torch.float64) - 1).clamp(min=0) * U * torch.as_tensor(magnitudes, dtype=torch.float64)
    assert bool(((got - want).abs() <= bound)[finite].all()), float(((got - want).abs() - bound)[finite].max())


def check_host(flow, gt, valid, score):
    from rnc.metrics import host_sparsification
    p = host_sparsification(flow, gt, valid, score)
    count, kept, ideal = numpy_sparsification(flow, gt, valid, score)
    assert p.count.dtype == torch.int64 and p.kept_epe.dtype == torch.float64 and p.count.shape == (flow.shape[0], K)
    assert np.array_equal(p.count.numpy(), count)
    # a bound on each sum's magnitude: the tail of the valid EPEs in either order is at most their total
    _, tot, _ = numpy_sparsification(flow, gt, valid, torch.zeros_like(score))
    mags = np.where(np.isfinite(tot[:, :1]), tot[:, :1], 0.0) * np.ones((1, K))
    assert_sums_close(p.kept_epe, kept, count, mags)
    assert_sums_close(p.ideal_epe, ideal, count, mags)
    return p


def rand(shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def test_heavily_tied_scores_with_invalid_pixels():
    flow, gt = rand((3, 2, 17, 23), 1, 4), rand((3, 2, 17, 23), 2, 4)
    score = torch.floor(torch.rand(3, 17, 23, generator=torch.Generator().manual_seed(3)) * 4) / 4    # 4 levels
    valid = (torch.rand(3, 17, 23, generator=torch.Generator().manual_seed(4)) > 0.3).float()
    valid[1] = 0                                                                   # an image without a valid pixel
    p = check_host(flow, gt, valid, score)
    assert p.count[1].tolist() == [0] * K and p.kept_epe[1].tolist() == [0.0] * K and p.ideal_epe[1].tolist() == [0.0] * K
    check_host(flow, gt, None, score)
    # kept pixels at k = 0 are all of them, in either order: the flow metrics' sum
    from rnc.metrics import host_partials
    h = host_partials(flow, gt, valid)
    assert torch.equal(p.count[:, 0], h.counts[:, 0])
    torch.testing.assert_close(p.kept_epe[:, 0], h.epe_sum, rtol=1e-12, atol=0)
    torch.testing.assert_close(p.ideal_epe[:, 0], h.epe_sum, rtol=1e-12, atol=0)


@pytest.mark.parametrize("n", [1, 99, 100, 101])
def test_valid_counts_around_the_fraction_count(n):
    from rnc.metrics import host_sparsification
    flow, gt = rand((1, 2, 13, 17), n, 3), rand((1, 2, 13, 17), n + 1, 3)
    score = rand((1, 13, 17), n + 2)
    valid = torch.zeros(1, 13 * 17)
    valid[0, torch.randperm(13 * 17, generator=torch.Generator().manual_seed(n))[:n]] = 1
    valid = valid.view(1, 13, 17)
    p = check_host(flow, gt, valid, score)
    assert p.count[0].tolist() == [n - k * n // K for k in range(K)]
    assert int(p.count.min()) >= 1                                               # at least one pixel is kept
    if n == 1:
        assert torch.equal(p.kept_epe, p.ideal_epe)
    one = host_sparsification(flow, gt, valid, score)
    assert torch.equal(one.kept_epe, p.kept_epe) and torch.equal(one.ideal_epe, p.ideal_epe)


def test_nan_and_inf_scores_and_flows():
    flow, gt = rand((2, 2, 11, 13), 5, 4), rand((2, 2, 11, 13), 6, 4)
    score = torch.floor(rand((2, 11, 13), 7, 2))
    score[0, 0, :4] = float("nan")
    score[0, 1, :3] = float("inf")
    score[0, 2, :3] = -float("inf")
    score[0, 3, :6] = torch.tensor([0.0, -0.0, 0.0, -0.0, -0.0, 0.0])             # -0 and +0 tie: index order
    score[1, 5, 5] = float("nan")
    flow[0, 0, 4, 4] = float("nan")                                              # a NaN EPE: first in the ideal order
    flow[0, 1, 6, 2] = float("inf")
    flow[1, 0, 9, 9] = float("inf")
    flow[1, 1, 9, 10] = float("inf")
    valid = torch.ones(2, 11, 13)
    valid[1, 9, 10] = 0                                                          # an invalid inf does not count
    p = check_host(flow, gt, valid, score)
    assert math.isnan(p.kept_epe[0, 0]) and math.isnan(p.ideal_epe[0, 0])
    assert math.isfinite(p.ideal_epe[0, 2]) and math.isinf(p.ideal_epe[0, 1])  # NaN removed first, then the inf
    assert math.isfinite(p.ideal_epe[1, 1]) and math.isinf(p.ideal_epe[1, 0])
    check_host(flow, gt, None, score)


def test_strided_views():
    base = rand((3, 19, 29, 2), 8, 5)
    flow = base.permute(0, 3, 1, 2)                                            # channel-last storage
    gt = rand((3, 2, 23, 29), 9, 5)[:, :, 2:21]                                # an unpadded view
    score = rand((3, 29, 19), 10).transpose(1, 2)
    valid = (rand((3, 19, 58), 11) > -0.5).float()[:, :, ::2]
    assert not (flow.is_contiguous() or gt.is_contiguous() or score.is_contiguous() or valid.is_contiguous())
    from rnc.metrics import host_sparsification
    p = check_host(flow, gt, valid, score)
    c = host_sparsification(flow.contiguous(), gt.contiguous(), valid.contiguous(), score.contiguous())
    assert all(torch.equal(a, b) for a, b in zip(p, c))


def test_summarize_hand_built_partials():
    from rnc.metrics import SparsPartials, summarize_sparsification
    k = torch.arange(K, dtype=torch.float64)
    ca, cb = 100 - torch.arange(K), 200 - 2 * torch.arange(K)                 # N = 100 and 200
    count = torch.stack([ca, torch.zeros(K, dtype=torch.int64), cb])          # the empty middle image does not count
    kept = torch.stack([3.0 * ca, torch.zeros(K), cb * (1 + 2 * k / 100)])     # per-image curves 3 and 1 + 2k/100
    ideal = torch.stack([1.0 * ca, torch.zeros(K), 1.0 * cb])                # ideal curves 1 and 1
    s = summarize_sparsification(SparsPartials(count, kept, ideal))
    assert list(s) == ["sparsification", "ideal", "ause"]
    assert s["sparsification"] == pytest.approx([2 + kk / 100 for kk in range(K)], rel=1e-15)
    assert s["ideal"] == [1.0] * K
    # sparsification - ideal = 1 + f_k on f_k = 0, 0.01, ..., 0.99: the trapezoid rule is exact on a line,
    # 0.99 * (1 + 1.99) / 2 = 1.48005
    assert s["ause"] == pytest.approx(1.48005, rel=1e-13)
    empty = summarize_sparsification(SparsPartials(count[1:2], kept[1:2], ideal[1:2]))
    assert math.isnan(empty["ause"]) and all(math.isnan(v) for v in empty["sparsification"] + empty["ideal"])


def test_confidence_score_is_the_float32_harmonic_mean():
    from rnc.metrics import confidence_score
    g = np.random.default_rng(3)
    c = g.random((2, 2, 7, 9)).astype(np.float32)
    c[0, :, 0, 0] = 0                                                        # c_u + c_v == 0: score 0
    c[1, 0, 1, 1] = 0                                                        # one plane 0: harmonic mean 0
    c[1, :, 2, 2] = [1e-30, 3e-30]
    with np.errstate(invalid="ignore"):
        want = np.where(c[:, 0] + c[:, 1] == 0, np.float32(0), (np.float32(2) * c[:, 0] * c[:, 1]) / (c[:, 0] + c[:, 1]))
    got = confidence_score(torch.from_numpy(c))
    assert got.dtype == torch.float32 and got.shape == (2, 7, 9)
    assert np.array_equal(got.numpy(), want.astype(np.float32))
    assert got[0, 0, 0] == 0 and got[1, 1, 1] == 0
    with pytest.raises(ValueError):
        confidence_score(torch.zeros(2, 3, 4, 5))


# ----------------------------------------------------------------------------- validate


class ConfStub(torch.nn.Module):
    """Flow = the first two channels of image1 - image2; confidence = image1's third channel and image2's, quantised (ties)."""

    def __init__(self):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))

    def forward(self, im1, im2, iters=12, test_mode=True, flow_init=None, return_confidence=False):
        flow = im1[:, :2] - im2[:, :2]
        if not return_confidence:
            return flow[:, :, ::8, ::8], flow
        conf = torch.stack([im1[:, 2], im2[:, 2]], 1).div(6).mul(8).floor().div(8)
        return flow[:, :, ::8, ::8], flow, conf


def conf_samples(sparse):
    from test_flow_metrics import stub_samples
    return stub_samples(sparse)


def expected(samples, sparse):
    from rnc.metrics import SparsPartials, confidence_score, host_sparsification, summarize_sparsification
    parts = []
    for s in samples:
        a, b, gt = s[0][None], s[1][None], s[2][None]
        _, flow, conf = ConfStub()(a, b, return_confidence=True)
        parts.append(host_sparsification(flow, gt, s[3][None] if sparse else None, confidence_score(conf)))
    return summarize_sparsification(SparsPartials(*(torch.cat(c) for c in zip(*parts))))


def per_image_mean_epe(samples, sparse):
    from rnc.metrics import host_partials
    means = []
    for s in samples:
        p = host_partials((s[0][:2] - s[1][:2])[None], s[2][None], s[3][None] if sparse else None)
        means.append(p.epe_sum[0].item() / p.counts[0, 0].item())
    return sum(means) / len(means)


@pytest.mark.parametrize("sparse", [False, True])
def test_validate_confidence_equals_the_host_definition(sparse):
    from rnc.harness import validate
    samples = conf_samples(sparse)
    want = expected(samples, sparse)
    plain = validate(ConfStub(), samples, iters=1, batch_size=3, device="cpu")
    assert set(plain) == ({"epe", "1px", "3px", "5px", "f1"} if sparse else {"epe", "1px", "3px", "5px"})
    for bs in (1, 7):
        res = validate(ConfStub(), samples, iters=1, batch_size=bs, device="cpu", confidence=True)
        assert {k: res[k] for k in plain} == plain                               # the existing keys, bit for bit
        assert res["sparsification"] == want["sparsification"] and res["ideal"] == want["ideal"]
        assert res["ause"] == want["ause"]
        assert len(res["sparsification"]) == K and res["ause"] > 0
        assert all(o <= s + 1e-12 for o, s in zip(res["ideal"], res["sparsification"]))
        assert res["sparsification"][0] == pytest.approx(per_image_mean_epe(samples, sparse), rel=1e-12)
        if sparse:
            assert res["sparsification"][0] == pytest.approx(plain["epe"], rel=1e-12)      # KITTI-style: the same mean


def test_validate_without_confidence_is_unchanged():
    from rnc.harness import validate
    from test_flow_metrics import Stub, assert_matches_reference, reference_metrics
    samples = conf_samples(True)
    res = validate(Stub(), samples, iters=1, mode="kitti", batch_size=4, device="cpu")
    assert list(res) == ["epe", "1px", "3px", "5px", "f1"]
    want = reference_metrics([a[:2] - b[:2] for a, b, *_ in samples], [s[2] for s in samples], [s[3] for s in samples])
    assert_matches_reference(res, want)


def _validate_worker(rank, world, port, sparse, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from rnc.harness import validate
        q.put((rank, validate(ConfStub(), conf_samples(sparse), iters=1, batch_size=2, device="cpu", confidence=True)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,sparse", [(2, True), (3, False)])
def test_validate_confidence_gloo_equals_world_1(world, sparse):
    from rnc.harness import validate
    want = validate(ConfStub(), conf_samples(sparse), iters=1, batch_size=2, device="cpu", confidence=True)
    for got in run_ranks(_validate_worker, world, sparse):
        assert got == want                                       # bit for bit, on every rank


# ----------------------------------------------------------------------------- argument checks and the C ABI


def test_python_entry_points_check_their_arguments():
    from rnc import native
    from rnc.metrics import sparsification
    f = torch.zeros(2, 2, 4, 5)
    n0 = native.launch_count()
    for args in ((f, f, None, torch.zeros(2, 5, 4)), (f, f, None, torch.zeros(1, 4, 5)), (f, f, None, None),
                 (f, torch.zeros(2, 2, 4, 6), None, torch.zeros(2, 4, 5)), (f, f, torch.zeros(2, 5, 4), torch.zeros(2, 4, 5)),
                 (torch.zeros(2, 3, 4, 5), torch.zeros(2, 3, 4, 5), None, torch.zeros(2, 4, 5))):
        with pytest.raises(ValueError):
            sparsification(*args)
    assert native.launch_count() == n0


def test_entry_point_rejects_bad_arguments():
    from rnc import native
    L = native.lib()
    ws = L.rnc_sparsification_workspace_bytes(8, 436, 1024)
    n = 8 * 436 * 1024
    assert ws >= n * (4 * 8 + 2 * 4) + (1 << 20) + n * 4
    assert L.rnc_sparsification_workspace_bytes(1, 1, 1) > 0
    assert L.rnc_sparsification_workspace_bytes(0, 4, 5) == 0 and L.rnc_sparsification_workspace_bytes(2, -1, 5) == 0
    assert L.rnc_sparsification_workspace_bytes(65536, 4, 5) == 0
    assert L.rnc_sparsification_workspace_bytes(1, 1 << 15, 1 << 15) == 0       # H*W too large for the key
    assert L.rnc_sparsification_workspace_bytes(4, 1 << 14, 1 << 15) == 0      # B*H*W beyond the sort's index range
    assert L.rnc_sparsification_workspace_bytes(1, 1 << 14, 1 << 15) > 0
    P = 1 << 20   # never dereferenced: every check fails on the host before a launch
    n0 = L.rnc_launch_count()

    def call(B=8, H=436, W=1024, flow=P, gt=P, valid=P, score=P, count=P, kept=P, orc=P, wsp=P, wsb=ws):
        return L.rnc_sparsification(flow, 40, 20, 5, 1, gt, 40, 20, 5, 1, valid, 20, 5, 1, score, 20, 5, 1, B, H, W, count, kept,
                                    orc, wsp, wsb, None)

    assert call(B=0) == -1 and call(B=-2) == -1 and call(H=0) == -1 and call(W=-1) == -1 and call(B=65536) == -1
    assert call(H=1 << 15, W=1 << 15) == -1 and call(B=4, H=1 << 14, W=1 << 15) == -1
    assert call(flow=0) == -2 and call(gt=0) == -2 and call(score=0) == -2 and call(count=0) == -2
    assert call(kept=0) == -2 and call(orc=0) == -2 and call(wsp=0) == -2
    assert call(flow=P + 2) == -2 and call(gt=P + 1) == -2 and call(valid=P + 2) == -2 and call(score=P + 2) == -2
    assert call(count=P + 4) == -2 and call(kept=P + 4) == -2 and call(orc=P + 4) == -2 and call(wsp=P + 8) == -2
    assert call(wsb=ws - 1) == -5 and call(valid=0, wsb=0) == -5
    assert L.rnc_launch_count() == n0


def test_sparsification_cu_does_not_spill(tmp_path):
    from rnc.build import ARCH, nvcc_path
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-c", os.path.join(CSRC, "sparsification.cu"), "-o", str(tmp_path / "s.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    ours = re.findall(r"Function properties for \S*(spars_\w+_kernel)", log)
    assert sorted(ours) == ["spars_keys_kernel", "spars_range_kernel", "spars_suffix_kernel"], ours
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)      # ours and the radix sort's
    assert len(spills) > 3 and all(a == "0" and b == "0" for a, b in spills), spills
