"""Frame interpolation on the GPU (rnc_interpolate, rnc_interp_error): the kernels against the host oracle bit for bit, batch
independence, interpolate_frames and validate_interpolation against one-pair-at-a-time host loops, and rnc_boundary_dist2,
whose kernels the fill shares, against its host restatement."""
import pytest
import torch

from conftest import build_model
from rnc.harness import bidirectional_flow, interpolate_frames, validate_interpolation
from rnc.interp import (host_interpolate, host_interpolation_error, interpolate, interpolation_error, InterpPartials,
                        summarize_interpolation)
from rnc.metrics import boundary_dist2, fb_consistency, host_boundary_dist2
from rnc.synth import frames, shift_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def random_inputs(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    I0, I1 = torch.rand(B, 3, H, W, generator=g) * 255, torch.rand(B, 3, H, W, generator=g) * 255
    F = torch.randn(B, 2, H, W, generator=g) * 6
    G = -F + torch.randn(B, 2, H, W, generator=g)
    F[:, :, ::7, ::5] *= 40                                # targets far out of the frame
    F[0, 0, 3, 4] = float("nan")
    G[-1, 1, 5, 6] = float("inf")
    occ = (torch.rand(B, H, W, generator=g) < 0.2).to(torch.uint8)
    occ_bw = (torch.rand(B, H, W, generator=g) < 0.2).to(torch.uint8)
    I0[:, :, 2:6, 2:6] = 128.0                             # flat patches: ties of e
    I1[:, :, 2:6, 2:6] = 128.0
    return I0, I1, F, G, occ, occ_bw


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H,W", [(37, 53), (64, 96)])
def test_kernels_equal_the_host_oracle(B, H, W):
    cpu = random_inputs(B, H, W, seed=B * 100 + H)
    times = (0.25, 0.5, 0.75)
    want = host_interpolate(*cpu, times)
    got = interpolate(*(t.to(DEV) for t in cpu), times).cpu()
    bad = (got != want) & ~(torch.isnan(got) & torch.isnan(want))
    assert not bad.any(), f"{int(bad.sum())} of {bad.numel()} values differ"


def test_kernels_equal_the_oracle_on_strided_inputs_and_consistent_masks():
    H, W = 48, 80
    f = shift_sequence(3, H, W, seed=4)
    g = torch.Generator().manual_seed(5)
    F = (torch.randn(2, 2, H + 2, W + 4, generator=g) * 3)[..., 1:H + 1, 2:W + 2]      # strided views
    G = (torch.randn(2, 2, H + 2, W + 4, generator=g) * 3)[..., 1:H + 1, 2:W + 2]
    I0, I1 = torch.stack([f[0], f[1]]), torch.stack([f[2], f[0]])
    occ, occ_bw, _, _ = fb_consistency(F.to(DEV), G.to(DEV))
    got = interpolate(I0.to(DEV), I1.to(DEV), F.to(DEV), G.to(DEV), occ, occ_bw, (0.3, 0.5)).cpu()
    assert torch.equal(got, host_interpolate(I0, I1, F, G, occ.cpu(), occ_bw.cpu(), (0.3, 0.5)))


def test_each_image_is_the_same_alone():
    cpu = random_inputs(3, 40, 64, seed=9)
    dev = [t.to(DEV) for t in cpu]
    times = (0.5, 0.2)
    full = interpolate(*dev, times)
    for b in range(3):
        assert torch.equal(interpolate(*(t[b:b + 1] for t in dev), times)[0], full[b]), b
    err = interpolation_error(full[:, 0], dev[1])
    for b in range(3):
        one = interpolation_error(full[b:b + 1, 0], dev[1][b:b + 1])
        assert torch.equal(one.sq_sum[0], err.sq_sum[b]) and one.count[0] == err.count[b], b


def test_interpolation_error_agrees_with_the_host():
    g = torch.Generator().manual_seed(6)
    pred, gt = torch.rand(5, 3, 436, 1024, generator=g) * 255, torch.rand(5, 3, 436, 1024, generator=g) * 255
    got = interpolation_error(pred.to(DEV), gt.to(DEV))
    want = host_interpolation_error(pred, gt)
    torch.testing.assert_close(got.sq_sum.cpu(), want.sq_sum, rtol=1e-12, atol=0)
    assert torch.equal(got.count.cpu(), want.count)
    again = interpolation_error(pred.to(DEV)[[3, 1]], gt.to(DEV)[[3, 1]])
    assert torch.equal(again.sq_sum.cpu(), got.sq_sum.cpu()[[3, 1]])


def test_boundary_dist2_is_unchanged():
    g = torch.Generator().manual_seed(8)
    for B, H, W in ((2, 64, 96), (1, 436, 1024), (3, 1, 17), (2, 33, 1)):
        occ = (torch.nn.functional.interpolate(torch.rand(B, 1, max(H // 8, 1), max(W // 8, 1), generator=g),
                                               size=(H, W)) > 0.6).float()[:, 0]
        assert torch.equal(boundary_dist2(occ.to(DEV)).cpu(), host_boundary_dist2(occ)), (B, H, W)
    flat = torch.zeros(2, 20, 30)
    assert (boundary_dist2(flat.to(DEV)).cpu() == host_boundary_dist2(flat)).all()


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def test_interpolate_frames_is_bidirectional_flow_then_interpolate():
    m = build_model("raft_nc_dbl").to(DEV)
    f0, f1 = (x.to(DEV) for x in frames(2, 100, 180, seed=3))       # not a multiple of 8: padded and unpadded
    with torch.no_grad():
        got = interpolate_frames(m, f0, f1, times=(0.5, 0.25), iters=6)
        r = bidirectional_flow(m, f0, f1, 6)
        want = interpolate(f0, f1, r["flow_up"], r["flow_up_bw"], r["occ"], r["occ_bw"], (0.5, 0.25))
    assert got.shape == (2, 2, 3, 100, 180)
    # the same forward twice: equal up to the flow's run-to-run spread; bit for bit with the exact lookup (below)
    assert (got - want).abs().mean().item() < 1.0


def test_interpolate_frames_bit_for_bit_with_the_exact_lookup(monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft").to(DEV)
    f0, f1 = (x.to(DEV) for x in frames(1, 64, 96, seed=4))
    with torch.no_grad():
        got = interpolate_frames(m, f0, f1, times=(0.5,), iters=4)
        r = bidirectional_flow(m, f0, f1, 4)
    want = host_interpolate(f0.cpu(), f1.cpu(), r["flow_up"].cpu(), r["flow_up_bw"].cpu(), r["occ"].cpu(), r["occ_bw"].cpu())
    assert torch.equal(got.cpu(), want)


LENS = [3, 4, 6, 2, 5]
H, W, ITERS = 64, 128, 6


def sequences():
    return [[f.to(DEV) for f in shift_sequence(n, H, W, seed=s, dy=1, dx=2)] for s, n in enumerate(LENS)]


@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_validate_interpolation_is_the_triplet_loop_for_any_batch_size(name, monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model(name).to(DEV)
    seqs = sequences()
    res = {bs: validate_interpolation(m, seqs, ITERS, batch_size=bs, device=DEV) for bs in (1, 3, 8)}
    assert res[1] == res[3] == res[8], res
    parts = []
    with torch.no_grad():
        for seq in seqs:
            for k in range(len(seq) - 2):
                r = bidirectional_flow(m, seq[k][None], seq[k + 2][None], ITERS)
                pred = host_interpolate(seq[k][None].cpu(), seq[k + 2][None].cpu(), r["flow_up"].cpu(),
                                        r["flow_up_bw"].cpu(), r["occ"].cpu(), r["occ_bw"].cpu())
                parts.append(host_interpolation_error(pred[:, 0], seq[k + 1][None].cpu()))
    want = summarize_interpolation(InterpPartials(torch.cat([p.sq_sum for p in parts]), torch.cat([p.count for p in parts])))
    assert res[1]["frames"] == want["frames"] == sum(n - 2 for n in LENS if n >= 3)
    assert abs(res[1]["ie"] - want["ie"]) <= 1e-12 * want["ie"] and abs(res[1]["psnr"] - want["psnr"]) <= 1e-10, (res[1], want)
    print(f"{name}: {res[1]}")


def test_validate_interpolation_warm_does_not_depend_on_batch_size(monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft_nc_dbl").to(DEV)
    seqs = sequences()
    a = validate_interpolation(m, seqs, ITERS, batch_size=2, warm_start=True, device=DEV)
    b = validate_interpolation(m, seqs, ITERS, batch_size=8, warm_start=True, device=DEV)
    assert a == b and a["frames"] == sum(n - 2 for n in LENS if n >= 3)
