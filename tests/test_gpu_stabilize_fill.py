"""Full-frame video stabilization on the GPU (csrc/stabilize_fill.cu): the residual transfer and the global re-add against
their host restatements bit for bit, on strided inputs, non-finite flows and maps that send points to w <= 0;
stabilize_videos(fill=True) against fill=False and against the host pipeline fed the flows run_sequences_bidirectional
yields; batch independence and determinism; validate_stabilization(fill=True) end to end."""
import numpy as np
import pytest
import torch

from conftest import build_model
from rnc.harness import run_sequences_bidirectional, stabilize_videos, validate_stabilization
from rnc.inpaint import SOURCE_KNOWN
from rnc.stabilize import (_inv, add_global_motion, flow_residual, host_add_global_motion, host_fill_uncovered,
                           host_flow_residual, host_smooth_path)
from rnc.synth import shaky_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def same(got, want):
    """Equal bits, NaN where NaN (a NaN's payload is not part of the rule)."""
    got = got.cpu()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(got[~nan].view(torch.int32), want[~nan].view(torch.int32))


def inputs(V, T, H, W, seed, perspective=False):
    """Flows [V,T-1,2,H,W] as strided views of a channel-last stack with NaN and +-inf values, motions near the identity,
    and maps of a zoom, roll and shift (with perspective that sends part of the frame to w <= 0 when asked)."""
    g = np.random.default_rng(seed)
    flows = []
    for _ in range(2):
        f = g.normal(0, 3, (V, T - 1, H, W, 2)).astype(np.float32)
        bad = g.random((V, T - 1, H, W))
        f[..., 0][bad < 0.01] = np.nan
        f[..., 1][(bad >= 0.01) & (bad < 0.015)] = np.inf
        f[..., 0][(bad >= 0.015) & (bad < 0.02)] = -np.inf
        flows.append(torch.from_numpy(f).permute(0, 1, 4, 2, 3))               # channel-last storage, [V,T-1,2,H,W] view
    A = np.tile(np.eye(3), (V, T - 1, 1, 1))
    A[..., :2, :2] += g.normal(0, 0.01, (V, T - 1, 2, 2))
    A[..., :2, 2] = g.normal(0, 3, (V, T - 1, 2))
    A[..., 2, :2] = g.normal(0, 1e-5, (V, T - 1, 2))
    M = np.tile(np.eye(3), (V, T, 1, 1))
    M[..., :2, :2] = g.uniform(0.9, 1.3) * np.eye(2) + g.normal(0, 0.02, (V, T, 2, 2))
    M[..., :2, 2] = g.normal(0, 4, (V, T, 2))
    if perspective:
        M[..., 2, 0] = g.choice([-1, 1], (V, T)) * 3.0 / W                   # w = 0 crosses the frame
    M = M / M[..., 2:3, 2:3]
    Minv = _inv(M)
    return (*flows, *(torch.from_numpy(x) for x in (A, M, Minv)))


@pytest.mark.parametrize("V,T,H,W,perspective", [(1, 2, 8, 8, False), (2, 3, 13, 37, True), (1, 3, 64, 96, True),
                                                 (1, 2, 480, 854, False), (1, 2, 375, 1242, True)])
def test_the_transfer_and_the_readd_equal_the_host_restatements(V, T, H, W, perspective):
    f, b, A, M, Mi = inputs(V, T, H, W, seed=H + W, perspective=perspective)
    got = flow_residual(*(t.to(DEV) for t in (f, b, A, M, Mi)))
    want = host_flow_residual(f, b, A, M, Mi)
    for g, w in zip(got, want):
        same(g, w)
    if perspective:
        assert bool(torch.isnan(want[0]).any()) and bool(torch.isfinite(want[0]).any())
    # the re-add of a residual with NaNs and values, on a strided view
    r = torch.where(torch.isnan(want[0]), torch.full_like(want[0], 0.25), want[0]).transpose(-1, -2).contiguous()
    r = r.transpose(-1, -2)
    got = add_global_motion(r.to(DEV), want[1].to(DEV), A.to(DEV), M.to(DEV), Mi.to(DEV))
    want = host_add_global_motion(r, want[1], A, M, Mi)
    for g, w in zip(got, want):
        same(g, w)


H, W, ITERS = 64, 128, 6
KW = dict(radius=4, sigma=2.0, stride=4, hypotheses=64)
FILL = dict(fill=True, sweeps=32, crop=False)


def split():
    return [[f.to(DEV) for f in shaky_sequence(n, H, W, seed=s)[0]] for s, n in enumerate((5, 3, 6))]


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def test_stabilize_videos_fill_keeps_fill_false_and_is_the_host_pipeline(monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft_nc_dbl").to(DEV)
    seqs = split()
    with torch.no_grad():
        rows = {(s, k): r for s, k, r in run_sequences_bidirectional(m, seqs, ITERS, batch_size=3, device=DEV)}
        plain = stabilize_videos(m, seqs, ITERS, batch_size=3, device=DEV, crop=False, **KW)
        got = stabilize_videos(m, seqs, ITERS, batch_size=3, device=DEV, **FILL, **KW)
        again = stabilize_videos(m, seqs, ITERS, batch_size=2, device=DEV, **FILL, **KW)
        alone = [stabilize_videos(m, [seq], ITERS, batch_size=1, device=DEV, **FILL, **KW)[0] for seq in seqs]
    holes = 0
    for s, (seq, r, p) in enumerate(zip(seqs, got, plain)):
        for key in ("motion", "transforms", "alpha", "inliers", "matched", "status", "valid"):
            assert torch.equal(r[key], p[key]), (s, key)
        v = r["valid"] != 0
        assert torch.equal(r["source"] == SOURCE_KNOWN, v)
        assert torch.equal(r["frames"][v[:, None].expand_as(r["frames"])], p["frames"][v[:, None].expand_as(p["frames"])])
        holes += int((~v).sum())
        n = len(seq)
        fw = torch.stack([rows[s, k]["flow_up"].cpu() for k in range(n - 1)])[None]
        bw = torch.stack([rows[s, k]["flow_up_bw"].cpu() for k in range(n - 1)])[None]
        Minv = host_smooth_path(p["motion"].cpu()[None], H, W, crop=False, **{k: KW[k] for k in ("radius", "sigma")})[1]
        want, src = host_fill_uncovered(p["frames"].cpu()[None], p["valid"].cpu()[None], fw, bw, p["motion"].cpu()[None],
                                        p["transforms"].cpu()[None], Minv, sweeps=32)
        assert torch.equal(r["frames"].cpu(), want[0]) and torch.equal(r["source"].cpu(), src[0]), s
        for other in (again[s], alone[s]):
            assert torch.equal(other["frames"], r["frames"]) and torch.equal(other["source"], r["source"]), s
    assert holes > 0


def test_validate_stabilization_fill_runs_end_to_end(monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft").to(DEV)
    res = validate_stabilization(m, split(), ITERS, batch_size=2, device=DEV, **FILL, **KW)
    assert res["videos"] == 3 and res["frames"] == 14
    assert 0 <= res["filled_spatial"] <= res["filled"] < 1
    assert 0 < res["itf"] <= 100 and 0 < res["input_itf"] <= 100
    print(res)
