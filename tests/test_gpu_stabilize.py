"""Video stabilization on the GPU (csrc/stabilize.cu): the fit, the path and the warp against their host restatements bit for
bit, on strided, non-finite and edge inputs; batch independence and determinism; stabilize_videos against the host pipeline
fed the flows run_sequences yields; validate_stabilization end to end."""
import math

import numpy as np
import pytest
import torch

from conftest import build_model
from rnc.harness import run_sequences, stabilize_videos, validate_stabilization
from rnc.stabilize import (FEW, OK, fit_homographies, host_fit_homographies, host_smooth_path, host_warp_frames, smooth_path,
                           warp_frames)
from rnc.synth import shaky_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def camera_flows(N, H, W, seed):
    """N forward flows of random camera homographies, with a moving block, NaN and +-inf values, and flows that land
    exactly on x = W - 1 and y = H - 1."""
    g = np.random.default_rng(seed)
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    out = np.empty((N, 2, H, W), dtype=np.float32)
    for n in range(N):
        A = np.eye(3)
        A[:2, :2] += g.normal(0, 0.01, (2, 2))
        A[:2, 2] = g.normal(0, 3, 2)
        A[2, :2] = g.normal(0, 2e-5, 2)
        X, Y, Wh = (A[r, 0] * xs + A[r, 1] * ys + A[r, 2] for r in range(3))
        out[n, 0], out[n, 1] = X / Wh - xs, Y / Wh - ys
        by, bx = g.integers(0, max(1, H // 2)), g.integers(0, max(1, W // 2))
        out[n, :, by:by + H // 3, bx:bx + W // 3] += g.uniform(6, 12, (2, 1, 1)).astype(np.float32)
        bad = g.random((H, W))
        out[n, 0][bad < 0.01] = np.nan
        out[n, 1][(bad >= 0.01) & (bad < 0.015)] = np.inf
        out[n, 0][(bad >= 0.015) & (bad < 0.02)] = -np.inf
        edge = (bad >= 0.02) & (bad < 0.03)
        out[n, 0][edge] = (W - 1 - xs[edge]).astype(np.float32)
        out[n, 1][edge] = (H - 1 - ys[edge]).astype(np.float32)
    return torch.from_numpy(out)


def assert_fit_equal(got, want):
    for g, w in zip(got, want):
        assert torch.equal(g.cpu(), w), (g, w)


@pytest.mark.parametrize("N,H,W,stride", [(1, 8, 8, 8), (3, 13, 37, 3), (2, 436, 1024, 8), (2, 480, 854, 8), (2, 375, 1242, 8)])
def test_the_fit_equals_the_host_restatement(N, H, W, stride):
    flows = camera_flows(N, H, W, seed=H)
    got = fit_homographies(flows.to(DEV), stride=stride)
    want = host_fit_homographies(flows, stride=stride)
    assert_fit_equal(got, want)
    if (H, W) == (8, 8):
        assert want[3].tolist() == [FEW]
    else:
        assert (want[3] == OK).all() and (want[1] > 0).all()
    # a strided slice of a channel-last stack, and the least-squares start (K = 0)
    stack = torch.zeros(2 * N, H, W, 2, device=DEV)
    stack[::2] = flows.to(DEV).permute(0, 2, 3, 1)
    view = stack[::2].permute(0, 3, 1, 2)
    assert_fit_equal(fit_homographies(view, stride=stride, hypotheses=100, tau=1.5, refine=2, seed=7),
                     host_fit_homographies(flows, stride=stride, hypotheses=100, tau=1.5, refine=2, seed=7))
    assert_fit_equal(fit_homographies(view, stride=stride, hypotheses=0, refine=3),
                     host_fit_homographies(flows, stride=stride, hypotheses=0, refine=3))


def test_degenerate_pairs_match_the_host():
    H, W = 40, 56
    nan = torch.full((H, W), math.nan)
    line = torch.full((2, H, W), math.nan)
    line[:, 4] = 1.5
    flows = torch.stack([torch.stack([nan, nan]), torch.full((2, H, W), 1e4), line, torch.zeros(2, H, W)])
    got = fit_homographies(flows.to(DEV))
    want = host_fit_homographies(flows)
    assert_fit_equal(got, want)
    assert want[3].tolist() == [FEW, FEW, FEW, OK]


def test_a_pairs_fit_does_not_depend_on_the_batch_and_is_deterministic():
    flows = camera_flows(5, 64, 96, seed=3).to(DEV)
    batch = fit_homographies(flows)
    again = fit_homographies(flows)
    assert all(torch.equal(a, b) for a, b in zip(batch, again))
    for i in range(5):
        alone = fit_homographies(flows[i:i + 1])
        assert all(torch.equal(a[0], b[i]) for a, b in zip(alone, batch)), i
    moved = fit_homographies(torch.cat([flows[3:], flows[:3]]))
    assert all(torch.equal(torch.cat([m[2:], m[:2]]), b) for m, b in zip(moved, batch))


def jittered_motion(V, T, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.eye(3, dtype=torch.float64).repeat(V, T - 1, 1, 1)
    A[..., :2, :2] += 0.01 * torch.randn(V, T - 1, 2, 2, generator=g, dtype=torch.float64)
    A[..., :2, 2] += 3 * torch.randn(V, T - 1, 2, generator=g, dtype=torch.float64) + torch.tensor([2.0, 0.5],
                                                                                                  dtype=torch.float64)
    A[..., 2, :2] += 1e-5 * torch.randn(V, T - 1, 2, generator=g, dtype=torch.float64)
    return A


@pytest.mark.parametrize("V,T,H,W,radius,sigma,crop,crop_min",
                         [(1, 2, 8, 8, 30, 10.0, True, 0.5), (3, 13, 13, 37, 4, 2.0, True, 0.5),
                          (2, 50, 480, 854, 30, 10.0, True, 0.5), (2, 50, 436, 1024, 30, 10.0, False, 0.5),
                          (2, 200, 375, 1242, 30, 10.0, True, 0.95), (1, 300, 64, 64, 0, 1.0, True, 0.5)])
def test_the_path_equals_the_host_restatement(V, T, H, W, radius, sigma, crop, crop_min):
    A = jittered_motion(V, T, seed=T)
    got = smooth_path(A.to(DEV), H, W, radius, sigma, crop, crop_min)
    want = host_smooth_path(A, H, W, radius, sigma, crop, crop_min)
    for g, w in zip(got, want):
        assert torch.equal(g.cpu(), w)
    for v in range(V):                                                  # a video's path does not depend on the batch
        alone = smooth_path(A[v:v + 1].to(DEV), H, W, radius, sigma, crop, crop_min)
        assert all(torch.equal(a[0], b[v]) for a, b in zip(alone, got))


@pytest.mark.parametrize("N,C,H,W", [(1, 1, 8, 8), (3, 2, 13, 37), (2, 3, 436, 1024), (2, 4, 480, 854), (1, 3, 375, 1242)])
def test_the_warp_equals_the_host_restatement(N, C, H, W):
    g = torch.Generator().manual_seed(C)
    frames = torch.rand(N, C, H, W, generator=g) * 255
    frames[0, 0, 0, :3] = torch.tensor([math.nan, math.inf, -math.inf])
    A = jittered_motion(1, N + 1, seed=W)
    _, Minv, _ = host_smooth_path(A, H, W, radius=2, sigma=1.0, crop_min=0.2)
    maps = Minv[0, :N].clone()
    if N > 1:
        maps[1] = torch.tensor([[0.5, 0, 6], [0, -1.0, 8], [0.05, 0.1, -0.4]], dtype=torch.float64)   # w < 0 over part
    stack = torch.zeros(N, C + 1, H, W + 3, device=DEV)
    stack[:, 1:, :, 3:] = frames.to(DEV)
    view = stack[:, 1:, :, 3:]                                          # a strided slice of a stack
    out, valid = warp_frames(view, maps.to(DEV))
    want_out, want_valid = host_warp_frames(frames, maps)
    assert torch.equal(out.cpu(), want_out) and torch.equal(valid.cpu(), want_valid)
    again = warp_frames(view, maps.to(DEV))
    assert torch.equal(again[0], out) and torch.equal(again[1], valid)


# ----------------------------------------------------------------------------------------------------------- harness


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


H, W, ITERS = 64, 128, 6
KW = dict(radius=4, sigma=2.0, stride=4, hypotheses=64)


def split():
    return [[f.to(DEV) for f in shaky_sequence(n, H, W, seed=s)[0]] for s, n in enumerate((5, 3, 6))]


@pytest.mark.parametrize("warm_start", [False, True])
def test_stabilize_videos_is_the_sequence_pass_then_the_host_pipeline(warm_start, monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft_nc_dbl").to(DEV)
    seqs = split()
    with torch.no_grad():
        flows = {(s, k): f.cpu() for s, k, f in run_sequences(m, seqs, ITERS, warm_start=warm_start, batch_size=3, device=DEV)}
        for bs in (1, 3):
            res = stabilize_videos(m, seqs, ITERS, warm_start=warm_start, batch_size=bs, device=DEV, **KW)
            assert len(res) == 3
            for s, (seq, r) in enumerate(zip(seqs, res)):
                F = torch.stack([flows[s, k] for k in range(len(seq) - 1)])
                A, inl, mat, st = host_fit_homographies(F, stride=4, hypotheses=64)
                M, Minv, alpha = host_smooth_path(A[None], H, W, radius=4, sigma=2.0)
                frames, valid = host_warp_frames(torch.stack(seq).cpu(), Minv[0])
                assert r["frames"].is_cuda and r["frames"].shape == (len(seq), 3, H, W)
                for key, want in (("motion", A), ("inliers", inl), ("matched", mat), ("status", st), ("transforms", M[0]),
                                  ("alpha", alpha[0]), ("frames", frames), ("valid", valid)):
                    assert torch.equal(r[key].cpu(), want), (bs, s, key)


def test_validate_stabilization_runs_end_to_end(monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft").to(DEV)
    res = validate_stabilization(m, split(), ITERS, batch_size=2, device=DEV, **KW)
    assert res["videos"] == 3 and res["frames"] == 14
    assert 0 < res["cropping"] <= 1 and 0 < res["distortion"] <= 1
    assert 0 <= res["stability"] <= 1 and 0 <= res["input_stability"] <= 1
    assert 0 < res["itf"] <= 100 and 0 < res["input_itf"] <= 100
    print(res)
