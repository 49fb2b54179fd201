"""Video stabilization on the host (rnc.stabilize, DESIGN §3.21): the fit against the known camera motion and an independent
least-squares solve, the degenerate inputs, the path and crop, the warp against a naive loop, the scores against direct
NumPy, the argument errors, the C ABI, the distributed validation and the kernels' compile properties."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from rnc import native
from rnc.stabilize import (FEW, OK, SHRINK, _inv, crop_alpha, fit_homographies, gaussian_taps, host_fit_homographies,
                           host_fit_pair, host_smooth_path, host_warp_frames, smooth_path, solve8, stabilization_metrics,
                           summarize_stabilization, warp_frames)
from rnc.synth import shaky_sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def project(M, H, W):
    """Every pixel of an H x W frame mapped by M: [2, H*W]."""
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    q = np.asarray(M) @ np.stack([xs.ravel(), ys.ravel(), np.ones(H * W)])
    return q[:2] / q[2]


def reprojection(A, G, H, W):
    return np.abs(project(A, H, W) - project(G, H, W)).max()


def truth(C, k):
    C = C.numpy()
    return C[k + 1] @ np.linalg.inv(C[k])


# ------------------------------------------------------------------------------------------------------------- the fit


def test_the_fit_recovers_the_camera_motion_from_exact_flows():
    _, C, flows = shaky_sequence(6, 96, 128, seed=1)
    A, inl, matched, status = host_fit_homographies(flows)
    assert status.tolist() == [OK] * 5
    for k in range(5):
        assert reprojection(A[k], truth(C, k), 96, 128) < 1e-6, k
        assert 0.9 * matched[k] <= inl[k] <= matched[k]


def test_a_moving_object_over_40_percent_of_the_frame_is_rejected_and_plain_least_squares_is_not():
    H, W = 96, 128
    _, C, flows = shaky_sequence(5, H, W, seed=2)
    g = torch.Generator().manual_seed(3)
    moved = flows.clone()
    moved[:, :, 8:8 + 64, 20:20 + 77] += (8 + 8 * torch.rand(4, 2, 1, 1, generator=g)) * torch.tensor([1.0, -1.0])[:, None, None]
    assert 64 * 77 >= 0.4 * H * W
    A, inl, matched, status = host_fit_homographies(moved)
    A_ls, *_ = host_fit_homographies(moved, hypotheses=0, refine=1)
    for k in range(4):
        assert status[k] == OK and reprojection(A[k], truth(C, k), H, W) < 1e-6, k
        assert inl[k] < 0.65 * matched[k]
        assert reprojection(A_ls[k], truth(C, k), H, W) > 1.0, k                 # the object drags the plain fit by pixels


def test_the_refit_is_numpys_least_squares_on_the_same_inliers():
    _, _, flows = shaky_sequence(3, 64, 96, seed=4)
    f = flows[0].numpy().copy()
    rng = np.random.default_rng(0)
    f += rng.normal(0, 0.3, f.shape).astype(np.float32)                     # noisy flow: the refit is a real compromise
    f[:, 10:40, 10:50] += np.float32(9.0)
    r = host_fit_pair(f, refine=3)
    L = r["L"]
    assert len(r["rounds"]) == 3
    for flags, h in r["rounds"]:
        x, y, u, v = (L[flags, k] for k in range(4))
        z, o = np.zeros_like(x), np.ones_like(x)
        D = np.concatenate([np.stack([x, y, o, z, z, z, -u * x, -u * y], 1), np.stack([z, z, z, x, y, o, -v * x, -v * y], 1)])
        want = np.linalg.lstsq(D, np.concatenate([u, v]), rcond=None)[0]
        assert np.abs(h - want).max() <= 1e-9 * np.abs(want).max()


def test_solve8_is_partial_pivoting_elimination():
    rng = np.random.default_rng(1)
    a = rng.normal(size=(50, 8, 9))
    ok, x = solve8(a.copy())
    assert ok.all()
    assert np.allclose(x, np.linalg.solve(a[:, :, :8], a[:, :, 8:])[..., 0], rtol=1e-9, atol=1e-12)
    a[:7, 3] = a[:7, 5]                                                     # singular: two equal rows
    ok, _ = solve8(a.copy())
    assert not ok[:7].any() and ok[7:].all()


def test_degenerate_inputs_give_few_and_the_identity():
    H, W = 40, 56
    ys, xs = np.mgrid[0:H, 0:W]
    nan = torch.full((1, 2, H, W), math.nan)
    leaving = torch.full((1, 2, H, W), 1e4)
    line = torch.full((1, 2, H, W), math.nan)                               # only row y = 4 of grid points is finite
    line[0, :, 4] = 1.5
    tiny = torch.zeros(1, 2, 8, 8)                                          # one grid point
    for f in (nan, leaving, line, tiny):
        A, inl, matched, status = host_fit_homographies(f)
        assert status.tolist() == [FEW] and inl.tolist() == [0] and torch.equal(A[0], torch.eye(3, dtype=torch.float64))
    assert host_fit_homographies(line)[2].tolist() == [7]
    assert host_fit_homographies(tiny)[2].tolist() == [1]


# ----------------------------------------------------------------------------------------------------- path and crop


def translation(dx, dy):
    return torch.tensor([[1.0, 0, dx], [0, 1.0, dy], [0, 0, 1.0]], dtype=torch.float64)


def test_a_constant_pan_is_left_as_it_is_on_interior_frames():
    T, r = 30, 6
    A = torch.stack([translation(3.0, -1.25)] * (T - 1))[None]
    M, Minv, alpha = host_smooth_path(A, 60, 80, radius=r, sigma=2.5, crop=False)
    for t in range(r, T - r):
        assert (M[0, t] - torch.eye(3, dtype=torch.float64)).abs().max() < 1e-9, t
    assert (M[0, 0] - torch.eye(3, dtype=torch.float64)).abs().max() > 1.0   # the truncated window at the ends
    assert torch.allclose(M[0] @ Minv[0], torch.eye(3, dtype=torch.float64).expand(T, 3, 3), atol=1e-12)


def inter_frame(M, A):
    B = M[1:] @ A @ torch.linalg.inv(M[:-1])
    return B / B[:, 2:3, 2:3]


def test_a_jittered_pan_is_smoothed_and_scores_as_more_stable():
    T, H, W, r = 48, 48, 64, 8
    _, C, flows = shaky_sequence(T, H, W, seed=5, pan=(2.0, 0.5))
    A, _, _, status = host_fit_homographies(flows)
    assert (status == OK).all()
    M, Minv, alpha = host_smooth_path(A[None], H, W, radius=r, sigma=3.0)
    pan = translation(-2.0, -0.5).numpy()                                   # the content moves against the camera
    dev_in = [reprojection(A[t], pan, H, W) for t in range(r, T - 1 - r)]
    dev_out = [reprojection(B, pan, H, W) for B in inter_frame(M[0], A)[r:T - 1 - r]]
    assert np.mean(dev_out) < np.mean(dev_in) / 5, (np.mean(dev_out), np.mean(dev_in))
    s = stabilization_metrics(A, M[0])
    assert s["stability"] > s["input_stability"] and s["stability_translation"] > s["input_stability_translation"]
    assert 0.5 <= float(alpha[0]) < 1 and 0 < s["cropping"] < 1 and 0.9 < s["distortion"] <= 1


def brute_alpha(S, H, W):
    """Bisection on corner containment (the feasible scales form an interval [0, alpha])."""
    P = np.linalg.inv(S)
    c = np.array([(W - 1) / 2, (H - 1) / 2])

    def inside(a):
        for sx in (-1, 1):
            for sy in (-1, 1):
                q = P @ np.array([c[0] + sx * a * c[0], c[1] + sy * a * c[1], 1.0])
                if not (q[2] > 0 and 0 <= q[0] / q[2] <= W - 1 and 0 <= q[1] / q[2] <= H - 1):
                    return False
        return True

    if inside(1.0):
        return 1.0
    if not inside(0.0):
        return 0.0
    lo, hi = 0.0, 1.0
    for _ in range(60):
        mid = (lo + hi) / 2
        lo, hi = (mid, hi) if inside(mid) else (lo, mid)
    return lo


def test_the_closed_form_crop_is_the_brute_force_search_and_leaves_every_pixel_valid():
    H, W = 36, 52
    rng = np.random.default_rng(7)
    S = np.tile(np.eye(3), (40, 1, 1))
    S[:, :2, :2] += rng.normal(0, 0.05, (40, 2, 2))
    S[:, :2, 2] += rng.normal(0, 4, (40, 2))
    S[:, 2, :2] += rng.normal(0, 2e-4, (40, 2))
    S[3] = np.array([[1.0, 0, 80], [0, 1, 0], [0, 0, 1]])                   # the centre leaves the frame: 0
    S[4] = np.eye(3)                                                        # nothing to crop: 1
    got = crop_alpha(S, H, W)
    want = np.array([brute_alpha(s, H, W) for s in S])
    assert got[3] == 0 and got[4] == 1 and np.abs(got - want).max() < 1e-9
    _, _, flows = shaky_sequence(12, H, W, seed=8, jitter_px=1.0)
    A, *_ = host_fit_homographies(flows, stride=4)
    frames = torch.rand(12, 2, H, W, generator=torch.Generator().manual_seed(0)) * 255
    M, Minv, alpha = host_smooth_path(A[None], H, W, radius=4, sigma=2.0, crop_min=0.3)
    assert alpha[0] >= 0.3
    _, valid = host_warp_frames(frames, Minv[0])
    assert bool(valid.all())
    M, Minv, alpha = host_smooth_path(A[None], H, W, radius=4, sigma=2.0, crop_min=0.3, crop=False)
    assert not bool(host_warp_frames(frames, Minv[0])[1].all())             # without the crop the borders are uncovered


# ------------------------------------------------------------------------------------------------------------ the warp


def naive_sample(img, px, py):
    H, W = img.shape
    f32 = np.float32
    px, py = min(max(px, f32(0)), f32(W - 1)), min(max(py, f32(0)), f32(H - 1))
    x0, y0 = np.floor(px), np.floor(py)
    ax, ay = f32(px - x0), f32(py - y0)
    bx, by = f32(1 - ax), f32(1 - ay)
    ix, iy = int(x0), int(y0)
    ix1, iy1 = min(ix + 1, W - 1), min(iy + 1, H - 1)
    s = f32(img[iy, ix] * f32(bx * by))
    s = f32(s + f32(img[iy, ix1] * f32(ax * by)))
    s = f32(s + f32(img[iy1, ix] * f32(bx * ay)))
    return f32(s + f32(img[iy1, ix1] * f32(ax * ay)))


def test_host_warp_frames_is_the_naive_per_pixel_loop():
    N, C, H, W = 3, 3, 9, 13
    frames = torch.rand(N, C, H, W, generator=torch.Generator().manual_seed(1)) * 255
    maps = torch.tensor([[[1.02, 0.03, -1.3], [-0.02, 0.98, 0.7], [1e-3, -2e-3, 1.0]],
                         [[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0]],
                         [[0.5, 0, 6], [0, -1.0, 8], [0.05, 0.1, -0.4]]], dtype=torch.float64)   # w < 0 over part of it
    out, valid = host_warp_frames(frames, maps)
    f = frames.numpy()
    for n in range(N):
        m = maps[n].numpy()
        for y in range(H):
            for x in range(W):
                X, Y, w = m @ np.array([x, y, 1.0])
                with np.errstate(all="ignore"):
                    qx, qy = np.float32(X / w), np.float32(Y / w)
                ok = w > 0 and 0 <= qx <= W - 1 and 0 <= qy <= H - 1
                assert valid[n, y, x] == ok
                for c in range(C):
                    want = naive_sample(f[n, c], qx, qy) if ok else 0.0
                    assert out[n, c, y, x].item() == want, (n, c, y, x)
    assert torch.equal(out[1], frames[1]) and bool(valid[1].all())
    assert 0 < valid[2].sum() < H * W


# --------------------------------------------------------------------------------------------------------- the scores


def test_each_score_is_its_direct_numpy_computation():
    rng = np.random.default_rng(2)
    T = 24
    A = np.tile(np.eye(3), (T - 1, 1, 1))
    A[:, :2, 2] = rng.normal(0, 2, (T - 1, 2))
    th = rng.normal(0, 0.02, T - 1)
    A[:, 0, 0] = A[:, 1, 1] = np.cos(th)
    A[:, 1, 0], A[:, 0, 1] = np.sin(th), -np.sin(th)
    M = np.tile(np.eye(3), (T, 1, 1))
    M[:, :2, :2] *= rng.uniform(1.1, 1.3, (T, 1, 1))
    M[:, 0, 1] = rng.normal(0, 0.05, T)
    M[:, :2, 2] = rng.normal(0, 3, (T, 2))
    s = stabilization_metrics(torch.from_numpy(A), torch.from_numpy(M))
    assert math.isclose(s["cropping"], np.mean([1 / abs(np.linalg.det(m[:2, :2])) for m in M]), rel_tol=1e-12)
    ratios = []
    for m in M:
        sv = np.linalg.svd(m[:2, :2], compute_uv=False)
        ratios.append(sv.min() / sv.max())
    assert math.isclose(s["distortion"], min(ratios), rel_tol=1e-12)

    def ratio(paths):
        spec = [np.abs(np.fft.fft(p)) ** 2 for p in paths]
        n = len(paths[0])
        low = sum(e[1:6].sum() for e in spec)
        return low / sum(e[1:n // 2 + 1].sum() for e in spec)

    B = np.stack([M[t + 1] @ A[t] @ np.linalg.inv(M[t]) for t in range(T - 1)])
    B /= B[:, 2:3, 2:3]
    for pre, X in (("", B), ("input_", A)):
        st = ratio([np.cumsum(X[:, 0, 2]), np.cumsum(X[:, 1, 2])])
        sr = ratio([np.cumsum(np.arctan2(X[:, 1, 0], X[:, 0, 0]))])
        assert math.isclose(s[pre + "stability_translation"], st, rel_tol=1e-9)
        assert math.isclose(s[pre + "stability_rotation"], sr, rel_tol=1e-9)
        assert s[pre + "stability"] == min(s[pre + "stability_translation"], s[pre + "stability_rotation"])
    eye = stabilization_metrics(torch.from_numpy(A), torch.eye(3, dtype=torch.float64).expand(T, 3, 3))
    assert eye["cropping"] == 1 and eye["distortion"] == 1
    assert eye["stability"] == eye["input_stability"]


def test_identity_maps_leave_the_video_and_its_itf_as_they_are():
    from rnc.interp import host_interpolation_error
    frames = torch.stack(shaky_sequence(5, 24, 32, seed=9)[0])
    out, valid = host_warp_frames(frames, torch.eye(3, dtype=torch.float64).expand(5, 3, 3))
    assert torch.equal(out, frames) and bool(valid.all())
    rows = [list(zip(*(t.tolist() for t in host_interpolation_error(v[1:], v[:-1])))) for v in (out, frames)]
    scores = stabilization_metrics(torch.eye(3, dtype=torch.float64).expand(4, 3, 3),
                                   torch.eye(3, dtype=torch.float64).expand(5, 3, 3))
    res = summarize_stabilization([(scores, *rows)])
    assert res["itf"] == res["input_itf"] and 10 < res["itf"] < 100 and res["frames"] == 5 and res["videos"] == 1
    assert math.isnan(summarize_stabilization([])["itf"])


def test_gaussian_taps():
    w = gaussian_taps(5, 2.0)
    assert w.dtype == torch.float64 and w.shape == (6,) and w[0] == 1
    assert torch.allclose(w, torch.exp(-torch.arange(6.0, dtype=torch.float64) ** 2 / 8))


# -------------------------------------------------------------------------------------------------------------- errors


def test_argument_errors_raise_before_any_launch():
    f = torch.zeros(2, 2, 16, 16)
    for kw in (dict(stride=0), dict(stride=257), dict(stride=2.0), dict(hypotheses=-1), dict(hypotheses=65537),
               dict(refine=-1), dict(refine=65), dict(hypotheses=0, refine=0), dict(tau=0.0), dict(tau=math.inf),
               dict(tau=math.nan), dict(seed=-1), dict(seed=1 << 64), dict(seed=1.5)):
        for fn in (fit_homographies, host_fit_homographies):
            with pytest.raises(ValueError):
                fn(f, **kw)
    for bad in (torch.zeros(2, 3, 4, 4), torch.zeros(2, 4, 4), torch.zeros(0, 2, 4, 4), torch.zeros(1, 2, 4097, 4)):
        with pytest.raises(ValueError):
            fit_homographies(bad)
    A = torch.eye(3, dtype=torch.float64).expand(1, 4, 3, 3)
    for args, kw in (((A, 0, 8), {}), ((A, 8, 4097), {}), ((A[0], 8, 8), {}), ((A[:, :0], 8, 8), {}),
                     ((A, 8, 8), dict(radius=-1)), ((A, 8, 8), dict(radius=1025)), ((A, 8, 8), dict(sigma=0.0)),
                     ((A, 8, 8), dict(sigma=math.nan)), ((A, 8, 8), dict(crop_min=0.0)), ((A, 8, 8), dict(crop_min=1.5))):
        for fn in (smooth_path, host_smooth_path):
            with pytest.raises(ValueError):
                fn(*args, **kw)
    fr = torch.zeros(2, 3, 8, 8)
    maps = torch.eye(3, dtype=torch.float64).expand(2, 3, 3)
    for args in ((torch.zeros(2, 5, 8, 8), maps), (torch.zeros(2, 0, 8, 8), maps), (fr, maps[:1]), (fr[0], maps),
                 (torch.zeros(2, 1, 4097, 2), maps)):
        for fn in (warp_frames, host_warp_frames):
            with pytest.raises(ValueError):
                fn(*args)
    with pytest.raises(ValueError):
        gaussian_taps(-1)


class _InferenceModel:
    def _needs_grad(self):
        return False


class _TrainingModel:
    def _needs_grad(self):
        return True


def test_stabilize_videos_and_validate_check_their_arguments(monkeypatch):
    from rnc import harness

    def boom(*a, **k):
        raise AssertionError("the flow pass ran")

    monkeypatch.setattr(harness, "run_sequences", boom)
    seqs = [[torch.zeros(3, 16, 16)] * 3]
    m = _InferenceModel()
    with pytest.raises(ValueError, match="inference only"):
        harness.stabilize_videos(_TrainingModel(), seqs)
    for kw in (dict(stride=0), dict(hypotheses=-1), dict(tau=-1.0), dict(refine=100), dict(seed=-1), dict(radius=-1),
               dict(sigma=0.0), dict(crop_min=2.0), dict(hypotheses=0, refine=0)):
        for fn in (harness.stabilize_videos, harness.validate_stabilization):
            with pytest.raises(ValueError):
                fn(m, seqs, device="cpu", **kw)
    for bad in ([[torch.zeros(3, 16, 16)]], [[torch.zeros(3, 4097, 8)] * 2]):
        with pytest.raises(ValueError):
            harness.stabilize_videos(m, bad, device="cpu")


# ----------------------------------------------------------------------- the harness under torch.distributed


def _stub_sequences(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                    return_confidence=False):
    """run_sequences' yields in its step order, on the CPU: each pair's flow is a rotation about the frame centre and a
    translation read off the frames' channel means, so any subset of the videos gets the same flows."""
    from rnc.harness import sequence_schedule
    for step in sequence_schedule([len(s) for s in sequences], batch_size):
        for c in step:
            if not c.idle:
                a, b = sequences[c.seq][c.pair], sequences[c.seq][c.pair + 1]
                _, H, W = a.shape
                d = (a.mean((1, 2)) - b.mean((1, 2))).double()
                th = float(d[2]) / 200
                ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64) - (H - 1) / 2,
                                        torch.arange(W, dtype=torch.float64) - (W - 1) / 2, indexing="ij")
                fx = math.cos(th) * xs - math.sin(th) * ys - xs + float(d[0]) / 4
                fy = math.sin(th) * xs + math.cos(th) * ys - ys + float(d[1]) / 4
                yield c.seq, c.pair, torch.stack([fx, fy]).float()


def stabilization_split():
    return [shaky_sequence(n, 24, 32, seed=k)[0] for k, n in enumerate((5, 3, 8, 4, 6))]


def _stabilization_worker(rank, world, port, q):
    import torch.distributed as dist
    from rnc import harness
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        harness.run_sequences = _stub_sequences
        q.put((rank, harness.validate_stabilization(_InferenceModel(), stabilization_split(), batch_size=2, device="cpu",
                                                    radius=3, sigma=1.5, stride=4, hypotheses=32)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_validate_stabilization_gloo_equals_world_1(world, monkeypatch):
    from test_flow_metrics import run_ranks
    from rnc import harness
    monkeypatch.setattr(harness, "run_sequences", _stub_sequences)
    seqs = stabilization_split()
    kw = dict(batch_size=2, device="cpu", radius=3, sigma=1.5, stride=4, hypotheses=32)
    want = harness.validate_stabilization(_InferenceModel(), seqs, **kw)
    assert want["videos"] == 5 and want["frames"] == sum(len(s) for s in seqs)
    assert all(math.isfinite(v) for v in want.values())
    got = harness.stabilize_videos(_InferenceModel(), seqs, **kw)
    for seq, r in zip(seqs, got):                                       # each video as the host pipeline defines it, alone
        flows = torch.stack([x[2] for x in _stub_sequences(None, [seq])])
        A, inl, mat, st = host_fit_homographies(flows, stride=4, hypotheses=32)
        M, Minv, alpha = host_smooth_path(A[None], 24, 32, radius=3, sigma=1.5)
        frames, valid = host_warp_frames(torch.stack(seq), Minv[0])
        assert torch.equal(r["motion"], A) and torch.equal(r["transforms"], M[0]) and torch.equal(r["alpha"], alpha[0])
        assert torch.equal(r["frames"], frames) and torch.equal(r["valid"], valid) and torch.equal(r["inliers"], inl)
        assert torch.equal(r["matched"], mat) and torch.equal(r["status"], st)
    for got in run_ranks(_stabilization_worker, world):
        assert got == want


# ----------------------------------------------------------------------------------------------------------- C ABI


_CTYPE = {"long long": native.C.c_longlong, "int": native.C.c_int, "size_t": native.C.c_size_t, "float": native.C.c_float,
          "double": native.C.c_double, "unsigned long long": native.C.c_ulonglong}
NAMES = ("rnc_homography_fit_workspace_bytes", "rnc_homography_fit", "rnc_stabilize_path", "rnc_stabilize_warp")


def test_declarations_match_the_binding():
    with open(os.path.join(ROOT, "include", "rnc.h")) as f:
        header = f.read()
    assert re.search(r"#define RNC_HOMOGRAPHY_OK 0\b", header) and re.search(r"#define RNC_HOMOGRAPHY_FEW 1\b", header)
    assert (native.HOMOGRAPHY_OK, native.HOMOGRAPHY_FEW) == (0, 1)
    for name in NAMES:
        m = re.search(r"\n(int|size_t) " + name + r"\(([^;]*)\);", header)
        assert m, name
        args = [a.strip() for a in m.group(2).replace("\n", " ").split(",")]
        want = [native.C.c_void_p if "*" in a else _CTYPE[a.rsplit(" ", 1)[0].replace("const ", "")] for a in args]
        res, argtypes = native.SIGNATURES[name]
        assert argtypes == want, name
        assert res is (native.C.c_int if m.group(1) == "int" else native.C.c_size_t), name


def test_entry_points_return_their_error_codes():
    L = native.lib()
    P = 1 << 20                                         # never dereferenced: every check fails on the host before a launch
    n0 = L.rnc_launch_count()
    ws = L.rnc_homography_fit_workspace_bytes(2, 40, 60, 8, 256)
    assert ws >= 2 * 5 * 7 * 4 * 8 + 2 * 256 * (8 * 8 + 4)
    for bad in ((0, 4, 4, 8, 1), (65536, 4, 4, 8, 1), (1, 0, 4, 8, 1), (1, 4, 4097, 8, 1), (1, 4, 4, 0, 1), (1, 4, 4, 257, 1),
                (1, 4, 4, 8, -1), (1, 4, 4, 8, 65537)):
        assert L.rnc_homography_fit_workspace_bytes(*bad) == 0, bad

    def fit(N=2, H=40, W=60, stride=8, K=256, tau=2.0, refine=4, f=P, A=P, i=P, m=P, s=P, wsp=P, wsb=ws):
        return L.rnc_homography_fit(f, 1, 1, 1, 1, N, H, W, stride, K, tau, refine, 0, A, i, m, s, wsp, wsb, None)

    for bad in (dict(N=0), dict(N=65536), dict(H=0), dict(W=4097), dict(stride=0), dict(stride=257), dict(K=-1),
                dict(K=65537), dict(refine=-1), dict(refine=65), dict(K=0, refine=0), dict(tau=0.0), dict(tau=-1.0),
                dict(tau=math.inf), dict(tau=math.nan)):
        assert fit(**bad) == -1, bad
    for bad in (dict(f=0), dict(A=0), dict(i=0), dict(m=0), dict(s=0), dict(wsp=0), dict(f=P + 2), dict(A=P + 4),
                dict(i=P + 2), dict(m=P + 1), dict(s=P + 2), dict(wsp=P + 8)):
        assert fit(**bad) == -2, bad
    assert fit(wsb=ws - 1) == -5

    def path(A=P, V=2, T=5, taps=P, radius=3, H=40, W=60, crop=1, crop_min=0.5, M=P, Mi=P, al=P):
        return L.rnc_stabilize_path(A, V, T, taps, radius, H, W, crop, crop_min, M, Mi, al, None)

    for bad in (dict(V=0), dict(V=65536), dict(T=1), dict(radius=-1), dict(radius=1025), dict(H=0), dict(W=4097),
                dict(crop_min=0.0), dict(crop_min=1.5), dict(crop_min=math.nan)):
        assert path(**bad) == -1, bad
    for bad in (dict(A=0), dict(taps=0), dict(M=0), dict(Mi=0), dict(al=0), dict(A=P + 4), dict(taps=P + 4), dict(M=P + 4),
                dict(Mi=P + 4), dict(al=P + 4)):
        assert path(**bad) == -2, bad

    def warp(fr=P, maps=P, N=2, C=3, H=40, W=60, out=P, valid=P):
        return L.rnc_stabilize_warp(fr, 1, 1, 1, 1, maps, N, C, H, W, out, 1, 1, 1, 1, valid, 1, 1, 1, None)

    for bad in (dict(N=0), dict(N=65536), dict(C=0), dict(C=5), dict(H=0), dict(W=4097)):
        assert warp(**bad) == -1, bad
    for bad in (dict(fr=0), dict(maps=0), dict(out=0), dict(valid=0), dict(fr=P + 2), dict(maps=P + 4), dict(out=P + 2)):
        assert warp(**bad) == -2, bad
    assert L.rnc_launch_count() == n0


BIT_EXACT = ("count_kernel", "scan_kernel", "write_kernel", "hyp_kernel", "argmax_kernel", "chunk_kernel", "solve_kernel",
             "path_kernel", "warp_kernel")


def _compile(tmp_path, name, *flags):
    from rnc.build import ARCH, CSRC, nvcc_path
    cubin = str(tmp_path / name)
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", *flags, "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-cubin", os.path.join(CSRC, "stabilize.cu"), "-o", cubin]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc_path()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    return out.stdout + out.stderr, re.sub(r"/\*[^*]*\*/", "", sass)


def test_stabilize_cu_has_no_atomics_no_contraction_and_does_not_spill(tmp_path):
    log, sass = _compile(tmp_path, "s.cubin")
    names = "|".join(BIT_EXACT)
    kernels = re.findall(r"Function properties for \S*?\d(" + names + r")\w*", log)
    assert sorted(kernels) == sorted(BIT_EXACT), kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == len(BIT_EXACT) and all(a == "0" and b == "0" for a, b in spills), spills
    assert re.findall(r"(\d+) bytes stack frame", log) == ["0"] * len(BIT_EXACT)
    assert not re.search(r"^\s*(@!?U?P\w+\s+)?(ATOM|ATOMS|ATOMG|RED)[.\s]", sass, re.M)
    # every DFMA left is inside __ddiv_rn's correctly rounded division
    _, strict = _compile(tmp_path, "f.cubin", "-fmad=false")
    assert sass == strict


def test_the_crop_margin_is_tiny():
    assert 1 - SHRINK == 2.0 ** -36
    S = torch.eye(3, dtype=torch.float64).expand(3, 3, 3).numpy()
    assert np.array_equal(_inv(S), S)
