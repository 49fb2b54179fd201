"""Full-frame video stabilization on the host (rnc.stabilize step 5, DESIGN §3.22): the residual transfer and the global re-add
against the analytic camera motion of rnc.synth.shaky_sequence, the unknown set of the transfer, the filled border against the
true canvas beside two simpler fills, the harness with and without crop, the argument errors, the C ABI, the distributed
validation and the kernels' compile properties."""
import math
import os
import re

import numpy as np
import pytest
import torch

from rnc import native
from rnc.inpaint import SOURCE_KNOWN, SOURCE_SPATIAL, host_harmonic_fill, host_inpaint
from rnc.stabilize import (add_global_motion, fill_uncovered, flow_residual, host_add_global_motion, host_fill_uncovered,
                           host_fit_homographies, host_flow_residual, host_smooth_path, host_warp_frames)
from rnc.synth import shaky_backward_flows, shaky_canvas, shaky_sequence
from test_stabilize import _CTYPE, _InferenceModel, _stub_sequences

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, H, W, SEED = 24, 96, 160, 0
SWEEPS = 64                     # the residuals start within 1e-5 px of their limit, and the spatial share is 0.1%


@pytest.fixture(scope="module")
def video():
    """One shaky video stabilized without crop on the host from its exact flows: a dict of the pipeline's tensors."""
    frames, C, flows = shaky_sequence(T, H, W, seed=SEED)
    bw = shaky_backward_flows(C, H, W)
    A, *_ = host_fit_homographies(flows)
    M, Minv, alpha = host_smooth_path(A[None], H, W, crop=False)
    warped, valid = host_warp_frames(torch.stack(frames), Minv[0])
    return dict(C=C, flow=flows[None], flow_bw=bw[None], A=A[None], M=M, Minv=Minv, alpha=float(alpha[0]), frames=warped[None],
                valid=valid[None])


def maps_args(v):
    return v["flow"], v["flow_bw"], v["A"], v["M"], v["Minv"]


def analytic_flow(v, a, b):
    """The output inter-frame flow from output frame a to b, pi(M_b C_b C_a^-1 M_a^-1 u) - u, in fp64 [2,H,W]."""
    C, M = v["C"].numpy(), v["M"][0].numpy()
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    P = np.stack([xs.ravel(), ys.ravel(), np.ones(H * W)])
    q = M[b] @ C[b] @ np.linalg.inv(C[a]) @ np.linalg.inv(M[a]) @ P
    return np.stack([q[0] / q[2] - P[0], q[1] / q[2] - P[1]]).reshape(2, H, W)


def truth(v):
    """The true content of every output pixel: the canvas at C_t^-1 M_t^-1 u, fp64 [T,3,H,W]."""
    C, M = v["C"].numpy(), v["M"][0].numpy()
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    P = np.stack([xs.ravel(), ys.ravel(), np.ones(H * W)])
    out = np.empty((T, 3, H, W))
    for t in range(T):
        q = np.linalg.inv(C[t]) @ np.linalg.inv(M[t]) @ P
        out[t] = shaky_canvas(q[0] / q[2], q[1] / q[2], SEED).reshape(3, H, W)
    return torch.from_numpy(out)


def psnr(x, gt, where):
    m = where[:, None].expand(-1, 3, -1, -1)
    return float(10 * torch.log10(255.0 ** 2 / ((x.double() - gt)[m] ** 2).mean()))


# ------------------------------------------------------------------------------------------------ transfer and re-add


def test_the_residual_is_zero_where_known_and_unknown_exactly_where_the_warp_is_invalid(video):
    R, Rb = host_flow_residual(*maps_args(video))
    hole = video["valid"][0] == 0
    assert 0.02 < float(hole.float().mean()) < 0.5 and video["alpha"] < 1          # a real border to fill
    for r, h in ((R[0], hole[:-1]), (Rb[0], hole[1:])):
        known = torch.isfinite(r)
        assert torch.equal(known[:, 0], known[:, 1])
        assert torch.equal(~known[:, 0], h)                                        # NaN exactly where valid == 0
        assert float(r[known].abs().max()) < 1e-3


def test_the_completed_flows_are_the_analytic_output_flows_across_the_border(video):
    R, Rb = host_flow_residual(*maps_args(video))
    hole = (video["valid"][0] == 0).to(torch.uint8)
    Rf, Rbf = host_harmonic_fill(R, hole[None, :-1], SWEEPS), host_harmonic_fill(Rb, hole[None, 1:], SWEEPS)
    F, G = host_add_global_motion(Rf, Rbf, *maps_args(video)[2:])
    err = max(max(np.abs(F[0, k].double().numpy() - analytic_flow(video, k, k + 1)).max(),
                  np.abs(G[0, k].double().numpy() - analytic_flow(video, k + 1, k)).max()) for k in range(T - 1))
    assert err < 1e-3, err
    # the full flow completed by the same fill bends near the border's free edges; the residual's does not
    Fg, _ = host_add_global_motion(R, Rb, *maps_args(video)[2:])
    full = host_harmonic_fill(Fg, hole[None, :-1], SWEEPS)
    err_full = max(np.abs(full[0, k].double().numpy() - analytic_flow(video, k, k + 1)).max() for k in range(T - 1))
    assert err_full > 20 * err, (err_full, err)


def test_add_global_motion_of_a_zero_residual_is_the_analytic_flow_of_the_fitted_motion(video):
    z = torch.zeros_like(video["flow"])
    F, G = add_global_motion(z, z, *maps_args(video)[2:])
    assert torch.isfinite(F).all() and torch.isfinite(G).all()
    assert max(np.abs(F[0, k].double().numpy() - analytic_flow(video, k, k + 1)).max() for k in range(T - 1)) < 1e-4


# ----------------------------------------------------------------------------------------------------- end to end


@pytest.fixture(scope="module")
def filled(video):
    return host_fill_uncovered(video["frames"], video["valid"], *maps_args(video), sweeps=SWEEPS)


def test_every_uncovered_pixel_is_filled_and_every_covered_pixel_keeps_its_bits(video, filled):
    out, source = filled
    valid = video["valid"] != 0
    assert torch.equal(source == SOURCE_KNOWN, valid)
    assert torch.isfinite(out).all()
    assert torch.equal(out[valid[:, :, None].expand_as(out)], video["frames"][valid[:, :, None].expand_as(out)])
    assert float((source == SOURCE_SPATIAL).float().sum() / (~valid).float().sum()) < 0.1


def test_the_filled_border_is_the_canvas_and_beats_a_spatial_fill(video, filled):
    """Measured (DESIGN §3.22): filled 45.9 dB, covered 57.4 dB, the full flows completed by rnc.inpaint.inpaint 45.9 dB,
    a spatial-only harmonic_fill 21.2 dB.  An affine camera's flow is harmonic, so the full-flow fill is within 4e-3 px of
    the truth here and ties; the residual's 1e-5 px shows in the flow test above, not in this PSNR."""
    out, _ = filled
    gt = truth(video)
    hole, valid = video["valid"][0] == 0, video["valid"][0] != 0
    p_fill, p_cov = psnr(out[0], gt, hole), psnr(out[0], gt, valid)
    R, Rb = host_flow_residual(*maps_args(video))
    Fg, Gg = host_add_global_motion(R, Rb, *maps_args(video)[2:])
    full, _ = host_inpaint(video["frames"], hole[None].to(torch.uint8), Fg, Gg, sweeps=SWEEPS)
    p_full = psnr(full[0], gt, hole)
    p_spatial = psnr(host_harmonic_fill(video["frames"][0], hole.to(torch.uint8), SWEEPS), gt, hole)
    print(f"PSNR filled {p_fill:.2f} covered {p_cov:.2f} full-flow {p_full:.2f} spatial {p_spatial:.2f}")
    assert p_fill > 42.0
    assert p_fill > p_spatial + 15.0
    assert p_fill > p_full - 0.2
    assert p_fill > p_cov - 15.0


# ------------------------------------------------------------------------------------------------------ the harness


def _stub_bidirectional(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                        return_confidence=False, alpha1=0.01, alpha2=0.5):
    """run_sequences_bidirectional's yields on the CPU: the forward flow is _stub_sequences' (a rotation about the centre and
    a translation from the frames' channel means), the backward flow that motion's inverse."""
    for s, k, f in _stub_sequences(model, sequences, iters, warm_start, batch_size, mode, device):
        a, b = sequences[s][k], sequences[s][k + 1]
        _, h, w = a.shape
        d = (a.mean((1, 2)) - b.mean((1, 2))).double()
        th = float(d[2]) / 200
        ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64) - (h - 1) / 2,
                                torch.arange(w, dtype=torch.float64) - (w - 1) / 2, indexing="ij")
        ux, uy = xs - float(d[0]) / 4, ys - float(d[1]) / 4
        bx = math.cos(th) * ux + math.sin(th) * uy - xs
        by = -math.sin(th) * ux + math.cos(th) * uy - ys
        yield s, k, {"flow_up": f, "flow_up_bw": torch.stack([bx, by]).float()}


def stub_split():
    return [shaky_sequence(n, 24, 32, seed=k)[0] for k, n in enumerate((5, 3, 8, 4, 6))]


KW = dict(batch_size=2, device="cpu", radius=3, sigma=1.5, stride=4, hypotheses=32, sweeps=16)


def _harness(monkeypatch):
    from rnc import harness
    monkeypatch.setattr(harness, "run_sequences", _stub_sequences)
    monkeypatch.setattr(harness, "run_sequences_bidirectional", _stub_bidirectional)
    return harness


@pytest.mark.parametrize("crop,crop_min", [(False, 0.5), (True, 0.99)])
def test_stabilize_videos_fill_is_the_host_pipeline_and_keeps_fill_false_where_valid(monkeypatch, crop, crop_min):
    harness = _harness(monkeypatch)
    seqs = stub_split()
    kw = dict(KW, crop=crop, crop_min=crop_min)
    plain = harness.stabilize_videos(_InferenceModel(), seqs, **{k: v for k, v in kw.items() if k != "sweeps"})
    got = harness.stabilize_videos(_InferenceModel(), seqs, fill=True, **kw)
    holes = 0
    for seq, r, p in zip(seqs, got, plain):
        for key in ("motion", "transforms", "alpha", "inliers", "matched", "status", "valid"):
            assert torch.equal(r[key], p[key]), key
        v = r["valid"] != 0
        assert torch.equal(r["source"] == SOURCE_KNOWN, v)
        assert torch.equal(r["frames"][v[:, None].expand_as(r["frames"])], p["frames"][v[:, None].expand_as(p["frames"])])
        holes += int((~v).sum())
        # alone, through the host pipeline
        rows = list(_stub_bidirectional(None, [seq]))
        fw = torch.stack([x[2]["flow_up"] for x in rows])[None]
        bw = torch.stack([x[2]["flow_up_bw"] for x in rows])[None]
        M, Minv = r["transforms"][None], host_smooth_path(r["motion"][None], 24, 32, 3, 1.5, crop, crop_min)[1]
        want, src = host_fill_uncovered(p["frames"][None], p["valid"][None], fw, bw, r["motion"][None], M, Minv, sweeps=16)
        assert torch.equal(r["frames"], want[0]) and torch.equal(r["source"], src[0])
    assert holes > 0


def test_crop_above_alpha_leaves_every_pixel_known_and_the_frames_as_they_were(monkeypatch):
    harness = _harness(monkeypatch)
    seqs = stub_split()
    plain = harness.stabilize_videos(_InferenceModel(), seqs, **{k: v for k, v in KW.items() if k != "sweeps"})
    got = harness.stabilize_videos(_InferenceModel(), seqs, fill=True, **KW)
    for r, p in zip(got, plain):
        assert float(p["alpha"]) >= 0.5 and bool((p["valid"] != 0).all())
        assert bool((r["source"] == SOURCE_KNOWN).all()) and torch.equal(r["frames"], p["frames"])


def _fill_worker(rank, world, port, q):
    import torch.distributed as dist
    from rnc import harness
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        harness.run_sequences = _stub_sequences
        harness.run_sequences_bidirectional = _stub_bidirectional
        q.put((rank, harness.validate_stabilization(_InferenceModel(), stub_split(), fill=True, crop=False, **KW)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_validate_stabilization_fill_gloo_equals_world_1(world, monkeypatch):
    from test_flow_metrics import run_ranks
    harness = _harness(monkeypatch)
    want = harness.validate_stabilization(_InferenceModel(), stub_split(), fill=True, crop=False, **KW)
    plain = harness.validate_stabilization(_InferenceModel(), stub_split(), crop=False,
                                           **{k: v for k, v in KW.items() if k != "sweeps"})
    assert set(want) == set(plain) | {"filled", "filled_spatial"}
    assert 0 < want["filled"] < 1 and 0 <= want["filled_spatial"] <= want["filled"]
    assert all(want[k] == plain[k] for k in plain if k not in ("itf",))
    for got in run_ranks(_fill_worker, world):
        assert got == want


# -------------------------------------------------------------------------------------------------------------- errors


def test_argument_errors_raise_before_any_launch(video):
    f, b, A, M, Mi = maps_args(video)
    for args in ((f[0], b, A, M, Mi), (f, b[:, 1:], A, M, Mi), (f, b, A[:, 1:], M, Mi), (f, b, A, M[:, 1:], Mi),
                 (f, b, A, M, Mi[..., :2]), (f[:, :0], b[:, :0], A[:, :0], M[:, :1], Mi[:, :1]),
                 (torch.zeros(1, 1, 2, 4097, 2), torch.zeros(1, 1, 2, 4097, 2), A[:, :1], M[:, :2], Mi[:, :2])):
        for fn in (flow_residual, host_flow_residual, add_global_motion, host_add_global_motion):
            with pytest.raises(ValueError):
                fn(*args)
    fr, va = video["frames"], video["valid"]
    for args, kw in (((fr[:, :, :2], va), {}), ((fr, va[:, 1:]), {}), ((fr, va), dict(sweeps=-1)),
                     ((fr, va), dict(max_distance=0)), ((fr, va), dict(alpha1=-1.0)), ((fr, va), dict(alpha2=math.nan)),
                     ((fr, va), dict(alpha1=math.inf))):
        for fn in (fill_uncovered, host_fill_uncovered):
            with pytest.raises(ValueError):
                fn(*args, f, b, A, M, Mi, **kw)


def test_stabilize_videos_checks_the_fill_arguments_before_the_flow_pass(monkeypatch):
    from rnc import harness

    def boom(*a, **k):
        raise AssertionError("the flow pass ran")

    monkeypatch.setattr(harness, "run_sequences", boom)
    monkeypatch.setattr(harness, "run_sequences_bidirectional", boom)
    seqs = [[torch.zeros(3, 16, 16)] * 3]
    for kw in (dict(sweeps=-1), dict(max_distance=0), dict(alpha1=-1.0), dict(alpha2=math.inf)):
        for fn in (harness.stabilize_videos, harness.validate_stabilization):
            with pytest.raises(ValueError):
                fn(_InferenceModel(), seqs, device="cpu", fill=True, **kw)


# ----------------------------------------------------------------------------------------------------------- C ABI


NAMES = ("rnc_stabilize_flow_residual", "rnc_stabilize_flow_readd")


def test_declarations_match_the_binding():
    with open(os.path.join(ROOT, "include", "rnc.h")) as f:
        header = f.read()
    for name in NAMES:
        m = re.search(r"\nint " + name + r"\(([^;]*)\);", header)
        assert m, name
        args = [a.strip() for a in m.group(1).replace("\n", " ").split(",")]
        want = [native.C.c_void_p if "*" in a else _CTYPE[a.rsplit(" ", 1)[0].replace("const ", "")] for a in args]
        res, argtypes = native.SIGNATURES[name]
        assert argtypes == want and res is native.C.c_int, name


def test_entry_points_return_their_error_codes():
    L = native.lib()
    P = 1 << 20                                         # never dereferenced: every check fails on the host before a launch
    n0 = L.rnc_launch_count()

    def res(V=2, T=5, H=40, W=60, f=P, b=P, A=P, M=P, Mi=P, r=P, rb=P):
        return L.rnc_stabilize_flow_residual(f, 1, 1, 1, 1, 1, b, 1, 1, 1, 1, 1, A, M, Mi, V, T, H, W, r, rb, None)

    def readd(V=2, T=5, H=40, W=60, A=P, M=P, Mi=P, r=P, rb=P):
        return L.rnc_stabilize_flow_readd(A, M, Mi, V, T, H, W, r, rb, None)

    for fn, ptrs in ((res, ("f", "b", "A", "M", "Mi", "r", "rb")), (readd, ("A", "M", "Mi", "r", "rb"))):
        for bad in (dict(V=0), dict(V=65536), dict(T=1), dict(T=65537), dict(H=0), dict(W=4097)):
            assert fn(**bad) == -1, bad
        for p in ptrs:
            assert fn(**{p: 0}) == -2, p
            assert fn(**{p: P + (4 if p in ("A", "M", "Mi") else 2)}) == -2, p
    assert L.rnc_launch_count() == n0


def test_stabilize_fill_cu_has_no_atomics_no_contraction_and_does_not_spill(tmp_path):
    log, sass = _compile_fill(tmp_path, "s.cubin")
    kernels = re.findall(r"Function properties for \S*?flow_kernelILb([01])", log)
    assert sorted(kernels) == ["0", "1"], kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 2 and all(a == "0" and b == "0" for a, b in spills), spills
    assert re.findall(r"(\d+) bytes stack frame", log) == ["0"] * 2
    assert not re.search(r"^\s*(@!?U?P\w+\s+)?(ATOM|ATOMS|ATOMG|RED)[.\s]", sass, re.M)
    _, strict = _compile_fill(tmp_path, "f.cubin", "-fmad=false")
    assert sass == strict


def _compile_fill(tmp_path, name, *flags):
    import subprocess
    from rnc.build import ARCH, CSRC, nvcc_path
    cubin = str(tmp_path / name)
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", *flags, "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-cubin", os.path.join(CSRC, "stabilize_fill.cu"), "-o", cubin]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc_path()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    return out.stdout + out.stderr, re.sub(r"/\*[^*]*\*/", "", sass)
