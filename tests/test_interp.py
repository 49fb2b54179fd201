"""Frame interpolation on the host (rnc.interp.host_interpolate, the kernels' reference) against the algorithm's stated
properties, the host feature transform against a brute-force search, the interpolation error against numpy, and the argument
checks of interpolate, interpolate_frames and validate_interpolation."""
import math

import numpy as np
import pytest
import torch

from rnc.interp import (host_interpolate, host_interpolation_error, interpolate, interpolation_error, summarize_interpolation,
                        InterpPartials)
from rnc.metrics import host_fb_consistency, nearest_site
from rnc.synth import shift_sequence


def zeros(B, H, W):
    return torch.zeros(B, 2, H, W), torch.zeros(B, 2, H, W), torch.zeros(B, H, W, dtype=torch.uint8), \
        torch.zeros(B, H, W, dtype=torch.uint8)


def test_zero_flow_without_occlusion_is_the_cross_fade():
    g = torch.Generator().manual_seed(1)
    I0, I1 = torch.rand(2, 3, 9, 13, generator=g) * 255, torch.rand(2, 3, 9, 13, generator=g) * 255
    out = interpolate(I0, I1, *zeros(2, 9, 13), times=(0.25, 0.5, 0.75))
    assert out.shape == (2, 3, 3, 9, 13) and out.dtype == torch.float32
    for k, t in enumerate((0.25, 0.5, 0.75)):
        assert torch.equal(out[:, k], (1 - t) * I0 + t * I1), t


@pytest.mark.parametrize("dy,dx", [(3, 4), (2, 6)])
def test_global_translation_reproduces_the_middle_frame(dy, dx):
    H, W = 40, 56
    f = shift_sequence(3, H, W, seed=3, dy=dy, dx=dx)
    F = torch.empty(1, 2, H, W)
    F[:, 0], F[:, 1] = 2 * dx, 2 * dy
    occ, occ_bw, _, _ = host_fb_consistency(F, -F)
    out = host_interpolate(f[0][None], f[2][None], F, -F, occ, occ_bw, (0.5,))[0, 0]
    # interior: both samples x -+ (dx, dy) lie in the frame
    ys, xs = slice(dy, H - dy), slice(dx, W - dx)
    assert torch.equal(out[:, ys, xs], f[1][:, ys, xs])


def moving_square(H=24, W=40, side=8, y0=8, x0=10, dx=8):
    """Frame 0: background 40, a square of 200 at (y0, x0); frame 1: background 60, the square (220) moved dx to the right.
    The frames' levels differ so that each output pixel shows which frame it came from (a blend gives the mean)."""
    I0, I1 = torch.full((1, 3, H, W), 40.0), torch.full((1, 3, H, W), 60.0)
    I0[..., y0:y0 + side, x0:x0 + side] = 200.0
    I1[..., y0:y0 + side, x0 + dx:x0 + dx + side] = 220.0
    F, G = torch.zeros(1, 2, H, W), torch.zeros(1, 2, H, W)
    F[:, 0, y0:y0 + side, x0:x0 + side] = dx
    G[:, 0, y0:y0 + side, x0 + dx:x0 + dx + side] = -dx
    occ, occ_bw, _, _ = host_fb_consistency(F, G)
    return I0, I1, F, G, occ, occ_bw


def test_moving_square_takes_the_visible_frame():
    H, W, side, y0, x0, dx = 24, 40, 8, 8, 10, 8
    I0, I1, F, G, occ, occ_bw = moving_square(H, W, side, y0, x0, dx)
    # the masks: frame 0's background that the square covers in frame 1 is occluded, frame 1's disoccluded background too
    rows = slice(y0, y0 + side)
    assert (occ[0, rows, x0 + side:x0 + side + dx] != 0).all() and (occ[0, rows, x0:x0 + side] == 0).all()
    assert (occ_bw[0, rows, x0:x0 + dx] != 0).all() and (occ_bw[0, rows, x0 + dx:x0 + dx + side] == 0).all()
    out = host_interpolate(I0, I1, F, G, occ, occ_bw, (0.5,))[0, 0, 0]
    h = dx // 2
    # the square at t = 0.5, seen by both frames: the blend of 200 and 220
    assert (out[rows, x0 + h:x0 + h + side] == 210.0).all()
    # the strip the square leaves (no proposal: frame 1's background there is disoccluded, frame 0 shows the square): x1
    # falls on frame 1's disoccluded pixels, so every pixel takes frame 0 alone (40 or 200, never a blend)
    trail = out[rows, x0:x0 + h]
    assert ((trail == 40.0) | (trail == 200.0)).all(), trail
    # the strip the square enters: x0 falls on frame 0's covered background, so every pixel takes frame 1 alone
    lead = out[rows, x0 + side + h:x0 + side + dx]
    assert ((lead == 60.0) | (lead == 220.0)).all(), lead
    # where the fill gives the square's motion (the half of each strip nearer the square, away from its corners) the
    # background shows
    inner = slice(y0 + 2, y0 + side - 2)
    assert (out[inner, x0 + h - 2:x0 + h] == 40.0).all() and (out[inner, x0 + side + h:x0 + side + h + 2] == 60.0).all()
    # everything else is background seen by both frames
    rest = torch.ones(H, W, dtype=torch.bool)
    rest[rows, x0:x0 + side + dx] = False
    assert (out[rest] == 50.0).all()


def isolated(W, f0=(), f1=()):
    """A 1xW pair where only the listed pixels are sources: f0 = [(x, F_u)] of frame 0, f1 = [(y, G_u)] of frame 1; every
    other pixel is occluded in both masks, so at the target the output is the winner's own pixel in its own frame (its
    sample in the other frame lands on an occluded pixel)."""
    I0, I1 = torch.zeros(1, 3, 1, W), torch.zeros(1, 3, 1, W)
    F, G = torch.zeros(1, 2, 1, W), torch.zeros(1, 2, 1, W)
    occ, occ_bw = torch.ones(1, 1, W, dtype=torch.uint8), torch.ones(1, 1, W, dtype=torch.uint8)
    for x, u in f0:
        F[0, 0, 0, x] = u
        occ[0, 0, x] = 0
    for y, u in f1:
        G[0, 0, 0, y] = u
        occ_bw[0, 0, y] = 0
    return I0, I1, F, G, occ, occ_bw


def test_smaller_error_wins_then_smaller_index():
    # frame-0 pixels 1 (F = +4) and 5 (F = -4) both land on pixel 3 at t = 0.5; e(1) = 3 |I1(5) - I0(1)|,
    # e(5) = 3 |I1(1) - I0(5)|; the output at 3 is the winner's I0
    I0, I1, F, G, occ, occ_bw = isolated(9, f0=[(1, 4.0), (5, -4.0)])
    I0[..., 1], I0[..., 5] = 10.0, 20.0

    def at3(i1_at_5, i1_at_1):
        I1[..., 5], I1[..., 1] = i1_at_5, i1_at_1
        return host_interpolate(I0, I1, F, G, occ, occ_bw, (0.5,))[0, 0, :, 0, 3]
    assert (at3(10.0, 0.0) == 10.0).all()           # e(1) = 0 < e(5) = 60
    assert (at3(0.0, 20.0) == 20.0).all()           # e(1) = 30 > e(5) = 0
    assert (at3(10.0, 20.0) == 10.0).all()          # equal e: the smaller index, 1


def test_frame_0_wins_a_tie_with_frame_1():
    # frame-0 pixel 1 (F = +4, u = +4) and frame-1 pixel 4 (G = -2, target rint(4 - 1) = 3, u = +2) both land on pixel 3;
    # e(frame 0) = 3 |I1(5) - I0(1)|, e(frame 1) = 3 |I0(2) - I1(4)|
    I0, I1, F, G, occ, occ_bw = isolated(9, f0=[(1, 4.0)], f1=[(4, -2.0)])
    I0[..., 1], I1[..., 4] = 10.0, 40.0
    I1[..., 5], I0[..., 2] = 10.0, 40.0             # both e = 0: frame 0's index 1 < HW + 4
    assert (host_interpolate(I0, I1, F, G, occ, occ_bw, (0.5,))[0, 0, :, 0, 3] == 10.0).all()
    I1[..., 5] = 11.0                               # e(frame 0) = 3 > 0: frame 1 wins
    assert (host_interpolate(I0, I1, F, G, occ, occ_bw, (0.5,))[0, 0, :, 0, 3] == 40.0).all()


def brute_nearest(s):
    N, H, W = s.shape
    out = np.full((N, H, W), -1)
    for n in range(N):
        ys, xs = np.nonzero(s[n])
        if len(ys) == 0:
            continue
        for y in range(H):
            for x in range(W):
                d = (ys - y) ** 2 + (xs - x) ** 2
                c = np.nonzero(d == d.min())[0]
                best = min(c, key=lambda i: (xs[i], ys[i]))
                out[n, y, x] = ys[best] * W + xs[best]
    return out


def test_hole_fill_is_the_nearest_site_with_the_tie_rule():
    rng = np.random.default_rng(0)
    for trial in range(40):
        H, W = rng.integers(1, 15, 2)
        s = rng.random((3, H, W)) < rng.choice([0.0, 0.03, 0.1, 0.4])
        if trial % 4 == 0:                         # equidistant sites
            s[:] = False
            s[:, H // 2, 0] = s[:, 0, W // 2] = s[:, H - 1, W - 1] = True
        assert (nearest_site(s) == brute_nearest(s)).all(), trial


def test_an_image_without_sources_has_zero_motion():
    g = torch.Generator().manual_seed(2)
    I0, I1 = torch.rand(1, 3, 6, 7, generator=g) * 255, torch.rand(1, 3, 6, 7, generator=g) * 255
    F = torch.randn(1, 2, 6, 7, generator=g) * 3
    occ = torch.ones(1, 6, 7, dtype=torch.uint8)
    out = host_interpolate(I0, I1, F, -F, occ, occ, (0.3,))[0, 0]
    assert torch.equal(out, 0.7 * I0[0] + 0.3 * I1[0])        # u = 0; both masks occluded everywhere: v0 == v1


def test_interpolation_error_equals_numpy():
    g = torch.Generator().manual_seed(3)
    pred, gt = torch.rand(4, 3, 17, 23, generator=g) * 255, torch.rand(4, 3, 17, 23, generator=g) * 255
    p = interpolation_error(pred, gt)
    d = pred.double().numpy() - gt.double().numpy()
    want = (d ** 2).sum(1).reshape(4, -1).sum(1)
    np.testing.assert_allclose(p.sq_sum.numpy(), want, rtol=1e-13)
    assert p.count.tolist() == [17 * 23] * 4
    s = summarize_interpolation(p)
    assert s["frames"] == 4
    assert math.isclose(s["ie"], float(np.mean(np.sqrt(want / (17 * 23)))), rel_tol=1e-12)
    assert math.isclose(s["psnr"], float(np.mean(10 * np.log10(255 ** 2 * 3 * 17 * 23 / want))), rel_tol=1e-12)
    assert host_interpolation_error(pred[:1], pred[:1]).sq_sum.item() == 0.0
    exact = summarize_interpolation(InterpPartials(torch.zeros(1, dtype=torch.float64), torch.tensor([5])))
    assert exact["ie"] == 0.0 and exact["psnr"] == math.inf
    assert math.isnan(summarize_interpolation(InterpPartials(torch.zeros(0), torch.zeros(0)))["ie"])


def test_argument_errors_raise_before_any_launch():
    I = torch.zeros(1, 3, 4, 5)
    F, G, o, ob = zeros(1, 4, 5)
    for bad in ((0.0,), (1.0,), (-0.2,), (0.5, 1.5), (), (0.999999999,)):
        with pytest.raises(ValueError, match="time"):
            interpolate(I, I, F, G, o, ob, bad)
    with pytest.raises(ValueError, match="frames"):
        interpolate(I, torch.zeros(1, 3, 4, 6), F, G, o, ob)
    with pytest.raises(ValueError, match="flow_bw"):
        interpolate(I, I, F, torch.zeros(1, 2, 5, 4), o, ob)
    with pytest.raises(ValueError, match="occ"):
        interpolate(I, I, F, G, torch.zeros(1, 4, 4, dtype=torch.uint8), ob)
    with pytest.raises(ValueError, match="one device"):
        interpolate(I, I, F, G.to("meta"), o, ob)
    with pytest.raises(ValueError, match="one \\[N,3,H,W\\] shape"):
        interpolation_error(I, torch.zeros(1, 3, 4, 6))
    with pytest.raises(ValueError, match="one device"):
        interpolation_error(I, I.to("meta"))


def test_interpolate_frames_is_inference_only_and_checks_times():
    from rnc.harness import interpolate_frames
    from rnc.synth import build_model
    m = build_model("raft")
    I = torch.zeros(1, 3, 16, 16)
    with pytest.raises(ValueError, match="inference only"):
        interpolate_frames(m, I, I)
    with torch.no_grad(), pytest.raises(ValueError, match="time"):
        interpolate_frames(m, I, I, times=(1.0,))


def test_validate_interpolation_checks_frame_sizes():
    from rnc.harness import validate_interpolation
    from rnc.synth import build_model
    seqs = [[torch.zeros(3, 16, 16)] * 3, [torch.zeros(3, 16, 24)] * 3]
    with pytest.raises(ValueError, match="same \\[3,H,W\\] size"):
        validate_interpolation(build_model("raft"), seqs)


def _stub_bidirectional(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda"):
    """run_sequences_bidirectional's yields in its step order, on the CPU: flows from the frames' first two channels, the
    masks of host_fb_consistency."""
    from rnc.harness import sequence_schedule
    for step in sequence_schedule([len(s) for s in sequences], batch_size):
        for c in step:
            if not c.idle:
                a, b = sequences[c.seq][c.pair], sequences[c.seq][c.pair + 1]
                fw, bw = ((b[:2] - a[:2]) / 8)[None], ((a[1:] - b[1:]) / 8)[None]
                occ, occ_bw, _, _ = host_fb_consistency(fw, bw)
                yield c.seq, c.pair, {"flow_up": fw[0], "flow_up_bw": bw[0], "occ": occ[0], "occ_bw": occ_bw[0]}


def interpolation_sequences():
    """Seven sequences of 2 to 9 frames, one without a triplet."""
    return [shift_sequence(n, 12, 20, seed=n, dy=k % 3, dx=2) for k, n in enumerate((5, 2, 9, 3, 6, 4, 7))]


def _interpolation_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    from rnc import harness
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        harness.run_sequences_bidirectional = _stub_bidirectional
        q.put((rank, harness.validate_interpolation(None, interpolation_sequences(), batch_size=2, device="cpu")))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_validate_interpolation_gloo_equals_world_1(world, monkeypatch):
    from test_flow_metrics import run_ranks
    from rnc import harness
    monkeypatch.setattr(harness, "run_sequences_bidirectional", _stub_bidirectional)
    seqs = interpolation_sequences()
    want = harness.validate_interpolation(None, seqs, batch_size=2, device="cpu")
    parts = []                                      # per triplet in (sequence, k) order, as the host defines it
    for seq in seqs:
        for k in range(len(seq) - 2):
            r = {name: v[None] for name, v in next(_stub_bidirectional(None, [[seq[k], seq[k + 2]]]))[2].items()}
            pred = host_interpolate(seq[k][None], seq[k + 2][None], r["flow_up"], r["flow_up_bw"], r["occ"], r["occ_bw"])
            parts.append(host_interpolation_error(pred[:, 0], seq[k + 1][None]))
    assert want == summarize_interpolation(InterpPartials(*(torch.cat(f) for f in zip(*parts))))
    assert want["frames"] == sum(len(s) - 2 for s in seqs if len(s) > 2)
    for got in run_ranks(_interpolation_worker, world):
        assert got == want                                  # bit for bit, on every rank


def test_interp_cu_does_not_spill(tmp_path):
    import os
    import re
    import subprocess
    from rnc.build import ARCH, CSRC, ROOT, nvcc_path
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-c", os.path.join(CSRC, "interp.cu"), "-o", str(tmp_path / "i.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    kernels = re.findall(r"Function properties for \S*?\d((?:dist2|interp|cta|image)_[a-z0-9_]+_kernel)", log)
    assert sorted(kernels) == ["cta_partials_kernel", "dist2_column_kernel", "dist2_row_kernel", "image_reduce_kernel",
                               "interp_composite_kernel", "interp_splat_kernel"], kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 6 and all(a == "0" and b == "0" for a, b in spills), spills
