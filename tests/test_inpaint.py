"""Video inpainting on the host (rnc.inpaint's restatements, the kernels' references): the harmonic fill against a direct
sparse solve of the Laplace equation, propagation along the true flows of a shifted video, the chains' stopping rules, the
masked bilinear colour and the distance weighting, SSIM against an fp64 scipy restatement, the PSNR cap and the summary, the
argument checks, validate_inpainting under gloo, the C entry points' error codes and declarations, and a compile of
inpaint.cu for sm_90a."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.ndimage as ndi
import scipy.sparse as sp
import scipy.sparse.linalg as spl
import torch

from rnc import native
from rnc.inpaint import (SOURCE_BACKWARD, SOURCE_BOTH, SOURCE_FORWARD, SOURCE_KNOWN, SOURCE_SPATIAL, SSIM_TAPS,
                         harmonic_fill, host_harmonic_fill, host_inpaint, host_inpaint_propagate, host_ssim, inpaint,
                         inpaint_propagate, omega, psnr, ssim, summarize_inpainting)
from rnc.synth import shift_sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ----------------------------------------------------------------------------------------------------------- harmonic fill


def laplace_solve(f, unk):
    """The discrete Laplace equation on the unknown pixels of f (fp64 [H,W]) with the known pixels as boundary values,
    each pixel's in-frame 4-neighbours only, by a direct sparse solve."""
    H, W = f.shape
    idx = -np.ones((H, W), np.int64)
    idx[unk] = np.arange(unk.sum())
    rows, cols, vals = [], [], []
    b = np.zeros(unk.sum())
    for y, x in zip(*np.nonzero(unk)):
        i = idx[y, x]
        n = 0
        for dy, dx in ((-1, 0), (0, -1), (0, 1), (1, 0)):
            yy, xx = y + dy, x + dx
            if 0 <= yy < H and 0 <= xx < W:
                n += 1
                if unk[yy, xx]:
                    rows.append(i), cols.append(idx[yy, xx]), vals.append(-1.0)
                else:
                    b[i] += f[yy, xx]
        rows.append(i), cols.append(i), vals.append(float(n))
    return spl.spsolve(sp.csr_matrix((vals, (rows, cols)), shape=(len(b), len(b))), b)


@pytest.mark.parametrize("side", [64, 128])
def test_the_fill_matches_a_direct_laplace_solve(side):
    H, W = side + 30, side + 36
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    f = np.stack([20 * np.sin(xs / 17.0) * np.cos(ys / 23.0), 15 * np.cos((xs + ys) / 29.0) - 5])   # smooth, within +-20
    unk = np.zeros((H, W), bool)
    unk[13:13 + side, 20:20 + side] = True
    v = torch.tensor(f, dtype=torch.float32)
    got = host_harmonic_fill(v[None], torch.tensor(unk)[None])[0].double().numpy()
    for c in range(2):
        want = laplace_solve(v[c].double().numpy(), unk)
        assert np.abs(got[c][unk] - want).max() < 1e-3, c
        assert np.array_equal(got[c][~unk], v[c].double().numpy()[~unk])       # known pixels copied through
    assert torch.equal(harmonic_fill(v[None], torch.tensor(unk)[None]), torch.from_numpy(got).float()[None])


def test_omega_gives_the_measured_factors():
    for L, w in ((64, 1.908), (128, 1.953), (200, 1.969), (300, 1.979)):
        assert abs(omega(L) - w) < 1e-3, L
    assert omega(64) == float(np.float32(2) / (np.float32(1) + np.float32(np.pi) / np.float32(65)))


def test_a_constant_field_stays_exactly_constant():
    unk = torch.zeros(2, 20, 24, dtype=torch.uint8)
    unk[0, 3:15, 4:20] = 1
    unk[1, :, 10:] = 1                                                  # touching three borders
    for c in (3.0, -1.25, 7.5):                                         # sums of these few-bit values are exact
        v = torch.full((2, 2, 20, 24), c)
        assert torch.equal(host_harmonic_fill(v, unk, 64), v), c


def test_an_image_without_a_known_pixel_is_zero_and_non_finite_values_are_unknown():
    v = torch.randn(2, 3, 9, 11)
    unk = torch.zeros(2, 9, 11, dtype=torch.uint8)
    unk[0] = 1
    v[1, 2, 4, 5] = float("nan")                                       # one channel: the whole pixel is unknown
    v[1, 0, 0, 0] = float("inf")
    got = host_harmonic_fill(v, unk, 0)
    assert torch.equal(got[0], torch.zeros(3, 9, 11))
    assert torch.equal(got[1, :, 4, 5], v[1, :, 4, 4])                 # of the four nearest, the smallest column
    assert torch.equal(got[1, :, 0, 0], v[1, :, 1, 0])                 # (1, 0) and (0, 1): column 0
    full = host_harmonic_fill(v, unk, 40)
    assert torch.equal(full[0], torch.zeros(3, 9, 11)) and torch.isfinite(full).all()
    mask = torch.ones(9, 11, dtype=torch.bool)
    mask[4, 5] = mask[0, 0] = False
    assert torch.equal(full[1][:, mask], v[1][:, mask])


def test_the_values_at_unknown_pixels_are_never_read():
    g = torch.Generator().manual_seed(1)
    v = torch.randn(3, 2, 17, 19, generator=g) * 5
    unk = (torch.rand(3, 17, 19, generator=g) < 0.3).to(torch.uint8)
    unk[1, 5:12, 3:16] = 1
    want = host_harmonic_fill(v, unk, 30)
    poisoned = v.clone()
    poisoned[unk[:, None].expand_as(v) != 0] = float("nan")
    assert torch.equal(host_harmonic_fill(poisoned, unk, 30), want)
    poisoned[unk[:, None].expand_as(v) != 0] = 1e30
    assert torch.equal(host_harmonic_fill(poisoned, unk, 30), want)
    stacked = host_harmonic_fill(v.view(1, 3, 2, 17, 19), unk.view(1, 3, 17, 19), 30)      # [V,T,...] is the same rule
    assert torch.equal(stacked[0], want)


# ----------------------------------------------------------------------------------------------------------- propagation


def shifted_video(T, H, W, dy, dx, seed=3):
    """Integer-valued frames whose content moves (dx, dy) a frame, and the true flows: F = (dx, dy), G = -F.  Integer
    colours and distances make the distance weighting exact, so propagated pixels equal the ground truth bit for bit."""
    seq = torch.stack([f.round() for f in shift_sequence(T, H, W, seed=seed, dy=dy, dx=dx)])
    F = torch.empty(T - 1, 2, H, W)
    F[:, 0], F[:, 1] = dx, dy
    return seq, F, -F


def test_true_flows_propagate_the_ground_truth_and_never_seen_content_is_spatial():
    T, H, W, dy, dx = 8, 40, 56, 1, 2
    frames, F, G = shifted_video(T, H, W, dy, dx)
    masks = torch.zeros(T, H, W, dtype=torch.uint8)
    masks[:, 12:24, 20:32] = 1                                          # a static square: the content slides under it
    for t in range(T):                                                  # a square moving with the content: never seen
        masks[t, 28 + t * dy:34 + t * dy, 4 + t * dx:10 + t * dx] = 1
    corrupted = torch.where(masks[:, None] != 0, float("nan"), frames)
    out, source = host_inpaint(corrupted[None], masks[None], F[None], G[None], sweeps=64)
    out, source = out[0], source[0]
    assert torch.equal(source == SOURCE_KNOWN, masks == 0)
    assert torch.equal(out[masks[:, None].expand_as(out) == 0], frames[masks[:, None].expand_as(out) == 0])
    temporal = (source >= SOURCE_FORWARD) & (source <= SOURCE_BOTH)
    assert temporal.sum() > 0.9 * (12 * 12 * T)
    for s in (SOURCE_FORWARD, SOURCE_BACKWARD, SOURCE_BOTH):
        assert (source == s).any(), s
    t_idx = temporal[:, None].expand_as(out)
    assert torch.equal(out[t_idx], frames[t_idx])                       # exactly the ground truth
    for t in range(T):
        assert (source[t, 28 + t * dy:34 + t * dy, 4 + t * dx:10 + t * dx] == SOURCE_SPATIAL).all(), t
    assert torch.isfinite(out).all()


def tiny(T=3, H=4, W=6, fx=1.0, fy=0.0):
    """A video of constant frames t * 10 + channel, zero holes, flows (fx, fy) forward and the negation backward, nothing
    occluded."""
    frames = (torch.arange(T, dtype=torch.float32).view(T, 1, 1, 1) * 10 + torch.arange(3.0).view(1, 3, 1, 1)).expand(
        T, 3, H, W).clone()
    masks = torch.zeros(T, H, W, dtype=torch.uint8)
    F = torch.empty(T - 1, 2, H, W)
    F[:, 0], F[:, 1] = fx, fy
    occ = torch.zeros(T - 1, H, W, dtype=torch.uint8)
    return frames, masks, F, -F, occ, occ.clone()


def prop(frames, masks, F, G, occ, occ_bw, max_distance=None):
    out, src = host_inpaint_propagate(frames[None], masks[None], F[None], G[None], occ[None], occ_bw[None], max_distance)
    return out[0], src[0]


def test_chains_stop_at_the_last_frame_the_border_an_occlusion_and_max_distance():
    frames, masks, F, G, occ, occ_bw = tiny()
    masks[0, 1, 1] = 1
    out, src = prop(frames, masks, F, G, occ, occ_bw)
    assert src[0, 1, 1] == SOURCE_FORWARD and torch.equal(out[0, :, 1, 1], frames[1, :, 1, 2])   # backward: k = 0 stops
    assert src[1].eq(SOURCE_KNOWN).all() and src[2].eq(SOURCE_KNOWN).all()
    masks[1:, :, :] = 1                                                 # every later frame a hole: the chain runs out
    out, src = prop(frames, masks, F, G, occ, occ_bw)
    assert src[0, 1, 1] == SOURCE_SPATIAL and out[0, :, 1, 1].eq(0).all()
    frames, masks, F, G, occ, occ_bw = tiny(fx=4.5)                     # 1 + 4.5 > W - 1: leaves the frame
    masks[0, 1, 1] = 1
    assert prop(frames, masks, F, G, occ, occ_bw)[1][0, 1, 1] == SOURCE_SPATIAL
    frames, masks, F, G, occ, occ_bw = tiny(fx=4.0)                     # 1 + 4 = W - 1: still inside
    masks[0, 1, 1] = 1
    assert prop(frames, masks, F, G, occ, occ_bw)[1][0, 1, 1] == SOURCE_FORWARD
    frames, masks, F, G, occ, occ_bw = tiny()
    masks[0, 1, 1] = 1
    occ[0, 1, 1] = 1                                                    # occluded where the chain starts
    assert prop(frames, masks, F, G, occ, occ_bw)[1][0, 1, 1] == SOURCE_SPATIAL
    frames, masks, F, G, occ, occ_bw = tiny()
    masks[0, 1, 1] = masks[1, 1, 2] = 1                                 # the first step lands in frame 1's hole
    out, src = prop(frames, masks, F, G, occ, occ_bw, max_distance=1)
    assert src[0, 1, 1] == SOURCE_SPATIAL
    out, src = prop(frames, masks, F, G, occ, occ_bw, max_distance=2)
    assert src[0, 1, 1] == SOURCE_FORWARD and torch.equal(out[0, :, 1, 1], frames[2, :, 1, 3])
    occ[1, 1, 2] = 1                                                    # the second step is occluded
    assert prop(frames, masks, F, G, occ, occ_bw)[1][0, 1, 1] == SOURCE_SPATIAL
    # backward: frame 2's pixel walks through G to frame 1, whose hole sends it on to frame 0
    frames, masks, F, G, occ, occ_bw = tiny()
    masks[2, 2, 3] = masks[1, 2, 2] = 1
    out, src = prop(frames, masks, F, G, occ, occ_bw)
    assert src[2, 2, 3] == SOURCE_BACKWARD and torch.equal(out[2, :, 2, 3], frames[0, :, 2, 1])
    occ_bw[0, 2, 2] = 1
    assert prop(frames, masks, F, G, occ, occ_bw)[1][2, 2, 3] == SOURCE_SPATIAL


def test_the_masked_bilinear_colour_renormalises_over_the_taps_outside_the_hole():
    frames, masks, F, G, occ, occ_bw = tiny(H=5, W=6, fx=0.5, fy=0.0)
    frames[1] = torch.arange(3 * 5 * 6, dtype=torch.float32).view(3, 5, 6) * 1.5
    masks[0, 1, 1] = masks[1, 1, 1] = 1
    masks[1, 0, 0] = 1                                                  # not a tap: changes nothing
    frames[1, :, 1, 1] = float("nan")                                   # the hole tap's colour is never read
    out, src = prop(frames, masks, F, G, occ, occ_bw)
    # x = 1.5 rounds to 2: frame 1's (1, 2) is not a hole; taps (1,1) hole, (1,2) w 0.5, (2,1) and (2,2) weight 0
    assert src[0, 1, 1] == SOURCE_FORWARD and torch.equal(out[0, :, 1, 1], frames[1, :, 1, 2])
    F[:, 0], F[:, 1] = 0.75, 0.25
    out, src = prop(frames, masks, F, -F, occ, occ_bw)
    w = {(1, 2): 0.5625, (2, 1): 0.0625, (2, 2): 0.1875}                # (1,1), weight 0.1875, is the hole
    want = sum(wi * frames[1, :, y, x].double() for (y, x), wi in w.items()) / sum(w.values())
    assert src[0, 1, 1] == SOURCE_FORWARD
    assert torch.allclose(out[0, :, 1, 1].double(), want, rtol=1e-6, atol=0)


def test_two_candidates_are_weighted_by_the_other_ones_distance():
    frames, masks, F, G, occ, occ_bw = tiny(T=4, fx=0.0)
    masks[1, 2, 2] = masks[2, 2, 2] = 1                                 # frame 1: backward 1 frame, forward 2 frames
    out, src = prop(frames, masks, F, G, occ, occ_bw)
    assert src[1, 2, 2] == SOURCE_BOTH and src[2, 2, 2] == SOURCE_BOTH
    # (d_b c_f + d_f c_b) / (d_f + d_b): frame 1 = (1 * 30 + 2 * 0) / 3, frame 2 = (2 * 30 + 1 * 0) / 3, plus the channel
    assert torch.equal(out[1, :, 2, 2], torch.tensor([10.0, 11.0, 12.0]))
    assert torch.equal(out[2, :, 2, 2], torch.tensor([20.0, 21.0, 22.0]))


def test_the_cpu_entry_points_are_the_host_restatements():
    T, H, W = 4, 14, 18
    g = torch.Generator().manual_seed(2)
    frames = torch.rand(2, T, 3, H, W, generator=g) * 255
    masks = (torch.rand(2, T, H, W, generator=g) < 0.2).to(torch.uint8)
    F, G = (torch.randn(2, T - 1, 2, H, W, generator=g) * 1.5 for _ in range(2))
    occ, occ_bw = ((torch.rand(2, T - 1, H, W, generator=g) < 0.1).to(torch.uint8) for _ in range(2))
    assert all(torch.equal(a, b) for a, b in zip(inpaint_propagate(frames, masks, F, G, occ, occ_bw),
                                                 host_inpaint_propagate(frames, masks, F, G, occ, occ_bw)))
    F0 = F.clone()
    got = inpaint(frames, masks, F, G, sweeps=20)
    assert torch.equal(F, F0)                                           # the inputs are not modified
    want = host_inpaint(frames, masks, F, G, sweeps=20)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    assert torch.isfinite(got[0]).all() and got[1].eq(SOURCE_SPATIAL).any()


# ----------------------------------------------------------------------------------------------------------- scoring


def scipy_ssim(a, b):
    """SSIM of two [3,H,W] frames in fp64 (scipy's separable correlation with the fp64 Gaussian), over the valid pixels."""
    x = np.exp(-(np.arange(-5, 6, dtype=np.float64) ** 2) / 4.5)
    g = x / x.sum()

    def filt(q):
        return ndi.correlate1d(ndi.correlate1d(q, g, axis=-1), g, axis=-2)[..., 5:-5, 5:-5]
    a, b = a.astype(np.float64), b.astype(np.float64)
    mx, my = filt(a), filt(b)
    sx, sy, sxy = filt(a * a) - mx * mx, filt(b * b) - my * my, filt(a * b) - mx * my
    C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2
    return float((((2 * mx * my + C1) * (2 * sxy + C2)) / ((mx * mx + my * my + C1) * (sx + sy + C2))).mean())


def test_ssim_is_one_for_identical_frames_and_matches_an_fp64_restatement():
    g = torch.Generator().manual_seed(4)
    noise = torch.rand(2, 3, 30, 41, generator=g) * 255
    smooth = torch.stack(shift_sequence(2, 30, 41, seed=9))
    s, c = host_ssim(noise, noise)
    assert torch.equal(s / c, torch.ones(2, dtype=torch.float64)) and c.tolist() == [3 * 20 * 31] * 2
    for a, b in ((noise[0:1], (noise[1:2] + noise[0:1]) / 2), (smooth[0:1], smooth[1:2]),
                 (smooth[0:1], (smooth[0:1] + torch.randn(1, 3, 30, 41, generator=g) * 8).clamp(0, 255))):
        s, c = ssim(a, b)
        assert abs(float(s[0] / c[0]) - scipy_ssim(a[0].numpy(), b[0].numpy())) < 1e-4
    assert abs(float(SSIM_TAPS.astype(np.float64).sum()) - 1) < 1e-6


def test_psnr_caps_at_100_and_unscored_videos_are_skipped():
    assert psnr(0.0, 10) == 100.0
    assert math.isclose(psnr(3 * 10 * 255.0 ** 2 / 100, 10), 20.0)      # MSE = 255^2 / 100
    rec = [[0.0, 10, 9.0, 10], [3 * 10 * 255.0 ** 2 / 100, 10, 5.0, 10]]
    s = summarize_inpainting([rec, [], [[0.0, 4, 4.0, 4]]])
    assert s["videos"] == 2 and s["frames"] == 3
    assert math.isclose(s["psnr"], ((100 + 20) / 2 + 100) / 2)
    assert math.isclose(s["ssim"], ((0.9 + 0.5) / 2 + 1.0) / 2)
    empty = summarize_inpainting([[], []])
    assert math.isnan(empty["psnr"]) and math.isnan(empty["ssim"]) and empty["videos"] == 0


# ----------------------------------------------------------------------------------------------------------- arguments


def test_argument_errors_raise_before_any_launch():
    v, u = torch.zeros(2, 2, 8, 9), torch.zeros(2, 8, 9, dtype=torch.uint8)
    with pytest.raises(ValueError, match="expected unknown"):
        harmonic_fill(v, u[:, 1:])
    with pytest.raises(ValueError, match="one device"):
        harmonic_fill(v, u.to("meta"))
    with pytest.raises(ValueError, match="channels"):
        harmonic_fill(torch.zeros(2, 5, 8, 9), u)
    with pytest.raises(ValueError, match="4096"):
        harmonic_fill(torch.zeros(1, 2, 1, 4097), torch.zeros(1, 1, 4097))
    with pytest.raises(ValueError, match="sweeps >= 0"):
        harmonic_fill(v, u, -1)
    with pytest.raises(ValueError, match="values"):
        harmonic_fill(v[0], u[0])
    frames, masks, F, G, occ, occ_bw = (t[None] for t in tiny(T=3))
    with pytest.raises(ValueError, match="masks"):
        inpaint_propagate(frames, masks[:, :2], F, G, occ, occ_bw)
    with pytest.raises(ValueError, match="flow_bw"):
        inpaint_propagate(frames, masks, F, G[..., 1:], occ, occ_bw)
    with pytest.raises(ValueError, match="occ_bw"):
        inpaint_propagate(frames, masks, F, G, occ, occ_bw[:, :1])
    with pytest.raises(ValueError, match="one device"):
        inpaint_propagate(frames, masks, F, G, occ.to("meta"), occ_bw)
    with pytest.raises(ValueError, match="T >= 2"):
        inpaint_propagate(frames[:, :1], masks[:, :1], F[:, :0], G[:, :0], occ[:, :0], occ_bw[:, :0])
    with pytest.raises(ValueError, match="max_distance"):
        inpaint_propagate(frames, masks, F, G, occ, occ_bw, max_distance=0)
    with pytest.raises(ValueError, match="4096"):
        inpaint_propagate(torch.zeros(1, 2, 3, 1, 4097), torch.zeros(1, 2, 1, 4097), torch.zeros(1, 1, 2, 1, 4097),
                          torch.zeros(1, 1, 2, 1, 4097), torch.zeros(1, 1, 1, 4097), torch.zeros(1, 1, 1, 4097))
    with pytest.raises(ValueError, match="sweeps >= 0"):
        inpaint(frames, masks, F, G, sweeps=-2)
    with pytest.raises(ValueError, match="max_distance"):
        inpaint(frames, masks, F, G, max_distance=0)
    with pytest.raises(ValueError, match="one device"):
        inpaint(frames, masks, F.to("meta"), G)
    with pytest.raises(ValueError, match="11x11"):
        ssim(torch.zeros(1, 3, 10, 20), torch.zeros(1, 3, 10, 20))
    with pytest.raises(ValueError, match="one \\[N,3,H,W\\] shape"):
        ssim(torch.zeros(1, 3, 20, 20), torch.zeros(1, 3, 20, 21))
    with pytest.raises(ValueError, match="one device"):
        ssim(torch.zeros(1, 3, 20, 20), torch.zeros(1, 3, 20, 20, device="meta"))


def test_inpaint_videos_and_validate_inpainting_check_their_arguments():
    from rnc.harness import inpaint_videos, validate_inpainting
    from rnc.synth import build_model
    m = build_model("raft")
    seqs = [[torch.zeros(3, 16, 16)] * 3]
    masks = [torch.zeros(3, 16, 16, dtype=torch.uint8)]
    with pytest.raises(ValueError, match="inference only"):
        inpaint_videos(m, seqs, masks)
    with torch.no_grad():
        with pytest.raises(ValueError, match="1 videos but 2 mask sets"):
            inpaint_videos(m, seqs, masks * 2)
        with pytest.raises(ValueError, match="T >= 2"):
            inpaint_videos(m, [seqs[0][:1]], [masks[0][:1]])
        with pytest.raises(ValueError, match="expected masks"):
            inpaint_videos(m, seqs, [masks[0][:2]])
        with pytest.raises(ValueError, match="sweeps >= 0"):
            inpaint_videos(m, seqs, masks, sweeps=-1)
        with pytest.raises(ValueError, match="max_distance"):
            inpaint_videos(m, seqs, masks, max_distance=0)
        with pytest.raises(ValueError, match="4096"):
            inpaint_videos(m, [[torch.zeros(3, 2, 4097)] * 2], [torch.zeros(2, 2, 4097)])
        assert inpaint_videos(m, [], []) == []
        with pytest.raises(ValueError, match="mask sets"):
            validate_inpainting(m, seqs, [])


# ----------------------------------------------------------------------------- validate_inpainting under torch.distributed


class _InferenceModel:
    def _needs_grad(self):
        return False


def _stub_bidirectional(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                        alpha1=0.01, alpha2=0.5):
    """run_sequences_bidirectional's yields in its step order, on the CPU: flows from the frames' first channels; one frame
    size per call, as the real one requires."""
    from rnc.harness import sequence_schedule
    assert len({tuple(f.shape) for s in sequences for f in s}) == 1
    for step in sequence_schedule([len(s) for s in sequences], batch_size):
        for c in step:
            if not c.idle:
                a, b = sequences[c.seq][c.pair], sequences[c.seq][c.pair + 1]
                yield c.seq, c.pair, {"flow_up": (b[:2] - a[:2]) / 40, "flow_up_bw": (a[1:] - b[1:]) / 40}


def inpainting_split():
    """Seven videos of 2 to 6 frames in two frame sizes, with a moving square hole (one video without a hole)."""
    seqs, masks = [], []
    for k, (n, H, W) in enumerate(((4, 16, 20), (3, 18, 14), (6, 16, 20), (2, 18, 14), (3, 16, 20), (5, 18, 14),
                                   (4, 16, 20))):
        seqs.append(shift_sequence(n, H, W, seed=k, dy=1, dx=k % 3))
        m = torch.zeros(n, H, W, dtype=torch.uint8)
        if k != 4:
            for t in range(n):
                m[t, 3 + t:9 + t, 2 + (t + k) % 5:8 + (t + k) % 5] = 1
        masks.append(m)
    return seqs, masks


def _inpainting_worker(rank, world, port, q):
    import torch.distributed as dist
    from rnc import harness
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        harness.run_sequences_bidirectional = _stub_bidirectional
        q.put((rank, harness.validate_inpainting(_InferenceModel(), *inpainting_split(), batch_size=2, device="cpu",
                                                 sweeps=16)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_validate_inpainting_gloo_equals_world_1(world, monkeypatch):
    from test_flow_metrics import run_ranks
    from rnc import harness
    monkeypatch.setattr(harness, "run_sequences_bidirectional", _stub_bidirectional)
    seqs, masks = inpainting_split()
    want = harness.validate_inpainting(_InferenceModel(), seqs, masks, batch_size=2, device="cpu", sweeps=16)
    assert want["videos"] == 6 and want["frames"] == sum(len(s) for s in seqs) - 3
    assert 10 < want["psnr"] < 100 and 0 < want["ssim"] < 1
    got = harness.inpaint_videos(_InferenceModel(), seqs, masks, batch_size=2, device="cpu", sweeps=16)
    for seq, m, (out, src) in zip(seqs, masks, got):                    # each video as inpaint defines it, alone
        x = torch.stack([torch.where(h != 0, 0.0, f) for f, h in zip(seq, m)])
        r = [p[2] for p in _stub_bidirectional(None, [list(x)])]
        F, G = (torch.stack([p[k] for p in r])[None] for k in ("flow_up", "flow_up_bw"))
        w_out, w_src = host_inpaint(torch.stack(seq)[None], m[None], F, G, sweeps=16)
        assert torch.equal(out, w_out[0]) and torch.equal(src, w_src[0])
    for got in run_ranks(_inpainting_worker, world):
        assert got == want                              # bit for bit, on every rank


# ----------------------------------------------------------------------------- C ABI


_CTYPE = {"long long": native.C.c_longlong, "int": native.C.c_int, "size_t": native.C.c_size_t, "float": native.C.c_float}
NAMES = ("rnc_harmonic_fill_workspace_bytes", "rnc_harmonic_fill", "rnc_inpaint_propagate",
         "rnc_ssim_partials_workspace_bytes", "rnc_ssim_partials")


def test_declarations_match_the_binding():
    with open(os.path.join(ROOT, "include", "rnc.h")) as f:
        header = f.read()
    assert f"#define RNC_HARMONIC_MAX_CHANNELS {native.HARMONIC_MAX_CHANNELS}" in header
    for name, value in (("KNOWN", SOURCE_KNOWN), ("FORWARD", SOURCE_FORWARD), ("BACKWARD", SOURCE_BACKWARD),
                        ("BOTH", SOURCE_BOTH), ("SPATIAL", SOURCE_SPATIAL)):
        assert f"#define RNC_INPAINT_{name} {value}" in header
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
    ws = L.rnc_harmonic_fill_workspace_bytes(2, 3, 2, 40, 60)
    assert ws >= 6 * 40 * 60 * 5
    for bad in ((0, 1, 2, 4, 4), (1, 0, 2, 4, 4), (256, 256, 2, 4, 4), (1, 1, 0, 4, 4), (1, 1, 5, 4, 4), (1, 1, 2, 0, 4),
                (1, 1, 2, 4, 4097)):
        assert L.rnc_harmonic_fill_workspace_bytes(*bad) == 0, bad

    def fill(A=2, B=3, C=2, H=40, W=60, sweeps=4, v=P, u=P, o=P, wsp=P, wsb=ws):
        return L.rnc_harmonic_fill(v, 1, 1, 1, 1, 1, u, 1, 1, 1, 1, A, B, C, H, W, sweeps, o, 1, 1, 1, 1, 1, wsp, wsb, None)

    for bad in (dict(A=0), dict(B=70000), dict(C=0), dict(C=5), dict(H=0), dict(W=4097), dict(sweeps=-1)):
        assert fill(**bad) == -1, bad
    for bad in (dict(v=0), dict(u=0), dict(o=0), dict(wsp=0), dict(v=P + 2), dict(o=P + 1), dict(wsp=P + 8)):
        assert fill(**bad) == -2, bad
    assert fill(wsb=ws - 1) == -5

    def prop(V=2, T=3, H=40, W=60, maxd=2, i=P, m=P, f=P, g=P, o=P, ob=P, out=P, src=P):
        return L.rnc_inpaint_propagate(i, 1, 1, 1, 1, 1, m, 1, 1, 1, 1, f, 1, 1, 1, 1, 1, g, 1, 1, 1, 1, 1, o, 1, 1, 1, 1,
                                       ob, 1, 1, 1, 1, V, T, H, W, maxd, out, src, None)

    for bad in (dict(V=0), dict(V=65536), dict(T=1), dict(H=0), dict(W=4097), dict(maxd=0)):
        assert prop(**bad) == -1, bad
    for bad in (dict(i=0), dict(m=0), dict(f=0), dict(g=0), dict(o=0), dict(ob=0), dict(out=0), dict(src=0), dict(f=P + 2),
                dict(out=P + 1)):
        assert prop(**bad) == -2, bad
    sws = L.rnc_ssim_partials_workspace_bytes(5, 40, 60)
    assert sws == 5 * 2 * 16
    for bad in ((0, 40, 60), (65536, 40, 60), (1, 10, 60), (1, 40, 10)):
        assert L.rnc_ssim_partials_workspace_bytes(*bad) == 0, bad

    def sim(N=5, H=40, W=60, p=P, g=P, s=P, c=P, wsp=P, wsb=sws):
        return L.rnc_ssim_partials(p, 1, 1, 1, 1, g, 1, 1, 1, 1, N, H, W, s, c, wsp, wsb, None)

    for bad in (dict(N=0), dict(H=10), dict(W=10)):
        assert sim(**bad) == -1, bad
    for bad in (dict(p=0), dict(g=0), dict(s=0), dict(c=0), dict(wsp=0), dict(s=P + 4), dict(c=P + 4), dict(wsp=P + 8)):
        assert sim(**bad) == -2, bad
    assert sim(wsb=sws - 1) == -5
    assert L.rnc_launch_count() == n0


BIT_EXACT = ("known_kernel", "list_offsets_kernel", "compact_kernel", "sor_kernel", "sor_kernel", "propagate_kernel",
             "dist2_column_kernel", "dist2_row_kernel", "cta_partials_kernel", "image_reduce_kernel")


def _compile(tmp_path, name, *flags):
    from rnc.build import ARCH, CSRC, nvcc_path
    cubin = str(tmp_path / name)
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", *flags, "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-cubin", os.path.join(CSRC, "inpaint.cu"), "-o", cubin]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc_path()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    return out.stdout + out.stderr, re.sub(r"/\*[^*]*\*/", "", sass)


def test_inpaint_cu_has_no_atomics_no_contraction_and_does_not_spill(tmp_path):
    log, sass = _compile(tmp_path, "i.cubin")
    names = "|".join(sorted(set(BIT_EXACT)))
    kernels = re.findall(r"Function properties for \S*?\d(" + names + r")\w*", log)
    assert sorted(kernels) == sorted(BIT_EXACT), kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == len(BIT_EXACT) and all(a == "0" and b == "0" for a, b in spills), spills
    assert re.findall(r"(\d+) bytes stack frame", log) == ["0"] * len(BIT_EXACT)
    # memory atomics as opcodes (BAR.RED.POPC, __syncthreads_count's barrier reduction, touches no memory)
    assert not re.search(r"^\s*(@!?U?P\w+\s+)?(ATOM|ATOMS|ATOMG|RED)[.\s]", sass, re.M)
    # every FFMA left is inside __fdiv_rn's correctly rounded division: forbidding contraction changes no instruction
    _, strict = _compile(tmp_path, "s.cubin", "-fmad=false")
    assert sass == strict
