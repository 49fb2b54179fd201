"""Blind video temporal consistency on the host (rnc.temporal): the restatement against naive per-pixel loops, the bits of P
where nothing is matched, the solve against scipy's direct solve, flicker removal on a shifted video, the warping error, the
argument errors, the C ABI, the harness under torch.distributed, and a compile check of csrc/temporal.cu."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl
import torch
from scipy.ndimage import zoom

from rnc import native
from rnc.restate import PI_F32
from rnc.temporal import (host_temporal_step, host_temporally_consistent, host_warping_error, omega, sigma, summarize_temporal,
                          temporal_step, temporally_consistent, warping_error)
from rnc.synth import shift_sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


# ----------------------------------------------------------------------------------------------- the rule, pixel by pixel


def naive_sample(img, c, px, py):
    H, W = img.shape[-2:]
    px, py = min(max(px, f32(0)), f32(W - 1)), min(max(py, f32(0)), f32(H - 1))
    x0, y0 = math.floor(px), math.floor(py)
    ax, ay = px - f32(x0), py - f32(y0)
    bx, by = f32(1) - ax, f32(1) - ay
    x1, y1 = min(x0 + 1, W - 1), min(y0 + 1, H - 1)
    s = img[c, y0, x0] * (bx * by)
    s = s + img[c, y0, x1] * (ax * by)
    s = s + img[c, y1, x0] * (bx * ay)
    return s + img[c, y1, x1] * (ax * ay)


def naive_step(O, P, I0, I1, G, occ, lam, alpha, sweeps):
    """The rule as written, one pixel at a time in numpy float32 scalars: O, P [C,H,W], I0, I1 [3,H,W], G [2,H,W] float32."""
    C, H, W = P.shape
    lam, alpha = f32(lam), f32(alpha)
    w = np.zeros((H, W), f32)
    r = np.zeros((C, H, W), f32)
    for y in range(H):
        for x in range(W):
            ux, uy = G[0, y, x], G[1, y, x]
            px, py = f32(x) + ux, f32(y) + uy
            if not (np.isfinite(ux) and np.isfinite(uy) and occ[y, x] == 0 and 0 <= px <= W - 1 and 0 <= py <= H - 1):
                continue
            d2 = f32(0)
            for c in range(3):
                e = (I1[c, y, x] - naive_sample(I0, c, px, py)) / f32(255)
                d2 = d2 + e * e
            w[y, x] = lam / (f32(1) + alpha * d2)
            if w[y, x] > 0:
                for c in range(C):
                    r[c, y, x] = w[y, x] * (naive_sample(O, c, px, py) - P[c, y, x])
    weak = w < lam * f32(0.25)
    strong = np.argwhere(~weak)
    d2max = 0
    if weak.any() and len(strong):
        for y, x in np.argwhere(weak):
            d2max = max(d2max, int(((strong - (y, x)) ** 2).sum(1).min()))
    s = f32(math.sqrt(float(lam) / 2))
    if d2max:
        L = 0
        while L * L < 4 * d2max:
            L += 1
        s = min(f32(PI_F32) / f32(L + 1), s)
    om = f32(2) / (f32(1) + s)
    D = np.zeros((C, H, W), f32)
    for _ in range(sweeps):
        for colour in (0, 1):
            for y in range(H):
                for x in range(W):
                    n = (y > 0) + (x > 0) + (x < W - 1) + (y < H - 1)
                    den = f32(n) + w[y, x]
                    if (x + y) % 2 != colour or den == 0:
                        continue
                    for c in range(C):
                        t = f32(-0.0)
                        for yy, xx in ((y - 1, x), (y, x - 1), (y, x + 1), (y + 1, x)):
                            if 0 <= yy < H and 0 <= xx < W:
                                t = t + D[c, yy, xx]
                        D[c, y, x] = D[c, y, x] + om * ((t + r[c, y, x]) / den - D[c, y, x])
    return P + D, om


def step_inputs(V, C, H, W, seed):
    """Frames in 0..255, fractional flows with NaN, +-inf and targets exactly on the last column and row, random
    occlusions, processed frames and previous outputs of another range."""
    g = torch.Generator().manual_seed(seed)
    I0, I1 = (torch.rand(V, 3, H, W, generator=g) * 255 for _ in range(2))
    I1 = 0.7 * I1 + 0.3 * I0                            # some pixels agree, some do not
    G = torch.randn(V, 2, H, W, generator=g) * 2
    G[0, 0, 0, 0] = float("nan")
    G[-1, 1, H // 2, W // 2] = float("inf")
    G[0, 0, H - 1, 0] = -float("inf")
    G[0, 0, H // 2, 0] = W - 1.0                        # p' exactly on x = W-1
    G[0, 1, H // 2, 0] = 0.0
    G[-1, 0, 0, W - 1] = 0.0                            # p' exactly on y = H-1
    G[-1, 1, 0, W - 1] = H - 1.0
    occ = (torch.rand(V, H, W, generator=g) < 0.15).to(torch.uint8)
    P = torch.randn(V, C, H, W, generator=g) * 3 + 10
    O = torch.randn(V, C, H, W, generator=g) * 3 + 12
    return O, P, I0, I1, G, occ


@pytest.mark.parametrize("C,H,W,lam,alpha,sweeps", [(1, 5, 7, 0.1, 50.0, 6), (3, 6, 5, 0.5, 4.0, 5), (2, 1, 6, 1.0, 50.0, 3),
                                                    (4, 1, 1, 0.1, 50.0, 2)])
def test_the_host_restatement_is_the_rule_pixel_by_pixel(C, H, W, lam, alpha, sweeps):
    O, P, I0, I1, G, occ = step_inputs(2, C, H, W, seed=H * 10 + C)
    got = host_temporal_step(O, P, I0, I1, G, occ, lam, alpha, sweeps)
    for v in range(2):
        want, _ = naive_step(*(t[v].numpy() for t in (O, P, I0, I1, G, occ)), lam, alpha, sweeps)
        assert np.array_equal(got[v].numpy().view(np.uint32), want.view(np.uint32)), v


def test_a_weak_region_sets_omega_from_its_distance_transform():
    O, P, I0, I1, G, occ = step_inputs(1, 2, 20, 24, seed=4)
    G.zero_()
    I1.copy_(I0)
    occ.zero_()
    occ[0, 2:18, 3:21] = 1                              # a weak 16x18 block: its centre is 8 px from the nearest strong pixel
    got = host_temporal_step(O, P, I0, I1, G, occ, 0.1, 50.0, 7)
    want, om = naive_step(*(t[0].numpy() for t in (O, P, I0, I1, G, occ)), 0.1, 50.0, 7)
    assert np.array_equal(got[0].numpy(), want)
    assert om == f32(omega(64, 0.1)) == f32(2) / (f32(1) + f32(PI_F32) / f32(17))
    occ[0, 2:18, 3:21] = 0
    occ[0, 4:8, 5:9] = 1                                # a small one: the screening's rate sigma is the smaller
    _, om = naive_step(*(t[0].numpy() for t in (O, P, I0, I1, G, occ)), 0.1, 50.0, 1)
    assert om == f32(omega(4, 0.1)) == f32(omega(0, 0.1)) == f32(2) / (f32(1) + f32(sigma(0.1)))


def test_omega_gives_the_measured_factors():
    assert abs(omega(0, 0.1) - 1.634) < 1e-3                             # no weak pixel: sigma = sqrt(0.05)
    assert abs(omega(12 ** 2, 0.1) - 1.777) < 1e-3                       # a 12-px strip on the border
    assert abs(omega(64 ** 2, 0.1) - 1.953) < 1e-3                       # a 128x128 block
    assert abs(omega(80 ** 2, 0.1) - 1.962) < 1e-3                       # a 160x160 block
    assert abs(omega(200 ** 2, 0.1) - 1.984) < 1e-3                      # a 200-px band on the border
    assert omega(1, 0.0) == 2.0 and omega(0, 0.0) == 2.0                # lam = 0: sigma = 0
    assert sigma(0.1) == float(f32(math.sqrt(float(f32(0.1)) / 2)))


def test_lam_zero_and_a_frame_without_a_match_return_the_processed_frame():
    O, P, I0, I1, G, occ = step_inputs(2, 3, 11, 13, seed=5)
    assert torch.equal(host_temporal_step(O, P, I0, I1, G, occ, 0.0, 50.0, 20), P)
    assert torch.equal(host_temporal_step(O, P, I0, I1, G, torch.ones_like(occ), 0.1, 50.0, 20), P)     # a scene cut
    G[:] = 1e6                                                          # every target leaves the frame
    assert torch.equal(host_temporal_step(O, P, I0, I1, G, occ, 0.3, 50.0, 20), P)
    O[:] = float("nan")                                                 # an unmatched pixel never reads O_k
    assert torch.equal(host_temporal_step(O, P, I0, I1, G, occ, 0.3, 50.0, 20), P)


# ----------------------------------------------------------------------------------------- the solve against scipy


def smooth_field(rng, H, W, scale):
    return torch.from_numpy(zoom(rng.random((H // 16 + 1, W // 16 + 1)), 16, order=3)[:H, :W] * scale).float()


def direct_solve(r, w):
    """(n + w) D - sum_q D_q = r on the 4-neighbour grid, by scipy's sparse LU in fp64."""
    H, W = w.shape
    idx = np.arange(H * W).reshape(H, W)
    a = np.concatenate([idx[:-1].ravel(), idx[:, :-1].ravel()])
    b = np.concatenate([idx[1:].ravel(), idx[:, 1:].ravel()])
    off = sp.csr_matrix((-np.ones(2 * len(a)), (np.concatenate([a, b]), np.concatenate([b, a]))), shape=(H * W, H * W))
    A = off + sp.diags(-np.asarray(off.sum(1)).ravel() + w.ravel())
    return spl.spsolve(A.tocsc(), r.ravel()).reshape(H, W)


# (frame, weak region, omega, the largest error after the default 512 sweeps), measured by this test's own solve; the last row
# is the documented limit of the default: a weak band on the border needs more sweeps
TABLE = [((480, 854), "none", 1.634, 1e-3),
         ((480, 854), "strips", 1.777, 1e-3),
         ((256, 448), "block128", 1.953, 1e-3),
         ((480, 854), "block160", 1.962, 1e-3),
         ((480, 854), "band200", 1.984, 4.0)]


@pytest.mark.parametrize("shape,region,om,bound", TABLE, ids=[t[1] for t in TABLE])
def test_the_default_sweeps_reach_scipys_direct_solve(shape, region, om, bound):
    """lam = 0.1, T - P a smooth field of about 16 in magnitude, weak pixels occluded (w = 0), the rest w = lam."""
    H, W = shape
    rng = np.random.default_rng(0)
    P = smooth_field(rng, H, W, 255.0)
    T = P + smooth_field(rng, H, W, 64.0) - 32.0
    occ = torch.zeros(H, W, dtype=torch.uint8)
    if region == "strips":                              # a 12-px strip along the top border, a 20-px one across the frame
        occ[:12] = 1
        occ[:, 400:420] = 1
    elif region == "block128":
        occ[64:192, 160:288] = 1
    elif region == "block160":
        occ[160:320, 347:507] = 1
    elif region == "band200":
        occ[:, :200] = 1
    I = torch.full((1, 3, H, W), 100.0)
    w = np.where(occ.numpy() == 0, f32(0.1), 0.0)
    want = direct_solve(w * (T - P).double().numpy(), w)
    got = host_temporal_step(T[None, None], P[None, None], I, I, torch.zeros(1, 2, H, W), occ[None], 0.1, 50.0, 512)
    err = np.abs((got[0, 0] - P).double().numpy() - want).max()
    d2 = {"none": 0, "strips": 12 ** 2, "block128": 64 ** 2, "block160": 80 ** 2, "band200": 200 ** 2}[region]
    assert abs(omega(d2, 0.1) - om) < 1e-3
    assert err < bound, err
    if region == "band200":
        assert err > 0.1                                # the default is not enough here, as documented


# ----------------------------------------------------------------------------------------------- flicker removal


def flickering_video(T=6, H=48, W=64, dy=1, dx=2, seed=1):
    """shift_sequence's smooth frames (frame t+1 is frame t moved by (dy, dx)), the exact backward flows (-dx, -dy) with no
    occlusion (pixels entering the frame are unmatched by the in-frame test), and P_t = a_t I_t + b_t + noise."""
    I = torch.stack(shift_sequence(T, H, W, seed=seed, dy=dy, dx=dx))[None]
    G = torch.zeros(1, T - 1, 2, H, W)
    G[:, :, 0], G[:, :, 1] = -dx, -dy
    occ = torch.zeros(1, T - 1, H, W, dtype=torch.uint8)
    g = torch.Generator().manual_seed(seed)
    a = 1 + 0.05 * torch.randn(T, generator=g)
    b = 6 * torch.randn(T, generator=g)
    P = a.view(1, T, 1, 1, 1) * I + b.view(1, T, 1, 1, 1) + torch.randn(I.shape, generator=g)
    return I, P, G, occ


def test_flicker_is_removed_and_the_output_stays_close_to_the_processed_frames():
    from rnc.inpaint import host_ssim, psnr
    from rnc.interp import host_interpolation_error
    I, P, G, occ = flickering_video()
    O = temporally_consistent(P, I, G, occ)
    assert torch.equal(O, host_temporally_consistent(P, I, G, occ)) and torch.equal(O[:, 0], P[:, 0])
    ep, cp = warping_error(P, G, occ)
    eo, co = warping_error(O, G, occ)
    assert torch.equal(cp, co) and (cp == 47 * 62).all()               # (H - dy) (W - dx) matched pixels per frame
    wp, wo = float((ep / cp).mean()), float((eo / co).mean())
    assert wo < 0.1 * wp, (wo, wp)
    err = host_interpolation_error(O[0, 1:], P[0, 1:])
    p = [psnr(s, c) for s, c in zip(err.sq_sum.tolist(), err.count.tolist())]
    s, c = host_ssim(O[0, 1:], P[0, 1:])
    assert min(p) > 25 and float((s / c).min()) > 0.9, (p, s / c)


def test_the_warping_error_is_the_naive_fp64_loop():
    O, P, I0, I1, G, occ = step_inputs(2, 1, 7, 9, seed=8)
    video = torch.stack([I0, I1, 0.5 * I0 + 0.5 * I1], 1)               # [2,3,3,7,9]
    flows = torch.stack([G, G.flip(-1)], 1)
    masks = torch.stack([occ, occ.flip(-2)], 1)
    s, c = host_warping_error(video, flows, masks)
    assert s.dtype == torch.float64 and c.dtype == torch.int64
    for v in range(2):
        for k in range(2):
            vid, g, m = video[v].numpy(), flows[v, k].numpy(), masks[v, k].numpy()
            tot, n = 0.0, 0
            for y in range(7):
                for x in range(9):
                    ux, uy = g[0, y, x], g[1, y, x]
                    px, py = f32(x) + ux, f32(y) + uy
                    if not (np.isfinite(ux) and np.isfinite(uy) and m[y, x] == 0 and 0 <= px <= 8 and 0 <= py <= 6):
                        continue
                    t = 0.0
                    for ch in range(3):
                        e = (float(vid[k + 1, ch, y, x]) - float(naive_sample(vid[k], ch, px, py))) / 255.0
                        t += e * e
                    tot += t
                    n += 1
            assert c[v, k] == n and math.isclose(s[v, k], tot, rel_tol=1e-13), (v, k)


def test_summarize_temporal_averages_frames_then_videos():
    nan = math.nan
    rows = [[[4.0, 1.0, 2, 0.0, 10, 9.0, 10], [0.0, 0.0, 0, 3 * 10 * 255.0 ** 2 / 100, 10, 5.0, 10]],
            [],
            [[1.0, 0.5, 1, nan, nan, nan, nan]]]
    s = summarize_temporal(rows)
    assert s["videos"] == 2 and s["frames"] == 3
    assert s["warping_error_processed"] == (2.0 + 1.0) / 2 and s["warping_error"] == (0.5 + 0.5) / 2
    assert math.isnan(s["psnr"]) and math.isnan(s["ssim"])             # video 2 has no fidelity partials
    one = summarize_temporal(rows[:1])
    assert math.isclose(one["psnr"], (100 + 20) / 2) and math.isclose(one["ssim"], (0.9 + 0.5) / 2)
    empty = summarize_temporal([[], []])
    assert all(math.isnan(empty[k]) for k in ("warping_error", "psnr", "ssim")) and empty["videos"] == 0


# ----------------------------------------------------------------------------------------------------------- arguments


def test_argument_errors_raise_before_any_launch():
    O, P, I0, I1, G, occ = step_inputs(2, 2, 8, 9, seed=1)
    with pytest.raises(ValueError, match="expected processed"):
        temporal_step(O, P[0], I0, I1, G, occ)
    with pytest.raises(ValueError, match="expected out_prev"):
        temporal_step(O[:1], P, I0, I1, G, occ)
    with pytest.raises(ValueError, match="expected frame_prev"):
        temporal_step(O, P, I0[:, :2], I1, G, occ)
    with pytest.raises(ValueError, match="expected frame "):
        temporal_step(O, P, I0, I1[..., 1:], G, occ)
    with pytest.raises(ValueError, match="expected flow_bw"):
        temporal_step(O, P, I0, I1, G[:, :1], occ)
    with pytest.raises(ValueError, match="expected occ_bw"):
        temporal_step(O, P, I0, I1, G, occ[:1])
    with pytest.raises(ValueError, match="one device"):
        temporal_step(O, P, I0, I1, G.to("meta"), occ)
    with pytest.raises(ValueError, match="processed channels"):
        temporal_step(torch.zeros(2, 5, 8, 9), torch.zeros(2, 5, 8, 9), I0, I1, G, occ)
    with pytest.raises(ValueError, match="4096"):
        temporal_step(*(torch.zeros(1, c, 1, 4097) for c in (1, 1, 3, 3, 2)), torch.zeros(1, 1, 4097))
    for bad in (dict(lam=-0.1), dict(lam=math.inf), dict(alpha=math.nan), dict(alpha=1e39), dict(lam="1")):
        with pytest.raises(ValueError, match="finite"):
            temporal_step(O, P, I0, I1, G, occ, **bad)
    for bad in (-1, 2.0, True):
        with pytest.raises(ValueError, match="sweeps >= 0"):
            temporal_step(O, P, I0, I1, G, occ, sweeps=bad)
    with pytest.raises(ValueError, match="expected out"):
        temporal_step(O, P, I0, I1, G, occ, out=torch.zeros(2, 2, 8, 8))
    I, Pv, Gv, ov = flickering_video(T=3, H=8, W=9)
    with pytest.raises(ValueError, match="T >= 2"):
        temporally_consistent(Pv[:, :1], I[:, :1], Gv[:, :0], ov[:, :0])
    with pytest.raises(ValueError, match="expected frames"):
        temporally_consistent(Pv, I[:, :2], Gv, ov)
    with pytest.raises(ValueError, match="expected occ_bw"):
        temporally_consistent(Pv, I, Gv, ov[:, :1])
    with pytest.raises(ValueError, match="one device"):
        temporally_consistent(Pv, I, Gv, ov.to("meta"))
    with pytest.raises(ValueError, match="expected processed"):
        temporally_consistent(Pv[0], I, Gv, ov)
    with pytest.raises(ValueError, match="sweeps >= 0"):
        host_temporally_consistent(Pv, I, Gv, ov, sweeps=-3)
    with pytest.raises(ValueError, match="T >= 2"):
        warping_error(I[:, :1], Gv[:, :0], ov[:, :0])
    with pytest.raises(ValueError, match="expected flow_bw"):
        warping_error(I, Gv[:, :1], ov)
    with pytest.raises(ValueError, match="expected occ_bw"):
        warping_error(I, Gv, ov[..., 1:])
    with pytest.raises(ValueError, match="one device"):
        warping_error(I, Gv.to("meta"), ov)
    with pytest.raises(ValueError, match="65535"):
        warping_error(torch.zeros(1, 65537, 1, 1, 1), torch.zeros(1, 65536, 2, 1, 1), torch.zeros(1, 65536, 1, 1))


def test_make_temporally_consistent_and_validate_check_their_arguments():
    from rnc.harness import make_temporally_consistent, validate_temporal_consistency
    from rnc.synth import build_model
    m = build_model("raft")
    seqs = [[torch.zeros(3, 16, 16)] * 3]
    procs = [torch.zeros(3, 2, 16, 16)]
    with pytest.raises(ValueError, match="inference only"):
        make_temporally_consistent(m, seqs, procs)
    with torch.no_grad():
        with pytest.raises(ValueError, match="1 videos but 2 processed videos"):
            make_temporally_consistent(m, seqs, procs * 2)
        with pytest.raises(ValueError, match="T >= 2"):
            make_temporally_consistent(m, [seqs[0][:1]], [procs[0][:1]])
        with pytest.raises(ValueError, match="expected processed frames"):
            make_temporally_consistent(m, seqs, [procs[0][:2]])
        with pytest.raises(ValueError, match="processed channels"):
            make_temporally_consistent(m, seqs, [torch.zeros(3, 5, 16, 16)])
        with pytest.raises(ValueError, match="finite lam"):
            make_temporally_consistent(m, seqs, procs, lam=-1.0)
        with pytest.raises(ValueError, match="sweeps >= 0"):
            make_temporally_consistent(m, seqs, procs, sweeps=-1)
        with pytest.raises(ValueError, match="4096"):
            make_temporally_consistent(m, [[torch.zeros(3, 2, 4097)] * 2], [torch.zeros(2, 1, 2, 4097)])
        assert make_temporally_consistent(m, [], []) == []
        with pytest.raises(ValueError, match="processed videos"):
            validate_temporal_consistency(m, seqs, [])


# ----------------------------------------------------------------------- the harness under torch.distributed


class _InferenceModel:
    def _needs_grad(self):
        return False


def _stub_bidirectional(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                        alpha1=0.01, alpha2=0.5):
    """run_sequences_bidirectional's yields in its step order, on the CPU: a backward flow from the frames' channels and an
    occlusion mask from their difference; one frame size per call, as the real one requires."""
    from rnc.harness import sequence_schedule
    assert len({tuple(f.shape) for s in sequences for f in s}) == 1
    for step in sequence_schedule([len(s) for s in sequences], batch_size):
        for c in step:
            if not c.idle:
                a, b = sequences[c.seq][c.pair], sequences[c.seq][c.pair + 1]
                yield c.seq, c.pair, {"flow_up_bw": (a[1:] - b[1:]) / 40, "occ_bw": ((a[0] - b[0]).abs() > 30).to(torch.uint8)}


def temporal_split():
    """Six videos of 2 to 6 frames of 16x20, processed with per-frame gain and offset; two with C = 3, the rest C = 1 or 2."""
    seqs, procs = [], []
    for k, n in enumerate((4, 3, 6, 2, 5, 3)):
        seq = shift_sequence(n, 16, 20, seed=k, dy=1, dx=k % 3)
        seqs.append(seq)
        C = (3, 1, 2, 3, 1, 2)[k]
        g = torch.Generator().manual_seed(k)
        procs.append(torch.stack([f[:C] * (1 + 0.1 * torch.randn(1, generator=g)) + 5 * torch.randn(1, generator=g)
                                  for f in seq]))
    return seqs, procs


def _temporal_worker(rank, world, port, q):
    import torch.distributed as dist
    from rnc import harness
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        harness.run_sequences_bidirectional = _stub_bidirectional
        q.put((rank, harness.validate_temporal_consistency(_InferenceModel(), *temporal_split(), batch_size=2, device="cpu",
                                                           sweeps=16)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_validate_temporal_consistency_gloo_equals_world_1(world, monkeypatch):
    from test_flow_metrics import run_ranks
    from rnc import harness
    monkeypatch.setattr(harness, "run_sequences_bidirectional", _stub_bidirectional)
    seqs, procs = temporal_split()
    want = harness.validate_temporal_consistency(_InferenceModel(), seqs, procs, batch_size=2, device="cpu", sweeps=16)
    assert want["videos"] == 6 and want["frames"] == sum(len(s) for s in seqs) - 6
    assert 0 < want["warping_error"] < want["warping_error_processed"]
    assert math.isnan(want["psnr"])                                     # C = 1 and 2 videos carry no fidelity partials
    got = harness.make_temporally_consistent(_InferenceModel(), seqs, procs, batch_size=2, device="cpu", sweeps=16)
    for seq, p, out in zip(seqs, procs, got):                           # each video as temporally_consistent defines it, alone
        r = [x[2] for x in _stub_bidirectional(None, [seq])]
        G, occ = (torch.stack([x[k] for x in r])[None] for k in ("flow_up_bw", "occ_bw"))
        assert torch.equal(out, host_temporally_consistent(p[None], torch.stack(seq)[None], G, occ, sweeps=16)[0])
    for got in run_ranks(_temporal_worker, world):                      # bit for bit, on every rank (NaN where C != 3)
        assert got.keys() == want.keys() and all(got[k] == want[k] or math.isnan(got[k]) and math.isnan(want[k]) for k in want)
    colour = harness.validate_temporal_consistency(_InferenceModel(), [seqs[0], seqs[3]], [procs[0], procs[3]],
                                                   batch_size=2, device="cpu", sweeps=16)
    assert 20 < colour["psnr"] < 100 and 0 < colour["ssim"] < 1


# ----------------------------------------------------------------------------- C ABI


_CTYPE = {"long long": native.C.c_longlong, "int": native.C.c_int, "size_t": native.C.c_size_t, "float": native.C.c_float}
NAMES = ("rnc_temporal_step_workspace_bytes", "rnc_temporal_step", "rnc_warping_error_partials_workspace_bytes",
         "rnc_warping_error_partials")


def test_declarations_match_the_binding():
    with open(os.path.join(ROOT, "include", "rnc.h")) as f:
        header = f.read()
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
    ws = L.rnc_temporal_step_workspace_bytes(2, 3, 40, 60)
    assert ws >= 2 * 40 * 60 * (2 * 3 * 4 + 4 + 4 + 1)
    for bad in ((0, 3, 4, 4), (65536, 1, 4, 4), (1, 0, 4, 4), (1, 5, 4, 4), (1, 1, 0, 4), (1, 1, 4, 4097)):
        assert L.rnc_temporal_step_workspace_bytes(*bad) == 0, bad

    def step(V=2, C=3, H=40, W=60, lam=0.1, alpha=50.0, sig=0.2, sweeps=4, o=P, p=P, i0=P, i1=P, g=P, m=P, q=P, wsp=P,
             wsb=ws):
        return L.rnc_temporal_step(o, 1, 1, 1, 1, p, 1, 1, 1, 1, i0, 1, 1, 1, 1, i1, 1, 1, 1, 1, g, 1, 1, 1, 1, m, 1, 1, 1,
                                   V, C, H, W, lam, alpha, sig, sweeps, q, 1, 1, 1, 1, wsp, wsb, None)

    for bad in (dict(V=0), dict(V=65536), dict(C=0), dict(C=5), dict(H=0), dict(W=4097), dict(sweeps=-1), dict(lam=-1.0),
                dict(lam=math.inf), dict(alpha=math.nan), dict(sig=-0.5)):
        assert step(**bad) == -1, bad
    for bad in (dict(o=0), dict(p=0), dict(i0=0), dict(i1=0), dict(g=0), dict(m=0), dict(q=0), dict(wsp=0), dict(o=P + 2),
                dict(g=P + 1), dict(q=P + 2), dict(wsp=P + 8)):
        assert step(**bad) == -2, bad
    assert step(wsb=ws - 1) == -5
    wws = L.rnc_warping_error_partials_workspace_bytes(2, 4, 3, 40, 60)
    assert wws == 2 * 3 * 2 * 16
    for bad in ((0, 4, 3, 40, 60), (1, 1, 3, 40, 60), (2, 32769, 3, 4, 4), (1, 2, 0, 4, 4), (1, 2, 1, 0, 4),
                (1, 2, 1, 32768, 32768)):
        assert L.rnc_warping_error_partials_workspace_bytes(*bad) == 0, bad

    def warp(V=2, T=4, C=3, H=40, W=60, v=P, g=P, m=P, s=P, c=P, wsp=P, wsb=wws):
        return L.rnc_warping_error_partials(v, 1, 1, 1, 1, 1, g, 1, 1, 1, 1, 1, m, 1, 1, 1, 1, V, T, C, H, W, s, c, wsp, wsb,
                                            None)

    for bad in (dict(V=0), dict(T=1), dict(C=0), dict(H=0)):
        assert warp(**bad) == -1, bad
    for bad in (dict(v=0), dict(g=0), dict(m=0), dict(s=0), dict(c=0), dict(wsp=0), dict(v=P + 2), dict(s=P + 4),
                dict(c=P + 4), dict(wsp=P + 8)):
        assert warp(**bad) == -2, bad
    assert warp(wsb=wws - 1) == -5
    assert L.rnc_launch_count() == n0


BIT_EXACT = ("target_kernel", "omega_kernel", "sor_kernel", "sor_kernel", "finish_kernel", "dist2_column_kernel",
             "dist2_row_kernel", "cta_partials_kernel", "image_reduce_kernel")


def _compile(tmp_path, name, *flags):
    from rnc.build import ARCH, CSRC, nvcc_path
    cubin = str(tmp_path / name)
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", *flags, "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-cubin", os.path.join(CSRC, "temporal.cu"), "-o", cubin]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc_path()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    return out.stdout + out.stderr, re.sub(r"/\*[^*]*\*/", "", sass)


def test_temporal_cu_has_no_atomics_no_contraction_and_does_not_spill(tmp_path):
    log, sass = _compile(tmp_path, "t.cubin")
    names = "|".join(sorted(set(BIT_EXACT)))
    kernels = re.findall(r"Function properties for \S*?\d(" + names + r")\w*", log)
    assert sorted(kernels) == sorted(BIT_EXACT), kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == len(BIT_EXACT) and all(a == "0" and b == "0" for a, b in spills), spills
    assert re.findall(r"(\d+) bytes stack frame", log) == ["0"] * len(BIT_EXACT)
    assert not re.search(r"^\s*(@!?U?P\w+\s+)?(ATOM|ATOMS|ATOMG|RED)[.\s]", sass, re.M)
    # every FFMA and DFMA left is inside __fdiv_rn's and __ddiv_rn's correctly rounded divisions
    _, strict = _compile(tmp_path, "s.cubin", "-fmad=false")
    assert sass == strict
