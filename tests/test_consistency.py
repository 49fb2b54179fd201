"""Forward-backward consistency on the host (rnc.metrics.host_fb_consistency, the kernel's test reference): against an fp64
F.grid_sample restatement, on analytic flows (a translation against its negation, a moving square, targets on and just past
the last row and column, NaN), the argument checks, the C entry point's own checks, and validate(consistency=True) with a
stub model."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from rnc.metrics import OCC_INCONSISTENT, OCC_OUTSIDE, fb_consistency, host_fb_consistency

A1, A2 = 0.01, 0.5


def fp64_consistency(f, g, a1=A1, a2=A2):
    """One direction in fp64 through F.grid_sample (zeros padding, align_corners=True on normalised coordinates).  The target is
    the float32 sum x + F(x) the definition rounds once: a coordinate near 1000 carries up to 3e-5 px of that rounding, which
    is part of the float32 input, not of the sampling.  Returns (err, occ, lhs, rhs, mag): mag = |F| + sum_taps w |G|, the
    magnitude of the terms whose rounding the bound scales with."""
    f, g = f.double(), g.double()
    B, _, H, W = f.shape
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    px = (xs + f[:, 0]).float().double()
    py = (ys + f[:, 1]).float().double()
    grid = torch.stack([2 * px / (W - 1) - 1, 2 * py / (H - 1) - 1], -1)
    gs = F.grid_sample(g, grid, mode="bilinear", padding_mode="zeros", align_corners=True)
    gabs = F.grid_sample(g.abs(), grid, mode="bilinear", padding_mode="zeros", align_corners=True)
    s = f + gs
    lhs = (s * s).sum(1)
    rhs = a1 * ((f * f).sum(1) + (gs * gs).sum(1)) + a2
    inside = (px >= 0) & (px <= W - 1) & (py >= 0) & (py <= H - 1)
    err = torch.where(inside, lhs.sqrt(), float("inf"))
    occ = torch.where(inside, (lhs > rhs).to(torch.uint8), 3)
    mag = f.pow(2).sum(1).sqrt() + gabs.pow(2).sum(1).sqrt()
    return err, occ, lhs, rhs, mag


def check_against_fp64(fw, bw, label, got=None):
    """err within 1e-6 of the magnitudes it cancels; occ equal wherever the fp64 margin from the threshold exceeds
    1e-5 (lhs + rhs) + 1e-6.  got: the (occ_fw, occ_bw, err_fw, err_bw) to check, by default host_fb_consistency's (CPU
    tensors).  Returns the number of near-threshold pixels."""
    got = host_fb_consistency(fw, bw, A1, A2) if got is None else [t.cpu() for t in got]
    near = 0
    for d, (f, g) in enumerate(((fw, bw), (bw, fw))):
        occ, err = got[d], got[2 + d]
        e64, o64, lhs, rhs, mag = fp64_consistency(f, g)
        inside = torch.isfinite(e64)
        assert torch.equal(torch.isfinite(err), inside), label
        bad = (err.double() - e64).abs()[inside] > 1e-6 * mag[inside] + 1e-12
        assert not bad.any(), f"{label} dir {d}: {int(bad.sum())} pixels beyond 1e-6 relative"
        far = (lhs - rhs).abs() > 1e-5 * (lhs + rhs) + 1e-6
        near += int((~far & inside).sum())
        assert torch.equal(occ[far | ~inside], o64[far | ~inside]), label
    print(f"{label}: {near} near-threshold pixels")
    return near


def smooth_flow(B, H, W, scale, seed):
    g = torch.Generator().manual_seed(seed)
    coarse = torch.randn(B, 2, 4, 5, generator=g) * scale
    return F.interpolate(coarse, size=(H, W), mode="bicubic", align_corners=True).float()


@pytest.mark.parametrize("H,W,B", [(23, 37, 3), (48, 64, 2)])
def test_host_against_fp64_grid_sample(H, W, B):
    fw = smooth_flow(B, H, W, 6.0, seed=H)
    # a backward flow that cancels the forward one except for a perturbation that crosses the threshold
    bw = -smooth_flow(B, H, W, 6.0, seed=H) + smooth_flow(B, H, W, 1.5, seed=W)
    check_against_fp64(fw, bw, f"smooth {B}x{H}x{W}")
    g = torch.Generator().manual_seed(H * W)
    check_against_fp64(torch.randn(B, 2, H, W, generator=g) * 4, torch.randn(B, 2, H, W, generator=g) * 4,
                       f"random {B}x{H}x{W}")


def translation(B, H, W, t):
    fw = torch.empty(B, 2, H, W)
    fw[:, 0], fw[:, 1] = t
    return fw, -fw


def test_translation_against_its_negation():
    H, W, t = 36, 52, (3.25, -2.5)
    fw, bw = translation(2, H, W, t)
    occ, occ_bw, err, err_bw = host_fb_consistency(fw, bw)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    for o, e, (tx, ty) in ((occ, err, t), (occ_bw, err_bw, (-t[0], -t[1]))):
        out = (xs + tx < 0) | (xs + tx > W - 1) | (ys + ty < 0) | (ys + ty > H - 1)
        assert torch.equal(o, torch.where(out, 3, 0).to(torch.uint8).expand_as(o))     # no interior pixel inconsistent
        assert torch.isinf(e[:, out]).all() and (e[:, ~out] < 1e-5).all()
    check_against_fp64(fw, bw, "translation")


def test_moving_square_flags_the_band_it_covers_and_uncovers():
    H, W, d = 40, 60, 6
    x0, y0, s = 20, 12, 14
    fw, bw = torch.zeros(1, 2, H, W), torch.zeros(1, 2, H, W)
    fw[0, 0, y0:y0 + s, x0:x0 + s] = d                   # the square moves d px right between the frames
    bw[0, 0, y0:y0 + s, x0 + d:x0 + d + s] = -d
    occ, occ_bw, _, _ = host_fb_consistency(fw, bw)
    covered = torch.zeros(H, W, dtype=torch.bool)
    covered[y0:y0 + s, x0 + s:x0 + s + d] = True         # background of frame 1 hidden in frame 2
    uncovered = torch.zeros(H, W, dtype=torch.bool)
    uncovered[y0:y0 + s, x0:x0 + d] = True               # background of frame 2 not visible in frame 1
    assert torch.equal(occ[0] & OCC_INCONSISTENT != 0, covered)
    assert torch.equal(occ_bw[0] & OCC_INCONSISTENT != 0, uncovered)
    assert not (occ & OCC_OUTSIDE).any() and not (occ_bw & OCC_OUTSIDE).any()


def test_targets_on_the_last_row_and_column_are_inside():
    H, W = 9, 13
    fw, bw = torch.zeros(1, 2, H, W), torch.zeros(1, 2, H, W)
    past = lambda v: float(np.nextafter(np.float32(v), np.float32(np.inf)))       # noqa: E731
    fw[0, :, 0, 0] = torch.tensor([W - 1.0, H - 1.0])    # exactly the last column and row
    fw[0, :, 1, 0] = torch.tensor([past(W - 1), 0.0])    # just past the last column
    fw[0, :, 0, 1] = torch.tensor([-1.0, past(H - 1)])   # pixel (1, 0) -> (0, just past the last row)
    fw[0, :, 3, 0] = torch.tensor([-0.0, 0.0])           # on column 0
    fw[0, :, 4, 0] = torch.tensor([-1e-30, 0.0])         # just before column 0
    fw[0, :, 5, 2] = torch.tensor([0.0, -5.0])           # pixel (2, 5) -> (2, 0), on row 0
    occ, _, err, _ = host_fb_consistency(fw, bw)
    at = [(0, 0), (1, 0), (0, 1), (3, 0), (4, 0), (5, 2)]
    assert [int(occ[0, y, x]) & OCC_OUTSIDE for y, x in at] == [0, 2, 2, 0, 2, 0]
    for y, x in at:
        outside = bool(occ[0, y, x] & OCC_OUTSIDE)
        assert bool(torch.isinf(err[0, y, x])) == outside and (occ[0, y, x] == 3) == outside


def test_nan_is_flagged():
    H, W = 10, 12
    fw, bw = torch.zeros(1, 2, H, W), torch.zeros(1, 2, H, W)
    fw[0, 1, 3, 4] = float("nan")                        # a NaN forward flow: its target is nowhere
    bw[0, 0, 6, 7] = float("nan")                        # a NaN backward flow, sampled by the forward pixel (7, 6)
    occ, occ_bw, err, err_bw = host_fb_consistency(fw, bw)
    assert occ[0, 3, 4] == 3 and torch.isinf(err[0, 3, 4])
    assert occ[0, 6, 7] == OCC_INCONSISTENT and torch.isinf(err[0, 6, 7])
    assert occ_bw[0, 6, 7] == 3 and occ_bw[0, 3, 4] == OCC_INCONSISTENT
    # a NaN tap spreads to every pixel whose bilinear reads it, also with weight 0 (0 * NaN), as in F.grid_sample: at zero
    # flow the taps of (x, y) are x..x+1, y..y+1
    reads = lambda y, x: {(y - dy, x - dx) for dy in (0, 1) for dx in (0, 1)}     # noqa: E731
    assert {tuple(p) for p in (occ[0] != 0).nonzero().tolist()} == reads(6, 7) | {(3, 4)}
    assert {tuple(p) for p in (occ_bw[0] != 0).nonzero().tolist()} == reads(3, 4) | {(6, 7)}
    assert not torch.isnan(err).any() and not torch.isnan(err_bw).any()


def test_alphas_are_arguments():
    fw, bw = translation(1, 16, 16, (1.0, 0.0))
    bw = bw + 0.6                                         # |F + G| = 0.6*sqrt(2): lhs 0.72 against 0.5 + alpha1 (...)
    assert (host_fb_consistency(fw, bw)[0][0, :, :15] == OCC_INCONSISTENT).all()
    assert (host_fb_consistency(fw, bw, alpha2=0.8)[0][0, :, :15] == 0).all()
    assert (host_fb_consistency(fw, bw, alpha1=1.0)[0][0, :, :15] == 0).all()


def test_arguments_are_checked():
    f = torch.zeros(2, 2, 4, 5)
    for a, b in ((f, torch.zeros(2, 2, 4, 6)), (torch.zeros(2, 3, 4, 5), torch.zeros(2, 3, 4, 5)), (f[0], f[0]),
                 (f, torch.zeros(1, 2, 4, 5)), (torch.zeros(0, 2, 4, 5), torch.zeros(0, 2, 4, 5)),
                 (f, torch.zeros(2, 2, 4, 5, device="meta"))):
        with pytest.raises(ValueError):
            fb_consistency(a, b)
        with pytest.raises(ValueError):
            host_fb_consistency(a, b)


def test_cpu_tensors_take_the_host_path():
    fw, bw = smooth_flow(2, 11, 14, 3.0, 1), smooth_flow(2, 11, 14, 3.0, 2)
    for x, y in zip(fb_consistency(fw, bw), host_fb_consistency(fw, bw)):
        assert torch.equal(x, y)
    # strided, unpadded views give the results of their contiguous copies
    big = smooth_flow(2, 15, 20, 3.0, 3).permute(0, 1, 3, 2).contiguous().permute(0, 1, 3, 2)
    v1, v2 = big[:, :, 2:13, 3:17], big.flip(0)[:, :, 1:12, 4:18]
    for x, y in zip(host_fb_consistency(v1, v2), host_fb_consistency(v1.contiguous(), v2.contiguous())):
        assert torch.equal(x, y)


def test_entry_point_rejects_bad_arguments():
    from rnc import native
    L = native.lib()
    P = 1 << 20   # never dereferenced: every check fails on the host before a launch
    n0 = L.rnc_launch_count()

    def call(B=2, H=436, W=1024, fw=P, bw=P, o1=P, o2=P, e1=P, e2=P):
        return L.rnc_fb_consistency(fw, 2 * H * W, H * W, W, 1, bw, 2 * H * W, H * W, W, 1, B, H, W, 0.01, 0.5, o1, o2, e1, e2,
                                    None)

    assert call(B=0) == -1 and call(H=0) == -1 and call(W=-1) == -1 and call(B=65536) == -1
    assert call(H=1 << 16, W=1 << 15) == -1
    assert call(fw=0) == -2 and call(bw=0) == -2 and call(o1=0) == -2 and call(o2=0) == -2 and call(e1=0) == -2
    assert call(e2=0) == -2 and call(fw=P + 2) == -2 and call(bw=P + 1) == -2 and call(e1=P + 2) == -2
    assert L.rnc_launch_count() == n0


# ----------------------------------------------------------------------------- validate(consistency=True)


class BidiStub(torch.nn.Module):
    """Flow = the first two channels of image1 - image2 plus a quarter of image1's third channel (so the two directions do
    not cancel exactly); the bidirectional pass stacks both directions."""

    def __init__(self):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))

    def forward(self, im1, im2, iters=12, test_mode=True, flow_init=None):
        flow = im1[:, :2] - im2[:, :2] + im1[:, 2:3] / 4
        return flow[:, :, ::8, ::8], flow

    def forward_bidirectional(self, im1, im2, iters=12, flow_init=None, return_confidence=False):
        lo1, up1 = self(im1, im2)
        lo2, up2 = self(im2, im1)
        return torch.cat([lo1, lo2]), torch.cat([up1, up2])


@pytest.mark.parametrize("sparse", [False, True])
def test_validate_consistency_equals_the_host_definition(sparse):
    from test_flow_metrics import stub_samples
    from rnc.harness import validate
    from rnc.metrics import SparsPartials, host_sparsification, summarize_sparsification
    samples = stub_samples(sparse)
    parts = []
    m = BidiStub()
    for s in samples:
        a, b, gt = s[0][None], s[1][None], s[2][None]
        flow, back = m(a, b)[1], m(b, a)[1]
        parts.append(host_sparsification(flow, gt, s[3][None] if sparse else None, -host_fb_consistency(flow, back)[2]))
    want = summarize_sparsification(SparsPartials(*(torch.cat(c) for c in zip(*parts))))
    plain = validate(m, samples, iters=1, mode="kitti" if sparse else "sintel", batch_size=3, device="cpu")
    for bs in (1, 4):
        res = validate(m, samples, iters=1, mode="kitti" if sparse else "sintel", batch_size=bs, device="cpu",
                       consistency=True)
        assert set(res) == set(plain) | {"fb_sparsification", "ideal", "fb_ause"}
        assert {k: res[k] for k in plain} == plain                               # the existing keys, bit for bit
        assert res["fb_sparsification"] == want["sparsification"] and res["ideal"] == want["ideal"]
        assert res["fb_ause"] == want["ause"] and np.isfinite(res["fb_ause"]) and res["fb_ause"] >= 0
