"""Unsupervised losses without a GPU (rnc/unsupervised.py, DESIGN §3.16): the host restatements against naive numpy loops and
fp64 gradcheck, the census on an exactly translated pair, argument errors, unsupervised_step's call of the bidirectional
forward, the binding of the new entry points and photometric.cu compiling for sm_90a without spills."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch
import torch.nn as nn

from conftest import ROOT, build_model
from rnc import native
from rnc.synth import smooth_shift_frames
from rnc.unsupervised import (_warp, census_loss, host_census_hamming, host_census_loss, host_smoothness_loss,
                              host_unsupervised_loss, smoothness_loss)

CSRC = os.path.join(ROOT, "raft-ncup_b200", "csrc")
ENTRY_POINTS = ("rnc_census_loss_workspace_bytes", "rnc_census_loss_fwd", "rnc_census_loss_bwd",
                "rnc_smoothness_workspace_bytes", "rnc_smoothness_fwd", "rnc_smoothness_bwd")


def rows(N, H, W, seed=0, scale=3.0, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    i1 = torch.rand(N, 3, H, W, generator=g, dtype=dtype) * 255
    i2 = torch.rand(N, 3, H, W, generator=g, dtype=dtype) * 255
    flow = torch.randn(N, 2, H, W, generator=g, dtype=dtype) * scale
    mask = torch.rand(N, H, W, generator=g) < 0.7
    return i1, i2, flow, mask


def naive_census(i1, i2, flow, mask):
    i1, i2, flow = (t.numpy() for t in (i1, i2, flow))
    N, _, H, W = i1.shape
    g1 = 0.2989 * i1[:, 0] + 0.5870 * i1[:, 1] + 0.1140 * i1[:, 2]
    g2 = 0.2989 * i2[:, 0] + 0.5870 * i2[:, 1] + 0.1140 * i2[:, 2]
    S = M = 0.0
    for n in range(N):
        def at(a, y, x):
            return a[n, y, x] if 0 <= x < W and 0 <= y < H else 0.0
        wh = np.zeros((H, W))
        for y in range(H):
            for x in range(W):
                px, py = x + flow[n, 0, y, x], y + flow[n, 1, y, x]
                if not (math.isfinite(px) and math.isfinite(py)):
                    continue                                            # samples nothing: W^ = 0
                x0, y0 = math.floor(px), math.floor(py)
                ax, ay = px - x0, py - y0
                wh[y, x] = ((1 - ay) * ((1 - ax) * at(g2, y0, x0) + ax * at(g2, y0, x0 + 1)) +
                            ay * ((1 - ax) * at(g2, y0 + 1, x0) + ax * at(g2, y0 + 1, x0 + 1)))
        for y in range(3, H - 3):
            for x in range(3, W - 3):
                if mask is not None and not mask[n, y, x]:
                    continue
                h = 0.0
                for dy in range(-3, 4):
                    for dx in range(-3, 4):
                        a = at(g1, y + dy, x + dx) - g1[n, y, x]
                        b = (wh[y + dy, x + dx] if 0 <= x + dx < W and 0 <= y + dy < H else 0.0) - wh[y, x]
                        e = a / math.sqrt(0.81 + a * a) - b / math.sqrt(0.81 + b * b)
                        h += e * e / (0.1 + e * e)
                S += (h + 0.01) ** 0.4
                M += 1
    return S / (M + 1e-6)


def naive_smoothness(im, flow, kappa=150.0):
    im, flow = im.numpy(), flow.numpy()
    N, _, H, W = flow.shape
    sx = sy = 0.0
    for n in range(N):
        for k in range(2):
            f = flow[n, k]
            for y in range(H):
                for x in range(W):
                    if 1 <= x <= W - 2:
                        d = f[y, x + 1] - 2 * f[y, x] + f[y, x - 1]
                        w = math.exp(-kappa * np.abs(im[n, :, y, x] - im[n, :, y, x - 1]).mean() / 255)
                        sx += math.sqrt(d * d + 1e-6) * w
                    if 1 <= y <= H - 2:
                        d = f[y + 1, x] - 2 * f[y, x] + f[y - 1, x]
                        w = math.exp(-kappa * np.abs(im[n, :, y, x] - im[n, :, y - 1, x]).mean() / 255)
                        sy += math.sqrt(d * d + 1e-6) * w
    return 0.5 * (sx / (N * 2 * H * (W - 2)) + sy / (N * 2 * (H - 2) * W))


@pytest.mark.parametrize("with_mask", [True, False])
def test_host_census_loss_matches_naive_loops(with_mask):
    i1, i2, flow, mask = rows(2, 9, 11, seed=1)
    mask = mask if with_mask else None
    got = float(host_census_loss(i1, i2, flow, mask))
    assert got == pytest.approx(naive_census(i1, i2, flow, mask), rel=1e-12)
    # non-finite flows sample nothing: W^ = 0 with a zero derivative; +-1e12 leaves the frame
    bad = flow.clone()
    for k, v in enumerate((math.nan, math.inf, -math.inf, 1e12, -1e12)):
        bad[0, k % 2, 2 + k, 1:9] = v
    bad[1, :, 4:7, 3:8] = math.nan
    f = bad.clone().requires_grad_()
    got = host_census_loss(i1, i2, f, mask)
    assert float(got) == pytest.approx(naive_census(i1, i2, bad, mask), rel=1e-12)
    got.backward()
    nonfinite = ~torch.isfinite(bad).all(1, keepdim=True).expand_as(bad)
    assert torch.isfinite(f.grad).all() and not f.grad[nonfinite].any()
    w = _warp(i2[:, 0], bad)
    assert not w[nonfinite[:, 0]].any() and torch.isfinite(w).all()


def test_host_smoothness_loss_of_a_non_finite_flow_is_not_finite():
    i1, _, flow, _ = rows(2, 9, 11, seed=3)
    for v in (math.nan, math.inf):
        bad = flow.clone()
        bad[1, 0, 4, 5] = v
        got, want = float(host_smoothness_loss(i1, bad)), naive_smoothness(i1, bad)
        assert not math.isfinite(got) and (math.isnan(got) == math.isnan(want) == math.isnan(v))


def test_host_census_loss_with_an_all_zero_mask_row():
    i1, i2, flow, mask = rows(2, 9, 11, seed=2)
    mask[0] = False
    got = float(host_census_loss(i1, i2, flow, mask))
    assert got == pytest.approx(naive_census(i1, i2, flow, mask), rel=1e-12)
    assert float(host_census_loss(i1, i2, flow, torch.zeros_like(mask))) == 0.0


def test_host_smoothness_loss_matches_naive_loops():
    i1, _, flow, _ = rows(2, 9, 11, seed=3)
    for kappa in (150.0, 10.0):
        got = float(host_smoothness_loss(i1, flow, kappa))
        assert got == pytest.approx(naive_smoothness(i1, flow, kappa), rel=1e-12)


def kink_free_flow(N, H, W, seed):
    """A flow whose sample positions x + F, y + F keep their fractional parts in [0.05, 0.95]: away from the bilinear kinks."""
    g = torch.Generator().manual_seed(seed)
    whole = torch.randint(-3, 4, (N, 2, H, W), generator=g).double()
    return whole + 0.05 + 0.9 * torch.rand(N, 2, H, W, generator=g, dtype=torch.float64)


def test_gradcheck_host_census_loss():
    i1, i2, _, mask = rows(2, 8, 9, seed=4)
    flow = kink_free_flow(2, 8, 9, seed=4).requires_grad_()
    assert torch.autograd.gradcheck(lambda f: host_census_loss(i1, i2, f, mask), (flow,), eps=1e-6, atol=1e-8, rtol=1e-5)


def test_gradcheck_host_smoothness_loss():
    i1, _, _, _ = rows(2, 8, 9, seed=5)
    flow = kink_free_flow(2, 8, 9, seed=5).requires_grad_()
    assert torch.autograd.gradcheck(lambda f: host_smoothness_loss(i1, f), (flow,), eps=1e-6, atol=1e-8, rtol=1e-5)


def test_the_true_translation_has_zero_hamming_distance_and_a_lower_loss():
    dy, dx = 3, 4
    i1, i2 = (t.double() for t in smooth_shift_frames(2, 32, 40, dy=dy, dx=dx))
    flow = torch.zeros(2, 2, 32, 40, dtype=torch.float64)
    flow[:, 0], flow[:, 1] = dx, dy
    h = host_census_hamming(i1, i2, flow)
    # every pixel of such a window, and its target, lies inside the frame
    assert torch.equal(h[:, 3:32 - 3 - dy, 3:40 - 3 - dx], torch.zeros_like(h[:, 3:32 - 3 - dy, 3:40 - 3 - dx]))
    assert float(host_census_loss(i1, i2, flow)) < float(host_census_loss(i1, i2, torch.zeros_like(flow)))


def test_argument_errors():
    i1, i2, flow, mask = rows(2, 9, 11, seed=6, dtype=torch.float32)
    for fn in (census_loss, host_census_loss):
        with pytest.raises(ValueError, match="image2"):
            fn(i1, i2[:1], flow)
        with pytest.raises(ValueError, match="mask"):
            fn(i1, i2, flow, mask[:, :5])
        with pytest.raises(ValueError, match="mask must be bool or uint8"):
            fn(i1, i2, flow, mask.float())
        with pytest.raises(ValueError, match="flow must be floating"):
            fn(i1, i2, flow.long())
        with pytest.raises(ValueError, match="image1 must be floating"):
            fn(i1.to(torch.uint8), i2, flow)
        with pytest.raises(ValueError, match="image1 requires grad"):
            fn(i1.clone().requires_grad_(), i2, flow)
        small = rows(1, 7, 11, dtype=torch.float32)
        with pytest.raises(ValueError, match="at least 8x8"):
            fn(*small[:3])
    for fn in (smoothness_loss, host_smoothness_loss):
        with pytest.raises(ValueError, match="flow"):
            fn(i1, flow[:, :1])
        with pytest.raises(ValueError, match="at least 8x8"):
            fn(i1[..., :7], flow[..., :7])
        with pytest.raises(ValueError, match="image requires grad"):
            fn(i1.clone().requires_grad_(), flow)


def test_cpu_tensors_do_not_reach_the_kernels():
    i1, i2, flow, mask = rows(2, 9, 11, dtype=torch.float32)
    with pytest.raises(native.RncUnavailable):
        census_loss(i1, i2, flow, mask)
    with pytest.raises(native.RncUnavailable):
        smoothness_loss(i1, flow)


def test_bidirectional_forward_rejects_a_malformed_flow_init():
    m = build_model("raft")
    im = torch.zeros(2, 3, 64, 64)
    good = torch.zeros(2, 2, 8, 8)
    for bad in (good, (good,), (good, torch.zeros(2, 2, 8, 9)), (torch.zeros(1, 2, 8, 8), None)):
        with pytest.raises(ValueError, match="flow_init"):
            m(im, im, iters=1, flow_init=bad, bidirectional=True)
    with pytest.raises(ValueError, match="one shape"):
        m(im, im[:1], iters=1, bidirectional=True)
    with pytest.raises(native.RncUnavailable):                 # a well-formed call still needs CUDA
        m(im, im, iters=1, flow_init=(good, None), bidirectional=True)


def test_unsupervised_step_trains_through_the_bidirectional_forward(monkeypatch):
    """unsupervised_step runs the model with bidirectional=True and the sequence loss on its 2B rows (here the host loss, on
    the CPU, in place of the kernels)."""
    from rnc import train

    class Stub(nn.Module):
        def __init__(self):
            super().__init__()
            self.flow = nn.Parameter(torch.full((2,), 0.5))
            self.calls = []

        def forward(self, image1, image2, iters=12, bidirectional=False):
            self.calls.append((iters, bidirectional))
            B, _, H, W = image1.shape
            f = self.flow.view(1, 2, 1, 1).expand(B, 2, H, W)
            return [torch.cat([f, -f]) * (i + 1) / iters for i in range(iters)]      # consistent: both directions visible

    monkeypatch.setattr(train, "unsupervised_loss", host_unsupervised_loss)
    i1, i2 = smooth_shift_frames(2, 16, 24, dy=1, dx=1)
    m = Stub()
    opt = torch.optim.SGD(m.parameters(), lr=1e-3)
    loss, metrics = train.unsupervised_step(m, opt, None, i1, i2, iters=3)
    assert m.calls == [(3, True)]
    assert torch.isfinite(loss) and set(metrics) == {"census", "smoothness", "occluded_fw", "occluded_bw"}
    assert not torch.equal(m.flow.detach(), torch.full((2,), 0.5))
    assert train.unsupervised_step(m, opt, None, i1, i2, iters=2, return_metrics=False)[1] is None


def test_entry_points_declared_and_bound():
    with open(os.path.join(ROOT, "include", "rnc.h")) as f:
        declared = set(re.findall(r"\b(rnc_\w+)\s*\(", f.read()))
    for n in ENTRY_POINTS:
        assert n in declared and n in native.SIGNATURES, n
    assert native.ABI_VERSION == 18


def test_entry_points_reject_bad_arguments():
    L = native.lib()
    assert L.rnc_census_loss_workspace_bytes(2, 9, 11) > 0 and L.rnc_smoothness_workspace_bytes(2, 9, 11) > 0
    for n, h, w in ((0, 9, 11), (2, 7, 11), (2, 9, 7), (70000, 9, 11)):
        assert L.rnc_census_loss_workspace_bytes(n, h, w) == 0 and L.rnc_smoothness_workspace_bytes(n, h, w) == 0
    P = 1 << 20   # never dereferenced: every check fails on the host before a launch
    n0 = L.rnc_launch_count()
    ws = L.rnc_census_loss_workspace_bytes(2, 9, 11)

    def census(N=2, H=9, W=11, img=P, flow=P, state=P, wsp=P, wsb=ws):
        return L.rnc_census_loss_fwd(img, 297, 99, 11, 1, img, 297, 99, 11, 1, flow, 198, 99, 11, 1, None, N, H, W, P, P, P,
                                     state, wsp, wsb, None)

    assert census(H=7) == -1 and census(img=None) == -2 and census(flow=P + 2) == -2 and census(wsb=ws - 1) == -5
    assert L.rnc_census_loss_bwd(P, 2, 9, 7, P, P, None) == -1 and L.rnc_census_loss_bwd(None, 2, 9, 11, P, P, None) == -2
    sws = L.rnc_smoothness_workspace_bytes(2, 9, 11)
    assert L.rnc_smoothness_fwd(P, 297, 99, 11, 1, P, 198, 99, 11, 1, 2, 9, 11, 150.0, P, P, P, P, sws - 1, None) == -5
    assert L.rnc_smoothness_fwd(P, 297, 99, 11, 1, P, 198, 99, 11, 1, 2, 9, 11, 150.0, None, P, P, P, sws, None) == -2
    assert L.rnc_smoothness_bwd(P, 297, 99, 11, 1, P, 198, 99, 11, 1, 2, 6, 11, 150.0, P, P, None) == -1
    assert L.rnc_launch_count() == n0


def test_photometric_kernels_do_not_spill(tmp_path):
    from rnc.build import ARCH, nvcc_path
    try:
        nvcc = nvcc_path()
    except RuntimeError:
        pytest.skip("nvcc not available")
    cmd = [nvcc, *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-c", os.path.join(CSRC, "photometric.cu"), "-o", str(tmp_path / "p.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", out.stdout + out.stderr)
    assert len(spills) >= 8
    assert all(s == ("0", "0") for s in spills), spills
