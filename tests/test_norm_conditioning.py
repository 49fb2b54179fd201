"""InstanceNorm statistics at controlled conditioning: the stimuli, the model transform and the comparators shared with
tests/test_gpu_norm_conditioning.py, and what can be checked without a GPU.

The three routes that feed fnet's InstanceNorm (the convolution epilogue's fused sums + rnc_instnorm_finalize,
rnc_instnorm_stats, rnc_instnorm_stats_det) take the variance as sum(x^2)/P - mean^2.  When |mean| >> std that difference
cancels the leading digits, and whatever rounding the sums carry becomes the variance's error.  A flat frame puts fnet's
norm1 there: the stem output is almost its bias (|mean|/std ~ 2000 on a mid-grey frame).  Here:
  - conditioned(): x = m + sigma * z per (image, channel) at |m|/sigma from 0 to 1e4, both signs, and constant channels;
  - near_uniform_frames(): grey, black, white, grey +- 1 and half-flat frames;
  - stats_bounds() / apply_bound(): the bounds of the GPU checks, independent of the conditioning;
  - trained_like(): a seeded model with BatchNorm statistics, per-channel weight scales and NConv weights spread like a
    trained network's, instead of the random init's identity statistics; compare_per_channel(): a pointwise comparator
    whose bound is taken per output channel;
  - CPU checks: the grey frame really reaches the regime, the bound rejects fp32 partial sums and accepts fp64 ones, the
    per-channel comparator sees a small channel, and the generators and the transform are deterministic.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from test_product_shapes import Mismatch

EPS = 1e-5                                   # nn.InstanceNorm2d's eps (rnc/encoder_umma.py EPS)
RSTD_CONST = float(np.float32(1.0 / np.sqrt(np.float64(np.float32(EPS)))))   # rstd of a constant channel
MEAN_REL, MEAN_FLOOR = 2.0 ** -23, 2.0 ** -126
RSTD_REL = 1e-6
APPLY_TOL = 2e-5                             # the suite's tolerance for one layer (test_product_shapes.TOL["conv"])

# ----------------------------------------------------------------------------------------------------------- (a) stimuli
RATIOS = (0.0, 1.0, 10.0, 100.0, 1000.0, 3000.0, 1e4)      # |m| / sigma
SIGMAS = (1.0, 0.01, 0.37, 1.9)                            # sigma per image: |m| <= 1.9e4 stays inside fp16's range
CONSTS = (0.0, 0.7301, 1234.5, -96.25)                     # the value of a constant (sigma = 0) channel


def conditioning(N, C):
    """Per (image, channel): ratio |m|/sigma (nan for a constant channel), m and sigma, all fp64 [N, C].  Every 16th channel
    is constant; the others cycle through RATIOS and both signs, shifted per image, so one tensor mixes all of them."""
    ratio = torch.full((N, C), math.nan, dtype=torch.float64)
    m = torch.zeros(N, C, dtype=torch.float64)
    s = torch.zeros(N, C, dtype=torch.float64)
    for n in range(N):
        for c in range(C):
            if c % 16 == 15:
                m[n, c] = CONSTS[(c // 16 + n) % len(CONSTS)]
                continue
            j = c - c // 16
            sign = -1.0 if (j // len(RATIOS) + n) % 2 else 1.0
            ratio[n, c] = RATIOS[(j + n) % len(RATIOS)]
            s[n, c] = SIGMAS[n % len(SIGMAS)]
            m[n, c] = sign * ratio[n, c] * s[n, c]
    return ratio, m, s


def conditioned(N, P, C, seed, device="cpu"):
    """x [N, P, C] fp32 = m + sigma * z (z standard normal, seeded), and the (ratio, m, sigma) of conditioning()."""
    ratio, m, s = conditioning(N, C)
    g = torch.Generator(device=device).manual_seed(seed)
    z = torch.randn(N, P, C, generator=g, device=device, dtype=torch.float32)
    x = (m.to(device)[:, None, :] + s.to(device)[:, None, :] * z.double()).float()
    return x, ratio, m, s


# ----------------------------------------------------------------------------------------------------------- (b) frames
FRAME_KINDS = ("grey", "black", "white", "grey+-1", "half")


def near_uniform_frames(n, H, W, seed=0):
    """n raw frames [n, 3, H, W] in 0..255 cycling through FRAME_KINDS: uniform 128, 0 and 255, 128 plus uniform noise in
    [-1, 1], and a frame whose left half is uniform 128 and whose right half is textured (uniform noise).  Returns the frames
    and the kind of each."""
    g = torch.Generator().manual_seed(seed)
    out, kinds = torch.empty(n, 3, H, W), []
    for i in range(n):
        k = FRAME_KINDS[i % len(FRAME_KINDS)]
        kinds.append(k)
        if k == "grey":
            out[i] = 128.0
        elif k == "black":
            out[i] = 0.0
        elif k == "white":
            out[i] = 255.0
        elif k == "grey+-1":
            out[i] = 128.0 + (torch.rand(3, H, W, generator=g) * 2 - 1)
        else:
            out[i] = 128.0
            out[i, :, :, W // 2:] = torch.rand(3, H, W - W // 2, generator=g) * 255
    return out, kinds


# ----------------------------------------------------------------------------------------------------------- (c) model
def _log_uniform(g, lo, hi, n):
    return torch.exp(math.log(lo) + (math.log(hi) - math.log(lo)) * torch.rand(n, generator=g, dtype=torch.float64))


def _calibrated(conv, bn, x):
    """conv -> eval-mode bn on fp64 x, after scaling conv's output channels so that on x they have bn's running statistics
    (mean running_mean, variance running_var), as a trained network's do.  Returns bn's fp64 output."""
    y = F.conv2d(x, conv.weight.double(), conv.bias.double(), conv.stride, conv.padding)
    mu, sd = y.mean((0, 2, 3)), y.std((0, 2, 3), unbiased=False)
    a = torch.where(sd > 0, bn.running_var.double().sqrt() / sd.clamp_min(1e-300), torch.zeros_like(sd))
    conv.weight.mul_(a.view(-1, 1, 1, 1).to(conv.weight.dtype))
    conv.bias.copy_((conv.bias.double() - mu) * a + bn.running_mean.double())
    y = (y - mu.view(1, -1, 1, 1)) * a.view(1, -1, 1, 1) + bn.running_mean.double().view(1, -1, 1, 1)
    return F.batch_norm(y, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(), bn.bias.double(),
                        False, 0.0, bn.eps)


def trained_like(model, seed):
    """Seeded in-place transform of a random-init model into one whose values look trained (returns the model):
      - every convolution: a per-output-channel factor log-uniform in [1e-3, 10], and two all-zero output channels (layers
        with at least 8 outputs: the flow head's two stay);
      - every BatchNorm (cnet, weights net): running_var log-uniform in [1e-3, 1e2], running_mean ~ N(0, 2^2), weight
        +-U[0.05, 3], bias ~ N(0, 1);
      - NConv weight_p uniform in [-3, 3] (softplus with beta = 10 maps it to [1e-13, 3]).
    Running statistics drawn independently of the activations they normalise compound over cnet's 15 BatchNorm layers (to
    ~1e18 on a smooth frame), far outside the fp16 range of the tensor-core operands; a trained network's running statistics
    describe its activations.  So the convolution feeding each BatchNorm is rescaled per output channel (weights and bias)
    so that its output has that BatchNorm's running mean and variance on a calibration input: a smooth frame for cnet, a
    random flow and guidance for the weights net."""
    from rnc.synth import smooth_shift_frames
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, nn.Conv2d):
                c = m.out_channels
                f = _log_uniform(g, 1e-3, 10.0, c)
                if c >= 8:
                    f[torch.randperm(c, generator=g)[:2]] = 0.0
                m.weight.mul_(f.view(-1, 1, 1, 1).to(m.weight.dtype))
            elif isinstance(m, nn.BatchNorm2d):
                c = m.num_features
                m.running_var.copy_(_log_uniform(g, 1e-3, 1e2, c))
                m.running_mean.copy_(torch.randn(c, generator=g, dtype=torch.float64) * 2)
                sign = torch.where(torch.rand(c, generator=g) < 0.5, -1.0, 1.0)
                m.weight.copy_(sign * (0.05 + 2.95 * torch.rand(c, generator=g)))
                m.bias.copy_(torch.randn(c, generator=g))
            if isinstance(getattr(m, "weight_p", None), torch.Tensor):
                m.weight_p.copy_(torch.rand(m.weight_p.shape, generator=g) * 6 - 3)
        # calibration: cnet (BasicEncoder, extractor.py:118-192) on a smooth frame
        enc = model.cnet
        im, _ = smooth_shift_frames(1, 96, 128, seed=seed)
        y = F.relu(_calibrated(enc.conv1, enc.norm1, 2 * (im.double() / 255.0) - 1.0))
        for layer in (enc.layer1, enc.layer2, enc.layer3):
            for blk in layer:
                t = F.relu(_calibrated(blk.conv1, blk.norm1, y))
                t = F.relu(_calibrated(blk.conv2, blk.norm2, t))
                if blk.downsample is not None:
                    y = _calibrated(blk.downsample[0], blk.downsample[1], y)
                y = F.relu(y + t)
        # the weights net (interp_weights_est.py Simple): conv -> BN -> ReLU layers on cat(flow x2, guidance)
        up = getattr(model, "upsampler", None)
        if up is not None:
            x = torch.cat([torch.randn(1, 2, 48, 64, generator=g, dtype=torch.float64) * 4,
                           torch.tanh(torch.randn(1, 128, 48, 64, generator=g, dtype=torch.float64))], 1)
            for seq in up.weights_est_net.conv:
                x = F.relu(_calibrated(seq[0], seq[1], x))
    return model


# ----------------------------------------------------------------------------------------------------------- bounds
def norm_ref(x):
    """Two-pass fp64 statistics of x [N, P, C] (any device): mean, variance (biased), rstd = 1/sqrt(var + eps), each [N, C]."""
    xd = x.double()
    mean = xd.mean(1)
    var = (xd - mean[:, None, :]).square().mean(1)
    return mean, var, 1.0 / torch.sqrt(var + float(np.float32(EPS)))


def stats_bounds(mr, mean, var, rstd):
    """mean_rstd [N, C, 2] of a kernel against norm_ref: (bad mask [N, C], relative errors of mean and rstd).  mean within
    2^-23 relative (+ the smallest normal), rstd within 1e-6 relative; a constant channel's rstd exactly float(1/sqrt(eps))."""
    mr = mr.double().to(mean.device)
    em = (mr[..., 0] - mean).abs()
    er = (mr[..., 1] - rstd).abs() / rstd
    bad = (em > MEAN_REL * mean.abs() + MEAN_FLOOR) | (er > RSTD_REL)
    const = var == 0
    bad |= const & (mr[..., 1] != RSTD_CONST)
    return bad, em / mean.abs().clamp_min(MEAN_FLOOR), er


def apply_ref(x, mean, rstd, mode, res=None):
    """fp64 rnc_instnorm_apply: (x - mean) * rstd, then relu (mode >= 1), then relu(res + .) (mode 2); x [N, P, C]."""
    y = (x.double() - mean[:, None, :]) * rstd[:, None, :]
    if mode >= 1:
        y = y.clamp_min(0)
    if mode == 2:
        y = (res.double() + y).clamp_min(0)
    return y


def apply_bound(x, mean, rstd, ref):
    """|err| <= 2e-5 + 2^-23 (|x| + |mean|) rstd (the unavoidable fp32 rounding of x and mean, scaled by rstd) + 2^-23 |ref|."""
    return (APPLY_TOL + 2.0 ** -23 * (x.double().abs() + mean.abs()[:, None, :]) * rstd[:, None, :]
            + 2.0 ** -23 * ref.abs())


def worst_at(bad_or_err, labels=None):
    """(image, channel) of the largest entry of an [N, C] tensor, and its label."""
    flat = int(bad_or_err.double().reshape(-1).argmax())
    n, c = divmod(flat, bad_or_err.shape[1])
    return n, c, (None if labels is None else float(labels[n, c]))


def compare_per_channel(what, got, ref, tol, floor=0.0, log=print):
    """compare() with the bound taken per output channel: |got - ref| <= tol * max(1, max|ref[:, c]|) + floor, so that a
    channel of small values is not judged against the largest channel's scale.  got, ref [B, C, H, W]; floor: a number or a
    per-channel tensor [C].  Returns the worst error relative to its channel's bound."""
    assert got.shape == ref.shape and got.dim() == 4, f"{what}: shape {tuple(got.shape)} != reference {tuple(ref.shape)}"
    ref = ref.double()
    err = (got.double().to(ref.device) - ref).abs()
    err = torch.where(torch.isfinite(got.to(ref.device)), err, torch.full_like(err, math.inf))
    scale = ref.abs().amax((0, 2, 3)).clamp_min(1.0)
    floor = torch.as_tensor(floor, dtype=ref.dtype, device=ref.device).expand(ref.shape[1])
    bound = (tol * scale + floor).view(1, -1, 1, 1)
    rel = err / bound
    B, C, H, W = err.shape
    flat = int(rel.reshape(-1).argmax())
    b, rem = divmod(flat, C * H * W)
    c, rem = divmod(rem, H * W)
    y, x = divmod(rem, W)
    worst = float(rel.reshape(-1)[flat])
    where = (f"image {b}, pixel (y={y}, x={x}), channel {c} (err {float(err[b, c, y, x]):.2e}, "
             f"channel bound {float(bound[0, c, 0, 0]):.2e}, channel max|ref| {float(scale[c]):.2e})")
    log(f"  {what:<34s} {B}x{C}x{H}x{W}: worst err/bound {worst:.2e} at {where}")
    nbad = int((rel > 1).sum())
    if nbad:
        chans = sorted({int(cc) for cc in (rel > 1).amax((0, 2, 3)).nonzero().reshape(-1).tolist()})
        raise Mismatch(f"{what}: {nbad} elements exceed their channel's bound; worst at {where}; bad channels: "
                       f"{chans[:16]}{' ...' if len(chans) > 16 else ''}")
    return worst


# ----------------------------------------------------------------------------------------------------------- emulation
def emulated_rstd(x, fp32_runs):
    """rstd of one channel x [P] (fp32 numpy) by the kernels' formula var = sum(x^2)/P - mean^2 in fp64, with the sums
    accumulated either in fp32 runs of 32 terms (fmaf for the squares) added in fp64, or in fp64 from the first term."""
    P = x.shape[0]
    xd = x.astype(np.float64)
    if fp32_runs:
        pad = np.zeros(-P % 32, np.float64)
        runs = np.concatenate([xd, pad]).reshape(-1, 32)
        s = np.zeros(runs.shape[0], np.float32)
        q = np.zeros(runs.shape[0], np.float32)
        for k in range(32):
            v = runs[:, k]
            s = (s.astype(np.float64) + v).astype(np.float32)
            q = (q.astype(np.float64) + v * v).astype(np.float32)          # fmaf: one rounding of v*v + q
        sm, sq = s.astype(np.float64).sum(), q.astype(np.float64).sum()
    else:
        sm, sq = xd.sum(), (xd * xd).sum()
    mean = sm / P
    var = max(sq / P - mean * mean, 0.0)
    return np.float32(1.0 / np.sqrt(var + np.float64(np.float32(EPS))))


def test_bound_rejects_fp32_partial_sums():
    """At fnet norm1's size (P = 220 x 512) the rstd bound fails the fp32-run formula at |mean|/std = 100 and passes fp64
    accumulation up to 1e4: the bound is what tells the two apart."""
    P = 220 * 512
    rng = np.random.default_rng(3)
    worst32, worst64 = {}, {}
    for ratio in (1.0, 100.0, 1000.0, 1e4):
        for sign in (1.0, -1.0):
            x = (sign * ratio + rng.standard_normal(P)).astype(np.float32)
            xd = x.astype(np.float64)
            ref = 1.0 / np.sqrt(((xd - xd.mean()) ** 2).mean() + np.float64(np.float32(EPS)))
            e32 = abs(float(emulated_rstd(x, True)) - ref) / ref
            e64 = abs(float(emulated_rstd(x, False)) - ref) / ref
            worst32[ratio] = max(worst32.get(ratio, 0.0), e32)
            worst64[ratio] = max(worst64.get(ratio, 0.0), e64)
    print("rstd rel err, fp32 runs:", {k: f"{v:.1e}" for k, v in worst32.items()},
          " fp64:", {k: f"{v:.1e}" for k, v in worst64.items()})
    assert worst32[100.0] > RSTD_REL and worst32[1e4] > RSTD_REL
    assert max(worst64.values()) <= RSTD_REL


def test_stats_bounds_flag_a_constant_channel():
    """A constant channel must come out with rstd exactly float(1/sqrt(eps)); a last-bit difference is flagged."""
    x = torch.full((1, 100, 4), 1234.5)
    mean, var, rstd = norm_ref(x)
    mr = torch.stack([mean.float(), rstd.float()], -1)
    assert float(rstd[0, 0]) == pytest.approx(RSTD_CONST, rel=1e-7)
    assert not stats_bounds(mr, mean, var, rstd)[0].any()
    mr[0, 2, 1] = float(np.nextafter(np.float32(RSTD_CONST), np.float32(0)))
    assert stats_bounds(mr, mean, var, rstd)[0].tolist() == [[False, False, True, False]]


def test_conditioned_stimulus():
    """Deterministic per seed; every ratio, both signs and constant channels present in one tensor; constant channels exact."""
    x, ratio, m, s = conditioned(3, 1000, 64, seed=5)
    x2, *_ = conditioned(3, 1000, 64, seed=5)
    assert torch.equal(x, x2) and not torch.equal(x, conditioned(3, 1000, 64, seed=6)[0])
    assert set(ratio[~ratio.isnan()].tolist()) == set(RATIOS)
    assert (m > 0).any() and (m < 0).any()
    const = ratio.isnan()
    assert const.sum() == 3 * 4 and set(m[const].tolist()) == set(CONSTS)
    assert torch.equal(x[const.nonzero()[:, 0], :, const.nonzero()[:, 1]],
                       m[const][:, None].float().expand(-1, 1000))
    mean, var, rstd = norm_ref(x)
    got = (mean.abs() / var.sqrt())[~const & (ratio > 0)]
    want = ratio[~const & (ratio > 0)]
    assert ((got / want - 1).abs() < 0.2).all()                    # the sample's |mean|/std is the label's


def test_near_uniform_frames_deterministic():
    a, kinds = near_uniform_frames(6, 24, 40, seed=1)
    b, _ = near_uniform_frames(6, 24, 40, seed=1)
    assert torch.equal(a, b) and kinds == list(FRAME_KINDS) + ["grey"]
    assert (a[0] == 128).all() and (a[1] == 0).all() and (a[2] == 255).all()
    assert (a[3] - 128).abs().max() <= 1 and a[3].std() > 0.3
    assert (a[4, :, :, :20] == 128).all() and a[4, :, :, 20:].std() > 50


def test_per_channel_comparator_sees_small_channels():
    """An error that the whole-tensor bound (tol * max|ref|) hides in a small channel fails the per-channel bound."""
    from test_product_shapes import compare
    ref = torch.ones(1, 2, 4, 4, dtype=torch.float64)
    ref[:, 0] *= 1000.0
    got = ref.clone()
    got[0, 1, 2, 3] += 1e-3
    compare("whole tensor", got, ref, 2e-5)
    with pytest.raises(Mismatch, match="channel 1"):
        compare_per_channel("per channel", got, ref, 2e-5)
    assert compare_per_channel("per channel, in bound", ref + 1e-6, ref, 2e-5) < 1
    assert compare_per_channel("per-channel floor", got, ref, 2e-5, torch.tensor([0.0, 2e-3])) < 1


def test_trained_like_deterministic_and_in_range():
    """Same seed -> the same weights; every BatchNorm drawn in its range; each BatchNorm's input on the calibration frame
    has the running statistics; NConv weights spread over [-3, 3]; two zero output channels per wide convolution."""
    from rnc.synth import build_model, smooth_shift_frames
    a = trained_like(build_model("raft_nc_dbl"), seed=4).state_dict()
    b = trained_like(build_model("raft_nc_dbl"), seed=4).state_dict()
    c = trained_like(build_model("raft_nc_dbl"), seed=5).state_dict()
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert any(not torch.equal(a[k], c[k]) for k in a if a[k].is_floating_point())
    m = trained_like(build_model("raft_nc_dbl"), seed=4)
    bns = [x for x in m.modules() if isinstance(x, nn.BatchNorm2d)]
    assert len(bns) == 15 + 2                                      # cnet + the weights net
    for bn in bns:
        assert 1e-3 <= bn.running_var.min() and bn.running_var.max() <= 1e2
        assert 0.05 <= bn.weight.abs().min() and bn.weight.abs().max() <= 3
    rv = torch.cat([bn.running_var for bn in bns])
    assert rv.min() < 1e-2 and rv.max() > 10
    wp = torch.cat([x.weight_p.reshape(-1) for x in m.modules() if isinstance(getattr(x, "weight_p", None), torch.Tensor)])
    assert wp.min() < -2 and wp.max() > 2 and wp.abs().max() <= 3
    for conv in (x for x in m.modules() if isinstance(x, nn.Conv2d) and x.out_channels >= 8):
        assert int((conv.weight.reshape(conv.out_channels, -1).abs().amax(1) == 0).sum()) >= 2
    # calibration: cnet's stem output on the calibration frame has norm1's running statistics
    im, _ = smooth_shift_frames(1, 96, 128, seed=4)
    y = F.conv2d(2 * (im.double() / 255.0) - 1.0, m.cnet.conv1.weight.double(), m.cnet.conv1.bias.double(), 2, 3)
    live = y.std((0, 2, 3)) > 0
    assert torch.allclose(y.mean((0, 2, 3)), m.cnet.norm1.running_mean.double(), atol=1e-4)
    assert torch.allclose(y.var((0, 2, 3), unbiased=False)[live], m.cnet.norm1.running_var.double()[live], rtol=1e-3)


def test_grey_frame_reaches_the_regime(monkeypatch):
    """The oracle's forward on a uniform mid-grey 440x1024 pair with the seeded model, in fp64: the input of fnet's first
    InstanceNorm (the oracle's own preprocessing and stem) has max |mean|/std > 1000 over its channels, so the GPU check on
    that frame exercises the cancellation.  The forward is stopped at that norm."""
    from oracle import raft_oracle as orc
    from rnc.synth import build_model

    class Reached(Exception):
        pass

    def first_norm(sd, name, x, kind):
        assert name == "fnet.norm1" and kind == "instance"
        raise Reached(x)

    monkeypatch.setattr(orc, "_norm", first_norm)
    sd = {k: v.detach().double() for k, v in build_model("raft_nc_dbl").state_dict().items()}
    img = torch.full((1, 3, 440, 1024), 128.0, dtype=torch.float64)
    with pytest.raises(Reached) as hit:
        orc.raft_forward(sd, img, img, iters=1)
    y = hit.value.args[0][:1]                                       # frame 1 (both frames are the same)
    ratio = (y.mean((2, 3)).abs() / y.std((2, 3), unbiased=False)).max().item()
    print(f"grey frame: fnet norm1 max |mean|/std = {ratio:.0f}")
    assert ratio > 1000
