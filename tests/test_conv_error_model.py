"""An fp64 model of the tensor-core convolution's arithmetic (csrc/conv_umma.cu, packed by rnc/engine_umma.py UmmaWeights),
and the elementwise error bound that follows from it.  tests/test_gpu_conv_error_model.py holds the kernel to this model.

What the kernel computes, and where it can lose accuracy:
  - every activation x is an exact-sum pair of halves, split_pair() in csrc/rnc_common.cuh: hi = rn_satfinite(x),
    lo = rn_satfinite(x - hi) (split_emulate below, bit for bit);
  - every weight is scaled by 2^s (the layer's largest |w| lands in [512, 1024)) and split the same way (pack_emulate);
  - each K step of 16 issues x_hi*w_hi into the main fp32 accumulator and x_hi*w_lo, x_lo*w_hi into the correction
    accumulator (x_lo*w_lo is dropped); the epilogue adds the two accumulators, then out = fma(acc, 2^-s, bias).

conv_split_ref() evaluates exactly those three products of the real pack in fp64; the bound has two parts:
  - R (representation): |conv(x, w) + b - conv_split_ref|, from the split rules alone (conv_split_ref's docstring);
  - A (accumulation and epilogue): |kernel - conv_split_ref| <= C_A * steps * 2^-24 * mag_a + 2^-24 * |ref| (C_A's
    comment; mag_a: mag with every half taken at no less than 2^-14, the tensor core's alignment of subnormal operands).
check_model() applies both through compare_mag (tests/test_train_shapes.py).
"""
import math
from typing import NamedTuple, Optional

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_product_shapes import Mismatch, compare
from test_train_shapes import compare_mag

U = 2.0 ** -24             # fp32 unit roundoff
HALF_MAX = 65504.0         # largest finite half
SPLIT_MAX = 2 * HALF_MAX   # largest hi + lo: both halves saturated
K_STEP = 16                # K of one wgmma (fp16 operands)

# Accumulation constant of bound A: |kernel - conv_split_ref| <= C_A * steps * 2^-24 * mag_a + 2^-24 * |ref|, with
# steps = K / 16 (the main accumulator's K steps).  The form is linear in steps, not sqrt(steps): the tensor core aligns the
# 16 products of a step to the largest exponent and truncates, so with operands of one sign every step errs the same way.
# Measured on an H100 SXM (80 GB, 700 W power limit) over tests/test_gpu_conv_error_model.py: all-positive operands need
# 1.93 at K = 64 (4 steps) and 1.79 at K = 2304 (144 steps), the same per step, as the linear form says, with a signed
# mean error of -0.8 and -1.5 (biased towards zero); random signs need 0.64 and 0.05.  C_A = 3 leaves a margin of 1.55x.
# C_A >= 1 also covers the epilogue's main + correction add, whose rounding is at most 2^-24 * mag.
# mag_a is mag with every operand half taken at no less than 2^-14 (zeros and subnormals included): the tensor core aligns a
# step's products and the running sum to the largest product *exponent*, and an fp16 subnormal carries the exponent of
# 2^-14 whatever its value.  Single-product launches on the H100 return every product of halves exactly (product exponents
# -48 .. 15, all three operand paths), but a sum of products with a subnormal w_hi keeps only the bits above 2^-23 of
# max |x| * 2^-14.  A two-product probe shows it: after a first step leaves 2^-24 + 2^-34 in the accumulator, the product
# 2^-14 made as x 2^10 * w 2^-24 (w subnormal) drops the 2^-34 bit, the same product made as x 1 * w 2^-14 keeps it.  In the
# weight-spread channels with a subnormal w_hi the kernel differs from conv_split_ref by up to 6.4 steps * 2^-24 * mag, and
# by 0.017 steps * 2^-24 * mag_a.
C_A = 3.0


# ----------------------------------------------------------------------------------------------------------- the split
def split_emulate(x):
    """split_pair() of csrc/rnc_common.cuh in torch: hi = rn(x) saturated to +-65504 (cvt.rn.satfinite: a finite result,
    never inf), lo = rn_satfinite(x - hi) with the difference in fp32.  Halves keep their subnormals.  Returns (hi, lo), fp16.
    |x| <= 65504: hi + lo = x to 22 bits (absolute floor 2^-25); up to 131008 lo carries the excess to 11 bits; beyond,
    both halves saturate."""
    x = x.float()
    hi = x.clamp(-HALF_MAX, HALF_MAX).half()          # rn, then the overflow to inf clamped back: the same as satfinite
    lo = (x - hi.float()).clamp(-HALF_MAX, HALF_MAX).half()
    return hi, lo


_HALVES = None


def _finite_halves():
    """Every finite half as (sorted float64 values, their bit patterns)."""
    global _HALVES
    if _HALVES is None:
        bits = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
        v = bits.view(np.float16).astype(np.float64)
        ok = np.isfinite(v) & ~((v == 0) & (bits == 0x8000))          # one zero: the sign is handled by the caller
        order = np.argsort(v[ok], kind="stable")
        _HALVES = v[ok][order], bits[ok][order]
    return _HALVES


def rn_satfinite_brute(v):
    """float64 array -> nearest finite half, ties to the even bit pattern, |v| beyond 65504 -> +-65504 (a zero keeps its
    sign): by search over every finite half, independent of any conversion routine."""
    vals, bits = _finite_halves()
    v = np.asarray(v, dtype=np.float64)
    a = np.clip(v, -HALF_MAX, HALF_MAX)
    j = np.clip(np.searchsorted(vals, a), 1, len(vals) - 1)
    lo_v, hi_v = vals[j - 1], vals[j]
    lo_b, hi_b = bits[j - 1], bits[j]
    d_lo, d_hi = a - lo_v, hi_v - a
    pick_hi = (d_hi < d_lo) | ((d_hi == d_lo) & (hi_b % 2 == 0))
    out = np.where(pick_hi, hi_b, lo_b).astype(np.uint16)
    out = np.where((out & 0x7FFF) == 0, np.where(np.signbit(v), 0x8000, 0), out).astype(np.uint16)   # a zero keeps v's sign
    return out.view(np.float16)


def split_brute(x):
    """split_pair() by brute force: x float32 array -> (hi, lo) float16 arrays."""
    x = np.asarray(x, dtype=np.float32)
    hi = rn_satfinite_brute(x.astype(np.float64))
    r = (x - hi.astype(np.float32)).astype(np.float32)          # the kernel's fp32 subtraction
    return hi, rn_satfinite_brute(r.astype(np.float64))


def split_bound(x):
    """Elementwise bound on |x - (hi + lo)| of split_emulate(x), from the split rules: |x| <= 65504: 2^-22 |x| (lo rounds a
    remainder of at most 2^-11 |x| to 11 bits) + 2^-25 (half the smallest subnormal: the floor of a subnormal lo or hi);
    (65504, 131008]: lo = rn(|x| - 65504) to 11 bits; beyond: |x| - 131008 (both halves saturate)."""
    a = x.double().abs()
    r = a - HALF_MAX
    return torch.where(a <= HALF_MAX, 2.0 ** -22 * a + 2.0 ** -25,
                       torch.where(r <= HALF_MAX, 2.0 ** -11 * r, a - SPLIT_MAX))


# ----------------------------------------------------------------------------------------------------------- the pack
def _coutpad(c):
    for p in (32, 64, 128, 192, 256):
        if c <= p:
            return p
    return -(-c // 192) * 192


def pack_emulate(weight, bias, segs, extra_cout=0, out_scale=1.0):
    """UmmaWeights restated: (w_hi, w_lo [coutpad, kh*kw*nblk*64] fp16, unscale, bias [coutpad] fp32).  Column
    (tap * nblk + block) * 64 + j holds input channel j of that 64-channel block of its segment at tap ky * kw + kx; the
    weights are multiplied by out_scale, then by 2^s with s = floor(log2(1000 / max|w|)), and split by split_emulate."""
    cout, cin, kh, kw = weight.shape
    w = weight.detach().float().cpu() * out_scale
    nblks = [-(-c // 64) for c in segs]
    nblk = sum(nblks)
    cp = _coutpad(cout + extra_cout)
    full = torch.zeros(cp, kh * kw, nblk * 64)
    ci = blk = 0
    for c, nb in zip(segs, nblks):
        for j in range(c):
            for ky in range(kh):
                for kx in range(kw):
                    full[:cout, ky * kw + kx, blk * 64 + j] = w[:, ci + j, ky, kx]
        ci += c
        blk += nb
    mx = float(full.abs().max())
    s = math.floor(math.log2(1000.0 / mx)) if mx > 0 else 0
    hi, lo = split_emulate(full.reshape(cp, -1) * 2.0 ** s)
    b = torch.zeros(cp)
    if bias is not None:
        b[:cout] = bias.detach().float().cpu() * out_scale
    return hi, lo, 2.0 ** -s, b


def unpack(planes, kh, kw):
    """[coutpad, kh*kw*nblk*64] -> [coutpad, nblk*64, kh, kw] (fp64): the pack as a convolution weight over the
    block-padded input channels."""
    cp = planes.shape[0]
    return planes.double().view(cp, kh, kw, -1).permute(0, 3, 1, 2)


def pad_segments(x, segs):
    """[B, sum(segs), H, W] -> [B, nblk*64, H, W]: each segment's channels at the start of its own 64-channel blocks."""
    B, _, H, W = x.shape
    out = x.new_zeros(B, sum(-(-c // 64) for c in segs) * 64, H, W)
    ci = col = 0
    for c in segs:
        out[:, col:col + c] = x[:, ci:ci + c]
        ci += c
        col += -(-c // 64) * 64
    return out


# ----------------------------------------------------------------------------------------------------------- the model
class SplitRef(NamedTuple):
    ref: torch.Tensor                  # fp64 sum of the three products of the pack, * unscale, + bias  [B, cout, Ho, Wo]
    mag: torch.Tensor                  # fp64 conv(|x_hi + x_lo|, |w_hi + w_lo|) * unscale + |bias|
    mag_a: torch.Tensor                # mag of the three products with every half taken at >= 2^-14 (bound A)
    steps: int                         # K steps of 16 of the main accumulator (all taps, all 64-channel blocks)
    exact: Optional[torch.Tensor]      # fp64 conv of the unsplit operands + bias (with weight=)
    R: torch.Tensor                    # bound on |conv(x, w) + b - ref| from the split rules, for the w the pack was made of


def conv_split_ref(x, pack, segs=None, weight=None, stride=1, dil=1, out_scale=1.0):
    """fp64 evaluation of what the tensor-core convolution computes with the pack `pack` (UmmaWeights: w_hi, w_lo,
    unscale, bias, cout, kh, kw) on the input x: sum over taps and channels of x_hi*w_hi + x_hi*w_lo + x_lo*w_hi, times
    unscale, plus the bias.

    x: fp32 [B, Cin, H, W] (split here by split_emulate, as rnc_f32_to_split and the epilogues do) or a (hi, lo) pair of
    [B, Cin, H, W] planes as a producer left them.  segs: the input segments the pack was built with (default one segment).
    weight: the unsplit [cout, Cin, kh, kw] weights; with it, also the fp64 convolution of the unsplit operands (x, or
    hi + lo of given planes; weight times out_scale, a power of two).  R bounds the distance of that convolution from ref
    for any weight the pack was split from:

        x = x^ + dx,  w = w^ + dw  (x^ = x_hi + x_lo, w^ = (w_hi + w_lo) 2^-s)
        x w - (x^ w^ - x_lo w_lo 2^-s) = x_lo w_lo 2^-s + dx w^ + x^ dw + dx dw
        |dx| <= split_bound(x) (0 for given planes),  |dw| <= (2^-22 |w_hi + w_lo| + 2^-25) 2^-s (the split rule on the
        scaled weights: 22 bits and the floor of a subnormal w_hi or w_lo)
        R = conv(|x_lo|, |w_lo|) 2^-s + conv(|dx|, |w^| + |dw|) + conv(|x^|, |dw|)

    times (1 + 2^-20), plus K 2^-52 mag for the fp64 evaluation itself.  Padding: kh // 2 * dil rows, kw // 2 * dil columns
    (zero outside the image, as the kernel's TMA boxes)."""
    kh, kw, cout = pack.kh, pack.kw, pack.cout
    if isinstance(x, (tuple, list)):
        hi, lo = (t.double() for t in x)
        dx = None
        x_unsplit = hi + lo
    else:
        h16, l16 = split_emulate(x)
        hi, lo = h16.double(), l16.double()
        dx = split_bound(x)
        x_unsplit = x.double()
    segs = [hi.shape[1]] if segs is None else segs
    dev = hi.device
    hi, lo = pad_segments(hi, segs), pad_segments(lo, segs)
    wh, wl = unpack(pack.w_hi, kh, kw)[:cout].to(dev), unpack(pack.w_lo, kh, kw)[:cout].to(dev)
    us = float(pack.unscale)
    b = pack.bias[:cout].double().to(dev)
    pad = (kh // 2 * dil, kw // 2 * dil)

    def conv(a, w, bias=None, padding=pad):
        return F.conv2d(a, w, bias, stride, padding, dil)
    wsum = wh + wl
    ref = (conv(hi, wsum) + conv(lo, wh)) * us + b.view(1, -1, 1, 1)
    xs = hi + lo
    mag = conv(xs.abs(), wsum.abs()) * us + b.abs().view(1, -1, 1, 1)
    steps = pack.ktot // K_STEP
    dw = (2.0 ** -22 * wsum.abs() + 2.0 ** -25) * us
    R = conv(lo.abs(), wl.abs()) * us + conv(xs.abs(), dw)
    if dx is not None:
        R = R + conv(pad_segments(dx, segs), wsum.abs() * us + dw)
    R = R * (1 + 2.0 ** -20) + pack.ktot * 2.0 ** -52 * mag
    exact = None
    if weight is not None:
        exact = conv(pad_segments(x_unsplit, segs), pad_segments(weight.double().to(dev) * out_scale, segs), b)
    # the halves as the tensor core aligns them: at no less than 2^-14 (zero-filled border pixels included)
    nu = lambda t: t.abs().clamp_min(2.0 ** -14)            # noqa: E731
    bord = lambda t: F.pad(nu(t), (pad[1], pad[1], pad[0], pad[0]), value=2.0 ** -14)      # noqa: E731
    mag_a = (conv(bord(hi), nu(wh) + nu(wl), padding=0) + conv(bord(lo), nu(wh), padding=0)) * us + b.abs().view(1, -1, 1, 1)
    return SplitRef(ref, mag, mag_a, steps, exact, R)


def fp64_floor(sref):
    """The fp64 evaluation's own error: K * 2^-53 * mag per element, at most (K = 16 * steps)."""
    return 16 * sref.steps * 2.0 ** -53 * sref.mag


def a_tol(steps, c_a=C_A):
    """The mag_a coefficient of bound A."""
    return c_a * steps * U


def check_model(what, got, sref, against="split", c_a=C_A, act=None, floor=0.0, log=print):
    """A kernel output [B, C, H, W] against the model.  against="split": |got - sref.ref| <= A (the kernel computes its own
    arithmetic); "exact": |got - sref.exact| <= R + A (the split operands stay within their rules).  act: the epilogue's
    activation (1-Lipschitz: it moves no error up), applied to the reference; A's epilogue term stays on the pre-activation
    |ref|.  floor: an extra elementwise allowance stated by the caller.  Returns the worst err / bound; raises Mismatch
    naming the worst image, pixel, channel and 128-pixel tile."""
    C = got.shape[1]
    ref = (sref.ref if against == "split" else sref.exact)[:, :C]
    if act is not None:
        ref = act(ref)
    floor = U * sref.ref[:, :C].abs() + fp64_floor(sref)[:, :C] + floor
    if against == "exact":
        floor = floor + sref.R[:, :C]
    return compare_mag(f"{what} [{against}]", got, ref, sref.mag_a[:, :C], a_tol(sref.steps, c_a), floor, log=log)


def a_ratio(got, sref):
    """(|got - ref| - 2^-24 |ref|) / (steps 2^-24 mag_a): the C_A a case needs, elementwise."""
    C = got.shape[1]
    err = (got.double() - sref.ref[:, :C]).abs() - U * sref.ref[:, :C].abs()
    den = sref.steps * U * sref.mag_a[:, :C]
    return torch.where(den > 0, err.clamp_min(0) / den.clamp_min(1e-300), torch.zeros_like(den))


# ----------------------------------------------------------------------------------------------------------- stimuli
def magnitude_sweep(B, C, H, W, seed, lo_log2=-24, hi_log2=16):
    """fp32 activations whose channels are log-spaced over 2^lo_log2 .. 2^hi_log2 (random signs, +-25% jitter), with two
    all-zero channels and two channels of fp16-subnormal values (below 2^-14)."""
    g = torch.Generator().manual_seed(seed)
    scale = 2.0 ** torch.linspace(lo_log2, hi_log2, C)
    x = scale.view(1, C, 1, 1) * (0.75 + 0.5 * torch.rand(B, C, H, W, generator=g))
    x = x * torch.where(torch.rand(B, C, H, W, generator=g) < 0.5, -1.0, 1.0)
    x[:, 1] = 0.0
    x[:, C // 2] = 0.0
    x[:, 2] = torch.randint(-1023, 1024, (B, H, W), generator=g).float() * 2.0 ** -24     # fp16 subnormals
    x[:, 3] = torch.rand(B, H, W, generator=g) * 2.0 ** -15
    return x.float()


def spread_weight(cout, cin, kh, kw, seed, lo_log2=-40):
    """Weights whose output channels carry factors 2^0 .. 2^lo_log2 of the layer's largest (log-spaced), two all-zero
    output channels; channel 0 keeps the factor 1."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    f = 2.0 ** torch.linspace(0, lo_log2, cout)
    f[torch.randperm(cout - 1, generator=g)[:2] + 1] = 0.0
    return (w * f.view(-1, 1, 1, 1)).float()


def signed_input(kind, B, C, H, W, seed):
    """Sign structure of an activation tensor: "positive" (|randn| + 0.1), "random" (randn), "cancelling" (positive; the
    matching weights cancel, see signed_weight)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g)
    return x if kind == "random" else x.abs() + 0.1


def signed_weight(kind, cout, cin, kh, kw, seed):
    """"positive": |randn|; "random": randn; "cancelling": the second half of the input channels carries the negated first
    half's weights times (1 - 1e-3 eps) with eps ~ U(-1, 1) per weight, so with a channel-pair-correlated input (see
    cancelling_input) the output is ~1e-3 of mag."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(cout, cin, kh, kw, generator=g)
    if kind == "positive":
        w = w.abs()
    elif kind == "cancelling":
        h = cin // 2
        w[:, h:2 * h] = -w[:, :h] * (1 - 1e-3 * (2 * torch.rand(cout, h, kh, kw, generator=g) - 1))
    return (w / (cin * kh * kw) ** 0.5).float()


def cancelling_input(B, C, H, W, seed):
    """Positive activations whose second half of channels repeats the first half: against signed_weight("cancelling")
    every pair of products nearly cancels."""
    x = signed_input("positive", B, C, H, W, seed)
    h = C // 2
    x[:, h:2 * h] = x[:, :h]
    return x


# ----------------------------------------------------------------------------------------------------------- CPU tests
def _split_inputs():
    """Every float32 exponent (subnormals to the largest finite) with several mantissas and both signs, +-0, 65504 and its
    neighbours, (65504, 131008], above 131008, and fp16-subnormal inputs."""
    rng = np.random.default_rng(0)
    vals = [0.0, -0.0, 65504.0, -65504.0, 65519.99, 65520.0, 131008.0, 131009.0, 131024.0, 2.0 ** 17, 3e38, -3e38,
            2.0 ** -24, 2.0 ** -25, 1.5 * 2.0 ** -25, 2.0 ** -26, 2.0 ** -14, 2.0 ** -14 * (1 - 2.0 ** -11)]
    for e in range(-149, 128):
        for m in (1.0, 1.0 + 2.0 ** -23, 1.5, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -12, 1.999999):
            v = m * 2.0 ** e
            if v < 3.4e38:
                vals += [v, -v]
    vals += list(rng.uniform(65504, 131008, 2000)) + list(rng.uniform(131008, 1e6, 200))
    vals += list(rng.integers(-1023, 1024, 2000) * 2.0 ** -24 + rng.uniform(-2.0 ** -25, 2.0 ** -25, 2000))
    vals += list(rng.standard_normal(4000) * 10.0 ** rng.uniform(-9, 5, 4000))
    x = np.array(vals, dtype=np.float64).astype(np.float32)
    return np.concatenate([x, -x])


def test_split_emulate_matches_brute_force():
    x = _split_inputs()
    hi, lo = split_emulate(torch.from_numpy(x))
    bh, bl = split_brute(x)
    bad = (hi.numpy().view(np.uint16) != bh.view(np.uint16)) | (lo.numpy().view(np.uint16) != bl.view(np.uint16))
    assert not bad.any(), f"split_emulate differs from the brute-force split at {x[bad][:8].tolist()}"
    # the bound and the saturation edges
    rec = hi.double() + lo.double()
    xd = torch.from_numpy(x).double()
    assert ((rec - xd).abs() <= split_bound(torch.from_numpy(x))).all()
    assert float(rec.max()) == SPLIT_MAX and float(rec.min()) == -SPLIT_MAX
    assert torch.isfinite(hi).all() and torch.isfinite(lo).all()
    v = torch.tensor([65504.0, 65600.0, 131008.0, 1e6])
    h, l = split_emulate(v)
    assert h.tolist() == [65504.0] * 4 and l.tolist() == [0.0, 96.0, 65504.0, 65504.0]


@pytest.mark.parametrize("case", ["plain", "segments", "spread", "extra-out-scale"])
def test_pack_emulate_matches_umma_weights(case):
    from rnc.engine_umma import UmmaWeights
    g = torch.Generator().manual_seed(5)
    segs, extra, osc, bias = [96], 0, 1.0, torch.randn(40, generator=g)
    w = torch.randn(40, 96, 3, 3, generator=g)
    if case == "segments":
        segs = [128, 70]
        w = torch.randn(40, 198, 1, 5, generator=g)
    elif case == "spread":
        w = spread_weight(40, 96, 3, 3, seed=6)
    elif case == "extra-out-scale":
        extra, osc = 2, 0.25
        w = torch.randn(30, 96, 1, 1, generator=g) * 1e-3
        bias = bias[:30]
    pk = UmmaWeights(w, bias, segs, extra_cout=extra, out_scale=osc)
    hi, lo, us, b = pack_emulate(w, bias, segs, extra, osc)
    assert pk.unscale == us and torch.equal(pk.bias, b)
    assert torch.equal(pk.w_hi.view(torch.int16), hi.view(torch.int16))
    assert torch.equal(pk.w_lo.view(torch.int16), lo.view(torch.int16))


class _Pack:
    """pack_emulate's planes in UmmaWeights' attributes (CPU self-tests of the model)."""

    def __init__(self, w, b, segs, extra_cout=0, out_scale=1.0):
        self.w_hi, self.w_lo, self.unscale, self.bias = pack_emulate(w, b, segs, extra_cout, out_scale)
        self.cout, _, self.kh, self.kw = w.shape
        self.coutpad = self.w_hi.shape[0]
        self.ktot = self.w_hi.shape[1]


# (name, x, weight, segs, stride, dil, out_scale)
def _r_cases():
    g = torch.Generator().manual_seed(9)
    B, H, W = 2, 9, 11
    out = [("magnitude sweep", magnitude_sweep(B, 96, H, W, 1), torch.randn(24, 96, 3, 3, generator=g) / 30, [96], 1, 1, 1.0),
           ("magnitude sweep 1x1 s2", magnitude_sweep(B, 64, H, W, 2), torch.randn(24, 64, 1, 1, generator=g) / 8, [64], 2, 1,
            1.0),
           ("weight spread", torch.randn(B, 64, H, W, generator=g), spread_weight(48, 64, 3, 3, 3), [64], 1, 1, 1.0),
           ("weight spread dil 2", torch.randn(B, 64, H, W, generator=g), spread_weight(48, 64, 3, 3, 4, -30), [64], 1, 2, 1.0),
           ("segments 1x5", torch.randn(B, 198, H, W, generator=g), torch.randn(32, 198, 1, 5, generator=g) / 30, [128, 70], 1,
            1, 1.0),
           ("out_scale 3x3 s2", torch.randn(B, 64, H, W, generator=g) * 300, torch.randn(20, 64, 3, 3, generator=g), [64], 2, 1,
            0.25)]
    for kind in ("positive", "cancelling", "random"):
        x = cancelling_input(B, 128, H, W, 7) if kind == "cancelling" else signed_input(kind, B, 128, H, W, 7)
        out.append((f"signs {kind}", x, signed_weight(kind, 32, 128, 3, 3, 8), [128], 1, 1, 1.0))
    return out


@pytest.mark.parametrize("case", range(9), ids=[c[0] for c in _r_cases()])
def test_split_ref_within_r(case):
    """|conv(x, w) + b - conv_split_ref| <= R on every stimulus family, and R is not vacuous: within 2^10 of the largest
    error of the family (the bound is linear in K, the error is not)."""
    name, x, w, segs, stride, dil, osc = _r_cases()[case]
    b = torch.randn(w.shape[0], generator=torch.Generator().manual_seed(case))
    pk = _Pack(w, b, segs, out_scale=osc)
    s = conv_split_ref(x, pk, segs, weight=w, stride=stride, dil=dil, out_scale=osc)
    err = (s.exact - s.ref).abs()
    ratio = float((err / s.R).max())
    print(f"{name}: worst |exact - split| / R {ratio:.3e}, max err {float(err.max()):.2e}")
    assert ratio <= 1.0
    assert ratio > 2.0 ** -10
    # the planes form of the same input: no activation split error, and the same split reference
    hi, lo = split_emulate(x)
    s2 = conv_split_ref((hi, lo), pk, segs, weight=w, stride=stride, dil=dil, out_scale=osc)
    assert torch.equal(s2.ref, s.ref) and ((s2.exact - s2.ref).abs() <= s2.R).all()


def test_comparator_rejects_what_the_flat_bound_accepts():
    """A 1e-6 error in a channel whose mag is 1e-2, inside a K = 2304 layer whose max|ref| is 10: compare() with the
    convolution tolerance (2e-5 * max(1, max|ref|)) passes it, check_model() does not."""
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 256, 6, 8, generator=g).abs()
    w = torch.randn(4, 256, 3, 3, generator=g) * 0.01
    w[1] *= 1e-4                                          # channel 1: mag ~ 1e-2
    pk = _Pack(w, None, [256])
    s = conv_split_ref(x, pk, weight=w)
    f = 10 / float(s.ref.abs().max())
    s = s._replace(ref=s.ref * f, mag=s.mag * f, mag_a=s.mag_a * f)
    assert 5e-3 < float(s.mag_a[:, 1].max()) < 5e-2
    got = s.ref.clone()
    got[0, 1, 2, 3] += 1e-6
    compare("flat", got, s.ref, 2e-5)                     # passes
    with pytest.raises(Mismatch, match=r"image 0, pixel \(y=2, x=3\), channel 1, tile 0"):
        check_model("model", got, s)
    assert check_model("model", s.ref.clone(), s) == 0.0


@pytest.mark.parametrize("bad", [math.nan, math.inf, -math.inf])
def test_comparator_rejects_non_finite(bad):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 64, 5, 130, generator=g)
    w = torch.randn(8, 64, 1, 1, generator=g)
    pk = _Pack(w, None, [64])
    s = conv_split_ref(x, pk, weight=w)
    got = s.ref.clone()
    got[0, 5, 4, 129] = bad
    for against in ("split", "exact"):
        with pytest.raises(Mismatch, match=r"image 0, pixel \(y=4, x=129\), channel 5, tile 5"):
            check_model("model", got, s, against)
