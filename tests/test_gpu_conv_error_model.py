"""The tensor-core convolution (rnc_conv2d_umma_fwd through UmmaEngine.uconv) against the fp64 model of its arithmetic in
tests/test_conv_error_model.py: every case runs one layer with RNC_EPI_LINEAR and an fp32 output and checks it against
conv_split_ref with bound A (the kernel computes the three products of its own pack) and against fp64 of the unsplit
operands with R + A.  Stimuli: activations over 2^-24 .. 2^16 with zeros and fp16 subnormals, weights spread over 2^0 ..
2^-40 of the layer's largest, all-positive / cancelling / random signs, and every layer signature the engine launches in a
test-mode forward of raft_nc_dbl and raft at S1-S4 (a coverage guard fails on a signature missing from the table)."""
import math

import numpy as np
import pytest
import torch

from conftest import build_model
from test_conv_error_model import (C_A, SPLIT_MAX, a_ratio, cancelling_input, check_model, conv_split_ref,
                                   magnitude_sweep, pack_emulate, signed_input, signed_weight, split_emulate,
                                   spread_weight)
from test_product_shapes import SHAPES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ueng():
    from rnc.engine_umma import UmmaEngine
    return UmmaEngine()


def cl(t):
    """[B, C, H, W] -> contiguous channel-last [B*H*W, C] on the device."""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1]).contiguous().to(DEV)


def nchw(t, B, H, W, C):
    return t[:, :C].reshape(B, H, W, C).permute(0, 3, 1, 2)


def device_split(x):
    """fp32 [B, C, H, W] -> (hi, lo) channel-last planes by rnc_f32_to_split, checked bit for bit against split_emulate."""
    from rnc.native import rnc
    xc = cl(x.float())
    M, C = xc.shape
    hi = torch.empty(M, C, dtype=torch.float16, device=DEV)
    lo = torch.empty_like(hi)
    rnc.f32_to_split(xc, C, C, M, hi, lo, C, 0)
    eh, el = split_emulate(xc)
    assert torch.equal(hi.view(torch.int16), eh.view(torch.int16)), "rnc_f32_to_split: hi differs from split_pair's rule"
    assert torch.equal(lo.view(torch.int16), el.view(torch.int16)), "rnc_f32_to_split: lo differs from split_pair's rule"
    return hi, lo


def run(ueng, planes, pk, B, H, W, segs=None, stride=1, hin=0, win=0, dil=1, flags=0, split_out=False):
    """One uconv of the pack pk on channel-last planes (hi, lo) [rows, Cin] (two input buffers for two segments), LINEAR,
    fp32 output.  H, W: output dims.  Returns the output [B, cout, H, W] (and its split planes, same layout, with
    split_out)."""
    from rnc import native
    hi, lo = planes
    cin = hi.shape[1]
    segs = segs or [cin]
    if len(segs) == 1 and cin % 8:                     # operand rows are 16-byte multiples: pad the pitch
        hi, lo = (torch.nn.functional.pad(t, (0, 8 - cin % 8)).contiguous() for t in (hi, lo))
        cin = hi.shape[1]
    kw = dict(stride=stride, hin=hin, win=win, dil=dil, flags=flags)
    c0, ld0 = segs[0], (cin if len(segs) == 1 else segs[0])
    bufs = []
    if len(segs) == 1:
        in0 = (hi.data_ptr(), lo.data_ptr())
    else:
        h0, l0 = hi[:, :segs[0]].contiguous(), lo[:, :segs[0]].contiguous()
        h1, l1 = hi[:, segs[0]:].contiguous(), lo[:, segs[0]:].contiguous()
        bufs += [h0, l0, h1, l1]
        in0 = (h0.data_ptr(), l0.data_ptr())
        kw.update(in1=(h1.data_ptr(), l1.data_ptr()), c1=segs[1], ld1=segs[1])
    M = B * H * W
    out = torch.full((M, pk.coutpad), math.nan, device=DEV)
    ueng.uconv(B, H, W, in0, c0, ld0, pk, native.EPI_LINEAR, out_f32=out.data_ptr(), ldo_f32=pk.coutpad, **kw)
    res = nchw(out, B, H, W, pk.cout)
    if not split_out:
        torch.cuda.synchronize()
        return res
    oh = torch.zeros(M, pk.coutpad, dtype=torch.float16, device=DEV)
    ol = torch.zeros_like(oh)
    ueng.uconv(B, H, W, in0, c0, ld0, pk, native.EPI_LINEAR, out_split=(oh.data_ptr(), ol.data_ptr()),
               ldo_split=pk.coutpad, **kw)
    torch.cuda.synchronize()
    return res, nchw(oh, B, H, W, pk.cout), nchw(ol, B, H, W, pk.cout)


def judge(what, got, s):
    """Both checks of one kernel output; prints the C_A it needed.  Returns (worst err/bound vs split, vs exact)."""
    need = float(a_ratio(got, s).max())
    ws = check_model(what, got, s, "split")
    we = check_model(what, got, s, "exact") if s.exact is not None else float("nan")
    d = (got.double() - s.ref).abs()
    print(f"  {what}: K steps {s.steps}, C_A needed {need:.3f} (C_A {C_A}), max err {float(d.max()):.2e}, worst err/bound "
          f"split {ws:.3f} exact {we:.3f}")
    return ws, we


# ----------------------------------------------------------------------------------------------------------- split producers
def test_split_producers_bit_exact(ueng):
    """rnc_f32_to_split and an epilogue's split output against split_emulate, bit for bit, over 2^-24 .. 2^20 with zeros,
    fp16 subnormals and the saturation range.  The epilogue case is a 1x1 layer of weight 4 * identity: its fp32 output is
    exactly 4 (hi + lo) (one exact product per output and accumulator), up to 4 * 131008, and its split output must be
    split_pair of that value."""
    from rnc.engine_umma import UmmaWeights
    B, C, H, W = 2, 64, 7, 33
    x = magnitude_sweep(B, C, H, W, seed=3, hi_log2=20)
    x[0, -1, 0, :4] = torch.tensor([65504.0, 65520.0, 131008.0, 3e38])
    hi, lo = device_split(x)
    assert float((hi.float() + lo.float()).abs().max()) == SPLIT_MAX
    pk = UmmaWeights(4 * torch.eye(C, device=DEV).view(C, C, 1, 1), None, [C])
    got, oh, ol = run(ueng, (hi, lo), pk, B, H, W, split_out=True)
    xh = nchw(hi.float() + lo.float(), B, H, W, C)
    assert torch.equal(got, 4 * xh), "4 * identity layer: the fp32 output is not exactly 4 (hi + lo)"
    eh, el = split_emulate(got)
    assert torch.equal(oh.contiguous().view(torch.int16), eh.view(torch.int16)), "epilogue split: hi differs"
    assert torch.equal(ol.contiguous().view(torch.int16), el.view(torch.int16)), "epilogue split: lo differs"
    assert float(got.abs().max()) > SPLIT_MAX


# ----------------------------------------------------------------------------------------------------------- stimuli
def test_activation_magnitude_sweep(ueng):
    """Input channels log-spaced over 2^-24 .. 2^16 (zeros, fp16 subnormals, values in the saturation range), a 3x3 layer;
    the split output of the same layer is split_pair of its fp32 output, bit for bit."""
    from rnc.engine_umma import UmmaWeights
    B, C, H, W = 2, 128, 13, 150
    x = magnitude_sweep(B, C, H, W, seed=4)
    g = torch.Generator().manual_seed(4)
    w = torch.randn(64, C, 3, 3, generator=g) / 34
    b = torch.randn(64, generator=g)
    hi, lo = device_split(x)
    pk = UmmaWeights(w.to(DEV), b.to(DEV), [C])
    got, oh, ol = run(ueng, (hi, lo), pk, B, H, W, split_out=True)
    judge("magnitude sweep 3x3", got, conv_split_ref(x.to(DEV), pk, weight=w))
    eh, el = split_emulate(got)
    assert torch.equal(oh.contiguous().view(torch.int16), eh.view(torch.int16))
    assert torch.equal(ol.contiguous().view(torch.int16), el.view(torch.int16))


@pytest.mark.parametrize("kh,kw", [(3, 3), (1, 1)])
def test_weight_spread(ueng, kh, kw):
    """Output channels at 2^0 .. 2^-40 of the layer's largest weight, two zero channels: the pack matches pack_emulate bit
    for bit (w_lo subnormal from 2^-13 down, w_hi from 2^-24, zero below), and every channel meets its own bound."""
    from rnc.engine_umma import UmmaWeights
    B, C, H, W = 2, 128, 11, 96
    g = torch.Generator().manual_seed(kh)
    x = torch.randn(B, C, H, W, generator=g)
    w = spread_weight(96, C, kh, kw, seed=kh)
    b = torch.randn(96, generator=g) * 2.0 ** -30
    pk = UmmaWeights(w.to(DEV), b.to(DEV), [C])
    eh, el, us, eb = pack_emulate(w, b, [C])
    assert pk.unscale == us and torch.equal(pk.bias.cpu(), eb)
    assert torch.equal(pk.w_hi.cpu().view(torch.int16), eh.view(torch.int16))
    assert torch.equal(pk.w_lo.cpu().view(torch.int16), el.view(torch.int16))
    hi, lo = device_split(x)
    got = run(ueng, (hi, lo), pk, B, H, W)
    s = conv_split_ref(x.to(DEV), pk, weight=w)
    judge(f"weight spread {kh}x{kw}", got, s)
    deep = w.abs().amax((1, 2, 3)) < float(w.abs().max()) * 2.0 ** -24      # channels with a subnormal w_hi
    e = (got.double() - s.ref).abs() / (s.steps * 2.0 ** -24)
    print(f"  weight spread {kh}x{kw}: in the {int(deep.sum())} channels with a subnormal w_hi err/(steps 2^-24 mag) "
          f"{float((e / s.mag)[:, deep].max()):.3f}, C_A needed {float(a_ratio(got, s)[:, deep].max()):.3f}; in the others "
          f"{float((e / s.mag)[:, ~deep].max()):.3f} and {float(a_ratio(got, s)[:, ~deep].max()):.3f}")


@pytest.mark.parametrize("kind", ["positive", "cancelling", "random"])
@pytest.mark.parametrize("cin,k", [(64, 1), (256, 3)])
def test_sign_structure(ueng, kind, cin, k):
    """All-positive operands (no cancellation: truncating accumulation errors all of one sign), cancelling halves of K
    (the output ~1e-3 of mag) and random signs.  Prints the signed mean error over steps * 2^-24 * mag next to the largest:
    a mean near the largest in magnitude means the accumulation is biased."""
    from rnc.engine_umma import UmmaWeights
    B, H, W = 2, 16, 130
    x = cancelling_input(B, cin, H, W, cin) if kind == "cancelling" else signed_input(kind, B, cin, H, W, cin)
    w = signed_weight(kind, 64, cin, k, k, cin + 1)
    pk = UmmaWeights(w.to(DEV), None, [cin])
    hi, lo = device_split(x)
    got = run(ueng, (hi, lo), pk, B, H, W)
    s = conv_split_ref(x.to(DEV), pk, weight=w)
    sig = (got.double() - s.ref) / (s.steps * 2.0 ** -24 * s.mag_a)
    print(f"  signs {kind} K={cin * k * k}: |ref|/mag median {float((s.ref.abs() / s.mag).median()):.1e}, "
          f"signed mean err/(steps 2^-24 mag_a) {float(sig.mean()):+.3e}, max |.| {float(sig.abs().max()):.3e}")
    judge(f"signs {kind} {cin}x{k}x{k}", got, s)


# ----------------------------------------------------------------------------------------------------------- signatures
EPI = dict(LINEAR=0, RELU=1, SIGMOID=2, GRU_ZR=3, GRU_Q=4, RELU_FLOW=5, RELU_ADD_RELU=6, TANH_RELU=7, FLOW_DELTA=8)
NO_HALO, WINDOW = 1, 128
MODES = ("tap", "rowhalo", "colhalo")


def _smem_fixed(bn):
    return 1024 + 512 + 8192 + 1024 + 4 * 4096 + 128 * (bn + 4) * 4       # csrc/conv_umma.cu, Cfg<BN>::kSmemFixed


def sm_count():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def launch_shape(c0, c1, coutpad, kh, kw, stride, epi, flags, B, H, W):
    """(A-staging mode, column tile) the kernel picks for one launch (H, W: its output dims), as conv_umma() and choose_bn()
    in csrc/conv_umma.cu (the column tile depends on the device's SM count).  The pixel-tile count of the mirrored mode is
    checked against the library's own, rnc_conv_umma_tiles, on every call."""
    from rnc.native import rnc
    halo = stride == 1 and not flags & NO_HALO
    mode = "rowhalo" if halo and kw > 1 and W > 64 else "colhalo" if halo and kw == 1 and kh > 1 and W >= 16 and H >= 8 else "tap"
    if mode == "rowhalo":
        tw, th, bw, bh = 128, 1, 136, 1
    elif mode == "colhalo":
        tw, th, bw, bh = 16, 8, 16, 8 + 2 * (kh // 2)
    else:
        tw = 8
        while tw < W and tw < 128:
            tw <<= 1
        th, bw, bh = 128 // tw, tw, 128 // tw
    ntiles = B * -(-W // tw) * -(-H // th)
    lib = rnc.conv_umma_tiles(kh, kw, stride, B, H, W, flags & NO_HALO)
    assert ntiles == lib, f"pixel tiles: mirror {ntiles}, library {lib} ({kh}x{kw} s{stride} {B}x{H}x{W}): re-sync launch_shape"
    bn0 = 32 if coutpad <= 32 else 64 if coutpad <= 64 else 128
    bn = bn0
    while bn > 32 and coutpad % bn:
        bn >>= 1
    if coutpad % bn:
        bn = bn0
    if coutpad % bn == 0 and epi not in (EPI["RELU_FLOW"], EPI["FLOW_DELTA"]):
        ksteps = kh * kw * (-(-c0 // 64) + -(-c1 // 64))
        sms = sm_count()
        best, best_cost = bn, np.float32(1e30)
        for cand, per_k in ((128, 1.0), (64, 0.68), (32, 0.57)):
            if cand > bn or coutpad % cand or (epi in (EPI["TANH_RELU"], EPI["GRU_ZR"]) and cand < 64):
                continue
            ntn = coutpad // cand
            rounds = -(-ntiles * ntn // sms)
            item = np.float32(ksteps) * np.float32(per_k) + np.float32(0.5)
            if ntn > 1:
                item = item * np.float32(1.08)
            cost = np.float32(rounds) * item
            if cost < best_cost * np.float32(0.97):
                best, best_cost = cand, cost
        bn = best
    a_plane = bw * bh * 128
    while bn > 32 and 4 * a_plane + 4 * bn * 128 > 226 * 1024 - _smem_fixed(bn) and coutpad % (bn >> 1) == 0:
        bn >>= 1
    return mode, bn


def signature(B, H, W, c0, wt, epi, c1=0, stride=1, dil=1, flags=0):
    """(segments, cout, coutpad, kh, kw, stride, dilation, mode, column tile, window) of one uconv call; mode and column
    tile of the first output phase of a dilated layer."""
    Hp, Wp = -(-H // dil), -(-W // dil)
    mode, bn = launch_shape(c0, c1, wt.coutpad, wt.kh, wt.kw, stride, epi, flags, B, Hp, Wp)
    segs = (c0, c1) if c1 else (c0,)
    return segs, wt.cout, wt.coutpad, wt.kh, wt.kw, stride, dil, mode, bn, bool(flags & WINDOW)


# Every signature the tensor-core engine launches in a test-mode forward of raft_nc_dbl and raft at S1-S4 (encoders, update
# block, mask head, weights net) on an H100 SXM (132 SMs: the column tiles depend on it), with a replay geometry (B, H, W of
# the output) that selects the same A-staging mode and column tile.  Collected by test_signature_table_covers_the_engine.
SIGNATURES = {
    ((128, 128), 128, 128, 1, 5, 1, 1, 'rowhalo', 128, False): (4, 9, 150),
    ((128, 128), 128, 128, 1, 5, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((128, 128), 128, 128, 1, 5, 1, 1, 'tap', 64, False): (3, 24, 40),
    ((128, 128), 128, 128, 5, 1, 1, 1, 'colhalo', 64, False): (6, 9, 40),
    ((128, 128), 128, 128, 5, 1, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((128, 128), 256, 256, 1, 5, 1, 1, 'rowhalo', 128, False): (2, 9, 150),
    ((128, 128), 256, 256, 1, 5, 1, 1, 'tap', 128, False): (3, 24, 40),
    ((128, 128), 256, 256, 1, 5, 1, 1, 'tap', 64, False): (4, 9, 40),
    ((128, 128), 256, 256, 5, 1, 1, 1, 'colhalo', 64, False): (3, 9, 40),
    ((128, 128), 256, 256, 5, 1, 1, 1, 'tap', 64, False): (3, 48, 12),
    ((128,), 128, 128, 1, 5, 1, 1, 'rowhalo', 128, False): (4, 9, 150),
    ((128,), 128, 128, 1, 5, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((128,), 128, 128, 1, 5, 1, 1, 'tap', 64, False): (3, 24, 40),
    ((128,), 128, 128, 3, 3, 1, 1, 'rowhalo', 128, False): (4, 9, 150),
    ((128,), 128, 128, 3, 3, 1, 1, 'tap', 128, False): (3, 48, 40),
    ((128,), 128, 128, 3, 3, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((128,), 128, 128, 3, 3, 1, 1, 'tap', 64, False): (3, 24, 40),
    ((128,), 128, 128, 5, 1, 1, 1, 'colhalo', 64, False): (6, 9, 40),
    ((128,), 128, 128, 5, 1, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((128,), 256, 256, 1, 1, 1, 1, 'tap', 128, False): (2, 9, 150),
    ((128,), 256, 256, 1, 1, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((128,), 256, 256, 1, 1, 1, 1, 'tap', 64, False): (1, 9, 150),
    ((128,), 256, 256, 1, 5, 1, 1, 'rowhalo', 128, False): (2, 9, 150),
    ((128,), 256, 256, 1, 5, 1, 1, 'tap', 128, False): (3, 24, 40),
    ((128,), 256, 256, 1, 5, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((128,), 256, 256, 3, 3, 1, 1, 'rowhalo', 128, False): (2, 9, 150),
    ((128,), 256, 256, 3, 3, 1, 1, 'tap', 128, False): (3, 24, 40),
    ((128,), 256, 256, 3, 3, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((128,), 256, 256, 5, 1, 1, 1, 'colhalo', 64, False): (3, 9, 40),
    ((128,), 256, 256, 5, 1, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((128,), 64, 64, 3, 3, 1, 1, 'rowhalo', 64, False): (4, 9, 150),
    ((128,), 64, 64, 3, 3, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((132,), 64, 64, 3, 3, 1, 1, 'rowhalo', 64, False): (4, 9, 150),
    ((132,), 64, 64, 3, 3, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((256,), 126, 128, 3, 3, 1, 1, 'rowhalo', 128, False): (4, 9, 150),
    ((256,), 126, 128, 3, 3, 1, 1, 'tap', 128, False): (3, 48, 40),
    ((256,), 18, 32, 1, 1, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((256,), 192, 192, 3, 3, 1, 1, 'rowhalo', 64, False): (1, 13, 150),
    ((256,), 192, 192, 3, 3, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((256,), 192, 192, 3, 3, 1, 1, 'tap', 64, False): (1, 48, 40),
    ((256,), 576, 576, 1, 1, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((256,), 576, 576, 1, 1, 1, 1, 'tap', 64, False): (4, 9, 12),
    ((352,), 256, 256, 1, 1, 1, 1, 'tap', 128, False): (2, 9, 150),
    ((352,), 256, 256, 1, 1, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((64,), 32, 32, 3, 3, 1, 1, 'rowhalo', 32, False): (1, 8, 96),
    ((64,), 32, 32, 3, 3, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((64,), 64, 64, 3, 3, 1, 1, 'rowhalo', 64, False): (4, 9, 150),
    ((64,), 64, 64, 3, 3, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((64,), 64, 64, 3, 3, 1, 1, 'tap', 64, False): (3, 48, 40),
    ((64,), 64, 64, 7, 1, 2, 1, 'tap', 32, True): (1, 8, 12),
    ((64,), 64, 64, 7, 1, 2, 1, 'tap', 64, True): (4, 9, 150),
    ((64,), 96, 128, 1, 1, 2, 1, 'tap', 128, False): (4, 9, 150),
    ((64,), 96, 128, 1, 1, 2, 1, 'tap', 32, False): (1, 8, 12),
    ((64,), 96, 128, 3, 3, 2, 1, 'tap', 128, False): (4, 9, 150),
    ((64,), 96, 128, 3, 3, 2, 1, 'tap', 32, False): (1, 8, 12),
    ((96,), 128, 128, 1, 1, 2, 1, 'tap', 128, False): (4, 9, 150),
    ((96,), 128, 128, 1, 1, 2, 1, 'tap', 32, False): (1, 8, 12),
    ((96,), 128, 128, 1, 1, 2, 1, 'tap', 64, False): (2, 9, 150),
    ((96,), 128, 128, 3, 3, 2, 1, 'tap', 128, False): (4, 9, 150),
    ((96,), 128, 128, 3, 3, 2, 1, 'tap', 32, False): (1, 8, 12),
    ((96,), 128, 128, 3, 3, 2, 1, 'tap', 64, False): (2, 9, 150),
    ((96,), 96, 128, 3, 3, 1, 1, 'rowhalo', 128, False): (4, 9, 150),
    ((96,), 96, 128, 3, 3, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((98,), 128, 128, 1, 1, 1, 1, 'tap', 128, False): (4, 9, 150),
    ((98,), 128, 128, 1, 1, 1, 1, 'tap', 32, False): (1, 8, 12),
    ((98,), 128, 128, 1, 1, 1, 1, 'tap', 64, False): (2, 9, 150),
}


def record_signatures(monkeypatch, eng, seen):
    orig = eng.uconv

    def uconv(B, H, W, in0, c0, ld0, wt, epi, **kw):
        seen.setdefault(signature(B, H, W, c0, wt, epi, kw.get("c1", 0), kw.get("stride", 1), kw.get("dil", 1), kw.get("flags", 0)),
                        (B, H, W))
        return orig(B, H, W, in0, c0, ld0, wt, epi, **kw)
    monkeypatch.setattr(eng, "uconv", uconv)


REPLAY_GEOMETRIES = sorted(((B, H, W) for B in (1, 2, 3, 4, 6, 8) for H in (8, 9, 13, 16, 24, 30, 48, 55)
                            for W in (12, 16, 40, 64, 96, 128, 150, 156)), key=lambda g: (g[0] * g[1] * g[2], g))


def replay_geometry(sig, seen_at):
    """The smallest of REPLAY_GEOMETRIES (and the geometry the engine ran it at) that selects sig's mode and column tile."""
    segs, cout, coutpad, kh, kw, stride, dil, mode, bn, window = sig
    for B, H, W in REPLAY_GEOMETRIES + [seen_at]:
        if launch_shape(segs[0], segs[1] if len(segs) > 1 else 0, coutpad, kh, kw, stride, EPI["LINEAR"], 0, B,
                        -(-H // dil), -(-W // dil)) == (mode, bn):
            return B, H, W
    return seen_at


def test_signature_table_covers_the_engine(monkeypatch):
    """Test-mode forwards of raft_nc_dbl and raft at S1-S4 (encoders included): every uconv signature is in SIGNATURES."""
    seen = {}
    for name in ("raft_nc_dbl", "raft"):
        m = build_model(name).to(DEV)
        eng = m.engine()
        assert eng.mode == "umma"
        with monkeypatch.context() as mp:
            record_signatures(mp, eng, seen)
            for sid, (B, H8, W8) in SHAPES.items():
                g = torch.Generator().manual_seed(B)
                im1, im2 = (torch.rand(B, 3, 8 * H8, 8 * W8, generator=g) * 255 for _ in range(2))
                with torch.no_grad():
                    m(im1.to(DEV), im2.to(DEV), iters=2, test_mode=True)
        torch.cuda.synchronize()
    missing = {s: replay_geometry(s, g) for s, g in seen.items() if s not in SIGNATURES}
    print(f"{len(seen)} signatures launched, {len(missing)} missing from the table")
    for s, g in sorted(missing.items(), key=str):
        print(f"    {s!r}: {g!r},")
    assert not missing, f"{len(missing)} launched signatures are not in SIGNATURES (listed above)"


def _pack_for(sig, seed):
    from rnc.engine_umma import UmmaWeights
    segs, cout, coutpad, kh, kw = sig[:5]
    g = torch.Generator().manual_seed(seed)
    cin = sum(segs)
    w = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    b = torch.randn(cout, generator=g)
    pk = UmmaWeights(w.to(DEV), b.to(DEV), list(segs), extra_cout=coutpad - cout)
    assert pk.coutpad == coutpad
    return pk, w, g


def _window_case(ueng, sig, geo, seed):
    """The encoders' stem: a 7x1 layer at stride 2 over a sliding-window view of the split image (RNC_CONV_WINDOW):
    output position x of row y reads the 64 halves from element 8x of image row y (16 pixels x 4 channels)."""
    from rnc import native
    from rnc.native import rnc
    pk, w, g = _pack_for(sig, seed)
    N, h, wo = geo
    Hin, Win = 2 * h, 2 * wo
    pitch = (Win + 7) & ~1
    img = torch.rand(N, 3, Hin, Win, generator=g) * 255
    hi = torch.zeros(N * Hin * pitch + 32, 4, dtype=torch.float16, device=DEV)
    lo = torch.zeros_like(hi)
    rnc.stem_window_prep(img.to(DEV), N, Hin, Win, pitch, hi, lo)
    win = dict(stride=2, hin=Hin, win=wo, win_pitch=4 * pitch, flags=native.CONV_WINDOW)
    out = torch.full((N * h * wo, pk.coutpad), math.nan, device=DEV)
    ueng.uconv(N, h, wo, (hi.data_ptr(), lo.data_ptr()), 64, 8, pk, native.EPI_LINEAR, out_f32=out.data_ptr(),
               ldo_f32=pk.coutpad, **win)
    torch.cuda.synchronize()
    view = lambda t: t.view(-1).as_strided((N, Hin, wo, 64), (Hin * pitch * 4, pitch * 4, 8, 1)).permute(0, 3, 1, 2)  # noqa
    s = conv_split_ref((view(hi), view(lo)), pk, weight=w, stride=(2, 1))
    return nchw(out, N, h, wo, pk.cout), s


@pytest.mark.parametrize("sig", list(SIGNATURES), ids=str)
def test_layer_signature(ueng, sig):
    """One launch of each engine signature, at a geometry that selects the same A-staging mode and column tile."""
    geo = SIGNATURES[sig]
    segs, cout, coutpad, kh, kw, stride, dil, mode, bn, window = sig
    B, H, W = geo
    if window:
        got, s = _window_case(ueng, sig, geo, seed=cout + kh)
    else:
        assert launch_shape(segs[0], segs[1] if len(segs) > 1 else 0, coutpad, kh, kw, stride, EPI["LINEAR"], 0, B,
                            -(-H // dil), -(-W // dil)) == (mode, bn), "the replay geometry selects another launch shape"
        pk, w, g = _pack_for(sig, seed=cout + kh + stride)
        Hin, Win = (2 * H, 2 * W) if stride == 2 else (H, W)
        x = torch.randn(B, sum(segs), Hin, Win, generator=g)
        hi, lo = device_split(x)
        got = run(ueng, (hi, lo), pk, B, H, W, list(segs), stride=stride, hin=Hin if stride == 2 else 0,
                  win=Win if stride == 2 else 0, dil=dil, flags=0)
        s = conv_split_ref(x.to(DEV), pk, list(segs), weight=w, stride=stride, dil=dil)
    judge(f"{sig}", got, s)


@pytest.mark.parametrize("flag", ["no-halo"])
@pytest.mark.parametrize("kh,kw,cin,cout", [(3, 3, 128, 256), (1, 5, 256, 128), (5, 1, 256, 256), (3, 3, 64, 64)])
def test_layer_flags(ueng, flag, kh, kw, cin, cout):
    """RNC_CONV_NO_HALO (one A tile per tap) on row-halo, column-halo and per-tap layers."""
    from rnc import native
    from rnc.engine_umma import UmmaWeights
    B, H, W = 2, 24, 130
    g = torch.Generator().manual_seed(kh * 10 + kw)
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    pk = UmmaWeights(w.to(DEV), torch.randn(cout, generator=g).to(DEV), [cin])
    hi, lo = device_split(x)
    got = run(ueng, (hi, lo), pk, B, H, W, flags=native.CONV_NO_HALO)
    judge(f"{flag} {kh}x{kw} {cin}->{cout}", got, conv_split_ref(x.to(DEV), pk, weight=w))
