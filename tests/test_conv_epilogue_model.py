"""The fused epilogues of both convolution engines (csrc/conv_umma.cu, csrc/conv_ffma.cu) against fp64: an elementwise bound
for every epilogue form the engines launch, built on the accumulator model of tests/test_conv_error_model.py.
tests/test_gpu_conv_epilogue_model.py holds the kernels to it and measures the gate activations it uses.

Pre-activation.  v^ is the fp64 value the accumulator model gives (conv_split_ref: SplitRef.ref, bias included; the exact
engine: fp64 conv of its fp32 operands), plus the hoisted `add` operand as the kernel read it.  Its bound:
    tensor cores: A_v = C_A steps u mag_a + u |ref| (+ u |v^| for the addend's fp32 add), + R against the unsplit operands;
    exact engine: A_v = K u mag + u |v^| (the fp32 FMA chain over K = kh kw cin terms, then the bias add).
Activation.  |act_kernel(v) - act(v^)| <= L(v^, A_v) A_v + E_act(v^, A_v): L is the largest |act'| over [v^ - A_v, v^ + A_v]
(taken at the point of the interval nearest 0: sigma(1 - sigma), 1 - tanh^2; 1 for relu), E_act the measured error of the
device function (E_SIG, E_TANH below) at the fp32 value the kernel evaluated, which lies in that interval.
Epilogue forms (every output an fp32 value, then split by split_pair where the launch writes halves: + split_bound):
    RELU / SIGMOID / LINEAR (also tile-blocked, the hoisted czr / cq): act(v^);
    GRU_ZR: z = sigma(v^) into the aux buffer; r*h = rn(sigma(v) h) split: |h| (L A_v + E_sig) + u |r h| + split_bound;
    GRU_Q: h' = (1 - z) h + z tanh(v) with the z and h the kernel read: |z| (L A_v + E_tanh) + C_BLEND u (|(1-z) h| + |z t|);
           the split copy of h' (hx) is split_pair(h') bit for bit;
    RELU_FLOW: relu below cout (A_v + split_bound); channels cout, cout + 1 are split_pair(coords1 - x / y) bit for bit;
    RELU_ADD_RELU: relu(res + relu(v^)), A_v + u (|res| + |relu v^| + A_v): valid where res cancels relu(v);
    TANH_RELU: tanh of the first half (fp32 and split, the split = split_pair(fp32)), relu of the second half (split only).
"""
import math
from typing import NamedTuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_conv_error_model import C_A, U, _Pack, conv_split_ref, fp64_floor, split_bound, split_emulate
from test_product_shapes import Mismatch
from test_train_shapes import compare_mag

FTZ = 2.0 ** -126          # rcp.approx.ftz / expf flush: results below the smallest normal float are returned as 0

# Measured error of the gate activations: |f(v) - f64(v)| <= (REL + LIN |v|) |f64(v)| + 2^-126, elementwise, over every
# 22-bit-significand fp32 value of every binade 2^-24 .. 2^8, both signs (test_gpu_conv_epilogue_model.py::
# test_activation_sweep_*).  The linear term is the argument rounding of exp: x log2(e) carries a relative error of u, so
# exp(x) one of u |x| (ln 2 log2(e) = 1).  Measured on an H100 SXM (80 GB HBM3, 700 W power limit); each constant is the
# measured maximum times about 1.5.
#   tensor-core epilogues, sigmoid_fast / tanh_fast (ex2.approx, rcp.approx.ftz; Taylor branch below |x| = 0.25):
#     sigmoid: relative error <= 1.82e-7 for |v| < 1, then growing with |v| (2.26e-7 at 2^0, 9.6e-7 at 2^3, 3.88e-6 at
#     2^6): at most 1.82e-7 + 1.06e-7 |v|; flushed to 0 for v <= -87.3366 (sigma < 2^-126).
#     tanh: relative error <= 8.9e-8 on the Taylor branch (|v| < 0.25), 4.27e-7 just above it (the largest: 1 - 2 / (e + 1)
#     cancels most there), 1.02e-7 at 2^0, exact (1) from |v| = 16.
#   exact engine, 1 / (1 + expf(-x)) and tanhf: relative error <= 2.11e-7 and 1.97e-7, not growing with |v|; sigmoid
#     flushed to 0 below -88.72 (expf overflows), where sigma < 2^-127.
E_SIG = (2.8e-7, 1.6e-7)            # (REL, LIN)
E_TANH = (6.4e-7, 1.0e-8)
E_SIG_EXACT = (3.2e-7, 1.0e-9)
E_TANH_EXACT = (3.0e-7, 1.0e-9)
C_BLEND = 3.0 * (1 + 2.0 ** -20)    # (1 - z) h + z t in fp32, contracted into FMAs or not: at most 3 roundings deep


def act64(kind, v):
    v = v.double()
    if kind == "sigmoid":
        return torch.sigmoid(v)
    if kind == "tanh":
        return torch.tanh(v)
    if kind == "relu":
        return v.clamp_min(0)
    return v


def lip(kind, v, a):
    """max |act'| over [v - a, v + a], elementwise: the derivative at the interval's point nearest 0."""
    v, a = v.double(), torch.as_tensor(a, dtype=torch.float64, device=v.device)
    t = torch.where((v - a <= 0) & (v + a >= 0), torch.zeros_like(v), torch.where(v > 0, v - a, v + a))
    if kind == "sigmoid":
        s = torch.sigmoid(t)
        return s * (1 - s)
    if kind == "tanh":
        return 1 - torch.tanh(t) ** 2
    return torch.ones_like(v)


def act_err(kind, v, a=0.0, exact=False):
    """E_act at the fp32 value the kernel evaluated, somewhere in [v - a, v + a]: (REL + LIN (|v| + a)) (|act(v)| + L a)
    + 2^-126.  relu / linear: 0."""
    if kind not in ("sigmoid", "tanh"):
        return torch.zeros_like(v, dtype=torch.float64)
    rel, lin = (E_SIG_EXACT if exact else E_SIG) if kind == "sigmoid" else (E_TANH_EXACT if exact else E_TANH)
    v = v.double()
    return (rel + lin * (v.abs() + a)) * (act64(kind, v).abs() + lip(kind, v, a) * a) + FTZ


class Pre(NamedTuple):
    v: torch.Tensor          # fp64 pre-activation [B, C, H, W]
    A: torch.Tensor          # elementwise bound on |kernel's fp32 pre-activation - v|


def pre_umma(sref, add=None, against="split"):
    """Pre-activation of a tensor-core launch: SplitRef plus the addend (fp32 [B, C, H, W] as the kernel read it)."""
    v = sref.ref if against == "split" else sref.exact
    A = C_A * sref.steps * U * sref.mag_a + U * sref.ref.abs() + fp64_floor(sref)
    if against != "split":
        A = A + sref.R
    if add is not None:
        v = v + add.double()[:, :v.shape[1]]
        A = A + U * v.abs()
    return Pre(v, A)


def pre_ffma(x, w, b, dil=1, add=None):
    """Pre-activation of an exact-engine launch: fp64 conv of the fp32 operands (x [B, Cin, H, W], w [Cout, Cin, kh, kw])."""
    K = w.shape[1] * w.shape[2] * w.shape[3]
    pad = (w.shape[2] // 2 * dil, w.shape[3] // 2 * dil)
    x, w = x.double(), w.double().to(x.device)
    b = torch.zeros(w.shape[0], dtype=torch.float64, device=x.device) if b is None else b.double().to(x.device)
    v = F.conv2d(x, w, b, padding=pad, dilation=dil)
    mag = F.conv2d(x.abs(), w.abs(), b.abs(), padding=pad, dilation=dil)
    A = (K + 1) * U * mag + U * v.abs()
    if add is not None:
        v = v + add.double()
        A = A + U * v.abs()
    return Pre(v, A)


def _sl(pre, c0, c1):
    return Pre(pre.v[:, c0:c1], pre.A[:, c0:c1])


def check(what, got, ref, bound, log=print):
    """|got - ref| <= bound elementwise (NaN / Inf fail); raises Mismatch naming the worst image, pixel, channel and tile."""
    return compare_mag(what, got, ref.to(got.device) if torch.is_tensor(ref) else ref, bound, 1.0, log=log)


def act_bound(kind, pre, exact=False):
    """Reference and bound of act(pre-activation) as an fp32 output."""
    return act64(kind, pre.v), lip(kind, pre.v, pre.A) * pre.A + act_err(kind, pre.v, pre.A, exact)


def check_act(what, kind, pre, f32=None, split=None, exact=False, log=print):
    """RELU / SIGMOID / tanh half / LINEAR: the fp32 output and / or the split output ((hi, lo) [B, C, H, W]).  With both,
    the split must be split_pair of the fp32 output, bit for bit.  Returns the worst err / bound."""
    ref, bnd = act_bound(kind, pre, exact)
    worst = 0.0
    if f32 is not None:
        worst = check(f"{what} fp32", f32, ref, bnd, log)
    if split is not None:
        hi, lo = split
        if f32 is not None:
            eh, el = split_emulate(f32)
            assert torch.equal(hi.contiguous().view(torch.int16), eh.view(torch.int16).to(hi.device)) and \
                torch.equal(lo.contiguous().view(torch.int16), el.view(torch.int16).to(lo.device)), \
                f"{what}: the split output is not split_pair of the fp32 output"
        val = hi.double() + lo.double()
        worst = max(worst, check(f"{what} split", val, ref, bnd + split_bound(ref + bnd), log))
    return worst


def check_gru_zr(what, pre, z, rh, h, exact=False, log=print):
    """GRU_ZR: pre [B, 2C, H, W]; z [B, C, H, W] (fp32, read back channel-last); rh the r*h output: (hi, lo) planes on the
    tensor cores, fp32 on the exact engine; h the fp32 state the kernel read."""
    C = pre.v.shape[1] // 2
    w = check_act(f"{what} z", "sigmoid", _sl(pre, 0, C), f32=z, exact=exact, log=log)
    r, rb = act_bound("sigmoid", _sl(pre, C, 2 * C), exact)
    h = h.double()
    ref = r * h
    bnd = h.abs() * rb + U * (ref.abs() + h.abs() * rb)
    if isinstance(rh, (tuple, list)):
        got = rh[0].double() + rh[1].double()
        bnd = bnd + split_bound(ref.abs() + bnd)
    else:
        got = rh
    return max(w, check(f"{what} r*h", got, ref, bnd, log))


def blend_bound(z, h, t):
    """Rounding of the fp32 blend (1 - z) h + z t, contracted or not: C_BLEND u (|(1 - z) h| + |z t|)."""
    z, h, t = z.double(), h.double(), t.double()
    return C_BLEND * U * (((1 - z) * h).abs() + (z * t).abs())


def check_gru_q(what, pre, z, h_old, h_new, hx=None, exact=False, log=print):
    """GRU_Q: h_new = (1 - z) h_old + z tanh(v), z and h_old as the kernel read them; hx: the split copy of h_new (the
    tensor-core engine), split_pair(h_new) bit for bit."""
    z, h_old = z.double(), h_old.double()
    t, tb = act_bound("tanh", pre, exact)
    ref = (1 - z) * h_old + z * t
    bnd = z.abs() * tb + blend_bound(z, h_old, t.abs() + tb)
    w = check(f"{what} h", h_new, ref, bnd, log)
    if hx is not None:
        eh, el = split_emulate(h_new)
        assert torch.equal(hx[0].contiguous().view(torch.int16), eh.view(torch.int16).to(hx[0].device)) and \
            torch.equal(hx[1].contiguous().view(torch.int16), el.view(torch.int16).to(hx[1].device)), \
            f"{what}: the split copy of h is not split_pair(h)"
    return w


def check_relu_flow(what, pre, out, flow, exact=False, log=print):
    """RELU_FLOW: out [B, cout + 2, H, W] as (hi, lo) planes (tensor cores) or fp32 (exact engine); flow [B, 2, H, W] the
    fp32 coords1 - (x, y) the kernel computes (exactly reproducible: one fp32 subtraction)."""
    cout = pre.v.shape[1]
    if isinstance(out, (tuple, list)):
        w = check_act(f"{what} relu", "relu", pre, split=(out[0][:, :cout], out[1][:, :cout]), log=log)
        eh, el = split_emulate(flow)
        assert torch.equal(out[0][:, cout:cout + 2].contiguous().view(torch.int16), eh.view(torch.int16).to(out[0].device)) \
            and torch.equal(out[1][:, cout:cout + 2].contiguous().view(torch.int16), el.view(torch.int16).to(out[1].device)), \
            f"{what}: the appended flow channels are not split_pair(coords1 - grid)"
        return w
    w = check_act(f"{what} relu", "relu", pre, f32=out[:, :cout], exact=exact, log=log)
    assert torch.equal(out[:, cout:cout + 2], flow.to(out.device)), f"{what}: the appended flow channels differ"
    return w


def check_relu_add_relu(what, pre, res, f32=None, split=None, log=print):
    """RELU_ADD_RELU: relu(res + relu(v)); res [B, C, H, W] fp32 as the kernel read it."""
    r = pre.v.clamp_min(0)
    res = res.double()
    ref = (res + r).clamp_min(0)
    bnd = pre.A + U * (res.abs() + r + pre.A)
    w = 0.0
    if f32 is not None:
        w = check(f"{what} fp32", f32, ref, bnd, log)
    if split is not None:
        if f32 is not None:
            eh, el = split_emulate(f32)
            assert torch.equal(split[0].contiguous().view(torch.int16), eh.view(torch.int16).to(split[0].device)) and \
                torch.equal(split[1].contiguous().view(torch.int16), el.view(torch.int16).to(split[1].device)), \
                f"{what}: the split output is not split_pair of the fp32 output"
        w = max(w, check(f"{what} split", split[0].double() + split[1].double(), ref, bnd + split_bound(ref + bnd), log))
    return w


def check_tanh_relu(what, pre, f32, split, log=print):
    """TANH_RELU: tanh of channels [0, C/2) to f32 [B, C/2, H, W] and the split, relu of [C/2, C) to the split only."""
    C = pre.v.shape[1]
    hi, lo = split
    w = check_act(f"{what} tanh", "tanh", _sl(pre, 0, C // 2), f32=f32, split=(hi[:, :C // 2], lo[:, :C // 2]), log=log)
    return max(w, check_act(f"{what} relu", "relu", _sl(pre, C // 2, C), split=(hi[:, C // 2:], lo[:, C // 2:]), log=log))


# ----------------------------------------------------------------------------------------------------------- CPU tests
@pytest.mark.parametrize("kind", ["sigmoid", "tanh", "relu"])
def test_lipschitz_against_grid(kind):
    """L(v, a) equals the largest |act'| over a fine grid of [v - a, v + a], intervals on either side of 0 and across it."""
    g = torch.Generator().manual_seed(1)
    v = torch.cat([torch.randn(300, generator=g) * 8, torch.tensor([0.0, -30.0, 30.0, 0.25, -0.25, 1e-3])]).double()
    a = torch.cat([torch.rand(300, generator=g).double() * 2.0 ** torch.randint(-20, 3, (300,), generator=g).double(),
                   torch.tensor([1.0, 1e-6, 1e-6, 0.3, 0.2, 0.0], dtype=torch.float64)])
    s = torch.linspace(-1, 1, 20001, dtype=torch.float64)
    pts = v[:, None] + a[:, None] * s[None, :]
    if kind == "sigmoid":
        d = torch.sigmoid(pts) * (1 - torch.sigmoid(pts))
    elif kind == "tanh":
        d = 1 - torch.tanh(pts) ** 2
    else:
        d = torch.ones_like(pts)
    brute = d.max(1).values
    L = lip(kind, v, a)
    assert (L >= brute * (1 - 1e-12)).all(), "L below the grid maximum"
    assert torch.allclose(L, brute, rtol=1e-6, atol=0), "L above the grid maximum beyond its spacing"


def _fp32(x):
    return np.float32(x)


def test_blend_bound_covers_both_contractions():
    """(1 - z) h + z t in fp32: plain (three roundings), fma((1 - z), h, z t) and fma(z, t, (1 - z) h), against the fp64
    value, over random z, h, t with z within 2^-24 of 0 and of 1, h over 2^-20 .. 2^4 with zeros, t over [-1, 1]."""
    rng = np.random.default_rng(3)
    n = 200000
    z = rng.random(n)
    z[:n // 8] = rng.integers(0, 4, n // 8) * 2.0 ** -26              # within 2^-24 of 0
    z[n // 8:n // 4] = 1 - rng.integers(0, 4, n // 8) * 2.0 ** -26    # within 2^-24 of 1
    h = rng.choice([-1, 1], n) * 2.0 ** rng.uniform(-20, 4, n)
    h[::50] = 0.0
    t = rng.uniform(-1, 1, n)
    z, h, t = (a.astype(np.float32) for a in (z, h, t))
    omz = (np.float32(1) - z).astype(np.float32)
    a32 = (omz * h).astype(np.float32)
    b32 = (z * t).astype(np.float32)
    zd, hd, td = (a.astype(np.float64) for a in (z, h, t))
    forms = {"plain": (a32 + b32).astype(np.float32),
             "fma(1-z, h, z t)": (omz.astype(np.float64) * hd + b32.astype(np.float64)).astype(np.float32),
             "fma(z, t, (1-z) h)": (zd * td + a32.astype(np.float64)).astype(np.float32)}
    ref = (1 - zd) * hd + zd * td
    bnd = blend_bound(torch.from_numpy(z), torch.from_numpy(h), torch.from_numpy(t)).numpy()
    for name, got in forms.items():
        r = np.abs(got.astype(np.float64) - ref) / np.where(bnd > 0, bnd, 1)
        r = np.where((bnd == 0) & (got == ref), 0, r)
        print(f"  blend {name}: worst err / bound {r.max():.3f}")
        assert r.max() <= 1.0, f"blend form {name} exceeds C_BLEND"
    # the bound is not loose by more than the form's depth: the plain form reaches a third of it
    assert np.abs(forms["plain"].astype(np.float64) - ref).max() > 0


def test_activation_bounds_reject_the_two_plausible_mistakes():
    """The activation bounds are tight enough to reject a tanh Taylor branch moved from 0.25 to 0.45 (truncation ~1.4e-6)
    and a sigmoid written as 0.5 + 0.5 tanh(x / 2) (0 at x = -20 where sigma = 2e-9)."""
    x = torch.linspace(0.25, 0.45, 2001, dtype=torch.float64)
    x2 = x * x
    poly = x * (1 + x2 * (-1 / 3 + x2 * (2 / 15 + x2 * (-17 / 315 + x2 * 62 / 2835))))
    err = (poly - torch.tanh(x)).abs()
    assert float((err / act_err("tanh", x)).max()) > 1.2
    v = torch.tensor([-20.0], dtype=torch.float64)
    assert float(torch.sigmoid(v)) > act_err("sigmoid", v).item()       # returning 0 fails
    # and the sound forms pass: fp64 itself, and the flush to zero below -87.3
    assert float(act_err("sigmoid", torch.tensor([-87.5], dtype=torch.float64))) >= float(torch.sigmoid(torch.tensor(-87.5)))


def _pre_case(seed=0, B=2, C=8, H=5, W=130):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 64, H, W, generator=g)
    w = torch.randn(C, 64, 3, 3, generator=g) / 24
    pk = _Pack(w, torch.randn(C, generator=g), [64])
    return pre_umma(conv_split_ref(x, pk, weight=w)), g


@pytest.mark.parametrize("form", ["sigmoid", "tanh-split", "gru-q", "gru-zr", "relu-add-relu"])
def test_perturbation_rejected_at_its_place(form):
    """The model's own fp32 rounding of the reference passes; one element moved by 1.01 x its bound is rejected, and the
    message names its image, pixel, channel and tile."""
    pre, g = _pre_case()
    B, C, H, W = pre.v.shape
    at = (1, 5, 3, 129)
    where = r"image 1, pixel \(y=3, x=129\), channel 5, tile 4"

    def bump(t, bnd):
        t = t.clone()
        t[at] += 1.01 * float(bnd[at]) * (1 if float(t[at]) <= 0 else -1)
        return t
    if form == "sigmoid":
        ref, bnd = act_bound("sigmoid", pre)
        check_act("ok", "sigmoid", pre, f32=ref.float())
        with pytest.raises(Mismatch, match=where):
            check_act("bad", "sigmoid", pre, f32=bump(ref, bnd).float().double())
    elif form == "tanh-split":
        ref, bnd = act_bound("tanh", pre)
        hi, lo = split_emulate(ref.float())
        check_act("ok", "tanh", pre, split=(hi, lo))
        bad = bump(hi.double() + lo.double(), bnd + split_bound(ref + bnd))
        with pytest.raises(Mismatch, match=where):
            check_act("bad", "tanh", pre, split=(bad, torch.zeros_like(bad)))
    elif form == "gru-q":
        z = torch.rand(B, C, H, W, generator=g)
        h = torch.randn(B, C, H, W, generator=g)
        ref = (1 - z.double()) * h.double() + z.double() * torch.tanh(pre.v)
        hn = ref.float()
        check_gru_q("ok", pre, z, h, hn, hx=split_emulate(hn))
        t, tb = act_bound("tanh", pre)
        bnd = z.double() * tb + blend_bound(z, h, t.abs() + tb)
        with pytest.raises(Mismatch, match=where):
            check_gru_q("bad", pre, z, h, bump(ref, bnd))
    elif form == "gru-zr":
        pre2 = Pre(torch.cat([pre.v, pre.v.flip(1)], 1), torch.cat([pre.A, pre.A.flip(1)], 1))
        h = torch.randn(B, C, H, W, generator=g)
        r = torch.sigmoid(pre2.v[:, C:])
        rh = split_emulate((r * h.double()).float())
        check_gru_zr("ok", pre2, torch.sigmoid(pre2.v[:, :C]).float(), rh, h)
        _, rb = act_bound("sigmoid", _sl(pre2, C, 2 * C))
        ref = r * h.double()
        bnd = h.double().abs() * rb + U * (ref.abs() + h.double().abs() * rb)
        bnd = bnd + split_bound(ref.abs() + bnd)
        bad = bump(ref, bnd)
        with pytest.raises(Mismatch, match=where):
            check_gru_zr("bad", pre2, torch.sigmoid(pre2.v[:, :C]).float(), (bad, torch.zeros_like(bad)), h)
    else:
        r = pre.v.clamp_min(0)
        res = -r * (1 + 1e-3 * torch.randn(B, C, H, W, generator=g).double())          # a share cancels relu(v)
        ref = (res + r).clamp_min(0)
        check_relu_add_relu("ok", pre, res.float(), f32=(res.float() + r.float()).clamp_min(0))
        bnd = pre.A + U * (res.abs() + r + pre.A)
        with pytest.raises(Mismatch, match=where):
            check_relu_add_relu("bad", pre, res.float(), f32=bump(ref, bnd))


def test_non_finite_and_flow_channels_rejected():
    pre, _ = _pre_case(1)
    ref, _ = act_bound("relu", pre)
    got = ref.clone()
    got[0, 2, 1, 7] = math.nan
    with pytest.raises(Mismatch, match=r"image 0, pixel \(y=1, x=7\), channel 2, tile 1"):
        check_act("nan", "relu", pre, f32=got)
    flow = torch.randn(2, 2, 5, 130)
    v = torch.cat([ref.float(), flow], 1)
    hi, lo = split_emulate(v)
    check_relu_flow("ok", pre, (hi, lo), flow)
    lo2 = lo.clone()
    lo2[0, -1, 0, 0] = lo2[0, -1, 0, 0] + 2.0 ** -24 if lo2[0, -1, 0, 0] == 0 else 0
    with pytest.raises(AssertionError, match="appended flow"):
        check_relu_flow("bad", pre, (hi, lo2), flow)
