"""The fused epilogues of both convolution engines against the fp64 model of tests/test_conv_epilogue_model.py:
  - the gate activations measured over every 22-bit-significand value of 2^-24 .. 2^8 (both signs), through the epilogues
    that ship (SIGMOID, TANH_RELU's tanh half, GRU_Q with z = 1, h = 0), on the tensor cores and on the exact engine;
  - every epilogue stage of the update block in real test-mode forwards, checked on the call's own input planes with the
    engine's own packs;
  - a synthetic stress of each epilogue form: saturating and flushed gates, tanh across +-0.25, h over 2^-20 .. 2^4 with
    zeros, z within 1e-6 of 0 and 1, residuals that cancel, both aux layouts, NaN-filled outputs that must stay NaN outside
    the written pixels and channels;
  - a coverage guard over the epilogue forms the forwards launch."""
import math

import pytest
import torch

from conftest import build_model
from test_conv_epilogue_model import (E_SIG, E_SIG_EXACT, E_TANH, E_TANH_EXACT, FTZ, act64, act_err, check_act,
                                      check_gru_q, check_gru_zr, check_relu_add_relu, check_relu_flow, check_tanh_relu,
                                      pre_ffma, pre_umma)
from test_conv_error_model import conv_split_ref, split_emulate
from test_gpu_product_shapes import Recorder, run_forward
from test_product_shapes import SHAPES, blocked_index, cl, tiles, unblock

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WORST = {}


def note(key, w):
    WORST[key] = max(WORST.get(key, 0.0), w)


@pytest.fixture(scope="module")
def ueng():
    from rnc.engine_umma import UmmaEngine
    return UmmaEngine()


def nchw(t2d, B, H, W, c0=0, c1=None):
    return cl(t2d[:B * H * W, c0:c1], B, H, W)


def nan_buf(rows, ld, dtype=torch.float32):
    return torch.full((rows, ld), math.nan, dtype=dtype, device=DEV)


def ffma_conv(x2d, c0, ld0, w, b, epi, out=None, ldo=0, B=1, H=1, W=1, in1=None, c1=0, ld1=0, h=None, ldh=0, aux0=None,
              ldaux=0):
    """One rnc_conv2d_cl_fwd launch of weight w [cout, cin, kh, kw] (packed as rnc.engine.pack_conv)."""
    from rnc import native
    from rnc.engine import pack_conv
    pw, pb = pack_conv(w.to(DEV), None if b is None else b.to(DEV))
    d = native.ConvDesc()
    d.in0, d.c0, d.ld0 = x2d.data_ptr(), c0, ld0
    d.in1, d.c1, d.ld1 = (in1.data_ptr() if in1 is not None else 0), c1, ld1
    d.weight, d.bias = pw.data_ptr(), pb.data_ptr()
    d.out, d.ldo = (out.data_ptr() if out is not None else 0), ldo
    d.h, d.ldh = (h.data_ptr() if h is not None else 0), ldh
    d.aux0, d.ldaux = (aux0.data_ptr() if aux0 is not None else 0), ldaux
    d.B, d.H, d.W = B, H, W
    d.cout, d.kh, d.kw, d.epilogue = w.shape[0], w.shape[2], w.shape[3], epi
    native.rnc.conv2d_cl_fwd(d)


# ----------------------------------------------------------------------------------------------------------- activations
SWEEP_BINADES = (-24, 7)        # every binade [2^e, 2^(e+1)) for e in this range


def binade_values(e_lo, e_hi):
    """Every fp32 value with a 22-bit significand in the binades 2^e_lo .. 2^e_hi, both signs: [binade][sign][2^21]."""
    m = torch.arange(1 << 21, device=DEV, dtype=torch.float32) + float(1 << 21)         # 22-bit integers, exact in fp32
    out = [s * m * 2.0 ** (e - 21) for e in range(e_lo, e_hi + 1) for s in (1.0, -1.0)]
    return torch.cat(out)


def measure(what, kind, v, got, exact, e_lo):
    """Per-binade worst relative error, the 0.25 branch and the flushed region; checks err <= E_act(v) everywhere."""
    ref = act64(kind, v)
    err = (got.double() - ref).abs()
    bound = act_err(kind, v, 0.0, exact)
    ratio = float((err / bound).max())
    normal = ref.abs() >= FTZ
    rel = torch.where(normal, err / ref.abs().clamp_min(1e-300), torch.zeros_like(err))
    nb = rel.numel() // (2 << 21)
    per = rel.view(nb, 2 << 21).amax(1).tolist()
    lin = torch.where(v.abs() >= 1, rel / v.abs().double(), torch.zeros_like(rel))
    print(f"  {what}: worst err/bound {ratio:.3f}; max rel err {max(per):.3e}, max rel err / |v| (|v| >= 1) "
          f"{float(lin.max()):.3e}")
    print("    per binade (2^e: max rel err): " + ", ".join(f"{e_lo + i}: {r:.2e}" for i, r in enumerate(per)))
    av = v.abs()
    for lo, hi in ((0.2, 0.25), (0.25, 0.3)):
        sel = (av >= lo) & (av < hi)
        if sel.any():
            print(f"    |v| in [{lo}, {hi}): max rel err {float(rel[sel].max()):.3e}")
    if kind == "sigmoid":
        zero = got == 0
        if zero.any():
            print(f"    flushed to 0 for v <= {float(v[zero].max()):.4f}; smallest v with a non-zero result "
                  f"{float(v[~zero].min()):.4f}; worst error there {float(err[zero].max()):.2e} (2^-126 = {FTZ:.2e})")
    note(what, ratio)
    assert ratio <= 1.0, f"{what}: the measured error exceeds E_act (worst err/bound {ratio:.3f})"
    return rel


def test_activation_sweep_umma(ueng):
    """A 1x1 layer of weight 2^k I over 64 channels: the pre-activation is exactly 2^k (hi + lo) (the LINEAR output is
    checked to be exactly the swept value), and SIGMOID, TANH_RELU's tanh half and GRU_Q with z = 1, h = 0 evaluate the
    device functions on it.  GRU_Q must return TANH_RELU's tanh bit for bit; TANH_RELU's split must be split_pair of its
    fp32 half, its relu half exact, and nothing written beyond the tanh half of the fp32 output."""
    from rnc import native
    from rnc.engine_umma import UmmaWeights
    sig, tnh, vals = [], [], []
    # (k, binades of v): the input 2^-k v lies in 2^-3 .. 2^15, where a 22-bit value is exactly hi + lo
    for k, (e_lo, e_hi) in ((-21, (-24, -7)), (-3, (-6, SWEEP_BINADES[1]))):
        v = binade_values(e_lo, e_hi)
        P = v.numel() // 64
        W = 1024
        H = P // W
        x = (v * 2.0 ** -k).view(P, 64)
        hi, lo = split_emulate(x)
        assert torch.equal(hi.float() + lo.float(), x)
        eye = torch.eye(64, device=DEV).view(64, 64, 1, 1) * 2.0 ** k
        pk = UmmaWeights(eye, None, [64])
        pk2 = UmmaWeights(torch.cat([eye, eye]), None, [64])
        planes = (hi.data_ptr(), lo.data_ptr())
        out = nan_buf(P, 64)
        ueng.uconv(1, H, W, planes, 64, 64, pk, native.EPI_LINEAR, out_f32=out.data_ptr(), ldo_f32=64, flags=0)
        torch.cuda.synchronize()
        assert torch.equal(out.view(-1), v), "the 2^k I layer's LINEAR output is not exactly the swept value"
        ueng.uconv(1, H, W, planes, 64, 64, pk, native.EPI_SIGMOID, out_f32=out.data_ptr(), ldo_f32=64, flags=0)
        s = out.clone()
        o2 = nan_buf(P, 128)
        sh, sl = nan_buf(P, 128, torch.float16), nan_buf(P, 128, torch.float16)
        ueng.uconv(1, H, W, planes, 64, 64, pk2, native.EPI_TANH_RELU, out_f32=o2.data_ptr(), ldo_f32=128,
                   out_split=(sh.data_ptr(), sl.data_ptr()), ldo_split=128, flags=0)
        z = torch.ones(P, 64, device=DEV)
        hq = torch.zeros(P, 64, device=DEV)
        ueng.uconv(1, H, W, planes, 64, 64, pk, native.EPI_GRU_Q, h=hq.data_ptr(), ldh=64, aux0=z.data_ptr(), ldaux=64,
                   flags=0)
        torch.cuda.synchronize()
        t = o2[:, :64]
        assert torch.isnan(o2[:, 64:]).all(), "TANH_RELU wrote fp32 outputs beyond its tanh half"
        assert torch.equal(hq, t), "GRU_Q with z = 1, h = 0 differs from TANH_RELU's tanh"
        eh, el = split_emulate(t)
        assert torch.equal(sh[:, :64], eh) and torch.equal(sl[:, :64], el), "TANH_RELU: split != split_pair(tanh)"
        rh, rl = split_emulate(x.clamp_min(0) * 2.0 ** k)
        assert torch.equal(sh[:, 64:], rh) and torch.equal(sl[:, 64:], rl), "TANH_RELU: relu half"
        sig.append(s.view(-1))
        tnh.append(t.reshape(-1))
        vals.append(v)
        del out, o2, sh, sl, hq, z, hi, lo, x
    v = torch.cat(vals)
    print(f"tensor-core epilogues: E_SIG {E_SIG}, E_TANH {E_TANH}")
    measure("sigmoid_fast (EPI_SIGMOID)", "sigmoid", v, torch.cat(sig), False, SWEEP_BINADES[0])
    measure("tanh_fast (EPI_TANH_RELU, EPI_GRU_Q)", "tanh", v, torch.cat(tnh), False, SWEEP_BINADES[0])


def test_activation_sweep_ffma():
    """The exact engine's 1 / (1 + expf(-x)) (EPI_SIGMOID and the GRU_ZR gates) and tanhf (EPI_GRU_Q with z = 1, h = 0)
    over the same values, through rnc_conv2d_cl_fwd with an identity 1x1 layer (its LINEAR output is the value, exactly)."""
    from rnc import native
    v = binade_values(*SWEEP_BINADES)
    P = v.numel() // 64
    W = 1024
    H = P // W
    x = v.view(P, 64)
    eye = torch.eye(64).view(64, 64, 1, 1)
    out = nan_buf(P, 64)
    ffma_conv(x, 64, 64, eye, None, native.EPI_LINEAR, out, 64, 1, H, W)
    torch.cuda.synchronize()
    assert torch.equal(out, x), "the identity layer's LINEAR output is not exactly the swept value"
    ffma_conv(x, 64, 64, eye, None, native.EPI_SIGMOID, out, 64, 1, H, W)
    z = torch.ones(P, 64, device=DEV)
    hq = torch.zeros(P, 64, device=DEV)
    ffma_conv(x, 64, 64, eye, None, native.EPI_GRU_Q, None, 0, 1, H, W, h=hq, ldh=64, aux0=z, ldaux=64)
    torch.cuda.synchronize()
    print(f"exact engine: E_SIG_EXACT {E_SIG_EXACT}, E_TANH_EXACT {E_TANH_EXACT}")
    measure("1/(1+expf(-x)) (exact EPI_SIGMOID)", "sigmoid", v, out.view(-1), True, SWEEP_BINADES[0])
    measure("tanhf (exact EPI_GRU_Q)", "tanh", v, hq.view(-1), True, SWEEP_BINADES[0])


# ----------------------------------------------------------------------------------------------------------- product launches
def _w_ffma(packed, cout, kh, kw):
    w, b = packed
    cin = w.shape[1]
    return w.view(kh, kw, cin, -1).permute(3, 2, 0, 1)[:cout], b[:cout]


class EpilogueRecorder(Recorder):
    """Recorder (tests/test_gpu_product_shapes.py) that checks every epilogue stage of the update block against the
    epilogue model, on the call's own input planes and the engine's own packs."""

    def __init__(self, monkeypatch, model, eng, B, H8, W8, check=True, tag=""):
        super().__init__(monkeypatch, model, eng, B, H8, W8, check=False, tag=tag)
        self.last = None
        self.snap = {}
        self.checked = set()
        name = "uconv" if self.umma else "conv"
        inner = getattr(eng, name)

        def capture(*a, **kw):
            self.last = (a, kw)
            return inner(*a, **kw)
        monkeypatch.setattr(eng, name, capture)

    def stage(self, st, when, args, out=None):
        super().stage(st, when, args, out)
        if when == "before" and st in ("q1", "q2"):
            self.snap["h_old"] = self.h32().clone()
        if when == "post" and st in EPILOGUE_STAGES:
            (self.check_umma if self.umma else self.check_ffma)(st)
            self.checked.add(st)

    # ---------------------------------------------------------------- readers
    def pl(self, buf, c0, c1):
        return nchw(buf.hi, self.B, self.H, self.W, c0, c1), nchw(buf.lo, self.B, self.H, self.W, c0, c1)

    def f(self, t, c0=0, c1=None):
        return nchw(t, self.B, self.H, self.W, c0, c1)

    def flow32(self):
        return self.ws.coords1 - self.grid.float()

    def blocked_read(self, buf, ld, C, kh, kw):
        return unblock(buf, ld, C, kh, kw, self.B, self.H, self.W)

    def check_umma(self, st):
        ws, tag = self.ws, f"{self.tag} {st}"
        a, kw = self.last
        wt = a[6]
        cat = lambda p, q: (torch.cat([p[0], q[0]], 1), torch.cat([p[1], q[1]], 1))     # noqa: E731
        relu_io = {"convc1": (ws.corr, 0, 352, ws.c1, 0), "convc2": (ws.c1, 0, 256, ws.corflo, 0),
                   "convf2": (ws.f1, 0, 128, ws.corflo, 192), "fh1": (ws.hx, 0, 128, ws.fh, 0)}
        if st == "m0":
            relu_io["m0"] = (ws.hx, 0, 128, ws.mh, 0)
        if st in relu_io:
            src, c0, c1, dst, o0 = relu_io[st]
            s = conv_split_ref(self.pl(src, c0, c1), wt)
            w = check_act(tag, "relu", pre_umma(s), split=self.pl(dst, o0, o0 + wt.cout))
        elif st == "conv":
            s = conv_split_ref(self.pl(ws.corflo, 0, 256), wt)
            w = check_relu_flow(tag, pre_umma(s), self.pl(ws.hx, 256, 256 + wt.cout + 2), self.flow32())
        elif st == "m2":
            s = conv_split_ref(self.pl(ws.mh, 0, 256), wt)
            w = check_act(tag, "linear", pre_umma(s), f32=self.f(ws.mask, 0, wt.cout))
        elif st in ("czr1", "cq1", "czr2", "cq2"):
            kh, kw_ = (1, 5) if st[-1] == "1" else (5, 1)
            s = conv_split_ref(self.pl(ws.hx, 128, 256), wt)
            got = self.f(self.blocked_read(getattr(ws, st), wt.coutpad, wt.coutpad, kh, kw_), 0, wt.cout)
            w = check_act(tag, "linear", pre_umma(s), f32=got)
        elif st in ("zr1", "zr2"):
            kh, kw_ = (1, 5) if st[-1] == "1" else (5, 1)
            s = conv_split_ref(cat(self.pl(ws.hx, 0, 128), self.pl(ws.hx, 256, 384)), wt, [128, 128])
            add = self.f(self.blocked_read(getattr(ws, "czr" + st[-1]), 256, 256, kh, kw_))
            w = check_gru_zr(tag, pre_umma(s, add), self.zgate(kh, kw_), self.pl(ws.rh, 0, 128), self.f(ws.h))
        elif st in ("q1", "q2"):
            kh, kw_ = (1, 5) if st[-1] == "1" else (5, 1)
            s = conv_split_ref(cat(self.pl(ws.rh, 0, 128), self.pl(ws.hx, 256, 384)), wt, [128, 128])
            add = self.f(self.blocked_read(getattr(ws, "cq" + st[-1]), 128, 128, kh, kw_))
            w = check_gru_q(tag, pre_umma(s, add), self.zgate(kh, kw_), self.f(self.snap.pop("h_old")), self.f(ws.h),
                            hx=self.pl(ws.hx, 0, 128))
        note(f"product {st} ({'umma' if self.umma else 'ffma'})", w)

    def check_ffma(self, st):
        ws, tag = self.ws, f"{self.tag} {st}"
        a, kw = self.last
        B_, H_, W_, in0, c0, ld0, packed, cout, kh, kw_ = a[:10]
        w, b = _w_ffma(packed, cout, kh, kw_)
        relu_io = {"convc1": (ws.corr, 0, 324, ws.c1, 0), "convc2": (ws.c1, 0, 256, ws.corflo, 0),
                   "convf2": (ws.f1, 0, 128, ws.corflo, 192), "fh1": (ws.hx, 0, 128, ws.fh, 0)}
        if st == "m0":
            relu_io["m0"] = (ws.hx, 0, 128, ws.mh, 0)
        if st in relu_io:
            src, c0_, c1_, dst, o0 = relu_io[st]
            pre = pre_ffma(self.f(src, c0_, c1_), w, b)
            r = check_act(tag, "relu", pre, f32=self.f(dst, o0, o0 + cout), exact=True)
        elif st == "m2":
            r = check_act(tag, "linear", pre_ffma(self.f(ws.mh, 0, 256), w, b), f32=self.f(ws.mask, 0, cout), exact=True)
        elif st == "conv":
            pre = pre_ffma(self.f(ws.corflo, 0, 256), w, b)
            r = check_relu_flow(tag, pre, self.f(ws.hx, 256, 256 + cout + 2), self.flow32(), exact=True)
        elif st in ("zr1", "zr2"):
            pre = pre_ffma(self.f(ws.hx, 0, 384), w, b)
            r = check_gru_zr(tag, pre, self.f(ws.z, 0, 128), self.f(ws.rh, 0, 128), self.f(ws.hx, 0, 128), exact=True)
        elif st in ("q1", "q2"):
            x = torch.cat([self.f(ws.rh, 0, 128), self.f(ws.hx, 128, 384)], 1)
            r = check_gru_q(tag, pre_ffma(x, w, b), self.f(ws.z, 0, 128), self.f(self.snap.pop("h_old")),
                            self.f(ws.hx, 0, 128), exact=True)
        else:
            return
        note(f"product {st} (ffma)", r)


EPILOGUE_STAGES = ("convc1", "convc2", "convf2", "conv", "czr1", "cq1", "czr2", "cq2", "zr1", "q1", "zr2", "q2", "fh1", "m0", "m2")
PRODUCT_CASES = ([("umma", m, s) for m in ("raft_nc_dbl", "raft") for s in SHAPES]
                 + [("ffma", m, s) for m in ("raft_nc_dbl", "raft") for s in ("S1", "S2")])


@pytest.mark.parametrize("cfg,model_name,sid", PRODUCT_CASES, ids=[f"{s}-{c}-{m}" for c, m, s in PRODUCT_CASES])
def test_product_epilogues(cfg, model_name, sid, monkeypatch):
    """Two iterations of a test-mode forward; every epilogue stage of the update block against the epilogue model on the
    call's own inputs (teacher forcing) and the engine's packs: relu layers, conv + flow append, the hoisted context
    addends (read back from their layout), z and r*h, the blended h and its split copy, the mask head's first layer."""
    import test_gpu_product_shapes as tps
    monkeypatch.setattr(tps, "Recorder", EpilogueRecorder)
    rec, *_ = run_forward(monkeypatch, cfg, model_name, sid)
    want = set(EPILOGUE_STAGES) - ({"m0", "m2"} if model_name == "raft_nc_dbl" else set())
    if cfg == "ffma":
        want -= {"czr1", "cq1", "czr2", "cq2"}
    assert rec.checked == want, f"stages not checked: {sorted(want - rec.checked)}"


# ----------------------------------------------------------------------------------------------------------- stress
GEOS = {"S2": (2, 47, 156), "S4": (3, 8, 12)}
BIAS_SET = [-95.0, -88.0, -60.0, -20.0, -5.0, 0.0, 0.0, 0.0, 0.25, -0.25, 5.0, 20.0, 30.0]


def _stim(B, H, W, C, g, scale=1.0):
    return (torch.randn(B, C, H, W, generator=g) * scale).to(DEV)


def _gates(shape, g):
    """Pre-activation offsets: a quarter below -87.3 (flushed gates), a quarter in [-30, 30], the rest 0 (the layer's own
    values, dense across +-0.25)."""
    u = torch.rand(shape, generator=g)
    off = torch.where(u < 0.25, -88.0 - 12 * torch.rand(shape, generator=g),
                      torch.where(u < 0.5, 60 * torch.rand(shape, generator=g) - 30, torch.zeros(shape)))
    return off.to(DEV)


def _h_state(shape, g):
    h = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0) * 2.0 ** (24 * torch.rand(shape, generator=g) - 20)
    h[torch.rand(shape, generator=g) < 0.05] = 0.0
    return h.float().to(DEV)


def _z_gate(shape, g):
    u = torch.rand(shape, generator=g)
    e = torch.rand(shape, generator=g) * 1e-6
    z = torch.where(u < 0.3, e, torch.where(u < 0.6, 1 - e, torch.rand(shape, generator=g)))
    z[u > 0.98] = 0.0
    z[(u > 0.96) & (u <= 0.98)] = 1.0
    return z.float().to(DEV)


def _to_cl(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1]).contiguous()


def _block(t_cl, ld, kh, kw, B, H, W):
    """Channel-last [M, C] -> a NaN-filled tile-blocked buffer (ld channels per tile) holding it."""
    tile, row = blocked_index(kh, kw, B, H, W)
    n = tiles(kh, kw, B, H, W)
    buf = torch.full((n * ld * 128,), math.nan, device=DEV)
    C = t_cl.shape[1]
    idx = (tile.to(DEV)[:, None] * ld + torch.arange(C, device=DEV)[None, :]) * 128 + row.to(DEV)[:, None]
    buf[idx.reshape(-1)] = t_cl.reshape(-1)
    return buf, idx


def _splitbuf(x_nchw, extra=0):
    hi, lo = split_emulate(_to_cl(x_nchw))
    if extra:
        hi, lo = (torch.nn.functional.pad(t, (0, extra)).contiguous() for t in (hi, lo))
    return hi, lo


STRESS = ["relu", "sigmoid", "linear-blocked", "relu-flow", "relu-add-relu", "tanh-relu", "gru-zr-blocked",
          "gru-zr-channel-last", "gru-q-blocked", "gru-q-channel-last"]


@pytest.mark.parametrize("geo", list(GEOS))
@pytest.mark.parametrize("form", STRESS)
def test_epilogue_stress_umma(ueng, form, geo):
    """One tensor-core launch of the epilogue form on synthetic stimuli (see _gates, _h_state, _z_gate), NaN-filled outputs:
    rows beyond the image and channels beyond the written width must stay NaN (the appended flow channels excepted)."""
    from rnc import native
    from rnc.engine_umma import UmmaWeights
    B, H, W = GEOS[geo]
    M = B * H * W
    g = torch.Generator().manual_seed(len(form) * 7 + H)
    gru = form.startswith("gru")
    blocked = form.endswith("-blocked")
    kh, kw = ((1, 5) if geo == "S2" else (5, 1)) if gru else (3, 3)
    segs = [128, 128] if gru else [96]
    cin = sum(segs)
    cout = {"relu": 96, "sigmoid": 96, "linear-blocked": 128, "relu-flow": 126, "relu-add-relu": 64, "tanh-relu": 128,
            "gru-zr-blocked": 256, "gru-zr-channel-last": 256, "gru-q-blocked": 128, "gru-q-channel-last": 128}[form]
    x = _stim(B, H, W, cin, g)
    w = torch.randn(cout, cin, kh, kw, generator=g) * (0.5 / (cin * kh * kw) ** 0.5)
    bias = None if gru else torch.tensor([BIAS_SET[c % len(BIAS_SET)] for c in range(cout)])
    pk = UmmaWeights(w.to(DEV), None if bias is None else bias.to(DEV), segs, extra_cout=2 if form == "relu-flow" else 0)
    flags = native.CONV_AUX_BLOCKED if blocked else 0
    if gru:
        hi0, lo0 = _splitbuf(x[:, :128])
        hi1, lo1 = _splitbuf(x[:, 128:])
        kwa = dict(in1=(hi1.data_ptr(), lo1.data_ptr()), c1=128, ld1=128)
        planes = (torch.cat([cl(hi0, B, H, W), cl(hi1, B, H, W)], 1), torch.cat([cl(lo0, B, H, W), cl(lo1, B, H, W)], 1))
    else:
        hi0, lo0 = _splitbuf(x)
        kwa = {}
        planes = (cl(hi0, B, H, W), cl(lo0, B, H, W))
    in0 = (hi0.data_ptr(), lo0.data_ptr())
    s = conv_split_ref(planes, pk, segs)
    rows = M + 256
    tag = f"[stress {form} {geo}]"
    if gru:
        add = _gates((B, cout, H, W), g)
        add_cl = _to_cl(add)
        if blocked:
            add_buf, _ = _block(add_cl, pk.coutpad, kh, kw, B, H, W)
        else:
            add_buf = add_cl
        pre = pre_umma(s, add)
        C = cout if form.startswith("gru-q") else cout // 2
        h = _h_state((B, C, H, W), g)
        h_cl = _to_cl(h)
        sh, sl = nan_buf(rows, 136, torch.float16), nan_buf(rows, 136, torch.float16)
        if form.startswith("gru-zr"):
            zbuf = (torch.full((tiles(kh, kw, B, H, W) * 128 * 128,), math.nan, device=DEV) if blocked
                    else nan_buf(rows, 128))
            ueng.uconv(B, H, W, in0, 128, 128, pk, native.EPI_GRU_ZR, out_split=(sh.data_ptr(), sl.data_ptr()),
                       ldo_split=136, h=h_cl.data_ptr(), ldh=C, aux0=zbuf.data_ptr(), ldaux=128, add=add_buf.data_ptr(),
                       ldadd=pk.coutpad, flags=flags, **kwa)
            torch.cuda.synchronize()
            z = unblock(zbuf, 128, 128, kh, kw, B, H, W) if blocked else zbuf[:M]
            assert int(torch.isfinite(zbuf).sum()) == M * 128, "GRU_ZR wrote z outside the image's pixels"
            w_ = check_gru_zr(tag, pre, nchw(z, B, H, W), (nchw(sh, B, H, W, 0, C), nchw(sl, B, H, W, 0, C)), h)
            assert torch.isnan(sh[M:]).all() and torch.isnan(sh[:, C:]).all(), "GRU_ZR wrote r*h beyond its pixels / channels"
        else:
            z = _z_gate((B, C, H, W), g)
            z_cl = _to_cl(z)
            zbuf = _block(z_cl, 128, kh, kw, B, H, W)[0] if blocked else z_cl
            hbuf = torch.cat([h_cl, torch.full((256, C), math.nan, device=DEV)])
            ueng.uconv(B, H, W, in0, 128, 128, pk, native.EPI_GRU_Q, out_split=(sh.data_ptr(), sl.data_ptr()),
                       ldo_split=136, h=hbuf.data_ptr(), ldh=C, aux0=zbuf.data_ptr(), ldaux=128, add=add_buf.data_ptr(),
                       ldadd=pk.coutpad, flags=flags, **kwa)
            torch.cuda.synchronize()
            w_ = check_gru_q(tag, pre, z, h, nchw(hbuf, B, H, W), hx=(nchw(sh, B, H, W, 0, C), nchw(sl, B, H, W, 0, C)))
            assert torch.isnan(hbuf[M:]).all() and torch.isnan(sh[M:]).all() and torch.isnan(sh[:, C:]).all()
        note(f"stress {form}", w_)
        return
    pre = pre_umma(s)
    sh, sl = nan_buf(rows, 136, torch.float16), nan_buf(rows, 136, torch.float16)
    f32 = nan_buf(rows, 128)
    split = (sh.data_ptr(), sl.data_ptr())
    ch32 = lambda c0, c1: nchw(f32, B, H, W, c0, c1)                                          # noqa: E731
    chs = lambda c0, c1: (nchw(sh, B, H, W, c0, c1), nchw(sl, B, H, W, c0, c1))              # noqa: E731
    if form in ("relu", "sigmoid"):
        epi = native.EPI_RELU if form == "relu" else native.EPI_SIGMOID
        ueng.uconv(B, H, W, in0, 96, 96, pk, epi, out_f32=f32.data_ptr(), ldo_f32=128, out_split=split, ldo_split=136,
                   flags=0)
        torch.cuda.synchronize()
        w_ = check_act(tag, form, pre, f32=ch32(0, 96), split=chs(0, 96))
        width = 96
    elif form == "linear-blocked":
        ob = torch.full((tiles(kh, kw, B, H, W) * 128 * 128,), math.nan, device=DEV)
        ueng.uconv(B, H, W, in0, 96, 96, pk, native.EPI_LINEAR, out_f32=ob.data_ptr(), ldo_f32=128,
                   flags=native.CONV_OUT_BLOCKED)
        torch.cuda.synchronize()
        assert int(torch.isfinite(ob).sum()) == M * 128, "the blocked output was written outside the image's pixels"
        w_ = check_act(tag, "linear", pre, f32=nchw(unblock(ob, 128, 128, kh, kw, B, H, W), B, H, W))
        note(f"stress {form}", w_)
        return
    elif form == "relu-flow":
        yy, xx = torch.meshgrid(torch.arange(H, device=DEV).float(), torch.arange(W, device=DEV).float(), indexing="ij")
        coords = torch.stack([xx, yy])[None] + (torch.randn(B, 2, H, W, generator=g) * 40).to(DEV)
        ueng.uconv(B, H, W, in0, 96, 96, pk, native.EPI_RELU_FLOW, out_split=split, ldo_split=136,
                   aux0=coords.data_ptr(), flags=0)
        torch.cuda.synchronize()
        flow = coords - torch.stack([xx, yy])[None]
        w_ = check_relu_flow(tag, pre, chs(0, 128), flow)
        width = 128
    elif form == "relu-add-relu":
        r = pre.v.clamp_min(0)
        res = torch.where(torch.rand(r.shape, generator=g).to(DEV) < 0.5,
                          -r * (1 + 1e-3 * torch.randn(r.shape, generator=g).to(DEV)), _stim(B, H, W, 64, g, 3.0).double())
        res = res.float()
        res_cl = _to_cl(res)
        ueng.uconv(B, H, W, in0, 96, 96, pk, native.EPI_RELU_ADD_RELU, out_f32=f32.data_ptr(), ldo_f32=128,
                   out_split=split, ldo_split=136, res=res_cl.data_ptr(), ldres=64, flags=0)
        torch.cuda.synchronize()
        w_ = check_relu_add_relu(tag, pre, res, f32=ch32(0, 64), split=chs(0, 64))
        width = 64
    else:   # tanh-relu
        ueng.uconv(B, H, W, in0, 96, 96, pk, native.EPI_TANH_RELU, out_f32=f32.data_ptr(), ldo_f32=128, out_split=split,
                   ldo_split=136, flags=0)
        torch.cuda.synchronize()
        w_ = check_tanh_relu(tag, pre, ch32(0, 64), chs(0, 128))
        assert torch.isnan(f32[:, 64:]).all(), "TANH_RELU wrote fp32 outputs beyond its tanh half"
        width = 128
    assert torch.isnan(sh[M:]).all() and torch.isnan(f32[M:]).all(), "outputs written beyond the image's pixels"
    assert torch.isnan(sh[:, width:]).all(), "split outputs written beyond the layer's channels"
    if form != "tanh-relu" and form != "relu-flow":
        assert torch.isnan(f32[:, width:]).all(), "fp32 outputs written beyond the layer's channels"
    note(f"stress {form}", w_)


@pytest.mark.parametrize("form", ["sigmoid", "relu-flow", "gru-zr", "gru-q"])
def test_epilogue_stress_ffma(form):
    """The exact engine's epilogues on the same kind of stimuli (fp32 operands, one segment or two)."""
    from rnc import native
    B, H, W = GEOS["S2"]
    M = B * H * W
    g = torch.Generator().manual_seed(len(form))
    gru = form.startswith("gru")
    kh, kw = (1, 5) if gru else (3, 3)
    cin = 256 if gru else 96
    cout = {"sigmoid": 96, "relu-flow": 126, "gru-zr": 256, "gru-q": 128}[form]
    x = _stim(B, H, W, cin, g)
    w = torch.randn(cout, cin, kh, kw, generator=g) * (0.5 / (cin * kh * kw) ** 0.5)
    b = torch.tensor([BIAS_SET[c % len(BIAS_SET)] for c in range(cout)])
    if gru:
        b = b + 30 * torch.rand(cout, generator=g) - 15
    pre = pre_ffma(x, w, b)
    tag = f"[stress exact {form}]"
    x0, x1 = _to_cl(x[:, :128] if gru else x), (_to_cl(x[:, 128:]) if gru else None)
    two = dict(in1=x1, c1=128, ld1=128) if gru else {}
    c0 = 128 if gru else 96
    if form == "sigmoid":
        out = nan_buf(M, 128)
        ffma_conv(x0, c0, c0, w, b, native.EPI_SIGMOID, out, 128, B, H, W)
        torch.cuda.synchronize()
        w_ = check_act(tag, "sigmoid", pre, f32=nchw(out, B, H, W, 0, cout), exact=True)
        assert torch.isnan(out[:, cout:]).all()
    elif form == "relu-flow":
        yy, xx = torch.meshgrid(torch.arange(H, device=DEV).float(), torch.arange(W, device=DEV).float(), indexing="ij")
        coords = torch.stack([xx, yy])[None] + (torch.randn(B, 2, H, W, generator=g) * 40).to(DEV)
        out = nan_buf(M, 136)
        ffma_conv(x0, c0, c0, w, b, native.EPI_RELU_FLOW, out, 136, B, H, W, aux0=coords)
        torch.cuda.synchronize()
        w_ = check_relu_flow(tag, pre, nchw(out, B, H, W, 0, cout + 2), coords - torch.stack([xx, yy])[None], exact=True)
        assert torch.isnan(out[:, cout + 2:]).all()
    elif form == "gru-zr":
        C = cout // 2
        h = _h_state((B, C, H, W), g)
        out, z = nan_buf(M, 128), nan_buf(M, 128)
        ffma_conv(x0, c0, c0, w, b, native.EPI_GRU_ZR, out, 128, B, H, W, h=_to_cl(h), ldh=C, aux0=z, ldaux=128, **two)
        torch.cuda.synchronize()
        w_ = check_gru_zr(tag, pre, nchw(z, B, H, W), nchw(out, B, H, W), h, exact=True)
    else:
        h = _h_state((B, cout, H, W), g)
        z = _z_gate((B, cout, H, W), g)
        hb = _to_cl(h)
        ffma_conv(x0, c0, c0, w, b, native.EPI_GRU_Q, None, 0, B, H, W, h=hb, ldh=cout, aux0=_to_cl(z), ldaux=cout, **two)
        torch.cuda.synchronize()
        w_ = check_gru_q(tag, pre, z, h, nchw(hb, B, H, W), exact=True)
    note(f"stress exact {form}", w_)


# ----------------------------------------------------------------------------------------------------------- coverage
# Every epilogue form (engine, epilogue, aux blocked, out blocked, add, h, res, fp32 out, split out) the forwards launch in
# test mode (both models, S1, on umma and ffma) -> the test that checks it against the model.
P, ST, SWP = "test_product_epilogues", "test_epilogue_stress", "test_activation_sweep"
_ERR = "test_gpu_conv_error_model.py (every launch signature, LINEAR fp32)"
EPILOGUE_COVERAGE = {
    ("umma", 0, False, False, False, False, False, True, False): f"{_ERR}; {P}: m2",
    ("umma", 0, False, True, False, False, False, True, False): f"{P}: czr1/cq1/czr2/cq2; {ST}_umma[linear-blocked]",
    ("umma", 1, False, False, False, False, False, False, True): f"{P}: convc1, convc2, convf2, fh1, m0; {ST}_umma[relu]",
    ("umma", 1, False, False, False, False, False, True, False): f"{ST}_umma[relu] (fp32 and split)",
    ("umma", 1, False, False, False, False, False, True, True): f"{ST}_umma[relu] (fp32 and split)",
    ("umma", 3, True, False, True, True, False, False, True): f"{P}[*-umma-*]: zr1, zr2; {ST}_umma[gru-zr-blocked]",
    ("umma", 4, True, False, True, True, False, False, True): f"{P}[*-umma-*]: q1, q2; {ST}_umma[gru-q-blocked]",
    ("umma", 5, False, False, False, False, False, False, True): f"{P}: conv; {ST}_umma[relu-flow]",
    ("umma", 6, False, False, False, False, True, False, True): f"{ST}_umma[relu-add-relu]",
    ("umma", 6, False, False, False, False, True, True, True): f"{ST}_umma[relu-add-relu]",
    ("umma", 7, False, False, False, False, False, True, True): f"{SWP}_umma; {ST}_umma[tanh-relu]",
    ("ffma", 0, False, False, False, False, False, True, False): f"{P}[*-ffma-raft]: m2",
    ("ffma", 1, False, False, False, False, False, True, False): f"{P}[*-ffma-*]: convc1, convc2, convf2, fh1, m0",
    ("ffma", 3, False, False, False, True, False, True, False): f"{P}[*-ffma-*]: zr1, zr2; {ST}_ffma[gru-zr]",
    ("ffma", 4, False, False, False, True, False, False, False): f"{P}[*-ffma-*]: q1, q2; {SWP}_ffma; {ST}_ffma[gru-q]",
    ("ffma", 5, False, False, False, False, False, True, False): f"{P}[*-ffma-*]: conv; {ST}_ffma[relu-flow]",
}


def _form(engine, epi, flags, kw):
    from rnc import native
    nz = lambda k: bool(kw.get(k)) and kw.get(k) != (0, 0)                                  # noqa: E731
    if engine == "umma":
        return ("umma", epi, bool(flags & native.CONV_AUX_BLOCKED), bool(flags & native.CONV_OUT_BLOCKED), nz("add"),
                nz("h"), nz("res"), nz("out_f32"), nz("out_split"))
    return ("ffma", epi, False, False, False, nz("h"), False, nz("out"), False)


def test_epilogue_coverage_guard(monkeypatch):
    """The epilogue forms of test-mode forwards of both models at S1 on umma and ffma are exactly the
    table's: a form added to an engine fails here until it has a check."""
    seen = {}
    for cfg, env in (("umma", {}), ("ffma", {"RNC_CONV": "ffma"})):
        for name in ("raft_nc_dbl", "raft"):
            with monkeypatch.context() as mp:
                for k, v in env.items():
                    mp.setenv(k, v)
                mp.setenv("RNC_GRAPH", "0")
                m = build_model(name).to(DEV)
                eng = m.engine()
                if eng.mode == "umma":
                    orig = eng.uconv

                    def uconv(B, H, W, in0, c0, ld0, wt, epi, _o=orig, **kw):
                        seen.setdefault(_form("umma", epi, kw.get("flags", 0), kw), cfg)
                        return _o(B, H, W, in0, c0, ld0, wt, epi, **kw)
                    mp.setattr(eng, "uconv", uconv)
                else:
                    orig = eng.conv

                    def conv(B, H, W, in0, c0, ld0, packed, cout, kh, kw_, epi, out=None, ldo=0, _o=orig, **kw):
                        seen.setdefault(_form("ffma", epi, 0, dict(kw, out=out)), cfg)
                        return _o(B, H, W, in0, c0, ld0, packed, cout, kh, kw_, epi, out, ldo, **kw)
                    mp.setattr(eng, "conv", conv)
                Bs, H8, W8 = SHAPES["S1"]
                gen = torch.Generator().manual_seed(1)
                im1, im2 = (torch.rand(Bs, 3, 8 * H8, 8 * W8, generator=gen) * 255 for _ in range(2))
                with torch.no_grad():
                    m(im1.to(DEV), im2.to(DEV), iters=2, test_mode=True)
                torch.cuda.synchronize()
    missing = {f: c for f, c in seen.items() if f not in EPILOGUE_COVERAGE}
    print(f"{len(seen)} epilogue forms launched, {len(missing)} missing from the table")
    for f, c in sorted(missing.items(), key=str):
        print(f"    {f!r}: '',  # {c}")
    assert not missing, f"{len(missing)} launched epilogue forms have no entry in EPILOGUE_COVERAGE (listed above)"
    stale = set(EPILOGUE_COVERAGE) - set(seen)
    assert not stale, f"forms in the table the forwards no longer launch: {sorted(stale, key=str)}"


def test_zz_summary():
    """Prints the worst err / bound of every epilogue check this session ran."""
    for k, v in sorted(WORST.items()):
        print(f"  {k:<48s} worst err/bound {v:.3f}")
