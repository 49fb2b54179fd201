"""Tensor-core variant of rnc.engine: the same loop body (raft_nc_dbl.py:148-165, update.py:130-141), with every
wide convolution on wgmma (rnc_conv2d_umma_fwd) and the 1/8-resolution activations resident as fp16 hi/lo split
planes (value = hi + lo).  Thin layers (7x7 on flow, 3x3 -> 2 flow head, 1x1 -> 2 confidence head) stay on CUDA cores.
"""
import math

import torch

from . import native
from .engine import CORR_CH, HX_LD, Engine, _Timed
from .native import UmmaConvDesc, rnc

CORR_LS = 88           # channels reserved per pyramid level in the resident corr row: 81 taps + 7 zero pads (16-byte groups)
CORR_LD = 4 * CORR_LS  # 352: row pitch of the corr halves planes; convc1 still needs only 6 K-blocks of 64


def corr_resident_index(device=None):
    """Reference channel k = l*81 + i*9 + j (corr.py:41-44)  ->  its position in the resident corr row of the tensor-core path:
    l*88 + (j*8 + i if i < 8 else 72 + j) — a pixel's 8 values of one window row are one aligned 16-byte group (rnc.h)."""
    idx = torch.empty(CORR_CH, dtype=torch.long)
    for lvl in range(4):
        for i in range(9):
            for j in range(9):
                idx[lvl * 81 + i * 9 + j] = lvl * CORR_LS + (j * 8 + i if i < 8 else 72 + j)
    return idx.to(device) if device is not None else idx


def expand_corr_weight(weight):
    """convc1 weight [Cout, 324, 1, 1] -> [Cout, 352, 1, 1] in the resident channel order (zeros at the pads)."""
    w = torch.zeros(weight.shape[0], CORR_LD, 1, 1, dtype=torch.float32, device=weight.device)
    w[:, corr_resident_index(weight.device)] = weight.detach().float()
    return w
GIN_LD = 136           # 2 + 128 (+2 zero) channels of the weights-net input, pitch multiple of 16 B


def _coutpad(cout):
    for c in (32, 64, 128, 192, 256):
        if cout <= c:
            return c
    return (cout + 191) // 192 * 192


class UmmaWeights:
    """[Cout,Cin,KH,KW] -> hi/lo operand planes [CoutPad][taps * blocks * bk] + fp32 bias [CoutPad] + unscale.
    fp16 (default): halves in 64-channel K blocks, scaled by 2^s (s chosen so the largest weight lands in [512, 1024): w_lo
    then stays a normal half), unscale = 2^-s.
    tf32: the RNC_CONV_TF32 format, fp32 planes in 32-channel K blocks (hi = w rounded to TF32, ties away from zero; lo = w - hi),
    unscale = 1: fp32's exponent range needs no scaling, and no device sync (training re-packs every step)."""

    def __init__(self, weight, bias, segs, extra_cout=0, out_scale=1.0, tf32=False):
        cout, cin, kh, kw = weight.shape
        w = weight.detach().float()
        if out_scale != 1.0:                                 # (training re-packs every step: no pass for a scale of 1)
            w = w * out_scale
        bk = 32 if tf32 else 64
        nblks = [(c + bk - 1) // bk for c in segs]
        nblk = sum(nblks)
        self.cout, self.kh, self.kw = cout, kh, kw
        self.coutpad = _coutpad(cout + extra_cout)
        self.ktot = kh * kw * nblk * bk
        wp = torch.zeros(self.coutpad, kh * kw, nblk * bk, dtype=torch.float32, device=w.device)
        ci = col = 0
        for c, nb in zip(segs, nblks):
            take = min(c, cin - ci)
            if take > 0:
                wp[:cout, :, col:col + take] = w[:, ci:ci + take].permute(0, 2, 3, 1).reshape(cout, kh * kw, take)
            ci += take
            col += nb * bk
        assert ci == cin, "segments do not cover the weight's input channels"
        ws = wp.reshape(self.coutpad, self.ktot)
        if tf32:
            self.w_hi = ((ws.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32).contiguous()
            self.w_lo = (ws - self.w_hi).contiguous()
            self.unscale = 1.0
        else:
            mx = float(wp.abs().max())                       # (one device sync; inference packs once per checkpoint)
            s = math.floor(math.log2(1000.0 / mx)) if mx > 0 else 0
            ws = ws * (2.0 ** s)
            self.w_hi = ws.half().contiguous()
            self.w_lo = (ws - self.w_hi.float()).half().contiguous()
            self.unscale = 2.0 ** (-s)
        self.bias = torch.zeros(self.coutpad, dtype=torch.float32, device=w.device)
        if bias is not None:
            self.bias[:cout] = bias.detach().float() * out_scale


class PackedUpdateUmma:
    def __init__(self, ub):
        e, g, fh = ub.encoder, ub.gru, ub.flow_head
        cat = torch.cat
        self.convc1 = UmmaWeights(expand_corr_weight(e.convc1.weight), e.convc1.bias, [CORR_LD])
        self.convc2 = UmmaWeights(e.convc2.weight, e.convc2.bias, [256])
        # convf1 (7x7, 2 -> 128) as a 1x1 layer over the im2col'ed flow neighbourhood: k = 2*(7*ky+kx)+c, K = 98 (+30)
        wf = e.convf1.weight.detach().float()
        self.convf1_mm = UmmaWeights(wf.permute(0, 2, 3, 1).reshape(wf.shape[0], 98, 1, 1), e.convf1.bias, [98])
        self.convf2 = UmmaWeights(e.convf2.weight, e.convf2.bias, [128])
        self.conv = UmmaWeights(e.conv.weight, e.conv.bias, [256], extra_cout=2)
        # SepConvGRU (update.py:33-60).  Its input cat([h, inp, motion]) holds 128 channels (`inp`, the context features) that do
        # not change over the iterations: their share of every gate pre-activation is computed once per forward (`*_c`,
        # biases included) and added in the per-iteration layers' epilogues, which then run over K = 256*5 instead of 384*5.
        def gate(convs):
            wt = cat([c.weight for c in convs], 0).detach().float()          # [Cout, 384 = h | inp | motion, kh, kw]
            bs = cat([c.bias for c in convs], 0)
            it = UmmaWeights(cat([wt[:, :128], wt[:, 256:]], 1), None, [128, 128])
            return it, UmmaWeights(wt[:, 128:256], bs, [128])
        self.zr1, self.zr1_c = gate([g.convz1, g.convr1])
        self.q1, self.q1_c = gate([g.convq1])
        self.zr2, self.zr2_c = gate([g.convz2, g.convr2])
        self.q2, self.q2_c = gate([g.convq2])
        self.fh1 = UmmaWeights(fh.conv1.weight, fh.conv1.bias, [128])
        # FlowHead.conv2 (3x3, 256 -> 2): as a 1x1 layer with one output pair per tap (18 -> 32 columns, K = 256 instead of
        # 2304), summed over the shifted neighbours by rnc_flow_tap_gather_fwd
        w2 = fh.conv2.weight.detach().float()                                # [2, 256, 3, 3]
        self.fh2 = UmmaWeights(w2.permute(2, 3, 0, 1).reshape(18, w2.shape[1], 1, 1), None, [256])
        self.fh2_bias = fh.conv2.bias.detach().float().contiguous()
        self.has_mask = len(ub.mask) > 0
        if self.has_mask:
            self.m0 = UmmaWeights(ub.mask[0].weight, ub.mask[0].bias, [128])
            self.m2 = UmmaWeights(ub.mask[2].weight, ub.mask[2].bias, [256], out_scale=0.25)   # update.py:140


def _ceil32(c):
    return (c + 31) // 32 * 32


class UmmaWnet:
    """The weights net's format on the tensor-core path: layer outputs of ceil32 columns (the epilogue writes whole 32-channel
    chunks; zero beyond the width) in split halves, or in fp32 where the conf head reads them; a convolution head's output
    [M, 32].  The input is the split staging of the guidance (GIN_LD), so a head without hidden layers is a convolution."""
    split, head_pitch = True, 32
    pitch = staticmethod(_ceil32)

    @staticmethod
    def pack(w, b, cin):
        return UmmaWeights(w, b, [cin])

    @staticmethod
    def buffer(M, layer, device):
        return SplitBuf(M, layer.pitch, device) if layer.split else torch.empty(M, layer.pitch, dtype=torch.float32, device=device)

    @staticmethod
    def conv(eng, B, H, W, x, c, ld, layer, epi, y):
        out = dict(out_split=y.ptrs(), ldo_split=layer.pitch) if layer.split else dict(out_f32=y.data_ptr(), ldo_f32=layer.pitch)
        eng.uconv(B, H, W, x.ptrs(), c, ld, layer.wt, epi, dil=layer.dil, **out)


class SplitBuf:
    """A CL activation stored as two planes of halves."""

    def __init__(self, rows, ld, device):
        self.hi = torch.zeros(rows, ld, dtype=torch.float16, device=device)
        self.lo = torch.zeros(rows, ld, dtype=torch.float16, device=device)
        self.ld = ld

    def ptrs(self, ch_off=0):
        """Addresses of channel ch_off in both planes (rnc_conv_umma_desc's in*_hi / in*_lo, out_hi / out_lo).  Computed rather
        than read off a view: uconv calls this on every layer of every iteration."""
        return self.hi.data_ptr() + ch_off * self.hi.element_size(), self.lo.data_ptr() + ch_off * self.lo.element_size()


class UmmaWorkspace:
    def __init__(self, device, B, H8, W8, with_mask, with_ncup):
        self.B, self.H8, self.W8 = B, H8, W8
        M = B * H8 * W8
        f = dict(dtype=torch.float32, device=device)
        self.corr = SplitBuf(M, CORR_LD, device)
        self.c1 = SplitBuf(M, 256, device)
        self.corflo = SplitBuf(M, 256, device)
        self.f1 = SplitBuf(M, 128, device)
        self.fcol = SplitBuf(M, 128, device)     # im2col of the flow for convf1
        self.hx = SplitBuf(M, HX_LD, device)
        self.rh = SplitBuf(M, 128, device)
        self.h = torch.zeros(M, 128, **f)            # fp32 master copy of the GRU state
        # Epilogue-only tensors live in the tile-blocked layout [tile][channel][128 px] of their layer's tiling (thread = pixel
        # then reads / writes full lines): the z gate, and the hoisted context-feature share of the GRU gate pre-activations
        # (valid until inp changes).  Horizontal (1x5) and vertical (5x1) layers tile differently; z serves both halves.
        th, tv = rnc.conv_umma_tiles(1, 5, 1, B, H8, W8, 0), rnc.conv_umma_tiles(5, 1, 1, B, H8, W8, 0)
        self.z = torch.empty(max(th, tv) * 128 * 128, **f)
        self.czr1, self.czr2 = torch.empty(th * 256 * 128, **f), torch.empty(tv * 256 * 128, **f)
        self.cq1, self.cq2 = torch.empty(th * 128 * 128, **f), torch.empty(tv * 128 * 128, **f)
        self.gru_const_valid = False
        self.fh = SplitBuf(M, 256, device)
        self.fh2p = torch.empty(M, 32, **f)      # FlowHead.conv2 per-tap partial sums
        self.tmp = torch.empty(M, 256, **f)
        self.coords1 = torch.empty(B, 2, H8, W8, **f)
        self.delta = torch.empty(B, 2, H8, W8, **f)
        self.f1_cl = self.f2_pyr = None
        if with_mask:
            self.mh = SplitBuf(M, 256, device)
            self.mask = torch.empty(M, 576, **f)
        if with_ncup:
            M4 = 4 * M
            self.x4 = torch.empty(B, 2, 2 * H8, 2 * W8, **f)
            self.gin = SplitBuf(M4, GIN_LD, device)
            self.conf = torch.empty(B, 2, 2 * H8, 2 * W8, **f)
        self.wnet = {}
        self.nconv_bufs = {}


class UmmaEngine(Engine):
    mode = "umma"
    PACK_UB, PACK_UP = PackedUpdateUmma, UmmaWnet
    WS = UmmaWorkspace

    def __init__(self):
        super().__init__()
        import os
        # RNC_LOOKUP=umma (default): wgmma lookup on fp16 features; RNC_LOOKUP=ffma: exact fp32 CUDA-core lookup
        self.lookup_mode = os.environ.get("RNC_LOOKUP", "umma").lower()
        if self.lookup_mode not in ("umma", "ffma"):
            raise ValueError(f"RNC_LOOKUP={self.lookup_mode!r}: expected 'umma' or 'ffma'")

    # ------------------------------------------------------------------ one tensor-core convolution
    def uconv(self, B, H, W, in0, c0, ld0, wt, epi, out_f32=0, ldo_f32=0, out_split=(0, 0), ldo_split=0, in1=(0, 0), c1=0, ld1=0,
              h=0, ldh=0, aux0=0, ldaux=0, stride=1, hin=0, win=0, res=0, ldres=0, flags=0, stats=0, add=0, ldadd=0, win_pitch=0,
              dil=1):
        """One rnc_conv2d_umma_fwd call.  H, W are the OUTPUT dims; for stride 2 pass the input dims as hin, win."""
        d = UmmaConvDesc()
        d.dil = dil
        d.stride, d.hin, d.win, d.res, d.ldres = stride, hin, win, res, ldres
        d.stats = stats
        d.add, d.ldadd = add, ldadd
        d.win_pitch = win_pitch
        d.flags = flags
        d.in0_hi, d.in0_lo, d.c0, d.ld0 = in0[0], in0[1], c0, ld0
        d.in1_hi, d.in1_lo, d.c1, d.ld1 = in1[0], in1[1], c1, ld1
        d.w_hi, d.w_lo, d.ktot, d.coutpad = wt.w_hi.data_ptr(), wt.w_lo.data_ptr(), wt.ktot, wt.coutpad
        d.bias, d.unscale = wt.bias.data_ptr(), wt.unscale
        d.out_f32, d.ldo_f32 = out_f32, ldo_f32
        d.out_hi, d.out_lo, d.ldo_split = out_split[0], out_split[1], ldo_split
        d.h, d.ldh, d.aux0, d.ldaux = h, ldh, aux0, ldaux
        d.B, d.H, d.W = B, H, W
        d.cout, d.kh, d.kw, d.epilogue = wt.cout, wt.kh, wt.kw, epi
        rnc.conv2d_umma_fwd(d)

    def fmap_prepare(self, ws, fmap1, fmap2, levels=4):
        super().fmap_prepare(ws, fmap1, fmap2, levels)
        self._refresh_halves(ws)     # halves copies of the CL feature map / pyramid: the tensor-core lookup's operands

    # ------------------------------------------------------------------ encoders on the tensor-core path
    def encoder(self):
        if getattr(self, "_encoder", None) is None:
            from .encoder_umma import EncoderRunner
            self._encoder = EncoderRunner(self)
        return self._encoder

    def finish_fmaps(self, ws, f1_slots=None):
        """Pool fmap2 into the pyramid (corr.py:18-21 on features) and refresh the halves copies (of fmap1: only the rows of
        batch items f1_slots when given, the others' halves being current)."""
        rnc.fmap_pyramid(ws.f2_pyr, ws.B, ws.D, ws.H8, ws.W8, ws.levels)
        self._refresh_halves(ws, f1_slots)

    def _refresh_halves(self, ws, f1_slots=None):
        if self.lookup_mode != "umma":
            return
        n1, n2 = ws.f1_cl.numel(), ws.f2_pyr.numel()
        if getattr(ws, "f1h", None) is None or ws.f1h.numel() != n1:
            dev = ws.f1_cl.device
            ws.f1h = torch.empty(n1, dtype=torch.float16, device=dev)
            ws.f2h = torch.empty(n2, dtype=torch.float16, device=dev)
            nbytes = rnc.corr_lookup_umma_workspace_bytes(ws.B, ws.H8, ws.W8)
            ws.lookup_flags = torch.zeros(nbytes // 4, dtype=torch.int32, device=dev)
        if f1_slots is None:
            rnc.f32_to_f16(ws.f1_cl, ws.f1h, n1)
        else:
            f1, f1h = ws.f1_cl.view(ws.B, -1), ws.f1h.view(ws.B, -1)
            for j in f1_slots:
                rnc.f32_to_f16(f1[j], f1h[j], n1 // ws.B)
        rnc.f32_to_f16(ws.f2_pyr, ws.f2h, n2)

    def lookup_resident(self, ws):
        """corr lookup straight into the split planes convc1 consumes."""
        if self.lookup_mode == "umma":
            with _Timed(self, "corr_lookup"):
                rnc.corr_lookup_umma_fwd(ws.f1h, ws.f2h, ws.f1_cl, ws.f2_pyr, ws.coords1, ws.B, ws.D, ws.H8, ws.W8, ws.levels, 4,
                                         ws.corr.hi, ws.corr.lo, CORR_LD, CORR_LS, ws.lookup_flags, ws.lookup_flags.numel() * 4)
            return
        with _Timed(self, "corr_lookup"):
            rnc.corr_lookup_split_fwd(ws.f1_cl, ws.f2_pyr, ws.coords1, ws.B, ws.D, ws.H8, ws.W8, ws.levels, 4, ws.corr.hi,
                                      ws.corr.lo, CORR_LD, CORR_LS)

    def _update_iter(self, ws, pk, want_mask, want_delta):
        B, H, W = ws.B, ws.H8, ws.W8
        E = native
        # BasicMotionEncoder (update.py:89-97)
        self.uconv(B, H, W, ws.corr.ptrs(), CORR_LD, CORR_LD, pk.convc1, E.EPI_RELU, out_split=ws.c1.ptrs(), ldo_split=256)
        self.uconv(B, H, W, ws.c1.ptrs(), 256, 256, pk.convc2, E.EPI_RELU, out_split=ws.corflo.ptrs(), ldo_split=256)
        # convf1 (7x7, 2 -> 128) as the im2col of the flow and a 1x1 layer
        rnc.flow_im2col7_split_fwd(ws.coords1, B, H, W, ws.fcol.hi, ws.fcol.lo, 128)
        self.uconv(B, H, W, ws.fcol.ptrs(), 98, 128, pk.convf1_mm, E.EPI_RELU, out_split=ws.f1.ptrs(), ldo_split=128)
        self.uconv(B, H, W, ws.f1.ptrs(), 128, 128, pk.convf2, E.EPI_RELU, out_split=ws.corflo.ptrs(192), ldo_split=256)
        self.uconv(B, H, W, ws.corflo.ptrs(), 256, 256, pk.conv, E.EPI_RELU_FLOW, out_split=ws.hx.ptrs(256), ldo_split=HX_LD,
                   aux0=ws.coords1.data_ptr())
        # SepConvGRU (update.py:45-60)
        hp = ws.h.data_ptr()
        if not ws.gru_const_valid:
            # the context channels' share of the gate pre-activations (+ biases): once per forward
            for wt, buf in ((pk.zr1_c, ws.czr1), (pk.q1_c, ws.cq1), (pk.zr2_c, ws.czr2), (pk.q2_c, ws.cq2)):
                self.uconv(B, H, W, ws.hx.ptrs(128), 128, HX_LD, wt, E.EPI_LINEAR, out_f32=buf.data_ptr(), ldo_f32=wt.coutpad,
                           flags=E.CONV_OUT_BLOCKED)
            ws.gru_const_valid = True
        for zr, q, czr, cq in ((pk.zr1, pk.q1, ws.czr1, ws.cq1), (pk.zr2, pk.q2, ws.czr2, ws.cq2)):
            self.uconv(B, H, W, ws.hx.ptrs(), 128, HX_LD, zr, E.EPI_GRU_ZR, in1=ws.hx.ptrs(256), c1=128, ld1=HX_LD,
                       out_split=ws.rh.ptrs(), ldo_split=128, h=hp, ldh=128, aux0=ws.z.data_ptr(), ldaux=128,
                       add=czr.data_ptr(), ldadd=256, flags=E.CONV_AUX_BLOCKED)
            self.uconv(B, H, W, ws.rh.ptrs(), 128, 128, q, E.EPI_GRU_Q, in1=ws.hx.ptrs(256), c1=128, ld1=HX_LD,
                       out_split=ws.hx.ptrs(), ldo_split=HX_LD, h=hp, ldh=128, aux0=ws.z.data_ptr(), ldaux=128,
                       add=cq.data_ptr(), ldadd=128, flags=E.CONV_AUX_BLOCKED)
        # FlowHead (update.py:13-14) + coords1 += delta (raft_nc_dbl.py:157)
        self.uconv(B, H, W, ws.hx.ptrs(), 128, HX_LD, pk.fh1, E.EPI_RELU, out_split=ws.fh.ptrs(), ldo_split=256)
        self.uconv(B, H, W, ws.fh.ptrs(), 256, 256, pk.fh2, E.EPI_LINEAR, out_f32=ws.fh2p.data_ptr(), ldo_f32=32)
        rnc.flow_tap_gather_fwd(ws.fh2p, 32, pk.fh2_bias, B, H, W, ws.delta if want_delta else None, ws.coords1)
        if want_mask:
            self.uconv(B, H, W, ws.hx.ptrs(), 128, HX_LD, pk.m0, E.EPI_RELU, out_split=ws.mh.ptrs(), ldo_split=256)
            self.uconv(B, H, W, ws.mh.ptrs(), 256, 256, pk.m2, E.EPI_LINEAR, out_f32=ws.mask.data_ptr(), ldo_f32=576)

    def load_state(self, ws, net, inp):
        ws.gru_const_valid = False
        B, _, H, W = net.shape
        rnc.nchw_to_cl(net, B, 128, H, W, ws.h, 128, 0)
        rnc.nchw_to_cl(net, B, 128, H, W, ws.tmp, 256, 0)
        rnc.nchw_to_cl(inp, B, 128, H, W, ws.tmp, 256, 128)
        rnc.f32_to_split(ws.tmp, 256, 256, B * H * W, ws.hx.hi, ws.hx.lo, HX_LD, 0)

    def load_corr(self, ws, corr_nchw):
        """seam path (BasicUpdateBlock.forward): NCHW corr -> split planes."""
        B, _, H, W = corr_nchw.shape
        tmp = torch.empty(B * H * W, CORR_CH, dtype=torch.float32, device=corr_nchw.device)
        rnc.nchw_to_cl(corr_nchw, B, CORR_CH, H, W, tmp, CORR_CH, 0)
        res = torch.zeros(B * H * W, CORR_LD, dtype=torch.float32, device=corr_nchw.device)     # layout plumbing: resident order
        res[:, corr_resident_index(res.device)] = tmp
        rnc.f32_to_split(res, CORR_LD, CORR_LD, B * H * W, ws.corr.hi, ws.corr.lo, CORR_LD, 0)

    def corr_nchw(self, ws):
        """The resident corr row back in the reference's layout [B, 324, H8, W8] (tests / debugging)."""
        v = (ws.corr.hi.float() + ws.corr.lo.float())[:, corr_resident_index(ws.corr.hi.device)]
        return v.view(ws.B, ws.H8, ws.W8, CORR_CH).permute(0, 3, 1, 2).contiguous()

    def net_nchw(self, ws):
        out = torch.empty(ws.B, 128, ws.H8, ws.W8, dtype=torch.float32, device=ws.h.device)
        rnc.cl_to_nchw(ws.h, 128, 0, ws.B, 128, ws.H8, ws.W8, out)
        return out

    def guidance(self, ws):
        return ws.h, 128

    def stage_guidance(self, ws, x_lowres, guid, ldg):
        rnc.ncup_guidance_split_fwd(x_lowres, guid, ldg, 128, ws.B, ws.H8, ws.W8, ws.gin.hi, ws.gin.lo, GIN_LD)
        return ws.gin, GIN_LD
