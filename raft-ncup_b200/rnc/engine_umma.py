"""Tensor-core variant of rnc.engine: the same loop body (raft_nc_dbl.py:148-165, update.py:130-141), with every
wide convolution on wgmma (rnc_conv2d_umma_fwd) and the 1/8-resolution activations resident as fp16 hi/lo split
planes (value = hi + lo).  Thin layers (7x7 on flow, 3x3 -> 2 flow head, 1x1 -> 2 confidence head) stay on CUDA cores.
"""
import ctypes as C
import math

import torch
import torch.nn.functional as F

from . import native
from .engine import CORR_CH, HX_LD, Engine, PackedUpsampler, _ptr, _stream, _Timed, pack_thin
from .native import UmmaConvDesc

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
    """[Cout,Cin,KH,KW] -> hi/lo halves planes [CoutPad][taps * blocks * 64] scaled by 2^s (s chosen so the largest
    weight lands in [512, 1024): w_lo then stays a normal half) + fp32 bias [CoutPad] + unscale = 2^-s."""

    def __init__(self, weight, bias, segs, extra_cout=0, out_scale=1.0, scale_log2=None):
        cout, cin, kh, kw = weight.shape
        w = weight.detach().float() * out_scale
        nblks = [(c + 63) // 64 for c in segs]
        nblk = sum(nblks)
        self.cout, self.kh, self.kw = cout, kh, kw
        self.coutpad = _coutpad(cout + extra_cout)
        self.ktot = kh * kw * nblk * 64
        wp = torch.zeros(self.coutpad, kh * kw, nblk * 64, dtype=torch.float32, device=w.device)
        ci = col = 0
        for c, nb in zip(segs, nblks):
            take = min(c, cin - ci)
            if take > 0:
                wp[:cout, :, col:col + take] = w[:, ci:ci + take].permute(0, 2, 3, 1).reshape(cout, kh * kw, take)
            ci += take
            col += nb * 64
        assert ci == cin, "segments do not cover the weight's input channels"
        if scale_log2 is None:
            mx = float(wp.abs().max())                       # (one device sync; inference packs once per checkpoint)
            s = math.floor(math.log2(1000.0 / mx)) if mx > 0 else 0
        else:
            s = scale_log2                                   # training re-packs every step: fixed scale, no sync (|w| < 2^(15-s))
        ws = wp.reshape(self.coutpad, self.ktot) * (2.0 ** s)
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
        self.convf1 = (pack_thin(e.convf1.weight), e.convf1.bias.detach().float().contiguous())    # CUDA-core form (RNC_CONVF1=ffma)
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


class PackedUpsamplerUmma(PackedUpsampler):
    def __init__(self, up):
        super().__init__(up)
        # re-pack the BN-folded 3x3 layers of the weights net for the tensor-core path
        wn = up.weights_est_net
        convs = []
        for blk in wn.conv:
            w, b = blk[0].weight.detach().float(), blk[0].bias.detach().float()
            if len(blk) == 3:
                bn = blk[1]
                s = bn.weight.detach() / torch.sqrt(bn.running_var + bn.eps)
                w, b = w * s.view(-1, 1, 1, 1), (b - bn.running_mean) * s + bn.bias.detach()
            convs.append((w, b))
        self.u0 = UmmaWeights(convs[0][0], convs[0][1], [132])
        self.u1 = UmmaWeights(convs[1][0], convs[1][1], [64])


class SplitBuf:
    """A CL activation stored as two planes of halves."""

    def __init__(self, rows, ld, device):
        self.hi = torch.zeros(rows, ld, dtype=torch.float16, device=device)
        self.lo = torch.zeros(rows, ld, dtype=torch.float16, device=device)
        self.ld = ld

    def ptrs(self, ch_off=0):
        return self.hi.data_ptr() + 2 * ch_off, self.lo.data_ptr() + 2 * ch_off


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
        L = native.lib()
        th = max(L.rnc_conv_umma_tiles(1, 5, 1, B, H8, W8, fl) for fl in (0, 1))      # with / without halo sharing (RNC_CONV_FLAGS)
        tv = max(L.rnc_conv_umma_tiles(5, 1, 1, B, H8, W8, fl) for fl in (0, 1))
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
        self.convf1_forked = False
        if with_mask:
            self.mh = SplitBuf(M, 256, device)
            self.mask = torch.empty(M, 576, **f)
        if with_ncup:
            M4 = 4 * M
            self.x4 = torch.empty(B, 2, 2 * H8, 2 * W8, **f)
            self.gin = SplitBuf(M4, GIN_LD, device)
            self.g1 = SplitBuf(M4, 64, device)
            self.g2 = torch.empty(M4, 32, **f)
            self.conf = torch.empty(B, 2, 2 * H8, 2 * W8, **f)


class UmmaEngine(Engine):
    mode = "umma"
    PACK_UB, PACK_UP = PackedUpdateUmma, PackedUpsamplerUmma
    WS = UmmaWorkspace

    def __init__(self):
        super().__init__()
        import os
        # RNC_LOOKUP=umma (default): wgmma lookup on fp16 features; RNC_LOOKUP=ffma: exact fp32 CUDA-core lookup
        self.lookup_mode = os.environ.get("RNC_LOOKUP", "umma").lower()
        if self.lookup_mode not in ("umma", "ffma"):
            raise ValueError(f"RNC_LOOKUP={self.lookup_mode!r}: expected 'umma' or 'ffma'")
        # RNC_CONV_FLAGS: bit 0 = one A tile per tap (no halo sharing), bit 1 = no descriptor base_offset (debug)
        self.conv_flags = int(os.environ.get("RNC_CONV_FLAGS", "0"))
        # RNC_CONVF1=mm (default): convf1 as flow im2col + 1x1 tensor-core layer on the main stream; ffma: the CUDA-core 7x7
        # kernel, forked onto a side stream underneath the lookup (RNC_FORK=0 keeps it on the main stream)
        self.convf1_mode = os.environ.get("RNC_CONVF1", "mm").lower()
        if self.convf1_mode not in ("mm", "ffma"):
            raise ValueError(f"RNC_CONVF1={self.convf1_mode!r}: expected 'mm' or 'ffma'")
        # RNC_BLOCKED=0: keep the z gate / hoisted addends channel-last instead of tile-blocked (developer A/B switch)
        self.blocked = os.environ.get("RNC_BLOCKED", "1") != "0"
        self.fork_convf1 = self.convf1_mode == "ffma" and os.environ.get("RNC_FORK", "1") != "0"
        self._side = None

    # ------------------------------------------------------------------ one tensor-core convolution
    def uconv(self, B, H, W, in0, c0, ld0, wt, epi, out_f32=0, ldo_f32=0, out_split=(0, 0), ldo_split=0, in1=(0, 0), c1=0, ld1=0,
              h=0, ldh=0, aux0=0, ldaux=0, stride=1, hin=0, win=0, res=0, ldres=0, flags=None, stats=0, add=0, ldadd=0, win_pitch=0):
        """One rnc_conv2d_umma_fwd call.  H, W are the OUTPUT dims; for stride 2 pass the input dims as hin, win."""
        d = UmmaConvDesc()
        d.stride, d.hin, d.win, d.res, d.ldres = stride, hin, win, res, ldres
        d.stats = stats
        d.add, d.ldadd = add, ldadd
        d.win_pitch = win_pitch
        d.flags = self.conv_flags if flags is None else flags
        d.in0_hi, d.in0_lo, d.c0, d.ld0 = in0[0], in0[1], c0, ld0
        d.in1_hi, d.in1_lo, d.c1, d.ld1 = in1[0], in1[1], c1, ld1
        d.w_hi, d.w_lo, d.ktot, d.coutpad = wt.w_hi.data_ptr(), wt.w_lo.data_ptr(), wt.ktot, wt.coutpad
        d.bias, d.unscale = wt.bias.data_ptr(), wt.unscale
        d.out_f32, d.ldo_f32 = out_f32, ldo_f32
        d.out_hi, d.out_lo, d.ldo_split = out_split[0], out_split[1], ldo_split
        d.h, d.ldh, d.aux0, d.ldaux = h, ldh, aux0, ldaux
        d.B, d.H, d.W = B, H, W
        d.cout, d.kh, d.kw, d.epilogue = wt.cout, wt.kh, wt.kw, epi
        native.check(self.L.rnc_conv2d_umma_fwd(C.byref(d), _stream()), "conv2d_umma")

    def fmap_prepare(self, ws, fmap1, fmap2, levels=4):
        super().fmap_prepare(ws, fmap1, fmap2, levels)
        self._refresh_halves(ws)     # halves copies of the CL feature map / pyramid: the tensor-core lookup's operands

    # ------------------------------------------------------------------ encoders on the tensor-core path
    def encoder(self):
        if getattr(self, "_encoder", None) is None:
            from .encoder_umma import EncoderRunner
            self._encoder = EncoderRunner(self)
        return self._encoder

    def alloc_fmaps(self, ws, B, D, H, W, levels):
        """Allocate the CL feature map / pyramid buffers that the encoder heads write into directly."""
        total = self.L.rnc_pyramid_offset(B, D, H, W, levels)
        if ws.f1_cl is None or ws.f1_cl.numel() != B * H * W * D:
            dev = ws.coords1.device
            ws.f1_cl = torch.empty(B * H * W, D, dtype=torch.float32, device=dev)
            ws.f2_pyr = torch.empty(total, dtype=torch.float32, device=dev)
        ws.D, ws.levels = D, levels

    def finish_fmaps(self, ws):
        """Pool fmap2 into the pyramid (corr.py:18-21 on features) and refresh the halves copies."""
        native.check(self.L.rnc_fmap_pyramid(_ptr(ws.f2_pyr), ws.B, ws.D, ws.H8, ws.W8, ws.levels, _stream()), "fmap_pyramid")
        self._refresh_halves(ws)

    def _refresh_halves(self, ws):
        if self.lookup_mode != "umma":
            return
        n1, n2 = ws.f1_cl.numel(), ws.f2_pyr.numel()
        if getattr(ws, "f1h", None) is None or ws.f1h.numel() != n1:
            dev = ws.f1_cl.device
            ws.f1h = torch.empty(n1, dtype=torch.float16, device=dev)
            ws.f2h = torch.empty(n2, dtype=torch.float16, device=dev)
            nbytes = self.L.rnc_corr_lookup_umma_workspace_bytes(ws.B, ws.H8, ws.W8)
            ws.lookup_flags = torch.zeros(nbytes // 4, dtype=torch.int32, device=dev)
        s = _stream()
        native.check(self.L.rnc_f32_to_f16(_ptr(ws.f1_cl), _ptr(ws.f1h), n1, s), "f32_to_f16(f1)")
        native.check(self.L.rnc_f32_to_f16(_ptr(ws.f2_pyr), _ptr(ws.f2h), n2, s), "f32_to_f16(f2)")

    def lookup_resident(self, ws):
        """corr lookup straight into the split planes convc1 consumes."""
        if self.lookup_mode == "umma":
            with _Timed(self, "corr_lookup"):
                native.check(self.L.rnc_corr_lookup_umma_fwd(
                    _ptr(ws.f1h), _ptr(ws.f2h), _ptr(ws.f1_cl), _ptr(ws.f2_pyr), _ptr(ws.coords1), ws.B, ws.D, ws.H8, ws.W8,
                    ws.levels, 4, _ptr(ws.corr.hi), _ptr(ws.corr.lo), CORR_LD, CORR_LS, _ptr(ws.lookup_flags),
                    ws.lookup_flags.numel() * 4, _stream()), "corr_lookup_umma")
            return
        with _Timed(self, "corr_lookup"):
            native.check(self.L.rnc_corr_lookup_split_fwd(_ptr(ws.f1_cl), _ptr(ws.f2_pyr), _ptr(ws.coords1), ws.B, ws.D, ws.H8,
                                                          ws.W8, ws.levels, 4, _ptr(ws.corr.hi), _ptr(ws.corr.lo), CORR_LD, CORR_LS,
                                                          _stream()), "corr_lookup_split")

    def _convf1(self, ws, pk):
        if self.convf1_mode == "mm":
            native.check(self.L.rnc_flow_im2col7_split_fwd(_ptr(ws.coords1), ws.B, ws.H8, ws.W8, _ptr(ws.fcol.hi), _ptr(ws.fcol.lo), 128,
                                                           _stream()), "flow_im2col7")
            self.uconv(ws.B, ws.H8, ws.W8, ws.fcol.ptrs(), 98, 128, pk.convf1_mm, native.EPI_RELU, out_split=ws.f1.ptrs(), ldo_split=128)
            return
        native.check(self.L.rnc_conv_flow7x7_split_fwd(_ptr(ws.coords1), _ptr(pk.convf1[0]), _ptr(pk.convf1[1]), ws.B, ws.H8, ws.W8,
                                                       128, _ptr(ws.f1.hi), _ptr(ws.f1.lo), 128, _stream()), "convf1")

    def begin_iter(self, ws, pk):
        """Fork: convf1 (7x7 on the flow, CUDA cores, ~1 KB of shared memory) depends only on coords1, so it runs on a side
        stream underneath the tensor-core lookup / convc1 / convc2 CTAs that own the SMs; _update_iter joins before convf2."""
        if not self.fork_convf1:
            return
        main = torch.cuda.current_stream()
        if self._side is None or self._side.device != main.device:
            self._side = torch.cuda.Stream(device=main.device)
        self._side.wait_stream(main)
        with torch.cuda.stream(self._side):
            self._convf1(ws, pk)
        ws.convf1_forked = True

    def _update_iter(self, ws, pk, want_mask, want_delta):
        B, H, W = ws.B, ws.H8, ws.W8
        s = _stream()
        E = native
        # BasicMotionEncoder (update.py:89-97)
        self.uconv(B, H, W, ws.corr.ptrs(), CORR_LD, CORR_LD, pk.convc1, E.EPI_RELU, out_split=ws.c1.ptrs(), ldo_split=256)
        self.uconv(B, H, W, ws.c1.ptrs(), 256, 256, pk.convc2, E.EPI_RELU, out_split=ws.corflo.ptrs(), ldo_split=256)
        if getattr(ws, "convf1_forked", False):
            torch.cuda.current_stream().wait_stream(self._side)       # join
            ws.convf1_forked = False
        else:
            self._convf1(ws, pk)
        self.uconv(B, H, W, ws.f1.ptrs(), 128, 128, pk.convf2, E.EPI_RELU, out_split=ws.corflo.ptrs(192), ldo_split=256)
        self.uconv(B, H, W, ws.corflo.ptrs(), 256, 256, pk.conv, E.EPI_RELU_FLOW, out_split=ws.hx.ptrs(256), ldo_split=HX_LD,
                   aux0=ws.coords1.data_ptr())
        # SepConvGRU (update.py:45-60)
        hp = ws.h.data_ptr()
        if not ws.gru_const_valid:
            # the context channels' share of the gate pre-activations (+ biases): once per forward
            for wt, buf in ((pk.zr1_c, ws.czr1), (pk.q1_c, ws.cq1), (pk.zr2_c, ws.czr2), (pk.q2_c, ws.cq2)):
                self.uconv(B, H, W, ws.hx.ptrs(128), 128, HX_LD, wt, E.EPI_LINEAR, out_f32=buf.data_ptr(), ldo_f32=wt.coutpad,
                           flags=self.conv_flags | (E.CONV_OUT_BLOCKED if self.blocked else 0))
            ws.gru_const_valid = True
        for zr, q, czr, cq in ((pk.zr1, pk.q1, ws.czr1, ws.cq1), (pk.zr2, pk.q2, ws.czr2, ws.cq2)):
            self.uconv(B, H, W, ws.hx.ptrs(), 128, HX_LD, zr, E.EPI_GRU_ZR, in1=ws.hx.ptrs(256), c1=128, ld1=HX_LD,
                       out_split=ws.rh.ptrs(), ldo_split=128, h=hp, ldh=128, aux0=ws.z.data_ptr(), ldaux=128,
                       add=czr.data_ptr(), ldadd=256, flags=self.conv_flags | (E.CONV_AUX_BLOCKED if self.blocked else 0))
            self.uconv(B, H, W, ws.rh.ptrs(), 128, 128, q, E.EPI_GRU_Q, in1=ws.hx.ptrs(256), c1=128, ld1=HX_LD,
                       out_split=ws.hx.ptrs(), ldo_split=HX_LD, h=hp, ldh=128, aux0=ws.z.data_ptr(), ldaux=128,
                       add=cq.data_ptr(), ldadd=128, flags=self.conv_flags | (E.CONV_AUX_BLOCKED if self.blocked else 0))
        # FlowHead (update.py:13-14) + coords1 += delta (raft_nc_dbl.py:157)
        self.uconv(B, H, W, ws.hx.ptrs(), 128, HX_LD, pk.fh1, E.EPI_RELU, out_split=ws.fh.ptrs(), ldo_split=256)
        self.uconv(B, H, W, ws.fh.ptrs(), 256, 256, pk.fh2, E.EPI_LINEAR, out_f32=ws.fh2p.data_ptr(), ldo_f32=32)
        native.check(self.L.rnc_flow_tap_gather_fwd(_ptr(ws.fh2p), 32, _ptr(pk.fh2_bias), B, H, W,
                                                    _ptr(ws.delta) if want_delta else None, _ptr(ws.coords1), s), "flow_tap_gather")
        if want_mask:
            self.uconv(B, H, W, ws.hx.ptrs(), 128, HX_LD, pk.m0, E.EPI_RELU, out_split=ws.mh.ptrs(), ldo_split=256)
            self.uconv(B, H, W, ws.mh.ptrs(), 256, 256, pk.m2, E.EPI_LINEAR, out_f32=ws.mask.data_ptr(), ldo_f32=576)

    def load_state(self, ws, net, inp):
        ws.gru_const_valid = False
        B, _, H, W = net.shape
        s = _stream()
        M = B * H * W
        L = self.L
        native.check(L.rnc_nchw_to_cl(_ptr(net), B, 128, H, W, _ptr(ws.h), 128, 0, s), "nchw_to_cl(net)")
        native.check(L.rnc_nchw_to_cl(_ptr(net), B, 128, H, W, _ptr(ws.tmp), 256, 0, s), "nchw_to_cl(net)")
        native.check(L.rnc_nchw_to_cl(_ptr(inp), B, 128, H, W, _ptr(ws.tmp), 256, 128, s), "nchw_to_cl(inp)")
        native.check(L.rnc_f32_to_split(_ptr(ws.tmp), 256, 256, M, _ptr(ws.hx.hi), _ptr(ws.hx.lo), HX_LD, 0, s), "f32_to_split")

    def load_corr(self, ws, corr_nchw):
        """seam path (BasicUpdateBlock.forward): NCHW corr -> split planes."""
        B, _, H, W = corr_nchw.shape
        tmp = torch.empty(B * H * W, CORR_CH, dtype=torch.float32, device=corr_nchw.device)
        native.check(self.L.rnc_nchw_to_cl(_ptr(corr_nchw), B, CORR_CH, H, W, _ptr(tmp), CORR_CH, 0, _stream()), "nchw_to_cl(corr)")
        res = torch.zeros(B * H * W, CORR_LD, dtype=torch.float32, device=corr_nchw.device)     # layout plumbing: resident order
        res[:, corr_resident_index(res.device)] = tmp
        native.check(self.L.rnc_f32_to_split(_ptr(res), CORR_LD, CORR_LD, B * H * W, _ptr(ws.corr.hi), _ptr(ws.corr.lo), CORR_LD, 0,
                                             _stream()), "f32_to_split(corr)")

    def corr_nchw(self, ws):
        """The resident corr row back in the reference's layout [B, 324, H8, W8] (tests / debugging)."""
        v = (ws.corr.hi.float() + ws.corr.lo.float())[:, corr_resident_index(ws.corr.hi.device)]
        return v.view(ws.B, ws.H8, ws.W8, CORR_CH).permute(0, 3, 1, 2).contiguous()

    def net_nchw(self, ws):
        out = torch.empty(ws.B, 128, ws.H8, ws.W8, dtype=torch.float32, device=ws.h.device)
        native.check(self.L.rnc_cl_to_nchw(_ptr(ws.h), 128, 0, ws.B, 128, ws.H8, ws.W8, _ptr(out), _stream()), "cl_to_nchw")
        return out

    def guidance(self, ws):
        return ws.h.data_ptr(), 128

    def ncup_from_lowres(self, ws, pu, x_lowres, guid_ptr, ldg, out_scale):
        B, H8, W8 = ws.B, ws.H8, ws.W8
        H4, W4 = 2 * H8, 2 * W8
        M4 = B * H4 * W4
        s = _stream()
        L = self.L
        native.check(L.rnc_ncup_guidance_split_fwd(_ptr(x_lowres), C.c_void_p(guid_ptr), ldg, 128, B, H8, W8, _ptr(ws.gin.hi),
                                                   _ptr(ws.gin.lo), GIN_LD, s), "ncup_guidance_split")
        self.uconv(B, H4, W4, ws.gin.ptrs(), 132, GIN_LD, pu.u0, native.EPI_RELU, out_split=ws.g1.ptrs(), ldo_split=64)
        self.uconv(B, H4, W4, ws.g1.ptrs(), 64, 64, pu.u1, native.EPI_RELU, out_f32=ws.g2.data_ptr(), ldo_f32=32)
        native.check(L.rnc_conf_head_fwd(_ptr(ws.g2), pu.c_mid1, 32, _ptr(pu.gout[0]), _ptr(pu.gout[1]), B, H4, W4, _ptr(ws.conf), s),
                     "conf_head")
        out = torch.empty(B, 2, 4 * H4, 4 * W4, dtype=torch.float32, device=x_lowres.device)
        with _Timed(self, "ncup"):
            native.check(L.rnc_ncup_fwd(_ptr(x_lowres), _ptr(ws.conf), pu.nconv_host, B, H4, W4, out_scale, _ptr(out), s), "ncup")
        return out
