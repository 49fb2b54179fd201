"""fnet / cnet (core/extractor.py:118-192 BasicEncoder, ResidualBlock :6-56) on the tensor-core convolution path.

The wide 3x3 / 1x1 layers run on rnc_conv2d_umma_fwd (fp16 hi/lo split operands, stride 1/2); so does the 7x7/2 stem: the
normalised image is repacked once as a zero-padded [H][W+8][4] plane of split halves and the convolution reads it through a
sliding-window tensor map (16-pixel windows 16 bytes apart: the TMA unit builds the im2col rows; 7 row taps x 64 = K 448 with
zero weights for the 9 phantom pixels and the phantom channel); InstanceNorm (fnet) is a statistics pass + an apply pass fused with
ReLU / residual add / re-splitting (under torch.use_deterministic_algorithms the statistics are per-CTA partials added in a
fixed order, rnc_instnorm_stats_det, instead of the convolution epilogue's fp64 atomics); BatchNorm (cnet, eval mode) is folded into the convolution weights.  The encoders write
their results straight into the loop's resident buffers: fmap1 -> f1_cl, fmap2 -> level 0 of f2_pyr, tanh(net) -> h and
hx[:, 0:128], relu(inp) -> hx[:, 128:256] (raft_nc_dbl.py:129-140).
"""
import torch

from . import native
from .engine import fold_bn
from .engine_umma import HX_LD, SplitBuf, UmmaWeights
from .native import rnc

EPS = 1e-5


class PackedEncoder:
    """Kernel-ready weights of one BasicEncoder.  kind = 'instance' (fnet) or 'batch' (cnet, BN folded)."""

    def __init__(self, enc):
        self.kind = enc.norm_fn
        if self.kind not in ("instance", "batch"):
            raise NotImplementedError("tensor-core encoder supports the reference's two configurations: instance / batch norm")
        bn = self.kind == "batch"
        if bn and any(m.training for m in enc.modules() if isinstance(m, torch.nn.BatchNorm2d)):
            raise NotImplementedError("cnet BatchNorm in training mode (batch statistics) is not built; call .eval() / freeze_bn()")
        w, b = fold_bn(enc.conv1, enc.norm1 if bn else None)
        # window form of the 7x7x3 filter: input "channel" e = 4 * px + c of the 16-pixel window, one tap per filter row
        wv = torch.zeros(w.shape[0], 16, 4, 7, dtype=torch.float32, device=w.device)
        wv[:, :7, :3, :] = w.permute(0, 3, 1, 2)              # [o][kx][c][ky]
        self.stem = UmmaWeights(wv.reshape(w.shape[0], 64, 7, 1), b, [64])
        self.blocks = []
        for layer in (enc.layer1, enc.layer2, enc.layer3):
            for blk in layer:
                cin, cout = blk.conv1.in_channels, blk.conv1.out_channels
                stride = blk.conv1.stride[0]
                w1 = UmmaWeights(*fold_bn(blk.conv1, blk.norm1 if bn else None), [cin])
                w2 = UmmaWeights(*fold_bn(blk.conv2, blk.norm2 if bn else None), [cout])
                wd = None
                if blk.downsample is not None:
                    wd = UmmaWeights(*fold_bn(blk.downsample[0], blk.norm3 if bn else None), [cin])
                self.blocks.append((cin, cout, stride, w1, w2, wd))
        self.head = UmmaWeights(enc.conv2.weight, enc.conv2.bias, [128])


class EncoderBuffers:
    """Scratch for one encoder pass over N images of Hin x Win (three resolution levels)."""

    def __init__(self, device, N, Hin, Win):
        self.key = (str(device), N, Hin, Win)
        f = dict(dtype=torch.float32, device=device)
        self.dims = []
        h, w = (Hin + 1) // 2, (Win + 1) // 2
        for c in (64, 96, 128):
            self.dims.append((h, w, c))
            h, w = (h + 1) // 2, (w + 1) // 2
        self.X32, self.XS, self.T32, self.AS, self.D32 = [], [], [], [], []
        for (h, w, c) in self.dims:
            rows = N * h * w
            self.X32.append(torch.empty(rows, c, **f))
            self.T32.append(torch.empty(rows, c, **f))
            self.D32.append(torch.empty(rows, c, **f) if c != 64 else None)
            self.XS.append(SplitBuf(rows, c, device))
            self.AS.append(SplitBuf(rows, c, device))
        # stem input: zero-padded pixel plane [N][Hin][pitch][4] of split halves (+ 32 zero pixels: the last windows run over)
        self.pitch = (Win + 7) & ~1
        npx = N * Hin * self.pitch + 32
        self.img_hi = torch.zeros(npx, 4, dtype=torch.float16, device=device)
        self.img_lo = torch.zeros(npx, 4, dtype=torch.float16, device=device)
        self.stats = torch.zeros(N * 128 * 2, dtype=torch.float64, device=device)   # kept zeroed by rnc_instnorm_finalize
        self.mr = torch.empty(N * 128 * 2, **f)
        self.parts = None                                  # rnc_instnorm_stats_det's partials, sized on first use

    def det_workspace(self):
        if self.parts is None:
            # sized for all N images of the buffers: a pass may run on fewer (cnet, sequence steps), but the first not always
            N = self.key[1]
            nbytes = max(rnc.instnorm_stats_det_workspace_bytes(N, h * w, c) for (h, w, c) in self.dims)
            self.parts = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=self.stats.device)
        return self.parts


class EncoderRunner:
    def __init__(self, engine):
        self.eng = engine
        self.L = engine.L
        self._bufs = None

    def packed(self, enc):
        return self.eng._packed_for("enc", enc, PackedEncoder)

    def buffers(self, device, N, Hin, Win):
        if self._bufs is None or self._bufs.key != (str(device), N, Hin, Win):
            self._bufs = None
            self._bufs = EncoderBuffers(device, N, Hin, Win)
        return self._bufs

    # ------------------------------------------------------------------ instance-norm helpers
    def _norm(self, bufs, x32, N, P, Cc, mode, res=None, out32=None, split=None, fused_stats=False):
        """fused_stats: the producing convolution already accumulated the sums into bufs.stats (rnc_conv_umma_desc.stats);
        otherwise the deterministic statistics pass reads x32."""
        if fused_stats:
            rnc.instnorm_finalize(bufs.stats, N, P, Cc, EPS, bufs.mr)
        else:
            ws = bufs.det_workspace()
            rnc.instnorm_stats_det(x32, N, P, Cc, EPS, ws, ws.numel() * 8, bufs.mr)
        rnc.instnorm_apply(x32, bufs.mr, res, N, P, Cc, mode, out32, split.hi if split else None, split.lo if split else None)

    def _trunk(self, pk, bufs, image, N, Hin, Win):
        """Stem + the six residual blocks.  Leaves the 128-channel features at 1/8 resolution in bufs.XS[2] (split)."""
        E, eng = native, self.eng
        inst = pk.kind == "instance"
        fused = not torch.are_deterministic_algorithms_enabled()    # epilogue statistics use fp64 atomics
        st = bufs.stats.data_ptr() if fused else 0
        h, w, _ = bufs.dims[0]
        rnc.stem_window_prep(image, N, Hin, Win, bufs.pitch, bufs.img_hi, bufs.img_lo)
        win = dict(stride=2, hin=Hin, win=w, win_pitch=4 * bufs.pitch, flags=E.CONV_WINDOW)
        img = (bufs.img_hi.data_ptr(), bufs.img_lo.data_ptr())
        if inst:
            eng.uconv(N, h, w, img, 64, 8, pk.stem, E.EPI_LINEAR, out_f32=bufs.T32[0].data_ptr(), ldo_f32=64,
                      stats=st, **win)
            self._norm(bufs, bufs.T32[0], N, h * w, 64, 1, out32=bufs.X32[0], split=bufs.XS[0], fused_stats=fused)
        else:
            eng.uconv(N, h, w, img, 64, 8, pk.stem, E.EPI_RELU, out_f32=bufs.X32[0].data_ptr(), ldo_f32=64,
                      out_split=bufs.XS[0].ptrs(), ldo_split=64, **win)
        lvl = 0
        for bi, (cin, cout, stride, w1, w2, wd) in enumerate(pk.blocks):
            # the fp32 copy of a block's output is only read as the next block's residual (blocks without a downsample branch)
            need32 = bi + 1 < len(pk.blocks) and pk.blocks[bi + 1][5] is None
            src = lvl
            if stride == 2:
                lvl += 1
            hi_, wi_, _ = bufs.dims[src]
            h, w, _ = bufs.dims[lvl]
            P = h * w
            xs_in, x32_in = bufs.XS[src], bufs.X32[src]
            if inst:
                eng.uconv(N, h, w, xs_in.ptrs(), cin, cin, w1, E.EPI_LINEAR, out_f32=bufs.T32[lvl].data_ptr(), ldo_f32=cout,
                          stride=stride, hin=hi_, win=wi_, stats=st)
                self._norm(bufs, bufs.T32[lvl], N, P, cout, 1, split=bufs.AS[lvl], fused_stats=fused)
                res = x32_in
                if wd is not None:
                    eng.uconv(N, h, w, xs_in.ptrs(), cin, cin, wd, E.EPI_LINEAR, out_f32=bufs.T32[lvl].data_ptr(), ldo_f32=cout,
                              stride=stride, hin=hi_, win=wi_, stats=st)
                    self._norm(bufs, bufs.T32[lvl], N, P, cout, 0, out32=bufs.D32[lvl], fused_stats=fused)
                    res = bufs.D32[lvl]
                eng.uconv(N, h, w, bufs.AS[lvl].ptrs(), cout, cout, w2, E.EPI_LINEAR, out_f32=bufs.T32[lvl].data_ptr(), ldo_f32=cout,
                          stats=st)
                self._norm(bufs, bufs.T32[lvl], N, P, cout, 2, res=res, out32=bufs.X32[lvl] if need32 else None, split=bufs.XS[lvl],
                           fused_stats=fused)
            else:
                eng.uconv(N, h, w, xs_in.ptrs(), cin, cin, w1, E.EPI_RELU, out_split=bufs.AS[lvl].ptrs(), ldo_split=cout,
                          stride=stride, hin=hi_, win=wi_)
                res = x32_in
                if wd is not None:
                    eng.uconv(N, h, w, xs_in.ptrs(), cin, cin, wd, E.EPI_LINEAR, out_f32=bufs.D32[lvl].data_ptr(), ldo_f32=cout,
                              stride=stride, hin=hi_, win=wi_)
                    res = bufs.D32[lvl]
                eng.uconv(N, h, w, bufs.AS[lvl].ptrs(), cout, cout, w2, E.EPI_RELU_ADD_RELU,
                          out_f32=bufs.X32[lvl].data_ptr() if need32 else 0, ldo_f32=cout, out_split=bufs.XS[lvl].ptrs(),
                          ldo_split=cout, res=res.data_ptr(), ldres=cout)
        return bufs.dims[2]

    # ------------------------------------------------------------------ public
    def run(self, model, ws, image1, image2):
        """image1/image2: raw [B,3,H,W] fp32 in 0..255 (the stem normalises).  Fills ws.f1_cl, ws.f2_pyr (level 0), ws.h,
        ws.hx[:, :256]; the caller finishes the pyramid."""
        eng, E = self.eng, native
        B, _, Hin, Win = image1.shape
        dev = image1.device
        pf, pc = self.packed(model.fnet), self.packed(model.cnet)
        bufs = self.buffers(dev, 2 * B, Hin, Win)
        # ---- fnet on both frames (extractor.py:168-172 concatenates them along the batch)
        both = torch.cat([image1, image2], 0).contiguous()
        h8, w8, _ = self._trunk(pf, bufs, both, 2 * B, Hin, Win)
        P = h8 * w8
        eng.alloc_fmaps(ws, B, 256, h8, w8, 4, dev)
        xs = bufs.XS[2]
        eng.uconv(B, h8, w8, xs.ptrs(), 128, 128, pf.head, E.EPI_LINEAR, out_f32=ws.f1_cl.data_ptr(), ldo_f32=256)
        # the second half of the batch inside the split planes
        eng.uconv(B, h8, w8, (xs.hi[B * P:].data_ptr(), xs.lo[B * P:].data_ptr()), 128, 128, pf.head, E.EPI_LINEAR,
                  out_f32=ws.f2_pyr.data_ptr(), ldo_f32=256)
        self._context(pc, bufs, ws, image1, h8, w8)
        return h8, w8

    def _context(self, pc, bufs, ws, image1, h8, w8):
        """cnet on frame 1 -> ws.h, ws.hx[:, :256]."""
        B, _, Hin, Win = image1.shape
        self._trunk(pc, bufs, image1.contiguous(), B, Hin, Win)
        ws.gru_const_valid = False                              # inp changes: the GRU's hoisted share must be recomputed
        self.eng.uconv(B, h8, w8, bufs.XS[2].ptrs(), 128, 128, pc.head, native.EPI_TANH_RELU, out_f32=ws.h.data_ptr(),
                       ldo_f32=128, out_split=ws.hx.ptrs(), ldo_split=HX_LD)

    def run_bidirectional(self, model, ws, image1, image2):
        """The encoders of the bidirectional pass (rnc.model.BidirectionalStage) on a workspace of 2B slots: fnet on the 2B
        frames cat(image1, image2), in the encoder buffers of an ordinary B-pair forward; its head writes ws.f1_cl for all 2B
        slots in frame order, and two device-to-device copies of the halves give level 0 of ws.f2_pyr (slot j: image2[j],
        slot B + j: image1[j]).  cnet on the same 2B frames -> ws.h, ws.hx[:, :256].  The caller finishes the pyramid."""
        eng, E = self.eng, native
        B, _, Hin, Win = image1.shape
        dev = image1.device
        pf, pc = self.packed(model.fnet), self.packed(model.cnet)
        bufs = self.buffers(dev, 2 * B, Hin, Win)
        both = torch.cat([image1, image2], 0).contiguous()
        h8, w8, _ = self._trunk(pf, bufs, both, 2 * B, Hin, Win)
        eng.alloc_fmaps(ws, 2 * B, 256, h8, w8, 4, dev)
        eng.uconv(2 * B, h8, w8, bufs.XS[2].ptrs(), 128, 128, pf.head, E.EPI_LINEAR, out_f32=ws.f1_cl.data_ptr(), ldo_f32=256)
        n = B * h8 * w8 * 256                               # elements of one half's feature maps
        f1 = ws.f1_cl.view(-1)
        ws.f2_pyr[:n].copy_(f1[n:])
        ws.f2_pyr[n:2 * n].copy_(f1[:n])
        self._context(pc, bufs, ws, both, h8, w8)
        return h8, w8

    def run_step(self, model, ws, image1, image2, carry, restart):
        """One step of sequence inference (rnc.model.SequenceStage): like run, but frame 1 of the `carry` slots is the last
        step's frame 2, whose features are still level 0 of ws.f2_pyr (and of ws.f2h, the tensor-core lookup's halves): they
        are copied into those slots' rows of ws.f1_cl / ws.f1h, then fnet runs on cat(image2 of every slot, image1 of the
        `restart` slots) and its head writes level 0 of f2_pyr for all slots and the f1_cl rows of the restarted ones.  Slots
        in neither list keep their f1 rows (an idle slot recomputes its last pair).  The caller converts only the restarted
        slots' f1 rows to halves (finish_fmaps(ws, f1_slots=restart))."""
        eng, E = self.eng, native
        B, _, Hin, Win = image1.shape
        dev = image1.device
        pf, pc = self.packed(model.fnet), self.packed(model.cnet)
        bufs = self.buffers(dev, 2 * B, Hin, Win)         # the size of an ordinary forward's: no reallocation as R varies
        h8, w8, _ = bufs.dims[2]
        n = h8 * w8 * 256                                   # elements of one slot's feature map
        eng.alloc_fmaps(ws, B, 256, h8, w8, 4, dev)
        f1, halves = ws.f1_cl.view(-1), eng.lookup_mode == "umma"
        for j0, k in _runs(carry):                          # before the fnet head overwrites level 0
            f1[j0 * n:(j0 + k) * n].copy_(ws.f2_pyr[j0 * n:(j0 + k) * n])
            if halves:
                ws.f1h[j0 * n:(j0 + k) * n].copy_(ws.f2h[j0 * n:(j0 + k) * n])
        both = torch.cat([image2] + [image1[j:j + 1] for j in restart]) if restart else image2
        self._trunk(pf, bufs, both.contiguous(), B + len(restart), Hin, Win)
        xs = bufs.XS[2]
        eng.uconv(B, h8, w8, xs.ptrs(), 128, 128, pf.head, E.EPI_LINEAR, out_f32=ws.f2_pyr.data_ptr(), ldo_f32=256)
        for r, j in enumerate(restart):
            i = (B + r) * h8 * w8                           # image B + r inside the 128-channel split planes
            eng.uconv(1, h8, w8, (xs.hi[i:].data_ptr(), xs.lo[i:].data_ptr()), 128, 128, pf.head, E.EPI_LINEAR,
                      out_f32=f1[j * n:].data_ptr(), ldo_f32=256)
        self._context(pc, bufs, ws, image1, h8, w8)
        return h8, w8

    def run_bidirectional_step(self, model, ws, image1, image2, carry, restart, ctx):
        """One step of bidirectional sequence inference (rnc.model.BidirectionalSequenceStage) on a workspace of 2B slots:
        slot j holds the forward pair (image1[j], image2[j]), slot B + j the backward pair (image2[j], image1[j]).  For the
        `carry` slots, frame 1 of the forward pair is the last step's frame 2, whose features are still level 0 of
        ws.f2_pyr: they are copied into slot j's rows of ws.f1_cl / ws.f1h and into level 0 of slot B + j.  Then fnet runs on
        cat(image2 of every slot, image1 of the `restart` slots), the images run_step encodes; its head writes level 0 of
        f2_pyr for slots 0..B-1, a copy of those gives the f1_cl rows of slots B..2B-1, and a restarted slot's own frame 1
        fills its f1_cl rows and level 0 of slot B + j.  cnet runs on the same B + R images: image2 is the context of the
        backward slots, a restarted slot's image1 that of its forward slot, and a carried forward slot takes the last step's
        backward context from ctx (h, hi, lo: [B*H8*W8, 128] fp32 and two [B*H8*W8, 256] fp16, the stage's buffer), which
        is then refilled with this step's.  Slots in neither list keep their forward f1 rows and backward f2 level 0 (an idle
        slot recomputes its last pair; its forward context is left as it is and its results are dropped).  The caller
        converts the f1 rows of the restarted forward slots and of every backward slot to halves."""
        eng, E = self.eng, native
        B, _, Hin, Win = image1.shape
        dev = image1.device
        pf, pc = self.packed(model.fnet), self.packed(model.cnet)
        bufs = self.buffers(dev, 2 * B, Hin, Win)         # B + R <= 2B images: an ordinary forward's buffers
        h8, w8, _ = bufs.dims[2]
        P = h8 * w8
        n = P * 256                                         # elements of one slot's feature map
        eng.alloc_fmaps(ws, 2 * B, 256, h8, w8, 4, dev)
        f1, halves = ws.f1_cl.view(-1), eng.lookup_mode == "umma"
        for j0, k in _runs(carry):                          # before the fnet head overwrites level 0
            src = ws.f2_pyr[j0 * n:(j0 + k) * n]
            f1[j0 * n:(j0 + k) * n].copy_(src)
            ws.f2_pyr[(B + j0) * n:(B + j0 + k) * n].copy_(src)
            if halves:
                ws.f1h[j0 * n:(j0 + k) * n].copy_(ws.f2h[j0 * n:(j0 + k) * n])
        both = (torch.cat([image2] + [image1[j:j + 1] for j in restart]) if restart else image2).contiguous()
        self._trunk(pf, bufs, both, B + len(restart), Hin, Win)
        xs = bufs.XS[2]
        eng.uconv(B, h8, w8, xs.ptrs(), 128, 128, pf.head, E.EPI_LINEAR, out_f32=ws.f2_pyr.data_ptr(), ldo_f32=256)
        f1[B * n:2 * B * n].copy_(ws.f2_pyr[:B * n])
        for r, j in enumerate(restart):
            i = (B + r) * P                                 # image B + r inside the 128-channel split planes
            eng.uconv(1, h8, w8, (xs.hi[i:].data_ptr(), xs.lo[i:].data_ptr()), 128, 128, pf.head, E.EPI_LINEAR,
                      out_f32=f1[j * n:].data_ptr(), ldo_f32=256)
            ws.f2_pyr[(B + j) * n:(B + j + 1) * n].copy_(f1[j * n:(j + 1) * n])
        # ---- cnet on the same images
        self._trunk(pc, bufs, both, B + len(restart), Hin, Win)
        ws.gru_const_valid = False                          # inp changes: the GRU's hoisted share must be recomputed
        xs = bufs.XS[2]
        hx_hi, hx_lo = ws.hx.hi[:, :256], ws.hx.lo[:, :256]
        eng.uconv(B, h8, w8, xs.ptrs(), 128, 128, pc.head, E.EPI_TANH_RELU, out_f32=ws.h[B * P:].data_ptr(), ldo_f32=128,
                  out_split=(ws.hx.hi[B * P:].data_ptr(), ws.hx.lo[B * P:].data_ptr()), ldo_split=HX_LD)
        for r, j in enumerate(restart):
            i = (B + r) * P
            eng.uconv(1, h8, w8, (xs.hi[i:].data_ptr(), xs.lo[i:].data_ptr()), 128, 128, pc.head, E.EPI_TANH_RELU,
                      out_f32=ws.h[j * P:].data_ptr(), ldo_f32=128,
                      out_split=(ws.hx.hi[j * P:].data_ptr(), ws.hx.lo[j * P:].data_ptr()), ldo_split=HX_LD)
        ch, chi, clo = ctx
        for j0, k in _runs(carry):
            rows = slice(j0 * P, (j0 + k) * P)
            ws.h[rows].copy_(ch[rows])
            hx_hi[rows].copy_(chi[rows])
            hx_lo[rows].copy_(clo[rows])
        ch.copy_(ws.h[B * P:])
        chi.copy_(hx_hi[B * P:])
        clo.copy_(hx_lo[B * P:])
        return h8, w8


def _runs(slots):
    """Sorted slot indices -> (first, count) of each run of consecutive ones: one copy per run."""
    out = []
    for j in sorted(slots):
        if out and out[-1][0] + out[-1][1] == j:
            out[-1][1] += 1
        else:
            out.append([j, 1])
    return out
