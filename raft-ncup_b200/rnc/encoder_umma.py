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
from .slot_plan import CARRY, NEW, SAVED, images, runs, slot_plan

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
    def run(self, model, ws, image1, image2, plan=None, saved=None):
        """One encoder call of rnc.slot_plan's `plan` (None: the pair plan, fnet on both frames and cnet on frame 1).
        image1/image2: raw [B,3,H,W] fp32 in 0..255 (the stem normalises).  Fills the slots' rows of ws.f1_cl, level 0 of
        ws.f2_pyr, ws.h and ws.hx[:, :256], then finishes the pyramid and the halves.  saved: (h, hx hi, hx lo) rows of the
        plan's `save` slots, restored into the slots that take a saved context and then refilled with this call's."""
        eng, E = self.eng, native
        B, _, Hin, Win = image1.shape
        dev = image1.device
        plan = plan or slot_plan(B)
        S = len(plan.f1)
        bufs = self.buffers(dev, 2 * B, Hin, Win)         # fnet_in and cnet_in have at most 2B images
        h8, w8, _ = bufs.dims[2]
        P = h8 * w8
        n = P * 256                                         # elements of one slot's feature map
        eng.alloc_fmaps(ws, S, 256, h8, w8, 4, dev)
        fmap = {"f1": ws.f1_cl.view(-1), "f2": ws.f2_pyr}
        # carried features are level 0 of the last call's f2: copy them before the fnet head overwrites it
        for name in ("f1", "f2"):
            for j, kind, s, k in runs(getattr(plan, name)):
                if kind == CARRY:
                    fmap[name][j * n:(j + k) * n].copy_(ws.f2_pyr[s * n:(s + k) * n])
                    if name == "f1" and eng.lookup_mode == "umma":
                        ws.f1h[j * n:(j + k) * n].copy_(ws.f2h[s * n:(s + k) * n])
        frames = (image1, image2)
        x = images(frames, plan.fnet_in)
        pf = self.packed(model.fnet)
        self._trunk(pf, bufs, x, len(plan.fnet_in), Hin, Win)
        xs = bufs.XS[2]
        written = {}                                        # fnet image -> (feature map, slot) it was first written to
        for name in ("f1", "f2"):
            for j, kind, i, k in runs(getattr(plan, name)):
                if kind != NEW:
                    continue
                # an image already written in this call is copied from there (encoded once); the others go through the head
                for t, src, s, m in runs([written.get(i + t, (None, i + t)) for t in range(k)]):
                    out = fmap[name][(j + t) * n:(j + t + m) * n]
                    if src is None:
                        eng.uconv(m, h8, w8, (xs.hi[s * P:].data_ptr(), xs.lo[s * P:].data_ptr()), 128, 128, pf.head,
                                  E.EPI_LINEAR, out_f32=out.data_ptr(), ldo_f32=256)
                        written.update((s + u, (name, j + t + u)) for u in range(m))
                    else:
                        out.copy_(fmap[src][s * n:(s + m) * n])
        pc = self.packed(model.cnet)
        self._trunk(pc, bufs, x if plan.cnet_in == plan.fnet_in else images(frames, plan.cnet_in), len(plan.cnet_in),
                    Hin, Win)
        xs = bufs.XS[2]
        hx_hi, hx_lo = ws.hx.hi[:, :256], ws.hx.lo[:, :256]
        for j, kind, i, k in runs(plan.ctx):
            if kind == NEW:
                eng.uconv(k, h8, w8, (xs.hi[i * P:].data_ptr(), xs.lo[i * P:].data_ptr()), 128, 128, pc.head,
                          E.EPI_TANH_RELU, out_f32=ws.h[j * P:].data_ptr(), ldo_f32=128,
                          out_split=(ws.hx.hi[j * P:].data_ptr(), ws.hx.lo[j * P:].data_ptr()), ldo_split=HX_LD)
            elif kind == SAVED:
                rows, src = slice(j * P, (j + k) * P), slice((i - plan.save.start) * P, (i + k - plan.save.start) * P)
                for buf, sv in zip((ws.h, hx_hi, hx_lo), saved):
                    buf[rows].copy_(sv[src])
        if plan.save:
            rows = slice(plan.save.start * P, plan.save.stop * P)
            for buf, sv in zip((ws.h, hx_hi, hx_lo), saved):
                sv.copy_(buf[rows])
        ws.gru_const_valid = False                          # inp changed: the GRU's hoisted share must be recomputed
        f1_slots = [j for j, s in enumerate(plan.f1) if s is not None and s[0] == NEW]
        eng.finish_fmaps(ws, f1_slots=None if len(f1_slots) == S else f1_slots)

