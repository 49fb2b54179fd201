"""Host-side driver of the per-iteration hot path: owns the resident channel-last (CL) workspace and issues the
librnc kernels in the order of the reference's loop body.

Reference control flow being replaced (file:line under /root/reference/core):
  raft_nc_dbl.py:148-165 / raft.py:121-138   for itr in range(iters): lookup -> update block -> coords += delta -> upsample
  update.py:130-141                          BasicUpdateBlock.forward
  raft_nc_dbl.py:107-112, upsampler.py:143-177   NCUP upsampling          raft.py:73-84  convex upsampling

PyTorch is used here only as plumbing: device memory (torch.empty), the current CUDA stream and weight
re-packing at load time.  All arithmetic of the path runs in librnc.so; there is no fallback.
"""
import ctypes as C
import os
import threading
from collections import OrderedDict

import torch
import torch.nn.functional as F

from . import native
from .native import ConvDesc

CORR_CH = 324          # 4 levels * 9 * 9
HX_LD = 384            # [h | inp | motion(126) flow(2)]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _require_cuda(*tensors):
    """Every tensor must live on one CUDA device (returned).  The kernels are launched on that device's current stream
    (callers wrap the launches in ``torch.cuda.device(dev)``), never on whatever device happens to be current."""
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise native.RncUnavailable(
                "the RAFT-NCUP hot path runs only on CUDA (sm_90a) tensors; got a CPU tensor and there is no CPU fallback")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise ValueError(f"tensors on different CUDA devices ({dev} and {t.device}): move them to one device first")
    return dev


def module_tensors(module):
    """Parameters and buffers a module tree computes with, also for nn.DataParallel replicas: a replica has empty
    ``_parameters`` and carries its per-device broadcast copies in ``_former_parameters`` (torch/nn/parallel/replicate.py)."""
    out = []
    for m in module.modules():
        out.extend(p for p in m._parameters.values() if p is not None)
        if getattr(m, "_is_replica", False):
            out.extend(p for p in getattr(m, "_former_parameters", {}).values() if p is not None)
        out.extend(b for b in m._buffers.values() if b is not None)
    return out


def module_device(module):
    for t in module_tensors(module):
        return t.device
    return None


def pack_conv(weight, bias, cin_pad=None, scale=1.0):
    """[Cout,Cin,KH,KW] -> ([KH*KW][CinPad][CoutPad], [CoutPad]) fp32, CoutPad = ceil64(Cout)."""
    cout, cin, kh, kw = weight.shape
    cin_pad = cin_pad or cin
    cout_pad = (cout + 63) // 64 * 64
    w = torch.zeros(kh * kw, cin_pad, cout_pad, dtype=torch.float32, device=weight.device)
    w[:, :cin, :cout] = (weight.detach().float() * scale).permute(2, 3, 1, 0).reshape(kh * kw, cin, cout)
    b = torch.zeros(cout_pad, dtype=torch.float32, device=weight.device)
    if bias is not None:
        b[:cout] = bias.detach().float() * scale
    return w.contiguous(), b


def pack_thin(weight):
    """[Cout,Cin,KH,KW] -> [KH*KW][Cin][Cout] (no padding) for the thin-channel kernels."""
    cout, cin, kh, kw = weight.shape
    return weight.detach().float().permute(2, 3, 1, 0).reshape(kh * kw, cin, cout).contiguous()


class PackedMotionEncoder:
    """Kernel-ready weights of BasicMotionEncoder (update.py:79-87) for the exact fp32 CUDA-core kernels."""

    def __init__(self, e):
        self.convc1 = pack_conv(e.convc1.weight, e.convc1.bias)
        self.convc2 = pack_conv(e.convc2.weight, e.convc2.bias)
        self.convf1 = (pack_thin(e.convf1.weight), e.convf1.bias.detach().float().contiguous())
        self.convf2 = pack_conv(e.convf2.weight, e.convf2.bias)
        self.conv = pack_conv(e.conv.weight, e.conv.bias)


class PackedGRU:
    """SepConvGRU (update.py:33-43): z and r of each half step share one 256-column layer."""

    def __init__(self, g):
        self.zr1 = pack_conv(torch.cat([g.convz1.weight, g.convr1.weight], 0), torch.cat([g.convz1.bias, g.convr1.bias], 0))
        self.q1 = pack_conv(g.convq1.weight, g.convq1.bias)
        self.zr2 = pack_conv(torch.cat([g.convz2.weight, g.convr2.weight], 0), torch.cat([g.convz2.bias, g.convr2.bias], 0))
        self.q2 = pack_conv(g.convq2.weight, g.convq2.bias)


class PackedFlowHead:
    """FlowHead (update.py:6-11)."""

    def __init__(self, fh):
        self.fh1 = pack_conv(fh.conv1.weight, fh.conv1.bias)
        self.fh2 = (pack_thin(fh.conv2.weight), fh.conv2.bias.detach().float().contiguous())


class PackedUpdateBlock:
    """Kernel-ready weights of BasicUpdateBlock (update.py:114-128)."""

    def __init__(self, ub):
        for part in (PackedMotionEncoder(ub.encoder), PackedGRU(ub.gru), PackedFlowHead(ub.flow_head)):
            self.__dict__.update(part.__dict__)
        self.has_mask = len(ub.mask) > 0
        if self.has_mask:
            self.m0 = pack_conv(ub.mask[0].weight, ub.mask[0].bias)
            self.m2 = pack_conv(ub.mask[2].weight, ub.mask[2].bias, scale=0.25)   # `.25 * self.mask(net)`, update.py:140


class PackedUpsampler:
    """Kernel-ready weights of NConvUpsampler (upsampler.py:75-141): BN-folded weights net + softplus'd NConv weights."""

    def __init__(self, up):
        wn = up.weights_est_net
        convs = []
        for blk in wn.conv:
            conv = blk[0]
            w, b = conv.weight.detach().float(), conv.bias.detach().float()
            if len(blk) == 3:   # Conv, BatchNorm, ReLU — eval-mode fold (interp_weights_est.py:26-30)
                bn = blk[1]
                s = bn.weight.detach() / torch.sqrt(bn.running_var + bn.eps)
                w = w * s.view(-1, 1, 1, 1)
                b = (b - bn.running_mean) * s + bn.bias.detach()
            convs.append((w, b))
        cin0 = convs[0][0].shape[1]
        self.cin0_pad = (cin0 + 3) // 4 * 4
        self.g0 = pack_conv(convs[0][0], convs[0][1], cin_pad=self.cin0_pad)
        self.g1 = pack_conv(convs[1][0], convs[1][1])
        self.c_mid0, self.c_mid1 = convs[0][0].shape[0], convs[1][0].shape[0]
        self.gout = (pack_thin(wn.out.weight), wn.out.bias.detach().float().contiguous())
        net = up.interpolation_net
        ws = [F.softplus(p.detach().float(), beta=10).reshape(-1).cpu() for p in
              (net.nconv_in.weight_p, net.nconv_x2[0].weight_p, net.decoder[0].weight_p, net.nconv_out.weight_p)]
        host = torch.cat(ws).contiguous()
        assert host.numel() == 224, "NCUP kernel is built for the shipped interp_net config (SURVEY.md §5)"
        self.nconv_host = (C.c_float * 224)(*host.tolist())


def _checksum(tensors):
    """Content checksum (one device sync): exact int64 sum of the fp32 bit patterns, position-weighted per tensor."""
    acc = None
    for i, t in enumerate(tensors):
        v = t.detach().reshape(-1)
        v = v.view(torch.int32) if v.dtype == torch.float32 else v.to(torch.int64)
        part = v.sum(dtype=torch.int64) * (2 * i + 1)
        acc = part if acc is None else acc + part
    return int(acc.item()) if acc is not None else 0


def _param_key(module):
    """Staleness key of a module's packed weights.  Ordinary modules: (storage pointer, version counter) of every parameter
    and buffer — load_state_dict, optimizer steps, .to() all change it.  In-place edits through ``.data`` bypass the version
    counter: call ``invalidate_packed()`` after them, or set RNC_PARAM_CHECK=checksum to key on the contents instead (costs
    one device sync per forward).  DataParallel replicas get fresh broadcast copies every forward (same addresses may hold
    new values), so they are always keyed by content."""
    ts = module_tensors(module)
    replica = any(getattr(m, "_is_replica", False) for m in module.modules())
    dev = str(ts[0].device) if ts else ""
    if replica or os.environ.get("RNC_PARAM_CHECK", "") == "checksum":
        return ("sum", dev, len(ts), _checksum(ts))
    return ("ptr", dev, _EPOCH[0]) + tuple((p.data_ptr(), p._version) for p in ts)


_EPOCH = [0]


def invalidate_packed():
    """Force every engine to re-pack weights on the next forward (needed only after in-place edits through ``.data``)."""
    _EPOCH[0] += 1


class Workspace:
    """Resident buffers for one (device, B, H8, W8).  Sized once; reused by every forward."""

    def __init__(self, device, B, H8, W8, with_mask, with_ncup):
        self.key = (str(device), B, H8, W8, with_mask, with_ncup)
        self.B, self.H8, self.W8 = B, H8, W8
        M = B * H8 * W8
        f = dict(dtype=torch.float32, device=device)
        self.hx = torch.zeros(M, HX_LD, **f)
        self.corr = torch.empty(M, CORR_CH, **f)
        self.c1 = torch.empty(M, 256, **f)
        self.corflo = torch.empty(M, 256, **f)
        self.f1 = torch.empty(M, 128, **f)
        self.z = torch.empty(M, 128, **f)
        self.rh = torch.empty(M, 128, **f)
        self.fh = torch.empty(M, 256, **f)
        self.coords1 = torch.empty(B, 2, H8, W8, **f)
        self.delta = torch.empty(B, 2, H8, W8, **f)
        self.f1_cl = None
        self.f2_pyr = None
        if with_mask:
            self.mh = torch.empty(M, 256, **f)
            self.mask = torch.empty(M, 576, **f)
        if with_ncup:
            M4 = 4 * M
            self.x4 = torch.empty(B, 2, 2 * H8, 2 * W8, **f)
            self.gin = torch.empty(M4, 132, **f)
            self.g1 = torch.empty(M4, 64, **f)
            self.g2 = torch.empty(M4, 32, **f)
            self.conf = torch.empty(B, 2, 2 * H8, 2 * W8, **f)


class _Timed:
    """CUDA-event bracket on the launching stream, active only while Engine.profile is a dict (bench.py)."""

    def __init__(self, eng, name):
        self.eng, self.name = eng, name

    def __enter__(self):
        if self.eng.profile is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *exc):
        if self.eng.profile is not None:
            self.e1.record()
            self.eng.profile.setdefault(self.name, []).append((self.e0, self.e1))
        return False


_ENGINES = {}
_ENGINES_LOCK = threading.Lock()
_ENGINE_ENV = ("RNC_CONV", "RNC_LOOKUP", "RNC_CONVF1", "RNC_FORK", "RNC_BLOCKED", "RNC_CONV_FLAGS")


def engine_for(device):
    """The engine of one CUDA device.  Engines (packed weights, workspaces, side streams) are per-device process-wide state
    that lives OUTSIDE the nn.Modules: modules stay deep-copyable / picklable, and nn.DataParallel replicas (one thread per
    device, shallow-copied module __dict__) never share packed weights or workspaces across devices."""
    device = torch.device(device)
    if device.type != "cuda":
        raise native.RncUnavailable("the RAFT-NCUP hot path runs only on CUDA (sm_90a) devices; there is no CPU fallback")
    idx = device.index if device.index is not None else torch.cuda.current_device()
    key = (idx,) + tuple(os.environ.get(k, "") for k in _ENGINE_ENV)      # developer switches select distinct engines
    eng = _ENGINES.get(key)
    if eng is None:
        with _ENGINES_LOCK:
            eng = _ENGINES.get(key)
            if eng is None:
                with torch.cuda.device(idx):
                    eng = _ENGINES[key] = make_engine()
                eng.device = torch.device("cuda", idx)
    return eng


def make_engine():
    """RNC_CONV=umma (default): wgmma tensor-core convolutions on fp16 hi/lo split operands;
    RNC_CONV=ffma: exact-fp32 CUDA-core convolutions (v1, kept as the on-GPU cross-check)."""
    mode = os.environ.get("RNC_CONV", "umma").lower()
    if mode == "ffma":
        return Engine()
    if mode == "umma":
        from .engine_umma import UmmaEngine
        return UmmaEngine()
    raise ValueError(f"RNC_CONV={mode!r}: expected 'umma' or 'ffma'")


class Engine:
    """Issues the kernels.  One per CUDA device (engine_for); keeps packed weights and workspaces.  ``lock`` serialises the
    forwards of one device (nn.DataParallel drives different devices from different threads: different engines)."""
    mode = "ffma"
    fork_convf1 = False
    PACK_UB, PACK_UP = PackedUpdateBlock, PackedUpsampler
    WS = Workspace
    MAX_WS, MAX_PACKED = 6, 64

    MAX_GRAPHS = 4

    def __init__(self):
        self.profile = None
        self._graphs = OrderedDict()        # forward signature -> captured CUDA graph (test-mode inference), LRU
        self._packed = OrderedDict()        # (kind, param key) -> packed weights, LRU
        self._ws = OrderedDict()            # workspace key -> workspace, LRU
        self.lock = threading.RLock()
        self.device = None
        self.L = native.lib()

    # ------------------------------------------------------------------ caches
    def _packed_for(self, kind, module, build):
        key = (kind,) + _param_key(module)
        hit = self._packed.get(key)
        if hit is None:
            hit = self._packed[key] = build(module)
            while len(self._packed) > self.MAX_PACKED:
                self._packed.popitem(last=False)
        else:
            self._packed.move_to_end(key)
        return hit

    def packed_update(self, ub):
        return self._packed_for("ub", ub, self.PACK_UB)

    def packed_upsampler(self, up):
        return self._packed_for("up", up, self.PACK_UP)

    def workspace(self, device, B, H8, W8, with_mask, with_ncup):
        """Resident buffers for one problem shape.  The least recently used one is dropped when a fifth shape shows up; the
        caller holds ``self.lock`` for the whole forward, so a workspace in use is never the one evicted."""
        key = (self.mode, str(device), B, H8, W8, with_mask, with_ncup)
        ws = self._ws.get(key)
        if ws is None:
            while len(self._ws) >= self.MAX_WS:
                self._ws.popitem(last=False)
            ws = self._ws[key] = self.WS(device, B, H8, W8, with_mask, with_ncup)
        else:
            self._ws.move_to_end(key)
        return ws

    # ------------------------------------------------------------------ whole-forward CUDA graphs (test-mode inference)
    def graphs_enabled(self, model):
        """A test-mode forward issues ~560 kernels; replaying them as one CUDA graph removes the host launch path (matters for
        single pairs, evaluate.py's usage, and for eight ranks sharing a host).  Off while bench.py brackets kernels with events
        (profile), for nn.DataParallel replicas (fresh weight copies every call) and with RNC_GRAPH=0."""
        if self.profile is not None or os.environ.get("RNC_GRAPH", "1") == "0":
            return False
        if os.environ.get("RNC_PARAM_CHECK", "") == "checksum" or getattr(model, "_is_replica", False):
            return False
        return not getattr(model.args, "mixed_precision", False) and os.environ.get("RNC_ENCODER", "umma").lower() == "umma" \
            and self.mode == "umma" and not self.fork_convf1

    def graph_forward(self, model, image1, image2, iters, flow_init):
        """Second and later forwards with the same signature (shape, iterations, warm start or not, weights) replay a captured
        graph: inputs are copied into the graph's static buffers, results are returned as fresh copies."""
        B, _, Him, Wim = image1.shape
        if flow_init is not None and tuple(flow_init.shape) != (B, 2, Him // 8, Wim // 8):
            raise ValueError("flow_init must be [N,2,H/8,W/8]")
        key = (type(model).__name__, tuple(image1.shape), iters, flow_init is not None, _param_key(model))
        ent = self._graphs.get(key)
        if ent is None:
            while len(self._graphs) >= self.MAX_GRAPHS:
                self._graphs.popitem(last=False)
            self._graphs[key] = {"seen": 1}
            return model._forward_eager(self, image1, image2, iters, flow_init, True)     # first sight: eager (also warms caches)
        self._graphs.move_to_end(key)
        if "graph" not in ent:
            ent["im1"], ent["im2"] = image1.detach().float().clone(), image2.detach().float().clone()
            ent["fi"] = flow_init.detach().float().clone() if flow_init is not None else None
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream(device=image1.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):                                                  # warm-up on a side stream
                model._forward_eager(self, ent["im1"], ent["im2"], iters, ent["fi"], True)
            cur.wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                ent["out"] = model._forward_eager(self, ent["im1"], ent["im2"], iters, ent["fi"], True)
                ent["net"] = model.update_block.net
            ent["graph"] = g
            # the graph addresses these buffers by pointer: keep them alive even if the LRU caches let go of them
            enc = getattr(self, "_encoder", None)
            ent["pins"] = (dict(self._ws), dict(self._packed), enc._bufs if enc is not None else None)
        ent["im1"].copy_(image1)
        ent["im2"].copy_(image2)
        if ent["fi"] is not None:
            ent["fi"].copy_(flow_init)
        ent["graph"].replay()
        model.update_block.net = ent["net"]
        lo, up = ent["out"]
        return lo.clone(), up.clone()

    # ------------------------------------------------------------------ single kernels
    def conv(self, B, H, W, in0, c0, ld0, packed, cout, kh, kw, epi, out=None, ldo=0, in1=None, c1=0, ld1=0,
             h=None, ldh=0, aux0=None, ldaux=0):
        d = ConvDesc()
        d.in0, d.c0, d.ld0 = in0, c0, ld0
        d.in1, d.c1, d.ld1 = (in1 or 0), c1, ld1
        d.weight, d.bias = packed[0].data_ptr(), packed[1].data_ptr()
        d.out, d.ldo = (out or 0), ldo
        d.h, d.ldh = (h or 0), ldh
        d.aux0, d.ldaux = (aux0 or 0), ldaux
        d.B, d.H, d.W = B, H, W
        d.cout, d.kh, d.kw, d.epilogue = cout, kh, kw, epi
        native.check(self.L.rnc_conv2d_cl_fwd(C.byref(d), _stream()), "conv2d_cl")

    def fmap_prepare(self, ws, fmap1, fmap2, levels=4):
        B, D, H, W = fmap1.shape
        total = self.L.rnc_pyramid_offset(B, D, H, W, levels)
        if ws.f1_cl is None or ws.f1_cl.numel() != B * H * W * D:
            ws.f1_cl = torch.empty(B * H * W, D, dtype=torch.float32, device=fmap1.device)
            ws.f2_pyr = torch.empty(total, dtype=torch.float32, device=fmap1.device)
        native.check(self.L.rnc_fmap_prepare(_ptr(fmap1), _ptr(fmap2), B, D, H, W, levels, _ptr(ws.f1_cl),
                                             _ptr(ws.f2_pyr), _stream()), "fmap_prepare")
        ws.D, ws.levels = D, levels

    def lookup(self, ws, coords, out, layout, ldo, radius=4):
        with _Timed(self, "corr_lookup"):
            native.check(self.L.rnc_corr_lookup_fwd(_ptr(ws.f1_cl), _ptr(ws.f2_pyr), _ptr(coords), ws.B, ws.D, ws.H8, ws.W8,
                                                    ws.levels, radius, _ptr(out), layout, ldo, _stream()), "corr_lookup")

    def begin_iter(self, ws, pk):
        """Hook called before the lookup of every iteration (the tensor-core engine forks independent work here)."""

    def lookup_resident(self, ws):
        """Per-iteration lookup at ws.coords1 into the resident corr buffer (CL fp32)."""
        self.lookup(ws, ws.coords1, ws.corr, 1, CORR_CH)

    def load_corr(self, ws, corr_nchw):
        B, _, H, W = corr_nchw.shape
        native.check(self.L.rnc_nchw_to_cl(_ptr(corr_nchw), B, CORR_CH, H, W, _ptr(ws.corr), CORR_CH, 0, _stream()), "nchw_to_cl(corr)")

    def guidance(self, ws):
        """(pointer, pixel stride) of the CL fp32 hidden state used as NCUP guidance (update.py:135, raft_nc_dbl.py:161)."""
        return ws.hx.data_ptr(), HX_LD

    # ------------------------------------------------------------------ update block on resident buffers
    def update_iter(self, ws, pk, want_mask=False, want_delta=False):
        """update.py:130-141 on the CL workspace: consumes ws.corr and ws.coords1, advances ws.hx[:, :128] (net) and
        ws.coords1 (raft_nc_dbl.py:157).  Optionally leaves the mask logits in ws.mask and delta in ws.delta."""
        with _Timed(self, "update_block"):
            self._update_iter(ws, pk, want_mask, want_delta)

    def _update_iter(self, ws, pk, want_mask, want_delta):
        self._motion_encoder_ffma(ws, pk)
        self._gru_ffma(ws, pk)
        self._flow_head_ffma(ws, pk, want_delta)
        if want_mask:
            # mask head (update.py:123-126,140), 0.25 folded into the 1x1 weights
            B, H, W = ws.B, ws.H8, ws.W8
            self.conv(B, H, W, ws.hx.data_ptr(), 128, HX_LD, pk.m0, 256, 3, 3, native.EPI_RELU, ws.mh.data_ptr(), 256)
            self.conv(B, H, W, ws.mh.data_ptr(), 256, 256, pk.m2, 576, 1, 1, native.EPI_LINEAR, ws.mask.data_ptr(), 576)

    # The three pieces below run the exact fp32 CUDA-core kernels on an `ffma` Workspace; they are the whole update block of
    # the RNC_CONV=ffma engine and the bodies of the operator seams FlowHead / SepConvGRU / BasicMotionEncoder.forward.
    def _motion_encoder_ffma(self, ws, pk):
        """BasicMotionEncoder (update.py:89-97): ws.corr, ws.coords1 -> hx[:, 256:384] = [motion(126) | flow(2)]."""
        B, H, W = ws.B, ws.H8, ws.W8
        mot_ptr = ws.hx.data_ptr() + 256 * 4
        self.conv(B, H, W, ws.corr.data_ptr(), CORR_CH, CORR_CH, pk.convc1, 256, 1, 1, native.EPI_RELU, ws.c1.data_ptr(), 256)
        self.conv(B, H, W, ws.c1.data_ptr(), 256, 256, pk.convc2, 192, 3, 3, native.EPI_RELU, ws.corflo.data_ptr(), 256)
        native.check(self.L.rnc_conv_flow7x7_fwd(_ptr(ws.coords1), _ptr(pk.convf1[0]), _ptr(pk.convf1[1]), B, H, W, 128,
                                                 _ptr(ws.f1), 128, _stream()), "convf1")
        self.conv(B, H, W, ws.f1.data_ptr(), 128, 128, pk.convf2, 64, 3, 3, native.EPI_RELU, ws.corflo.data_ptr() + 192 * 4, 256)
        self.conv(B, H, W, ws.corflo.data_ptr(), 256, 256, pk.conv, 126, 3, 3, native.EPI_RELU_FLOW, mot_ptr, HX_LD,
                  aux0=ws.coords1.data_ptr(), ldaux=0)

    def _gru_ffma(self, ws, pk):
        """SepConvGRU (update.py:45-60): horizontal (1x5) then vertical (5x1) half steps on hx = [h | x]; h in place."""
        B, H, W = ws.B, ws.H8, ws.W8
        hx = ws.hx.data_ptr()
        x_ptr = hx + 128 * 4          # channels 128.. = [inp | motion | flow]
        for zr, q, kh, kw in ((pk.zr1, pk.q1, 1, 5), (pk.zr2, pk.q2, 5, 1)):
            self.conv(B, H, W, hx, HX_LD, HX_LD, zr, 256, kh, kw, native.EPI_GRU_ZR, ws.rh.data_ptr(), 128,
                      h=hx, ldh=HX_LD, aux0=ws.z.data_ptr(), ldaux=128)
            self.conv(B, H, W, ws.rh.data_ptr(), 128, 128, q, 128, kh, kw, native.EPI_GRU_Q, in1=x_ptr, c1=256, ld1=HX_LD,
                      h=hx, ldh=HX_LD, aux0=ws.z.data_ptr(), ldaux=128)

    def _flow_head_ffma(self, ws, pk, want_delta):
        """FlowHead (update.py:13-14) + coords1 += delta (raft_nc_dbl.py:157)."""
        B, H, W = ws.B, ws.H8, ws.W8
        self.conv(B, H, W, ws.hx.data_ptr(), 128, HX_LD, pk.fh1, 256, 3, 3, native.EPI_RELU, ws.fh.data_ptr(), 256)
        native.check(self.L.rnc_flow_head2_fwd(_ptr(ws.fh), 256, 256, _ptr(pk.fh2[0]), _ptr(pk.fh2[1]), B, H, W,
                                               _ptr(ws.delta) if want_delta else C.c_void_p(0), _ptr(ws.coords1), _stream()),
                     "flow_head2")

    def ffma_workspace(self, device, B, H8, W8, with_mask=False, with_ncup=False):
        """Workspace of the exact fp32 CUDA-core kernels (operator seams), whatever this engine's own mode is."""
        key = ("ffma", str(device), B, H8, W8, with_mask, with_ncup)
        ws = self._ws.get(key)
        if ws is None:
            while len(self._ws) >= self.MAX_WS:
                self._ws.popitem(last=False)
            ws = self._ws[key] = Workspace(device, B, H8, W8, with_mask, with_ncup)
        else:
            self._ws.move_to_end(key)
        return ws

    def load_state(self, ws, net, inp):
        """NCHW net/inp (raft_nc_dbl.py:137-140) -> resident hx buffer."""
        B, _, H, W = net.shape
        s = _stream()
        native.check(self.L.rnc_nchw_to_cl(_ptr(net), B, 128, H, W, _ptr(ws.hx), HX_LD, 0, s), "nchw_to_cl(net)")
        native.check(self.L.rnc_nchw_to_cl(_ptr(inp), B, 128, H, W, _ptr(ws.hx), HX_LD, 128, s), "nchw_to_cl(inp)")

    def net_nchw(self, ws):
        out = torch.empty(ws.B, 128, ws.H8, ws.W8, dtype=torch.float32, device=ws.hx.device)
        native.check(self.L.rnc_cl_to_nchw(_ptr(ws.hx), HX_LD, 0, ws.B, 128, ws.H8, ws.W8, _ptr(out), _stream()), "cl_to_nchw")
        return out

    def flow_low(self, ws):
        out = torch.empty_like(ws.coords1)
        native.check(self.L.rnc_coords_to_flow(_ptr(ws.coords1), _ptr(out), ws.B, ws.H8, ws.W8, _stream()), "coords_to_flow")
        return out

    # ------------------------------------------------------------------ upsamplers
    def convex_upsample(self, ws, flow_low, mask_cl, ldm):
        out = torch.empty(ws.B, 2, 8 * ws.H8, 8 * ws.W8, dtype=torch.float32, device=flow_low.device)
        with _Timed(self, "convex"):
            native.check(self.L.rnc_convex_upsample_fwd(_ptr(flow_low), _ptr(mask_cl), ldm, ws.B, ws.H8, ws.W8, _ptr(out),
                                                        _stream()), "convex_upsample")
        return out

    def ncup_from_lowres(self, ws, pu, x_lowres, guid_ptr, ldg, out_scale):
        """NConvUpsampler.forward (upsampler.py:143-177) on x_lowres NCHW [B,2,H4,W4] with CL guidance at H8."""
        B, H8, W8 = ws.B, ws.H8, ws.W8
        H4, W4 = 2 * H8, 2 * W8
        s = _stream()
        native.check(self.L.rnc_ncup_guidance_fwd(_ptr(x_lowres), C.c_void_p(guid_ptr), ldg, 128, B, H8, W8, _ptr(ws.gin),
                                                  132, s), "ncup_guidance")
        self.conv(B, H4, W4, ws.gin.data_ptr(), pu.cin0_pad, 132, pu.g0, pu.c_mid0, 3, 3, native.EPI_RELU, ws.g1.data_ptr(), 64)
        self.conv(B, H4, W4, ws.g1.data_ptr(), pu.c_mid0, 64, pu.g1, pu.c_mid1, 3, 3, native.EPI_RELU, ws.g2.data_ptr(), 32)
        native.check(self.L.rnc_conf_head_fwd(_ptr(ws.g2), pu.c_mid1, 32, _ptr(pu.gout[0]), _ptr(pu.gout[1]), B, H4, W4,
                                              _ptr(ws.conf), s), "conf_head")
        out = torch.empty(B, 2, 4 * H4, 4 * W4, dtype=torch.float32, device=x_lowres.device)
        with _Timed(self, "ncup"):
            native.check(self.L.rnc_ncup_fwd(_ptr(x_lowres), _ptr(ws.conf), pu.nconv_host, B, H4, W4, out_scale, _ptr(out), s), "ncup")
        return out
