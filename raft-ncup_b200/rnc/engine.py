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
from collections import OrderedDict, namedtuple

import torch
import torch.nn.functional as F

from . import native
from .native import ConvDesc, rnc
from .nconv_unet import PackedUNet, is_fused

CORR_CH = 324          # 4 levels * 9 * 9
HX_LD = 384            # [h | inp | motion(126) flow(2)]


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


def fold_bn(conv, bn=None):
    """fp32 (weight, bias) of nn.Conv2d `conv` followed by an eval-mode BatchNorm2d `bn` (running statistics), or of `conv`
    alone when bn is None: s = gamma / sqrt(var + eps), weight * s, (bias - mean) * s + beta."""
    w, b = conv.weight.detach().float(), conv.bias.detach().float()
    if bn is None:
        return w, b
    s = bn.weight.detach() / torch.sqrt(bn.running_var + bn.eps)
    return w * s.view(-1, 1, 1, 1), (b - bn.running_mean) * s + bn.bias.detach()


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


def conv_dilation(conv):
    """The dilation a kernel applies for nn.Conv2d `conv` (square, odd filter): a 1x1 filter reads one pixel whatever it is."""
    return conv.dilation[0] if conv.kernel_size[0] > 1 else 1


def _ceil4(c):
    return (c + 3) // 4 * 4


class ExactWnet:
    """The weights net's format on the exact fp32 kernels: fp32 channel-last layer outputs of ceil4 channels, a convolution
    head's output [M, 4]."""
    split, head_pitch = False, 4
    pitch = staticmethod(_ceil4)

    @staticmethod
    def pack(w, b, cin):
        return pack_conv(w, b, cin_pad=cin)

    @staticmethod
    def buffer(M, layer, device):
        # the next layer reads the whole pitch: zero the columns the kernel does not write
        return (torch.empty if layer.pitch == layer.cout else torch.zeros)(M, layer.pitch, dtype=torch.float32, device=device)

    @staticmethod
    def conv(eng, B, H, W, x, c, ld, layer, epi, y):
        eng.conv(B, H, W, x.data_ptr(), c, ld, layer.wt, layer.cout, layer.k, layer.k, epi, y.data_ptr(), layer.pitch, dil=layer.dil)


# one convolution of the weights net: packed weights, filter size, dilation, output width, and its output's form (split
# halves or fp32) and pitch
WnetLayer = namedtuple("WnetLayer", "wt cout k dil split pitch")


class PackedSimple:
    """Kernel-ready weights of the weights net Simple (interp_weights_est.py:10-47) in one engine format fmt (ExactWnet,
    engine_umma.UmmaWnet).  It reads cin channels of its input (zero beyond in_ch); its hidden layers, eval-mode BatchNorm folded
    in, each read the previous output's pitch columns.  The head `out` + sigmoid: a 1x1 head on an fp32 input runs on
    rnc_conf_head_fwd (conf_head, its weight rows padded to that pitch), any other is a convolution with a sigmoid epilogue
    (conv_head).  The last hidden layer writes fp32 when the conf head reads it."""

    def __init__(self, wn, fmt):
        self.fmt, self.cin = fmt, _ceil4(wn.in_ch)
        out, n = wn.out, len(wn.conv)
        conf = out.kernel_size[0] == 1 and (n > 0 or not fmt.split)
        self.layers, pitch = [], self.cin
        for i, blk in enumerate(wn.conv):
            w, b = fold_bn(blk[0], blk[1] if len(blk) == 3 else None)      # Conv, BatchNorm, ReLU or Conv, ReLU (:26-30)
            cout = w.shape[0]
            self.layers.append(WnetLayer(fmt.pack(w, b, pitch), cout, blk[0].kernel_size[0], conv_dilation(blk[0]),
                                         fmt.split and not (conf and i == n - 1), fmt.pitch(cout)))
            pitch = self.layers[-1].pitch
        self.conf_head = self.conv_head = None
        if conf:
            w = pack_thin(out.weight)
            self.conf_head = (F.pad(w, (0, 0, 0, pitch - w.shape[1])), out.bias.detach().float().contiguous())
        else:
            self.conv_head = WnetLayer(fmt.pack(out.weight, out.bias, pitch), 2, out.kernel_size[0], conv_dilation(out), False,
                                       fmt.head_pitch)
        self.outputs = self.layers + ([self.conv_head] if self.conv_head else [])
        self.layout = tuple((l.cout, l.split, l.pitch) for l in self.outputs)

    def buffers(self, M, device):
        """The outputs of the layers, then of a convolution head, for M pixels."""
        return [self.fmt.buffer(M, l, device) for l in self.outputs]


class PackedUpsampler:
    """Kernel-ready weights of NConvUpsampler (upsampler.py:75-141): the BN-folded weights net in one engine format (wnet) and
    the NConvUNet: the fused network's softplus'd NConv weights (nconv_host) or the per-level chain (unet)."""

    def __init__(self, up, fmt):
        self.wnet = PackedSimple(up.weights_est_net, fmt)
        net = up.interpolation_net
        self.nconv_host = self.unet = None
        if is_fused(net):
            ws = [F.softplus(p.detach().float(), beta=10).reshape(-1).cpu() for p in
                  (net.nconv_in.weight_p, net.nconv_x2[0].weight_p, net.decoder[0].weight_p, net.nconv_out.weight_p)]
            self.nconv_host = (C.c_float * 224)(*torch.cat(ws).tolist())
        else:
            self.unet = PackedUNet(net)       # every other configuration: the per-level chain of rnc/nconv_unet.py


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


def _lru_get(cache, key, capacity, build):
    """cache[key] of an OrderedDict used as an LRU cache, marked most recently used; on a miss the least recently used entries
    are dropped to make room for build(), which is stored under key."""
    hit = cache.get(key)
    if hit is None:
        while len(cache) >= capacity:
            cache.popitem(last=False)
        hit = cache[key] = build()
    else:
        cache.move_to_end(key)
    return hit


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
            self.conf = torch.empty(B, 2, 2 * H8, 2 * W8, **f)
        self.wnet = {}              # weights-net layer outputs at 1/4 resolution, per PackedSimple.layout
        self.nconv_bufs = {}        # NConvUNet chain intermediates (PackedUNet.run)


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
_ENGINE_ENV = ("RNC_CONV", "RNC_LOOKUP")


def engine_for(device):
    """The engine of one CUDA device.  Engines (packed weights, workspaces) are per-device process-wide state
    that lives OUTSIDE the nn.Modules: modules stay deep-copyable / picklable, and nn.DataParallel replicas (one thread per
    device, shallow-copied module __dict__) never share packed weights or workspaces across devices."""
    device = torch.device(device)
    if device.type != "cuda":
        raise native.RncUnavailable("the RAFT-NCUP hot path runs only on CUDA (sm_90a) devices; there is no CPU fallback")
    idx = device.index if device.index is not None else torch.cuda.current_device()
    key = (idx,) + tuple(os.environ.get(k, "") for k in _ENGINE_ENV)      # RNC_CONV / RNC_LOOKUP select distinct engines
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
    PACK_UB, PACK_UP = PackedUpdateBlock, ExactWnet         # PACK_UP: the upsampler's weights-net format
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
        self.L = native.lib()               # the raw handle, for code that calls an entry point directly; see native.rnc

    # ------------------------------------------------------------------ caches
    def _packed_for(self, kind, module, build):
        return _lru_get(self._packed, (kind,) + _param_key(module), self.MAX_PACKED, lambda: build(module))

    def packed_update(self, ub):
        return self._packed_for("ub", ub, self.PACK_UB)

    def packed_upsampler(self, up):
        return self._packed_for("up", up, lambda m: PackedUpsampler(m, self.PACK_UP))

    def workspace(self, device, B, H8, W8, with_mask=False, with_ncup=False, mode=None):
        """Resident buffers for one problem shape, in the format of this engine's kernels, or with mode="ffma" of the exact
        fp32 CUDA-core kernels whatever this engine's mode is (the operator seams).  The least recently used workspace is
        dropped when a seventh one is needed; the caller holds ``self.lock`` for the whole forward, so a workspace in use is
        never the one evicted."""
        mode = mode or self.mode
        ws_cls = Workspace if mode == "ffma" else self.WS
        return _lru_get(self._ws, (mode, str(device), B, H8, W8, with_mask, with_ncup), self.MAX_WS,
                        lambda: ws_cls(device, B, H8, W8, with_mask, with_ncup))

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
            and self.mode == "umma"

    def graph_forward(self, model, image1, image2, iters, flow_init, return_confidence=False, bidirectional=False):
        """Second and later forwards with the same signature (shape, iterations, warm start or not, weights, confidence or
        not, bidirectional or not) replay a captured graph: inputs are copied into the graph's static buffers, results are
        returned as fresh copies.  bidirectional: the pass of model.forward_bidirectional, flow_init [2B,2,H/8,W/8]."""
        B, _, Him, Wim = image1.shape
        if flow_init is not None and tuple(flow_init.shape) != ((2 if bidirectional else 1) * B, 2, Him // 8, Wim // 8):
            raise ValueError("flow_init must be [N,2,H/8,W/8]")
        # a graph records one mode's kernels: the deterministic mode gets its own (torch.use_deterministic_algorithms)
        key = (type(model).__name__, tuple(image1.shape), iters, flow_init is not None, _param_key(model),
               torch.are_deterministic_algorithms_enabled(), return_confidence) + (("bidirectional",) if bidirectional else ())
        first = key not in self._graphs
        ent = _lru_get(self._graphs, key, self.MAX_GRAPHS, dict)
        conf = dict(return_confidence=True) if return_confidence else {}

        def eager(im1, im2, fi):
            if bidirectional:
                return model._forward_bidirectional(self, im1, im2, iters, fi, return_confidence)
            return model._forward_eager(self, im1, im2, iters, fi, True, **conf)
        if first:       # first sight: eager (also warms caches)
            return eager(image1, image2, flow_init)
        if "graph" not in ent:
            ent["im1"], ent["im2"] = image1.detach().float().clone(), image2.detach().float().clone()
            ent["fi"] = flow_init.detach().float().clone() if flow_init is not None else None
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream(device=image1.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):                                                  # warm-up on a side stream
                eager(ent["im1"], ent["im2"], ent["fi"])
            cur.wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                ent["out"] = eager(ent["im1"], ent["im2"], ent["fi"])
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
        return tuple(t.clone() for t in ent["out"])

    # ------------------------------------------------------------------ single kernels
    def conv(self, B, H, W, in0, c0, ld0, packed, cout, kh, kw, epi, out=None, ldo=0, in1=None, c1=0, ld1=0,
             h=None, ldh=0, aux0=None, ldaux=0, dil=1):
        d = ConvDesc()
        d.in0, d.c0, d.ld0 = in0, c0, ld0
        d.in1, d.c1, d.ld1 = (in1 or 0), c1, ld1
        d.weight, d.bias = packed[0].data_ptr(), packed[1].data_ptr()
        d.out, d.ldo = (out or 0), ldo
        d.h, d.ldh = (h or 0), ldh
        d.aux0, d.ldaux = (aux0 or 0), ldaux
        d.B, d.H, d.W = B, H, W
        d.cout, d.kh, d.kw, d.epilogue = cout, kh, kw, epi
        if dil > 1:
            rnc.conv2d_cl_dil_fwd(d, dil)
        else:
            rnc.conv2d_cl_fwd(d)

    def alloc_fmaps(self, ws, B, D, H, W, levels, device):
        """Allocate the CL feature map / pyramid buffers of ws, which fmap_prepare fills and the tensor-core encoder heads
        write into directly."""
        total = rnc.pyramid_offset(B, D, H, W, levels)
        if ws.f1_cl is None or ws.f1_cl.numel() != B * H * W * D:
            ws.f1_cl = torch.empty(B * H * W, D, dtype=torch.float32, device=device)
            ws.f2_pyr = torch.empty(total, dtype=torch.float32, device=device)
        ws.D, ws.levels = D, levels

    def fmap_prepare(self, ws, fmap1, fmap2, levels=4):
        B, D, H, W = fmap1.shape
        self.alloc_fmaps(ws, B, D, H, W, levels, fmap1.device)
        rnc.fmap_prepare(fmap1, fmap2, B, D, H, W, levels, ws.f1_cl, ws.f2_pyr)

    def lookup(self, ws, coords, out, layout, ldo, radius=4):
        with _Timed(self, "corr_lookup"):
            rnc.corr_lookup_fwd(ws.f1_cl, ws.f2_pyr, coords, ws.B, ws.D, ws.H8, ws.W8, ws.levels, radius, out, layout, ldo)

    def lookup_resident(self, ws):
        """Per-iteration lookup at ws.coords1 into the resident corr buffer (CL fp32)."""
        self.lookup(ws, ws.coords1, ws.corr, 1, CORR_CH)

    def load_corr(self, ws, corr_nchw):
        B, _, H, W = corr_nchw.shape
        rnc.nchw_to_cl(corr_nchw, B, CORR_CH, H, W, ws.corr, CORR_CH, 0)

    def guidance(self, ws):
        """(tensor, pixel stride) of the CL fp32 hidden state used as NCUP guidance (update.py:135, raft_nc_dbl.py:161)."""
        return ws.hx, HX_LD

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
        mot_ptr = ws.hx[:, 256:].data_ptr()
        self.conv(B, H, W, ws.corr.data_ptr(), CORR_CH, CORR_CH, pk.convc1, 256, 1, 1, native.EPI_RELU, ws.c1.data_ptr(), 256)
        self.conv(B, H, W, ws.c1.data_ptr(), 256, 256, pk.convc2, 192, 3, 3, native.EPI_RELU, ws.corflo.data_ptr(), 256)
        rnc.conv_flow7x7_fwd(ws.coords1, pk.convf1[0], pk.convf1[1], B, H, W, 128, ws.f1, 128)
        self.conv(B, H, W, ws.f1.data_ptr(), 128, 128, pk.convf2, 64, 3, 3, native.EPI_RELU, ws.corflo[:, 192:].data_ptr(), 256)
        self.conv(B, H, W, ws.corflo.data_ptr(), 256, 256, pk.conv, 126, 3, 3, native.EPI_RELU_FLOW, mot_ptr, HX_LD,
                  aux0=ws.coords1.data_ptr(), ldaux=0)

    def _gru_ffma(self, ws, pk):
        """SepConvGRU (update.py:45-60): horizontal (1x5) then vertical (5x1) half steps on hx = [h | x]; h in place."""
        B, H, W = ws.B, ws.H8, ws.W8
        hx = ws.hx.data_ptr()
        x_ptr = ws.hx[:, 128:].data_ptr()          # channels 128.. = [inp | motion | flow]
        for zr, q, kh, kw in ((pk.zr1, pk.q1, 1, 5), (pk.zr2, pk.q2, 5, 1)):
            self.conv(B, H, W, hx, HX_LD, HX_LD, zr, 256, kh, kw, native.EPI_GRU_ZR, ws.rh.data_ptr(), 128,
                      h=hx, ldh=HX_LD, aux0=ws.z.data_ptr(), ldaux=128)
            self.conv(B, H, W, ws.rh.data_ptr(), 128, 128, q, 128, kh, kw, native.EPI_GRU_Q, in1=x_ptr, c1=256, ld1=HX_LD,
                      h=hx, ldh=HX_LD, aux0=ws.z.data_ptr(), ldaux=128)

    def _flow_head_ffma(self, ws, pk, want_delta):
        """FlowHead (update.py:13-14) + coords1 += delta (raft_nc_dbl.py:157)."""
        B, H, W = ws.B, ws.H8, ws.W8
        self.conv(B, H, W, ws.hx.data_ptr(), 128, HX_LD, pk.fh1, 256, 3, 3, native.EPI_RELU, ws.fh.data_ptr(), 256)
        rnc.flow_head2_fwd(ws.fh, 256, 256, pk.fh2[0], pk.fh2[1], B, H, W, ws.delta if want_delta else None, ws.coords1)

    def load_state(self, ws, net, inp):
        """NCHW net/inp (raft_nc_dbl.py:137-140) -> resident hx buffer."""
        B, _, H, W = net.shape
        rnc.nchw_to_cl(net, B, 128, H, W, ws.hx, HX_LD, 0)
        rnc.nchw_to_cl(inp, B, 128, H, W, ws.hx, HX_LD, 128)

    def net_nchw(self, ws):
        out = torch.empty(ws.B, 128, ws.H8, ws.W8, dtype=torch.float32, device=ws.hx.device)
        rnc.cl_to_nchw(ws.hx, HX_LD, 0, ws.B, 128, ws.H8, ws.W8, out)
        return out

    def flow_low(self, ws):
        out = torch.empty_like(ws.coords1)
        rnc.coords_to_flow(ws.coords1, out, ws.B, ws.H8, ws.W8)
        return out

    # ------------------------------------------------------------------ upsamplers
    def convex_upsample(self, ws, flow_low, mask_cl, ldm):
        out = torch.empty(ws.B, 2, 8 * ws.H8, 8 * ws.W8, dtype=torch.float32, device=flow_low.device)
        with _Timed(self, "convex"):
            rnc.convex_upsample_fwd(flow_low, mask_cl, ldm, ws.B, ws.H8, ws.W8, out)
        return out

    def stage_guidance(self, ws, x_lowres, guid, ldg):
        """The weights net's input [x_lowres | guidance upsampled x2 | 0 0] at 1/4 resolution, written to ws.gin -> (ws.gin,
        its pitch)."""
        rnc.ncup_guidance_fwd(x_lowres, guid, ldg, 128, ws.B, ws.H8, ws.W8, ws.gin, 132)
        return ws.gin, 132

    def ncup_from_lowres(self, ws, pu, x_lowres, guid, ldg, out_scale, want_conf=False):
        """NConvUpsampler.forward (upsampler.py:143-177) on x_lowres NCHW [B,2,H4,W4] with CL guidance guid at H8 (pixel
        stride ldg); want_conf: (out, output confidence) as ncup_chain."""
        x, ld = self.stage_guidance(ws, x_lowres, guid, ldg)
        wn = pu.wnet
        bufs = ws.wnet.get(wn.layout)
        if bufs is None:            # allocated by the first (eager) forward of a shape, reused by graph capture
            bufs = ws.wnet[wn.layout] = wn.buffers(4 * ws.B * ws.H8 * ws.W8, ws.conf.device)
        self.weights_net(wn, ws.B, 2 * ws.H8, 2 * ws.W8, x, ld, bufs, ws.conf)
        return self.ncup_chain(ws, pu, x_lowres, ws.conf, out_scale, want_conf=want_conf)

    def weights_net(self, pk, B, H, W, x, ld, bufs, conf):
        """Simple.forward (interp_weights_est.py:39-47) on the kernels of pk's format: x CL [B*H*W, >= pk.cin] of pitch ld
        (zero beyond the input channels) -> conf NCHW [B,2,H,W]; bufs = pk.buffers(B*H*W)."""
        c = pk.cin
        for layer, y in zip(pk.layers, bufs):
            pk.fmt.conv(self, B, H, W, x, c, ld, layer, native.EPI_RELU, y)
            x, c, ld = y, layer.pitch, layer.pitch
        if pk.conf_head is not None:
            rnc.conf_head_fwd(x, c, ld, *pk.conf_head, B, H, W, conf)
            return
        y = bufs[-1]
        pk.fmt.conv(self, B, H, W, x, c, ld, pk.conv_head, native.EPI_SIGMOID, y)
        rnc.cl_to_nchw(y, pk.conv_head.pitch, 0, B, 2, H, W, conf)

    def ncup_chain(self, ws, pu, x_lowres, conf, out_scale, want_conf=False):
        """Zero-stuffing + NConvUNet + out_scale (upsampler.py:150-177) on x_lowres, conf NCHW [B,2,H4,W4] -> [B,2,4*H4,4*W4]:
        the fused rnc_ncup_fwd for the shipped network, the per-level chain of rnc/nconv_unet.py for any other.  Neither
        synchronises with the host, so graph capture records either.  want_conf: return (out, confidence), the network's
        output confidence (the cout upsampler.py:168 discards) in the layout of out, without out_scale; out is the same
        either way."""
        B, _, H4, W4 = x_lowres.shape
        if pu.unet is None:
            out = torch.empty(B, 2, 4 * H4, 4 * W4, dtype=torch.float32, device=x_lowres.device)
            cout = torch.empty_like(out) if want_conf else None
            with _Timed(self, "ncup"):
                rnc.ncup_fwd(x_lowres, conf, pu.nconv_host, B, H4, W4, out_scale, out, cout)
            return (out, cout) if want_conf else out
        # intermediates live in the workspace (allocated by the first, eager forward of a shape; graph capture reuses them)
        bufs = ws.nconv_bufs
        if "stuffed" not in bufs:
            # zero-stuffing (upsampler.py:179-210): only the lattice is ever written, so the zeros are laid down once
            bufs["stuffed"] = torch.zeros(2, B * 2, 1, 4 * H4, 4 * W4, dtype=torch.float32, device=x_lowres.device)
        xh, ch = bufs["stuffed"]
        with _Timed(self, "ncup"):
            xh.view(B, 2, 4 * H4, 4 * W4)[:, :, 2::4, 2::4] = x_lowres
            ch.view(B, 2, 4 * H4, 4 * W4)[:, :, 2::4, 2::4] = conf
            out, cout = pu.unet.run(xh, ch, out_scale, bufs)
        out = out.view(B, 2, 4 * H4, 4 * W4)
        # nconv_out's outputs are new tensors (PackedUNet.run), not workspace buffers: the next call does not overwrite them
        return (out, cout.view(B, 2, 4 * H4, 4 * W4)) if want_conf else out
