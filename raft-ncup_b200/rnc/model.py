"""RAFT / RAFT-NCUP model shells: the drop-in boundary (SURVEY.md §8b).

Mirrors ``RAFT(nn.Module)`` of core/raft.py:24-143 (convex upsampler) and core/raft_nc_dbl.py:26-173 (NCUP upsampler):
same ctor Namespace, ``forward(image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False)``, return values
and state_dict keys.  The iteration loop runs entirely on resident channel-last buffers through librnc.so.  The NCUP model
also returns the upsampler's output confidence on request (``return_confidence=True``).
"""
import os
from collections import OrderedDict

import torch
import torch.nn as nn

from .engine import _Timed, _require_cuda, engine_for, module_device, module_tensors
from .modules import BasicEncoder, BasicUpdateBlock, get_upsampler
from .native import rnc
from .slot_plan import CARRY, NEW, images, runs, slot_plan


class _RAFTBase(nn.Module):
    ncup = False

    def __init__(self, args):
        super().__init__()
        self.args = args
        if args.small:
            # the reference's --small path crashes (raft.py:134 passes align_corners= to upflow8, SURVEY.md C7)
            raise NotImplementedError("--small is out of scope: it is broken in the reference and unused by its scripts")
        self.hidden_dim = self.context_dim = 128
        args.corr_levels = 4
        args.corr_radius = 4
        args.dropout = 0     # raft.py:41-42: `'dropout' not in args._get_kwargs()` is always true -> dropout forced to 0
        self.fnet = BasicEncoder(output_dim=256, norm_fn="instance", dropout=args.dropout)
        self.cnet = BasicEncoder(output_dim=256, norm_fn="batch", dropout=args.dropout)
        self.update_block = BasicUpdateBlock(self.args, hidden_dim=128)

    # ------------------------------------------------------------------ reference helpers kept verbatim in meaning
    def freeze_bn(self):
        for m in self.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.eval()

    def initialize_flow(self, img):
        """raft.py:63-71: two identical coordinate grids at 1/8 resolution (flow = coords1 - coords0)."""
        N, _, H, W = img.shape
        ys, xs = torch.meshgrid(torch.arange(H // 8, device=img.device), torch.arange(W // 8, device=img.device), indexing="ij")
        g = torch.stack([xs, ys], 0).float()[None].repeat(N, 1, 1, 1)
        return g, g.clone()

    def engine(self, device=None):
        """The per-device engine (rnc.engine.engine_for) this model's forwards run on.  Nothing is cached on the module:
        it stays deep-copyable / picklable, and nn.DataParallel replicas resolve their own device's engine."""
        return engine_for(device if device is not None else module_device(self))

    # ------------------------------------------------------------------ forward
    def _needs_grad(self):
        return torch.is_grad_enabled() and any(t.requires_grad for t in module_tensors(self))

    def forward(self, image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False, return_confidence=False):
        """Estimate optical flow between a pair of frames (raft_nc_dbl.py:115-173 / raft.py:87-143).

        return_confidence (NCUP model only): also return the NCUP upsampler's per-pixel output confidence in [0, 1], shaped
        like flow_up ([N,2,H,W], one plane per flow component): (flow_low, flow_up, confidence_up) in test mode, else
        (flow_predictions, confidence_predictions), one entry per iteration.  The flows are the same as without it."""
        if return_confidence and not self.ncup:
            raise ValueError("return_confidence: the convex-upsampling RAFT has no NCUP upsampler and so no output confidence")
        dev = _require_cuda(image1, image2, flow_init)
        pdev = module_device(self)
        if pdev != dev:
            raise ValueError(f"model parameters are on {pdev} but the images are on {dev}")
        eng = engine_for(dev)
        # the kernels launch on `dev`'s current stream whatever device is current in the calling thread (nn.DataParallel
        # worker threads, a model on cuda:1 in a cuda:0 process); one forward at a time per device
        with torch.cuda.device(dev), eng.lock:
            return self._forward(eng, image1, image2, iters, flow_init, test_mode, bool(return_confidence))

    def _forward(self, eng, image1, image2, iters, flow_init, test_mode, conf=False):
        if iters < 1:
            raise ValueError("iters must be >= 1")
        if hasattr(self, "data_idx"):
            self.data_idx += 1
        if image1.shape[2] % 8 or image1.shape[3] % 8:
            raise ValueError("image height/width must be multiples of 8 (pad with utils.utils.InputPadder, evaluate.py:125)")
        if self._needs_grad():
            # training path (train.py:215): the same graph with autograd, exact-fp32 kernels forward and backward
            if frozen_trunk(self, image1, image2, flow_init):
                # only the upsampler trains: the trunk runs on the inference engine, the upsampler on autograd
                return self._forward_eager(eng, image1, image2, iters, flow_init, test_mode, upsample=self._upsample_frozen,
                                           return_confidence=conf)
            from .train import raft_forward_train
            return raft_forward_train(self, image1, image2, iters, flow_init, test_mode, return_confidence=conf)
        if test_mode and eng.graphs_enabled(self):
            return eng.graph_forward(self, image1, image2, iters, flow_init, return_confidence=conf)
        return self._forward_eager(eng, image1, image2, iters, flow_init, test_mode, return_confidence=conf)

    def _forward_eager(self, eng, image1, image2, iters, flow_init, test_mode, upsample=None, encode=None, ws=None,
                       return_confidence=False):
        """The iteration loop on the engine's resident buffers.  upsample(eng, ws, pu) produces each full-resolution prediction
        from the workspace; the default is the inference upsampler (self._upsample on packed weights).  encode(eng, ws, image1,
        image2) fills the feature maps and the GRU state; the default is EncoderStage's pair plan (fnet on both frames, cnet on
        frame 1).  ws: a workspace the caller owns instead of the engine's shared one of this shape; with an encode that fills
        more slots than the images' batch (the bidirectional plan), flow_init is [ws.B,2,H/8,W/8].  return_confidence:
        upsample(eng, ws, pu, True) returns (flow, confidence), and the forward returns the confidences next to the flows
        (forward's return_confidence)."""
        B, _, Him, Wim = image1.shape
        H8, W8 = Him // 8, Wim // 8
        pk = eng.packed_update(self.update_block)
        pu = None
        if upsample is None:
            upsample = self._upsample
            pu = eng.packed_upsampler(self.upsampler) if self.ncup else None
            if self.ncup and any(isinstance(m, nn.BatchNorm2d) and m.training for m in self.upsampler.modules()):
                raise NotImplementedError("weights-net BatchNorm with batch statistics needs the training path (enable grad) "
                                          "or eval mode: call .eval() / freeze_bn()")
        if ws is None:
            ws = eng.workspace(image1.device, B, H8, W8, pk.has_mask, self.ncup)
        (encode or EncoderStage(self))(eng, ws, image1, image2)
        fi = None
        if flow_init is not None:
            fi = flow_init.to(image1.device).float().contiguous()
            if fi.shape != (ws.B, 2, H8, W8):
                raise ValueError("flow_init must be [N,2,H/8,W/8]")
        rnc.coords_init(ws.coords1, fi, ws.B, H8, W8)

        preds, confs = [], []
        flow_up = conf_up = None
        for itr in range(iters):
            last = itr == iters - 1
            need_up = last or not test_mode     # inference upsamples once (SURVEY.md finding 9); list mode needs all
            eng.lookup_resident(ws)
            eng.update_iter(ws, pk, want_mask=(pk.has_mask and need_up))
            if need_up:
                if return_confidence:
                    flow_up, conf_up = upsample(eng, ws, pu, True)
                    confs.append(conf_up)
                else:
                    flow_up = upsample(eng, ws, pu)
                preds.append(flow_up)
        self.update_block.net = eng.net_nchw(ws)
        if test_mode:
            return (eng.flow_low(ws), flow_up, conf_up) if return_confidence else (eng.flow_low(ws), flow_up)
        return (preds, confs) if return_confidence else preds

    def forward_bidirectional(self, image1, image2, iters=12, flow_init=None, return_confidence=False):
        """Test-mode flow in both directions of B pairs from one encoder pass (rnc.harness.bidirectional_flow pads, unpads and
        checks consistency on top).  image1, image2: [B,3,H,W] in 0..255, H and W multiples of 8.  flow_init: None or a pair
        (fw, bw), each [B,2,H/8,W/8] or None (a cold start for that direction).  Returns (flow_low, flow_up), with
        return_confidence (NCUP model) (flow_low, flow_up, confidence), of 2B rows: row j is image1[j] -> image2[j], row B + j
        image2[j] -> image1[j], each what forward(..., test_mode=True) gives for that order of the frames.  Inference only."""
        if return_confidence and not self.ncup:
            raise ValueError("return_confidence: the convex-upsampling RAFT has no NCUP upsampler and so no output confidence")
        if self._needs_grad():
            raise ValueError("forward_bidirectional is inference only: call it under torch.no_grad() (training through the "
                             "bidirectional pass is not built)")
        if image1.shape != image2.shape or image1.dim() != 4:
            raise ValueError(f"forward_bidirectional: expected two [B,3,H,W] images of one shape, got {tuple(image1.shape)} "
                             f"and {tuple(image2.shape)}")
        B, _, Him, Wim = image1.shape
        fi = None
        if flow_init is not None:
            if not isinstance(flow_init, (tuple, list)) or len(flow_init) != 2:
                raise ValueError("flow_init: expected a pair (fw, bw), each [B,2,H/8,W/8] or None")
            fw, bw = flow_init
            for f in (fw, bw):
                if f is not None and tuple(f.shape) != (B, 2, Him // 8, Wim // 8):
                    raise ValueError(f"flow_init: expected [B,2,H/8,W/8] = {(B, 2, Him // 8, Wim // 8)}, got {tuple(f.shape)}")
            if fw is not None or bw is not None:
                ref = fw if fw is not None else bw
                # a missing direction starts cold: coords0 + 0.0 is exactly coords0, as with no flow_init
                fi = torch.cat([(f if f is not None else torch.zeros_like(ref)).float() for f in (fw, bw)])
        dev = _require_cuda(image1, image2, fi)
        pdev = module_device(self)
        if pdev != dev:
            raise ValueError(f"model parameters are on {pdev} but the images are on {dev}")
        eng = engine_for(dev)
        conf = bool(return_confidence)
        with torch.cuda.device(dev), eng.lock:
            if iters < 1:
                raise ValueError("iters must be >= 1")
            if Him % 8 or Wim % 8:
                raise ValueError("image height/width must be multiples of 8 (pad with utils.utils.InputPadder, evaluate.py:125)")
            if hasattr(self, "data_idx"):
                self.data_idx += 1
            if eng.graphs_enabled(self):
                return eng.graph_forward(self, image1, image2, iters, fi, return_confidence=conf, bidirectional=True)
            return self._forward_bidirectional(eng, image1, image2, iters, fi, conf)

    def _forward_bidirectional(self, eng, image1, image2, iters, flow_init, return_confidence=False):
        """The bidirectional pass on the engine: _forward_eager over 2B slots of the engine's workspace, slot j holding
        (image1[j], image2[j]) and slot B + j (image2[j], image1[j]), encoded by EncoderStage's bidirectional plan.  flow_init:
        [2B,2,H/8,W/8] or None."""
        B, _, Him, Wim = image1.shape
        pk = eng.packed_update(self.update_block)
        ws = eng.workspace(image1.device, 2 * B, Him // 8, Wim // 8, pk.has_mask, self.ncup)
        return self._forward_eager(eng, image1, image2, iters, flow_init, True,
                                   encode=EncoderStage(self, slot_plan(B, bidirectional=True)), ws=ws,
                                   return_confidence=return_confidence)

    def _umma_encoders(self, eng):
        """Do the encoders run on the tensor-core path (else on torch modules: RNC_ENCODER=cudnn, RNC_CONV=ffma, amp)?"""
        amp = bool(getattr(self.args, "mixed_precision", False))
        return eng.mode == "umma" and not amp and os.environ.get("RNC_ENCODER", "umma").lower() == "umma"

    def _upsample(self, eng, ws, pu):
        raise NotImplementedError


class RAFTConvex(_RAFTBase):
    """core/raft.py:24-143 — baseline RAFT with the convex-combination upsampler."""
    ncup = False

    def _upsample(self, eng, ws, pu):
        return eng.convex_upsample(ws, eng.flow_low(ws), ws.mask, 576)

    def upsample_flow(self, flow, mask):
        """raft.py:73-84: flow [N,2,H8,W8], mask [N,576,H8,W8] (NCHW) -> [N,2,8*H8,8*W8]."""
        dev = _require_cuda(flow, mask)
        eng = engine_for(dev)
        B, _, H8, W8 = flow.shape
        with torch.cuda.device(dev), eng.lock:
            m_cl = torch.empty(B * H8 * W8, 576, dtype=torch.float32, device=dev)
            rnc.nchw_to_cl(mask.detach().float().contiguous(), B, 576, H8, W8, m_cl, 576, 0)
            ws = _Dims(B, H8, W8)
            return eng.convex_upsample(ws, flow.detach().float().contiguous(), m_cl, 576)


class RAFTNcup(_RAFTBase):
    """core/raft_nc_dbl.py:26-173 — RAFT with the NCUP (normalized-convolution) upsampler."""
    ncup = True

    def __init__(self, args):
        super().__init__(args)
        if getattr(args, "load_pretrained", None) is not None:
            # raft_nc_dbl.py:58-66: strict load of a baseline-RAFT checkpoint (keys carry the DataParallel `module.` prefix)
            state = torch.load(args.load_pretrained, map_location="cpu")
            self.load_state_dict(OrderedDict((k[7:], v) for k, v in state.items()))
        self.update_block.mask = nn.Sequential()             # raft_nc_dbl.py:68
        if getattr(args, "freeze_raft", False):
            for p in self.parameters():
                p.requires_grad = False
        self.upsampler = get_upsampler(2, 128, args)
        self.data_idx = 0

    def _upsample(self, eng, ws, pu, want_conf=False):
        rnc.flow_x2_fwd(ws.coords1, ws.B, ws.H8, ws.W8, ws.x4)
        g, gld = eng.guidance(ws)
        return eng.ncup_from_lowres(ws, pu, ws.x4, g, gld, 8.0, want_conf=want_conf)   # `8 *` of raft_nc_dbl.py:161 (not on the conf)

    def _upsample_frozen(self, eng, ws, pu, want_conf=False):
        """Upsampling step of the frozen-trunk forward: snapshots what the upsampler consumes into tensors of this forward
        (the workspace is overwritten by the next iteration, and autograd's backward runs after the engine lock is released),
        then runs the differentiable upsampler on them.  want_conf: (flow, confidence), both differentiable."""
        from .train import ncup_upsampler_frozen
        B, H8, W8 = ws.B, ws.H8, ws.W8
        dev = ws.coords1.device
        x4 = torch.empty(B, 2, 2 * H8, 2 * W8, dtype=torch.float32, device=dev)
        rnc.flow_x2_fwd(ws.coords1, B, H8, W8, x4)
        # the weights-net input cat(x4, area-resized guidance) built straight from the fp32 guidance, channels padded to 136:
        # the tensor of to_cl(cat(x4, g4), pad_to=136) in ncup_upsampler_train
        g, gld = eng.guidance(ws)
        gin = torch.empty(B, 2 * H8, 2 * W8, 136, dtype=torch.float32, device=dev)
        rnc.ncup_guidance_fwd(x4, g, gld, 128, B, H8, W8, gin, 136)
        return ncup_upsampler_frozen(self.upsampler, x4, gin, 8.0, want_conf)   # `8 *` of raft_nc_dbl.py:161

    def upsample_flow(self, flow_lr, guidance):
        """raft_nc_dbl.py:107-112 (without the caller's x8): nearest x2, then the NConv upsampler."""
        x4 = torch.nn.functional.interpolate(flow_lr, scale_factor=2, mode="nearest")
        return self.upsampler(x4, guidance)


def frozen_trunk(model, image1=None, image2=None, flow_init=None):
    """Does this forward train the NCUP upsampler of a frozen RAFT only (the reference's --freeze_raft, train.py:295,
    raft_nc_dbl.py:70-72)?  Then the trunk runs on the inference engine and only the upsampler on autograd.  True when grad is
    enabled, the model is RAFTNcup, no parameter of fnet / cnet / update_block requires grad while some upsampler parameter
    does, no input requires grad, every trunk BatchNorm is in eval mode (the tensor-core encoder has no batch statistics) and
    mixed precision is off."""
    if not torch.is_grad_enabled() or not isinstance(model, RAFTNcup):
        return False
    trunk = (model.fnet, model.cnet, model.update_block)
    if any(p.requires_grad for m in trunk for p in m.parameters()):
        return False
    if not any(p.requires_grad for p in model.upsampler.parameters()):
        return False
    if any(t is not None and t.requires_grad for t in (image1, image2, flow_init)):
        return False
    if any(isinstance(m, nn.BatchNorm2d) and m.training for t in trunk for m in t.modules()):
        return False
    return not getattr(model.args, "mixed_precision", False)


class EncoderStage:
    """Encoder stage of a forward, for _forward_eager(encode=...): runs `plan` (rnc.slot_plan; None: the pair plan) on the
    tensor-core encoders (EncoderRunner.run) or on the torch modules (RNC_ENCODER=cudnn, RNC_CONV=ffma, mixed_precision).
    The sequence drivers set `plan` before each step.  The object keeps what crosses calls: the saved context rows of the
    tensor-core route, and the last call's NCHW fmap1 / fmap2 / net / inp of the torch route; the feature maps in the
    workspace are the rest, so one stage belongs to one workspace."""

    def __init__(self, model, plan=None):
        self.model, self.plan = model, plan
        self.saved = None       # tensor-core route: (h, hx hi, hx lo) rows of plan.save
        self.rows = None        # torch route: (fmap1, fmap2, net, inp) of the last call

    def __call__(self, eng, ws, image1, image2):
        m = self.model
        plan = self.plan or slot_plan(image1.shape[0])
        if m._umma_encoders(eng):
            if plan.save and self.saved is None:
                rows, dev = len(plan.save) * ws.H8 * ws.W8, image1.device
                self.saved = (torch.empty(rows, 128, dtype=torch.float32, device=dev),
                              torch.empty(rows, 256, dtype=torch.float16, device=dev),
                              torch.empty(rows, 256, dtype=torch.float16, device=dev))
            with _Timed(eng, "encoders"):
                eng.encoder().run(m, ws, image1.float().contiguous(), image2.float().contiguous(), plan, self.saved)
            return
        frames = (image1, image2)
        x = (2 * (images(frames, plan.fnet_in) / 255.0) - 1.0).contiguous()
        xc = x if plan.cnet_in == plan.fnet_in else (2 * (images(frames, plan.cnet_in) / 255.0) - 1.0).contiguous()
        with torch.autocast("cuda", enabled=bool(getattr(m.args, "mixed_precision", False))):
            f = m.fnet(x)
            net, inp = torch.split(m.cnet(xc), [128, 128], dim=1)      # raft_nc_dbl.py:137-140
            net, inp = torch.tanh(net), torch.relu(inp)
        f, net, inp = f.float().contiguous(), net.float().contiguous(), inp.float().contiguous()
        last = self.rows or (None,) * 4

        def rows(sources, new, prev):
            """One field's S rows: views of this call's outputs and of the last call's rows, concatenated by runs."""
            pieces = [{NEW: new, CARRY: last[1]}.get(kind, prev)[i:i + k] for _, kind, i, k in runs(sources)]
            return pieces[0] if len(pieces) == 1 else torch.cat(pieces)
        self.rows = (rows(plan.f1, f, last[0]), rows(plan.f2, f, last[1]), rows(plan.ctx, net, last[2]),
                     rows(plan.ctx, inp, last[3]))
        eng.fmap_prepare(ws, *self.rows[:2], 4)
        eng.load_state(ws, *self.rows[2:])


class _Dims:
    def __init__(self, B, H8, W8):
        self.B, self.H8, self.W8 = B, H8, W8
