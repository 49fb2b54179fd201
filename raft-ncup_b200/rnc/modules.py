"""The reference's module surface (same class names, ctor args, forward signatures, state_dict keys), with every
hot-path forward routed to librnc.so through rnc.engine.  Parameter containers are ordinary nn.Modules created in
the reference's construction order, so ``torch.manual_seed(s); RAFT(args)`` yields the reference's exact weights.

Reference surfaces mirrored here (under /root/reference/core):
  corr.py:6-55 CorrBlock        update.py:6-141 FlowHead/SepConvGRU/BasicMotionEncoder/BasicUpdateBlock
  extractor.py:6-56,118-192 ResidualBlock/BasicEncoder      interp_weights_est.py:10-47 Simple
  nconv_modules.py:25-215 NConvUNet/NConv2d                 upsampler.py:10-210 get_upsampler/NConvUpsampler
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.modules.utils import _pair

from .nconv_unet import PackedUNet, is_fused, nconv_fwd
from .engine import (CORR_CH, HX_LD, Engine, ExactWnet, PackedFlowHead, PackedGRU, PackedMotionEncoder, PackedSimple,
                     _require_cuda, engine_for, module_tensors)
from .native import rnc

# --------------------------------------------------------------------------------------------- encoders (C6)
# RAFT.forward runs the encoders on the tensor-core path (rnc/encoder_umma.py).  The nn.Module forwards below are the
# reference's own layer graph on cuDNN in strict fp32: used only when a caller invokes fnet/cnet directly, with
# RNC_ENCODER=cudnn, or under args.mixed_precision.


def _grad_needed(module, *tensors):
    return torch.is_grad_enabled() and (any(t is not None and t.requires_grad for t in tensors)
                                        or any(p.requires_grad for p in module_tensors(module)))


class _Seam:
    """Common prologue of the operator seams: one CUDA device for all inputs, that device's engine, its lock."""

    def __init__(self, *tensors):
        self.dev = _require_cuda(*tensors)
        self.eng = engine_for(self.dev)
        self._guard = torch.cuda.device(self.dev)

    def __enter__(self):
        self._guard.__enter__()
        self.eng.lock.acquire()
        return self.eng

    def __exit__(self, *exc):
        self.eng.lock.release()
        return self._guard.__exit__(*exc)


def _make_norm(kind, ch):
    if kind == "instance":
        return nn.InstanceNorm2d(ch)
    if kind == "batch":
        return nn.BatchNorm2d(ch)
    if kind == "group":
        return nn.GroupNorm(num_groups=ch // 8, num_channels=ch)
    if kind == "none":
        return nn.Sequential()
    raise ValueError(kind)


class ResidualBlock(nn.Module):
    def __init__(self, in_planes, planes, norm_fn="group", stride=1):
        super().__init__()
        self.conv1 = nn.Conv2d(in_planes, planes, 3, padding=1, stride=stride)
        self.conv2 = nn.Conv2d(planes, planes, 3, padding=1)
        self.relu = nn.ReLU(inplace=True)
        self.norm1, self.norm2 = _make_norm(norm_fn, planes), _make_norm(norm_fn, planes)
        self.downsample = None
        if stride != 1:
            self.norm3 = _make_norm(norm_fn, planes)
            self.downsample = nn.Sequential(nn.Conv2d(in_planes, planes, 1, stride=stride), self.norm3)

    def forward(self, x):
        y = self.relu(self.norm1(self.conv1(x)))
        y = self.relu(self.norm2(self.conv2(y)))
        skip = x if self.downsample is None else self.downsample(x)
        return self.relu(skip + y)


class BasicEncoder(nn.Module):
    def __init__(self, output_dim=128, norm_fn="batch", dropout=0.0):
        super().__init__()
        self.norm_fn = norm_fn
        self.norm1 = nn.GroupNorm(8, 64) if norm_fn == "group" else _make_norm(norm_fn, 64)
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3)
        self.relu1 = nn.ReLU(inplace=True)
        widths = [(64, 64, 1), (64, 96, 2), (96, 128, 2)]
        for i, (cin, cout, stride) in enumerate(widths, 1):
            setattr(self, f"layer{i}", nn.Sequential(ResidualBlock(cin, cout, norm_fn, stride),
                                                     ResidualBlock(cout, cout, norm_fn, 1)))
        self.conv2 = nn.Conv2d(128, output_dim, 1)
        self.dropout = nn.Dropout2d(p=dropout) if dropout > 0 else None
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, (nn.BatchNorm2d, nn.InstanceNorm2d, nn.GroupNorm)):
                if m.weight is not None:
                    nn.init.constant_(m.weight, 1)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)

    def forward(self, x):
        pair = isinstance(x, (tuple, list))
        if pair:
            n = x[0].shape[0]
            x = torch.cat(x, 0)
        # strict fp32: TF32 convolutions alone move the final flow by ~1e-2 px (SURVEY.md Appendix D)
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            x = self.relu1(self.norm1(self.conv1(x)))
            x = self.layer3(self.layer2(self.layer1(x)))
            x = self.conv2(x)
        if self.training and self.dropout is not None:
            x = self.dropout(x)
        return torch.split(x, [n, n], 0) if pair else x


# --------------------------------------------------------------------------------------------- CorrBlock (A1-A3)


class CorrBlock:
    """Drop-in for core/corr.py:6-44.  The constructor stores CL feature maps and the pooled fmap2 pyramid (never the
    4-D volume); ``__call__(coords)`` returns the reference's [N, levels*(2r+1)^2, H, W] fp32 tensor."""

    def __init__(self, fmap1, fmap2, num_levels=4, radius=4, engine=None):
        self.dev = _require_cuda(fmap1, fmap2)
        self.num_levels, self.radius = num_levels, radius
        self.engine = engine or engine_for(self.dev)
        B, D, H, W = fmap1.shape
        self.ws = _LookupState(B, D, H, W)
        self.fmap1, self.fmap2 = fmap1, fmap2            # kept for the training path (gradients flow to the feature maps)
        with torch.cuda.device(self.dev), self.engine.lock:
            self.engine.fmap_prepare(self.ws, fmap1.detach().float().contiguous(), fmap2.detach().float().contiguous(), num_levels)

    def __call__(self, coords):
        if _require_cuda(coords) != self.dev:
            raise ValueError("coords must live on the feature maps' device")
        if torch.is_grad_enabled() and (self.fmap1.requires_grad or self.fmap2.requires_grad):
            from .train import corr_lookup_autograd
            return corr_lookup_autograd(self, coords)
        ws = self.ws
        side = 2 * self.radius + 1
        with torch.cuda.device(self.dev), self.engine.lock:
            out = torch.empty(ws.B, self.num_levels * side * side, ws.H8, ws.W8, dtype=torch.float32, device=coords.device)
            self.engine.lookup(ws, coords.detach().float().contiguous(), out, 0, 0, self.radius)
        return out

    @staticmethod
    def corr(fmap1, fmap2):
        raise NotImplementedError("the all-pairs volume (corr.py:47-55) is never materialised by this implementation")


class _LookupState:
    def __init__(self, B, D, H, W):
        self.B, self.D, self.H8, self.W8 = B, D, H, W
        self.f1_cl = self.f2_pyr = None
        self.levels = 4


# --------------------------------------------------------------------------------------------- update block (A5-A8)


class FlowHead(nn.Module):
    """core/update.py:6-14: conv2(relu(conv1(x))), x NCHW [B,128,H,W] -> [B,2,H,W]."""

    def __init__(self, input_dim=128, hidden_dim=256):
        super().__init__()
        self.conv1 = nn.Conv2d(input_dim, hidden_dim, 3, padding=1)
        self.conv2 = nn.Conv2d(hidden_dim, 2, 3, padding=1)

    def forward(self, x):
        if _grad_needed(self, x):
            from .train import flow_head_train
            return flow_head_train(self, x)
        if x.shape[1] != 128 or self.conv1.out_channels != 256:
            raise NotImplementedError("kernels are built for the reference's FlowHead(128, 256)")
        with _Seam(x) as eng:
            B, _, H, W = x.shape
            ws = eng.workspace(x.device, B, H, W, mode="ffma")
            pk = eng._packed_for("flow_head", self, PackedFlowHead)
            rnc.nchw_to_cl(x.detach().float().contiguous(), B, 128, H, W, ws.hx, HX_LD, 0)
            eng._flow_head_ffma(ws, pk, want_delta=True)       # also advances the workspace's scratch coords1 (unused here)
            return ws.delta.clone()


class SepConvGRU(nn.Module):
    """core/update.py:33-60: forward(h [B,128,H,W], x [B,256,H,W]) -> h."""

    def __init__(self, hidden_dim=128, input_dim=192 + 128):
        super().__init__()
        for tag, k, p in (("1", (1, 5), (0, 2)), ("2", (5, 1), (2, 0))):
            for gate in "zrq":
                setattr(self, f"conv{gate}{tag}", nn.Conv2d(hidden_dim + input_dim, hidden_dim, k, padding=p))

    def forward(self, h, x):
        if _grad_needed(self, h, x):
            from .train import sep_conv_gru_train
            return sep_conv_gru_train(self, h, x)
        if h.shape[1] != 128 or x.shape[1] != 256:
            raise NotImplementedError("kernels are built for the reference's SepConvGRU(128, 256)")
        with _Seam(h, x) as eng:
            B, _, H, W = h.shape
            ws = eng.workspace(h.device, B, H, W, mode="ffma")
            pk = eng._packed_for("gru", self, PackedGRU)
            rnc.nchw_to_cl(h.detach().float().contiguous(), B, 128, H, W, ws.hx, HX_LD, 0)
            rnc.nchw_to_cl(x.detach().float().contiguous(), B, 256, H, W, ws.hx, HX_LD, 128)
            eng._gru_ffma(ws, pk)
            return Engine.net_nchw(eng, ws)          # the exact kernels' hidden state, whatever the engine's mode


class BasicMotionEncoder(nn.Module):
    """core/update.py:79-97: forward(flow [B,2,H,W], corr [B,324,H,W]) -> cat([conv features (126), flow (2)])."""

    def __init__(self, args):
        super().__init__()
        cor_planes = args.corr_levels * (2 * args.corr_radius + 1) ** 2
        self.convc1 = nn.Conv2d(cor_planes, 256, 1, padding=0)
        self.convc2 = nn.Conv2d(256, 192, 3, padding=1)
        self.convf1 = nn.Conv2d(2, 128, 7, padding=3)
        self.convf2 = nn.Conv2d(128, 64, 3, padding=1)
        self.conv = nn.Conv2d(64 + 192, 128 - 2, 3, padding=1)

    def forward(self, flow, corr):
        if _grad_needed(self, flow, corr):
            from .train import motion_encoder_train
            return motion_encoder_train(self, flow, corr)
        if corr.shape[1] != CORR_CH:
            raise NotImplementedError("kernels are built for 4 levels x radius 4 = 324 correlation channels")
        with _Seam(flow, corr) as eng:
            B, _, H, W = flow.shape
            ws = eng.workspace(flow.device, B, H, W, mode="ffma")
            pk = eng._packed_for("motion_encoder", self, PackedMotionEncoder)
            rnc.nchw_to_cl(corr.detach().float().contiguous(), B, CORR_CH, H, W, ws.corr, CORR_CH, 0)
            rnc.coords_init(ws.coords1, flow.detach().float().contiguous(), B, H, W)
            eng._motion_encoder_ffma(ws, pk)
            out = torch.empty(B, 128, H, W, dtype=torch.float32, device=flow.device)
            rnc.cl_to_nchw(ws.hx, HX_LD, 256, B, 128, H, W, out)
            return out


class BasicUpdateBlock(nn.Module):
    """Drop-in for core/update.py:114-141: forward(net, inp, corr, flow) -> (net, mask, delta_flow), all NCHW."""

    def __init__(self, args, hidden_dim=128, input_dim=128):
        super().__init__()
        self.args = args
        if hidden_dim != 128 or args.corr_levels != 4 or args.corr_radius != 4:
            raise NotImplementedError("kernels are built for the reference's only live config: hidden 128, 4 levels, radius 4")
        self.encoder = BasicMotionEncoder(args)
        self.gru = SepConvGRU(hidden_dim=hidden_dim, input_dim=128 + hidden_dim)
        self.flow_head = FlowHead(hidden_dim, hidden_dim=256)
        self.mask = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 64 * 9, 1, padding=0))
        self.net = []

    def engine(self, device=None):
        from .engine import module_device
        return engine_for(device if device is not None else module_device(self))

    def forward(self, net, inp, corr, flow, upsample=True):
        if _grad_needed(self, net, inp, corr, flow):
            from .train import update_block_train
            return update_block_train(self, net, inp, corr, flow)
        with _Seam(net, inp, corr, flow) as eng:
            return self._forward(eng, net, inp, corr, flow)

    def _forward(self, eng, net, inp, corr, flow):
        B, _, H, W = net.shape
        pk = eng.packed_update(self)
        ws = eng.workspace(net.device, B, H, W, pk.has_mask, False)
        eng.load_state(ws, net.float().contiguous(), inp.float().contiguous())
        eng.load_corr(ws, corr.float().contiguous())
        # the kernels read flow as coords1 - grid: rebuild coords1 from the flow argument
        rnc.coords_init(ws.coords1, flow.float().contiguous(), B, H, W)
        eng.update_iter(ws, pk, want_mask=pk.has_mask, want_delta=True)
        net_out = eng.net_nchw(ws)
        self.net = net_out                                  # guidance tap read by raft_nc_dbl.py:161
        mask = None
        if pk.has_mask:
            mask = torch.empty(B, 576, H, W, dtype=torch.float32, device=net.device)
            rnc.cl_to_nchw(ws.mask, 576, 0, B, 576, H, W, mask)
        else:
            mask = 0.25 * net_out                           # `.25 * Sequential()(net)` of the reference (update.py:140)
        return net_out, mask, ws.delta.clone()


# --------------------------------------------------------------------------------------------- NCUP (U2-U7)


class NConv2d(nn.Module):
    """core/nconv_modules.py:140-215: stores ``weight_p``; the effective kernel is softplus(weight_p, beta=10) (EnforcePos,
    :218-269), recomputed at every forward.  forward((data, conf)) -> (nconv, conf_out), NCHW, through rnc_nconv2d_fwd.
    With bias, ``nconv += bias`` follows the division and the confidence is unaffected (:175-179)."""

    def __init__(self, in_channels, out_channels, kernel_size, pos_fn="softplus", bias=False):
        super().__init__()
        if pos_fn.lower() != "softplus":
            raise NotImplementedError(f"NConv2d pos_fn={pos_fn!r}: only SoftPlus is built")
        self.in_channels, self.out_channels, self.kernel_size = in_channels, out_channels, tuple(kernel_size)
        self.eps = 1e-20
        w = torch.empty(out_channels, in_channels, *self.kernel_size)
        # _ConvNd.reset_parameters draws the weight, then the bias; both are drawn again by init_parameters (:201-215)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        bound = 1 / math.sqrt(in_channels * self.kernel_size[0] * self.kernel_size[1])
        if bias:
            torch.empty(out_channels).uniform_(-bound, bound)
        n = self.kernel_size[0] * self.kernel_size[1] * out_channels
        w.normal_(2, math.sqrt(2.0 / n))
        if bias:
            self.bias = nn.Parameter(torch.empty(out_channels).uniform_(-bound, bound))
        else:
            self.register_parameter("bias", None)
        self.weight_p = nn.Parameter(F.softplus(w, beta=10))

    @property
    def weight(self):
        return F.softplus(self.weight_p, beta=10)

    def forward(self, inpt):
        data, conf = inpt[0], inpt[1]
        if _grad_needed(self, data, conf):
            from .train import nconv2d_autograd
            return nconv2d_autograd(data, conf, self.weight, self.eps, self.bias)
        return nconv2d_forward(data, conf, self.weight.detach(), self.eps, self.bias)


def nconv2d_forward(data, conf, weight, eps=1e-20, bias=None):
    """One normalized convolution through the C ABI (nconv_modules.py:164-199); weight = the positive kernel."""
    with _Seam(data, conf, weight):
        b = None if bias is None else bias.detach().float().contiguous()
        return nconv_fwd(data.detach().float().contiguous(), conf.detach().float().contiguous(),
                         weight.detach().float().contiguous(), b, eps)


class NConvUNet(nn.Module):
    """core/nconv_modules.py:25-136 for in_ch 1, groups 1, SoftPlus, channels_multiplier <= 4 and odd filters <= 7, with
    the reference's module structure, state_dict keys (incl. the ``encoder.*`` aliases of shared layers) and RNG draws.
    forward((data, conf)) -> (xout, cout) runs the live path of rnc/nconv_unet.py: the decoder reads x[i+N] (index quirk
    at :128-131), so the deepest level never reaches the output and is not computed."""

    def __init__(self, in_ch=1, channels_multiplier=2, num_downsampling=3, encoder_filter_sz=5, decoder_filter_sz=3,
                 out_filter_sz=1, pos_fn="SoftPlus", groups=1, use_bias=False, data_pooling="conf_based",
                 shared_encoder=True, use_double_conv=True):
        super().__init__()
        self.__name__ = "NConvUNet"
        if in_ch != 1:
            raise NotImplementedError(f"NConvUNet in_ch={in_ch}: only in_ch 1 is built")
        if groups != 1:
            raise NotImplementedError(f"NConvUNet groups={groups}: only groups 1 is built")
        if pos_fn.lower() != "softplus":
            raise NotImplementedError(f"NConvUNet pos_fn={pos_fn!r}: only SoftPlus is built")
        if not 1 <= channels_multiplier <= 4:
            raise NotImplementedError(f"NConvUNet channels_multiplier={channels_multiplier}: the kernels take 1 to 4")
        for name, k in (("encoder_filter_sz", encoder_filter_sz), ("decoder_filter_sz", decoder_filter_sz),
                        ("out_filter_sz", out_filter_sz)):
            if not isinstance(k, int) or k < 1 or k > 7 or k % 2 == 0:
                raise NotImplementedError(f"NConvUNet {name}={k}: the kernels take odd square filters up to 7")
        if num_downsampling < 0:
            raise ValueError(f"NConvUNet num_downsampling={num_downsampling}")
        if data_pooling not in ("conf_based", "max_pooling"):
            raise NotImplementedError("Choose `self.data_pooling` from [conf_based, max_pooling]!")
        c = in_ch * channels_multiplier
        self.channels, self.num_downsampling, self.data_pooling = c, num_downsampling, data_pooling
        self.shared_encoder, self.use_double_conv, self.use_bias = shared_encoder, use_double_conv, use_bias
        self.use_double_conf = use_double_conv                  # the reference's attribute name
        self.filter_sizes = (encoder_filter_sz, decoder_filter_sz, out_filter_sz)
        ek, dk, ok = ((k, k) for k in self.filter_sizes)
        self.nconv_in = NConv2d(in_ch, c, ek, pos_fn, bias=use_bias)
        self.nconv_x2 = nn.Sequential(*[NConv2d(c, c, ek, pos_fn, bias=use_bias) for _ in range(2 if use_double_conv else 1)])
        self.encoder = nn.ModuleList([nn.Sequential(self.nconv_in, self.nconv_x2)])
        for _ in range(num_downsampling):
            self.encoder.append(self.nconv_x2[0] if shared_encoder else NConv2d(c, c, ek, pos_fn, bias=use_bias))
        self.decoder = nn.ModuleList([NConv2d(2 * c, c, dk, pos_fn, bias=use_bias) for _ in range(num_downsampling)])
        self.nconv_out = NConv2d(c, in_ch, ok, pos_fn, bias=False)

    def forward(self, inpt):
        if is_fused(self):
            x, c = self.nconv_in((inpt[0], inpt[1]))
            x, c = self.nconv_x2[0]((x, c))
            x, c = self.decoder[0]((torch.cat((x, x), 1), torch.cat((c, c), 1)))
            return self.nconv_out((x, c))
        if _grad_needed(self, inpt[0], inpt[1]):
            from .train import nconv_unet_train
            return nconv_unet_train(self, inpt[0], inpt[1])
        with _Seam(inpt[0], inpt[1]):
            return PackedUNet(self).run(inpt[0].detach().float().contiguous(), inpt[1].detach().float().contiguous())


class Simple(nn.Module):
    """core/interp_weights_est.py:10-47: forward(x [B,in_ch,h,w]) -> final_act(out(conv[n-1](...conv[0](x)))), for 0 to 6
    hidden layers of widths 1 to 256 and, in every layer, odd filter sizes 1 to 7 and dilations 1 to 4 (None: 1), with the
    reference's module structure, padding, state_dict keys and RNG draws."""

    def __init__(self, num_ch, out_ch, filter_sz, dilation=None, final_act=torch.sigmoid, use_bn=False):
        super().__init__()
        self.__name__ = "Simple"
        num_ch, filter_sz = list(num_ch), list(filter_sz)
        dilation = [1] * len(num_ch) if dilation is None else list(dilation)
        if len(filter_sz) != len(num_ch) or len(dilation) != len(num_ch):
            raise ValueError(f"Simple: num_ch {num_ch}, filter_sz {filter_sz} and dilation {dilation} must have one entry per layer")
        if not 1 <= len(num_ch) <= 7 or any(not isinstance(c, int) or not 1 <= c <= 256 for c in num_ch[1:]):
            raise NotImplementedError(f"Simple num_ch={num_ch[1:]}: the kernels take 0 to 6 hidden layers of widths 1 to 256")
        if any(not isinstance(k, int) or k < 1 or k > 7 or k % 2 == 0 for k in filter_sz):
            raise NotImplementedError(f"Simple filter_sz={filter_sz}: the kernels take odd square filters up to 7")
        if any(not isinstance(d, int) or not 1 <= d <= 4 for d in dilation):
            raise NotImplementedError(f"Simple dilation={dilation}: the kernels take dilations 1 to 4")
        self.in_ch = num_ch[0]  # Number of Input channels is added at the beginning of num_ch
        self.num_layers = len(num_ch) - 1

        def conv(i, cin, cout):       # interp_weights_est.py:25,36
            return nn.Conv2d(cin, cout, filter_sz[i], padding=_pair(int(filter_sz[i] // 2 + ((filter_sz[i] - 1) * (dilation[i] - 1)) / 2)),
                             dilation=dilation[i], stride=1)

        self.conv = nn.ModuleList()
        for i in range(self.num_layers):
            layers = [conv(i, num_ch[i], num_ch[i + 1])]
            if use_bn:
                layers.append(nn.BatchNorm2d(num_ch[i + 1]))
            layers.append(nn.ReLU(inplace=True))
            self.conv.append(nn.Sequential(*layers))
        self.out = conv(-1, num_ch[-1], out_ch)
        self.final_act = final_act

    def forward(self, x):
        if _grad_needed(self, x):
            from .train import simple_train
            return simple_train(self, x)
        if self.final_act is not torch.sigmoid or self.out.out_channels != 2:
            raise NotImplementedError("the fused confidence head applies the sigmoid the reference wires in (upsampler.py:44-46)")
        if any(isinstance(m, nn.BatchNorm2d) and m.training for m in self.modules()):
            raise NotImplementedError("weights-net BatchNorm with batch statistics needs the training path (enable grad)")
        B, Cin, h, w = x.shape
        if Cin != self.in_ch:
            raise ValueError(f"Simple: expected {self.in_ch} input channels, got {Cin}")
        with _Seam(x) as eng:
            pk = eng._packed_for("simple", self, lambda wn: PackedSimple(wn, ExactWnet))
            cpad = pk.cin
            M = B * h * w
            xin = torch.zeros(M, cpad, dtype=torch.float32, device=x.device) if cpad != Cin else torch.empty(M, cpad, dtype=torch.float32, device=x.device)
            rnc.nchw_to_cl(x.detach().float().contiguous(), B, Cin, h, w, xin, cpad, 0)
            conf = torch.empty(B, 2, h, w, dtype=torch.float32, device=x.device)
            eng.weights_net(pk, B, h, w, xin, cpad, pk.buffers(M, x.device), conf)
            return conf


class NConvUpsampler(nn.Module):
    """Drop-in for core/upsampler.py:75-210.  forward(x_lowres [B,2,h,w], x_guidance [B,128,h/2,w/2]) -> [B,2,4h,4w];
    with return_confidence=True -> (out, confidence): the interpolation network's output confidence in [0, 1] (the cout
    upsampler.py:168 discards), shaped like out and not multiplied by out_scale."""

    def __init__(self, scale=None, size=None, interpolation_net=None, weights_est_net=None, use_data_for_guidance=True,
                 channels_to_batch=True, use_residuals=False, est_on_high_res=False):
        super().__init__()
        self.__name__ = "NConvUpsampler"
        if scale is None and size is None:
            raise ValueError("Either scale or size needs to be set!")
        if scale is not None and size is not None:
            raise ValueError("You can set either scale or size at a time!")
        if interpolation_net is None:
            raise ValueError("An interpolation network mush be provided!")
        for name, bad in (("scale", scale != 4), ("use_data_for_guidance", not use_data_for_guidance),
                          ("channels_to_batch", not channels_to_batch), ("use_residuals", use_residuals),
                          ("est_on_high_res", est_on_high_res), ("weights_est_net", weights_est_net is None)):
            if bad:
                raise NotImplementedError(f"NConvUpsampler {name}: the NCUP kernels are built for scale 4, data for guidance, "
                                          "channels to batch, no residuals, estimation at low resolution and a weights net")
        self.scaleH = self.scaleW = float(scale)
        self.interpolation_net, self.weights_est_net = interpolation_net, weights_est_net
        self.use_data_for_guidance, self.channels_to_batch = use_data_for_guidance, channels_to_batch
        self.use_residuals, self.est_on_high_res = use_residuals, est_on_high_res

    def engine(self, device=None):
        from .engine import module_device
        return engine_for(device if device is not None else module_device(self))

    def forward(self, x_lowres, x_guidance=None, out_scale=1.0, return_confidence=False):
        if _grad_needed(self, x_lowres, x_guidance):
            from .train import ncup_upsampler_train
            return ncup_upsampler_train(self, x_lowres, x_guidance, out_scale, return_confidence=bool(return_confidence))
        if any(isinstance(m, nn.BatchNorm2d) and m.training for m in self.weights_est_net.modules()):
            raise NotImplementedError("weights-net BatchNorm with batch statistics needs the training path (enable grad)")
        B, C, h, w = x_lowres.shape
        if C != 2 or x_guidance is None or x_guidance.shape[1] != 128 or h != 2 * x_guidance.shape[2] or w != 2 * x_guidance.shape[3]:
            raise ValueError("expected x_lowres [B,2,h,w] with guidance [B,128,h/2,w/2]")
        with _Seam(x_lowres, x_guidance) as eng:
            pu = eng.packed_upsampler(self)
            ws = eng.workspace(x_lowres.device, B, h // 2, w // 2, False, True)
            g_cl = torch.empty(B * (h // 2) * (w // 2), 128, dtype=torch.float32, device=x_lowres.device)
            rnc.nchw_to_cl(x_guidance.float().contiguous(), B, 128, h // 2, w // 2, g_cl, 128, 0)
            return eng.ncup_from_lowres(ws, pu, x_lowres.float().contiguous(), g_cl, 128, out_scale,
                                        want_conf=bool(return_confidence))


def get_upsampler(in_ch, guidance_ch, args):
    """core/upsampler.py:10-72 — the factory is hard-wired to the NConv upsampler (:12)."""
    interpolation_net = NConvUNet(in_ch=1, channels_multiplier=args.interp_net_channels_multiplier,
                                  num_downsampling=args.interp_net_num_downsampling,
                                  encoder_filter_sz=args.interp_net_encoder_filter_sz,
                                  decoder_filter_sz=args.interp_net_decoder_filter_sz,
                                  out_filter_sz=args.interp_net_out_filter_sz, use_bias=args.interp_net_use_bias,
                                  data_pooling=args.interp_net_data_pooling, shared_encoder=args.interp_net_shared_encoder,
                                  use_double_conv=args.interp_net_use_double_conv, pos_fn="SoftPlus", groups=1)
    num_channels = list(args.weights_est_net_num_ch)
    num_channels.insert(0, guidance_ch + in_ch if args.final_upsampling_use_data_for_guidance else guidance_ch)
    use_bn = args.dataset == "sintel"                        # upsampler.py:42
    if args.weights_est_net.lower() != "simple":
        raise NotImplementedError(f"weights_est_net={args.weights_est_net!r}: only the `Simple` weights-estimation net is "
                                  "built (every reference script selects it)")
    weights_est_net = Simple(num_ch=num_channels, out_ch=in_ch, use_bn=use_bn, filter_sz=args.weights_est_net_filter_sz,
                             dilation=args.weights_est_net_dilation, final_act=torch.sigmoid)
    return NConvUpsampler(scale=args.final_upsampling_scale, interpolation_net=interpolation_net,
                          weights_est_net=weights_est_net, use_data_for_guidance=args.final_upsampling_use_data_for_guidance,
                          channels_to_batch=args.final_upsampling_channels_to_batch,
                          use_residuals=args.final_upsampling_use_residuals, est_on_high_res=args.final_upsampling_est_on_high_res)
