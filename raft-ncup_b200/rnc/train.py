"""Training path of RAFT / RAFT-NCUP (SURVEY.md §8f-3, Appendix G; BASELINE config #5): the forward of
``RAFT.forward`` in train mode (raft_nc_dbl.py:115-173, raft.py:87-143) as an autograd graph whose heavy nodes are
``torch.autograd.Function``s running librnc's exact-fp32 kernels forward AND backward:

    ConvCL          every nn.Conv2d (update.py, extractor.py, interp_weights_est.py): rnc_conv2d_cl_fwd; data gradient = the same
                    kernel on the (zero-dilated, for stride 2) output gradient with flipped / transposed weights; weight and bias
                    gradient = rnc_conv2d_cl_wgrad_det (fixed-order sum of the K-split partials)
    CorrPyramid     CorrBlock.__init__ on features (corr.py:7-21): rnc_fmap_pyramid / adjoint rnc_pyramid_pool_bwd
    CorrLookup      CorrBlock.__call__ (corr.py:23-44): rnc_corr_lookup_fwd / rnc_corr_lookup_bwd (d fmap1, d fmap2 pyramid; coords
                    are detached, raft_nc_dbl.py:149)
    NConv2dFn       NConv2d.forward (nconv_modules.py:164-199): rnc_nconv2d_fwd / rnc_nconv2d_bwd (quotient rule, confidence path)
    NConvPoolFn     NConvUNet.downsample_data_conf (nconv_modules.py:94-104): rnc_nconv_pool2_fwd / rnc_nconv_pool2_bwd
    NcupChainFn     the whole NConvUNet chain after the weights net at the shipped configuration: rnc_ncup_train_fwd /
                    rnc_ncup_bwd (fused, deterministic); used by the frozen-trunk forward (rnc.model.frozen_trunk), which runs the
                    trunk on the inference engine.  Other configurations run the NConv2dFn / NConvPoolFn chain of
                    rnc/nconv_unet.py there too.  With want_conf it also returns the chain's output confidence (the same
                    entry points, given conf_out / g_conf_out); the frozen-trunk forward asks for it when the confidence is
                    requested.

Under torch.use_deterministic_algorithms(True) the lookup backward, which otherwise scatters d fmap2 with floating-point
atomics, switches to its fixed-order form rnc_corr_lookup_bwd_det (deterministic()); the weight gradient sums in a fixed order
in both modes.  Identical steps then give bit-identical gradients.

Activations stay channel-last ([B, H, W, C] fp32) between convolutions.  Pointwise glue (ReLU / sigmoid / tanh / gate blend,
cat, nearest x2, zero-stuffing, the loss) and the normalisation layers (InstanceNorm / BatchNorm: library kernels, like cuDNN
in the reference) are plain torch ops — plumbing around the kernels above.  `sequence_loss`, `fetch_optimizer` and
`train_step` restate train.py:46-71, :83-99, :203-227; `ddp_model` replaces nn.DataParallel (train.py:169-175) with one
process per GPU and a bucketed NCCL all-reduce of the 4.9 M fp32 gradients.
"""
import copy
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import native
from .engine import CORR_CH, _require_cuda, engine_for, pack_conv
from .engine_umma import UmmaWeights, _ceil32
from .native import rnc
from .nconv_unet import is_fused, live_chain, nconv_fwd, pool_fwd, unused_parameters

_PACK_CACHE = {}          # (id(weight), version, kind, fmt, cin_pad) -> (weight, packed); flushed at every training forward


def _packed(weight, kind, cin_pad, fmt="ffma"):
    """Kernel-ready copy of a convolution weight ('fwd') or of its flipped transpose ('dgrad'), cached for the 12 iterations of a
    step, in the operand format of the exact kernel (fmt 'ffma': pack_conv) or of the TF32 tensor-core kernel ('tf32':
    UmmaWeights(tf32=True)).  The entry keeps the weight tensor alive, so neither its id nor its storage can be recycled while
    the entry exists."""
    key = (id(weight), weight._version, kind, fmt, cin_pad)
    hit = _PACK_CACHE.get(key)
    if hit is None or hit[0] is not weight:
        if len(_PACK_CACHE) > 512:
            _PACK_CACHE.clear()
        w = weight.detach().float()
        if kind == "dgrad":          # Wd[ci, co, ky, kx] = W[co, ci, kh-1-ky, kw-1-kx]
            w = w.flip(2, 3).transpose(0, 1)
        w = w.contiguous()
        packed = pack_conv(w, None, cin_pad=cin_pad) if fmt == "ffma" else UmmaWeights(w, None, [cin_pad], tf32=True)
        hit = _PACK_CACHE[key] = (weight, packed)
    return hit[1]


def deterministic():
    """torch.use_deterministic_algorithms(True) is in force: the lookup backward gathers d fmap2 in a fixed order instead of
    scattering it with atomics."""
    return torch.are_deterministic_algorithms_enabled()


def _ceil4(c):
    return (c + 3) // 4 * 4


def _conv_mode():
    """RNC_TRAIN_CONV selects how the training path's convolutions (forward and data gradient) run:
      ffma (default)  exact fp32 on CUDA cores (rnc_conv2d_cl_fwd): per-layer error 1.5e-7; every non-fnet parameter's gradient
                      within 1e-3 of the reference's autograd
      tf32            wgmma .tf32 on TF32 hi/lo operand planes, 3 MMAs per K step (x_hi*w_hi + x_hi*w_lo + x_lo*w_hi):
                      ~2^-21 per product (per-layer 1e-6 .. 5e-6) with fp32's exponent range, so output gradients of 1e-9
                      survive; 112 ms per step, ill-conditioned parameters (cnet.conv1) move to 5e-3
    The inference kernels' fp16 hi/lo split is not offered: output gradients fall below its normal range (DESIGN.md §3.8).
    Parity first: the default is the exact path; the tensor-core form is opt-in and reported beside it by bench.py.  Read at
    every call, so a process may switch between steps."""
    mode = os.environ.get("RNC_TRAIN_CONV", "ffma")
    if mode not in ("ffma", "tf32"):
        raise ValueError(f"RNC_TRAIN_CONV={mode!r}: expected 'ffma' or 'tf32'")
    return mode


def _tf32_ok(eng, Cx, cout):
    """Does this layer run on the TF32 tensor-core convolution (RNC_TRAIN_CONV=tf32 on the tensor-core engine)?  The kernel
    stores whole 32-channel chunks of fp32 output, so the output row must not need wider padding than the channel-last tensors
    use, and the operand planes need a pitch of 4 floats."""
    return _conv_mode() == "tf32" and eng.mode == "umma" and _ceil32(cout) == _ceil4(cout) and Cx % 4 == 0


def _padded_bias(packed_bias, bias):
    """This call's bias in the zero-padded layout of a packed weight's bias (packs are cached per weight; biases are tiny and
    change with it)."""
    b = torch.zeros_like(packed_bias)
    b[:bias.shape[0]] = bias.detach()
    return b


def _conv_launch_tf32(eng, x, wt, cout, stride=1, bias=None, dil=1):
    """Same contract as _conv_launch on the TF32 tensor-core path: x fp32 CL -> TF32 hi/lo operand planes -> rnc_conv2d_umma_fwd
    with an fp32 channel-last output; stride 2 is native (TMA element strides), no subsampling pass."""
    B, H, W, Cx = x.shape
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    M = B * H * W
    hi = torch.empty(M, Cx, dtype=torch.float32, device=x.device)
    lo = torch.empty(M, Cx, dtype=torch.float32, device=x.device)
    rnc.f32_to_tf32_split(x, Cx, Cx, M, hi, lo, Cx, 0)
    ldo = _ceil4(cout)
    out = torch.empty(B, Ho, Wo, ldo, dtype=torch.float32, device=x.device)
    if bias is not None:
        wt = copy.copy(wt)
        wt.bias = _padded_bias(wt.bias, bias)
    eng.uconv(B, Ho, Wo, (hi.data_ptr(), lo.data_ptr()), Cx, Cx, wt, native.EPI_LINEAR, out_f32=out.data_ptr(), ldo_f32=ldo,
              stride=stride, hin=H, win=W, flags=native.CONV_TF32, dil=dil)
    return out


def _conv_launch(eng, x, packed, cout, kh, kw, bias=None, dil=1):
    """x CL [B,H,W,C] contiguous (C % 4 == 0) -> CL [B,H,W,ceil4(cout)] (pad channels zero), stride 1, dilation dil, zero
    padding (k/2)*dil."""
    B, H, W, Cx = x.shape
    ldo = _ceil4(cout)
    alloc = torch.empty if ldo == cout else torch.zeros          # pad channels must read as zero downstream
    out = alloc(B, H, W, ldo, dtype=torch.float32, device=x.device)
    if bias is not None:
        packed = (packed[0], _padded_bias(packed[1], bias))
    eng.conv(B, H, W, x.data_ptr(), Cx, Cx, packed, cout, kh, kw, native.EPI_LINEAR, out.data_ptr(), ldo, dil=dil)
    return out


def _conv(eng, x, weight, kind, cout, stride=1, bias=None, dil=1):
    """x CL [B,H,W,Cx] -> CL [B,Ho,Wo,ceil4(cout)]: the convolution by `weight` ('fwd') or by its flipped transpose ('dgrad'),
    on the TF32 tensor-core form where _tf32_ok allows it, else exact fp32."""
    Cx = x.shape[-1]
    if _tf32_ok(eng, Cx, cout):
        return _conv_launch_tf32(eng, x, _packed(weight, kind, Cx, "tf32"), cout, stride, bias, dil)
    kh, kw = weight.shape[2:]
    y = _conv_launch(eng, x, _packed(weight, kind, Cx), cout, kh, kw, bias, dil)
    return y[:, ::2, ::2].contiguous() if stride == 2 else y      # same padding: out(y, x) of the strided conv = full(2y, 2x)


class ConvCL(torch.autograd.Function):
    """y = conv2d(x, weight, bias, stride, padding = (k // 2) * dil, dilation = dil) on channel-last tensors (dil > 1: stride 1).
    x [B,H,W,Cx] (Cx = ceil4(Cin); channels beyond Cin must be zero), weight [Cout,Cin,kh,kw] -> y [B,Ho,Wo,ceil4(Cout)]."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, dil=1):
        x = x.contiguous()
        eng = engine_for(x.device)
        cout, cin, kh, kw = weight.shape
        Cx = x.shape[-1]
        if Cx % 4 or Cx < cin:
            raise ValueError("ConvCL: input must be channel-last with ceil4(Cin) channels")
        if stride not in (1, 2) or (dil > 1 and stride != 1):
            raise NotImplementedError("stride 1 or 2; dilated layers at stride 1")
        y = _conv(eng, x, weight, "fwd", cout, stride, bias, dil)
        ctx.save_for_backward(x, weight)
        ctx.stride, ctx.dil, ctx.has_bias = stride, dil, bias is not None
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight = ctx.saved_tensors
        eng = engine_for(x.device)
        cout, cin, kh, kw = weight.shape
        B, H, W, Cx = x.shape
        gy = gy.contiguous()
        ldg = gy.shape[-1]
        gx = gw = gb = None
        dil = ctx.dil
        with torch.cuda.device(x.device):
            if ctx.needs_input_grad[0]:
                g_full = gy
                if ctx.stride == 2:
                    g_full = torch.zeros(B, H, W, ldg, dtype=torch.float32, device=x.device)
                    g_full[:, ::2, ::2] = gy
                # the same (dilated) convolution with the flipped, transposed weights: its padding (k // 2) * dil is symmetric
                gx = _conv(eng, g_full, weight, "dgrad", cin, dil=dil)
                if gx.shape[-1] != Cx:               # Cx > ceil4(cin) never happens; equal by construction
                    gx = F.pad(gx, (0, Cx - gx.shape[-1]))
            if ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2]):
                gwp, gbp = _wgrad(x, gy, cout, kh, kw, ctx.stride, ctx.has_bias, dil)
                gw = gwp.view(kh, kw, Cx, cout)[:, :, :cin].permute(3, 2, 0, 1).contiguous()
                gb = gbp
        return gx, gw, gb, None, None


def _wgrad(x, gy, cout, kh, kw, stride, has_bias, dil=1):
    """Weight / bias gradient of ConvCL: [kh*kw, Cx, cout], [cout] (or None).  rnc_conv2d_cl_wgrad_det (rnc_conv2d_cl_wgrad_dil_det
    for a dilated layer) sums the K-split partials in a fixed order (in either mode: it is no slower than adding them with atomics
    was) and writes its outputs."""
    B, H, W, Cx = x.shape
    gwp = torch.empty(kh * kw, Cx, cout, dtype=torch.float32, device=x.device)
    gbp = torch.empty(cout, dtype=torch.float32, device=x.device) if has_bias else None
    nbytes_fn, wgrad_fn, arg = ((rnc.conv2d_cl_wgrad_dil_workspace_bytes, rnc.conv2d_cl_wgrad_dil_det, dil) if dil > 1 else
                                (rnc.conv2d_cl_wgrad_workspace_bytes, rnc.conv2d_cl_wgrad_det, stride))
    nbytes = nbytes_fn(Cx, cout, B, H, W, kh, kw, arg)
    ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=x.device)
    wgrad_fn(x, Cx, Cx, gy, gy.shape[-1], cout, B, H, W, kh, kw, arg, gwp, cout, gbp, ws, ws.numel() * 4)
    return gwp, gbp


def conv_cl(x, conv, stride=None):
    """nn.Conv2d `conv` on a channel-last tensor: zero padding (k // 2) * dilation, as every convolution of the reference (the
    weights net's dilated ones included, interp_weights_est.py:25,36)."""
    s = conv.stride[0] if stride is None else stride
    kh, kw = conv.kernel_size
    dil = conv.dilation[0] if max(kh, kw) > 1 else 1
    if conv.dilation[0] != conv.dilation[1] or tuple(conv.padding) != ((kh // 2) * dil, (kw // 2) * dil):
        raise NotImplementedError(f"conv_cl: padding {conv.padding}, dilation {conv.dilation}: the kernels pad (k // 2) * dilation")
    return ConvCL.apply(x, conv.weight, conv.bias, s, dil)


def to_cl(x, pad_to=None):
    """NCHW -> contiguous channel-last, channels zero-padded to a multiple of 4 (or to pad_to)."""
    y = x.permute(0, 2, 3, 1)
    c = y.shape[-1]
    tgt = pad_to or _ceil4(c)
    if tgt != c:
        y = F.pad(y, (0, tgt - c))
    return y.contiguous()


def to_nchw(x, c=None):
    y = x if c is None else x[..., :c]
    return y.permute(0, 3, 1, 2).contiguous()


# --------------------------------------------------------------------------------------------- correlation


class CorrPyramid(torch.autograd.Function):
    """fmap2 (CL) -> pooled feature pyramid (corr.py:18-21 on features; SURVEY.md finding 7).  Output: flat pyramid buffer."""

    @staticmethod
    def forward(ctx, fmap2_cl, levels):
        _require_cuda(fmap2_cl)
        B, H, W, D = fmap2_cl.shape
        total = rnc.pyramid_offset(B, D, H, W, levels)
        pyr = torch.empty(total, dtype=torch.float32, device=fmap2_cl.device)
        pyr[:B * H * W * D] = fmap2_cl.reshape(-1)
        rnc.fmap_pyramid(pyr, B, D, H, W, levels)
        ctx.dims = (B, H, W, D, levels)
        return pyr

    @staticmethod
    def backward(ctx, g_pyr):
        B, H, W, D, levels = ctx.dims
        g = g_pyr.clone()
        with torch.cuda.device(g.device):
            rnc.pyramid_pool_bwd(g, B, D, H, W, levels)
        return g[:B * H * W * D].view(B, H, W, D), None


class CorrLookup(torch.autograd.Function):
    """corr.py:23-44 on (fmap1 CL, fmap2 pyramid): -> CL [B,H,W,324] in the reference channel order."""

    @staticmethod
    def forward(ctx, f1_cl, f2_pyr, coords, levels):
        _require_cuda(f1_cl)
        B, H, W, D = f1_cl.shape
        coords = coords.detach().float().contiguous()
        out = torch.empty(B, H, W, CORR_CH, dtype=torch.float32, device=f1_cl.device)
        rnc.corr_lookup_fwd(f1_cl, f2_pyr, coords, B, D, H, W, levels, 4, out, 1, CORR_CH)
        ctx.save_for_backward(f1_cl, f2_pyr, coords)
        ctx.levels = levels
        return out

    @staticmethod
    def backward(ctx, g_out):
        f1_cl, f2_pyr, coords = ctx.saved_tensors
        with torch.cuda.device(f1_cl.device):
            g_f1, g_f2 = _lookup_bwd(f1_cl, f2_pyr, coords, g_out.contiguous(), ctx.levels)
        return g_f1, g_f2, None, None


def _lookup_bwd(f1_cl, f2_pyr, coords, g_out, levels):
    """(d fmap1, d fmap2 pyramid) of CorrLookup.  Deterministic mode gathers d fmap2 per pyramid position in a fixed order
    (rnc_corr_lookup_bwd_det, which writes every position); otherwise every pixel scatters into it with atomics."""
    B, H, W, D = f1_cl.shape
    args = (f1_cl, f2_pyr, coords, g_out, g_out.shape[-1], B, D, H, W, levels, 4)
    g_f1 = torch.empty_like(f1_cl)
    if deterministic():
        g_f2 = torch.empty_like(f2_pyr)
        nbytes = rnc.corr_lookup_bwd_workspace_bytes(B, H, W, levels)
        ws = torch.empty((nbytes + 15) // 16, 4, dtype=torch.float32, device=f1_cl.device)
        rnc.corr_lookup_bwd_det(*args, g_f1, g_f2, ws, ws.numel() * 4)
    else:
        g_f2 = torch.zeros_like(f2_pyr)
        rnc.corr_lookup_bwd(*args, g_f1, g_f2)
    return g_f1, g_f2


def corr_lookup_autograd(corr_block, coords):
    """Seam CorrBlock.__call__ with gradients to the NCHW feature maps it was built from."""
    f1 = to_cl(corr_block.fmap1.float())
    pyr = CorrPyramid.apply(to_cl(corr_block.fmap2.float()), corr_block.num_levels)
    out = CorrLookup.apply(f1, pyr, coords, corr_block.num_levels)
    return to_nchw(out)


# --------------------------------------------------------------------------------------------- normalized convolution


class NConv2dFn(torch.autograd.Function):
    """(data, conf, W > 0[, bias, up_data, up_conf]) -> (nconv, conf_out), nconv_modules.py:164-199.  up_data / up_conf: the
    decoder's coarse half, read through the nearest-index map as input channels [0, Cup) (nconv_modules.py:129-131)."""

    @staticmethod
    def forward(ctx, data, conf, weight, eps, bias=None, up_data=None, up_conf=None):
        dev = _require_cuda(data, conf, weight, bias, up_data, up_conf)
        data, conf, weight = data.contiguous(), conf.contiguous(), weight.contiguous()
        bias = None if bias is None else bias.contiguous()
        up = None if up_data is None else (up_data.contiguous(), up_conf.contiguous())
        with torch.cuda.device(dev):
            y, c = nconv_fwd(data, conf, weight, bias, eps, up)
        ctx.save_for_backward(data, conf, weight, bias, y, c, *(up or (None, None)))
        ctx.eps = eps
        return y, c

    @staticmethod
    def backward(ctx, gy, gc):
        data, conf, weight, bias, y, c, ux, uc = ctx.saved_tensors
        N, Cin, H, W = data.shape
        Cout, _, kh, kw = weight.shape
        Cup, Hup, Wup = (ux.shape[1], ux.shape[2], ux.shape[3]) if ux is not None else (0, 0, 0)
        need = ctx.needs_input_grad
        with torch.cuda.device(data.device):
            nbytes = rnc.nconv2d_bwd_workspace_bytes(N, Cin, Cup, Cout, H, W, kh)
            ws = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=data.device)
            g_data = torch.empty_like(data) if need[0] else None
            g_conf = torch.empty_like(conf) if need[1] else None
            g_w = torch.empty_like(weight) if need[2] or (bias is not None and need[4]) else None
            g_b = torch.empty_like(bias) if bias is not None and need[4] else None
            g_ux = torch.empty_like(ux) if ux is not None and need[5] else None
            g_uc = torch.empty_like(uc) if uc is not None and need[6] else None
            rnc.nconv2d_bwd(data, conf, weight, bias, y, c, gy.contiguous() if gy is not None else None,
                            gc.contiguous() if gc is not None else None, N, Cin, Cout, H, W, kh, kw, ctx.eps, ux, uc, Cup, Hup, Wup,
                            g_data, g_conf, g_ux, g_uc, g_w, g_b, ws, ws.numel() * 8)
        return g_data, g_conf, g_w if need[2] else None, None, g_b, g_ux, g_uc


def nconv2d_autograd(data, conf, weight, eps=1e-20, bias=None):
    _require_cuda(data, conf, weight)
    return NConv2dFn.apply(data.float(), conf.float(), weight.float(), eps, None if bias is None else bias.float())


class NConvPoolFn(torch.autograd.Function):
    """NConvUNet.downsample_data_conf (nconv_modules.py:94-104), ds_factor 2: rnc_nconv_pool2_fwd / rnc_nconv_pool2_bwd."""

    @staticmethod
    def forward(ctx, data, conf, max_pool_data):
        dev = _require_cuda(data, conf)
        data, conf = data.contiguous(), conf.contiguous()
        with torch.cuda.device(dev):
            xo, co, idx = pool_fwd(data, conf, max_pool_data)
        ctx.save_for_backward(idx)
        ctx.shape = tuple(data.shape)
        ctx.mark_non_differentiable(idx)
        return xo, co

    @staticmethod
    def backward(ctx, gx, gc):
        (idx,) = ctx.saved_tensors
        N, C, H, W = ctx.shape
        need = ctx.needs_input_grad
        g_data = torch.empty(ctx.shape, dtype=torch.float32, device=idx.device) if need[0] else None
        g_conf = torch.empty(ctx.shape, dtype=torch.float32, device=idx.device) if need[1] else None
        if g_data is None and g_conf is None:
            return None, None, None
        with torch.cuda.device(idx.device):
            rnc.nconv_pool2_bwd(idx, gx.contiguous() if gx is not None else None, gc.contiguous() if gc is not None else None,
                                N, C, H, W, g_data, g_conf)
        return g_data, g_conf, None


# --------------------------------------------------------------------------------------------- module graphs (channel-last)


def _norm_cl(x, norm):
    """InstanceNorm2d / BatchNorm2d / identity on a channel-last tensor (library kernels on a strided NCHW view)."""
    if isinstance(norm, nn.Sequential) and len(norm) == 0:
        return x
    v = x.permute(0, 3, 1, 2)
    if isinstance(norm, nn.InstanceNorm2d):
        v = F.instance_norm(v, eps=norm.eps)
    elif isinstance(norm, nn.BatchNorm2d):
        v = F.batch_norm(v, norm.running_mean, norm.running_var, norm.weight, norm.bias, norm.training, norm.momentum, norm.eps)
    else:
        raise NotImplementedError(type(norm).__name__)
    return v.permute(0, 2, 3, 1).contiguous()


def res_block_cl(blk, x):
    """extractor.py:6-56."""
    y = F.relu(_norm_cl(conv_cl(x, blk.conv1), blk.norm1))
    y = F.relu(_norm_cl(conv_cl(y, blk.conv2), blk.norm2))
    if blk.downsample is not None:
        x = _norm_cl(conv_cl(x, blk.downsample[0]), blk.downsample[1])
    return F.relu(x + y)


def encoder_cl(enc, x_cl):
    """BasicEncoder.forward (extractor.py:160-192) on a channel-last image batch [N,H,W,4] (3 channels + 1 zero)."""
    x = F.relu(_norm_cl(conv_cl(x_cl, enc.conv1), enc.norm1))
    for layer in (enc.layer1, enc.layer2, enc.layer3):
        for blk in layer:
            x = res_block_cl(blk, x)
    x = conv_cl(x, enc.conv2)
    if enc.training and enc.dropout is not None:
        x = enc.dropout(x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1).contiguous()
    return x


def motion_encoder_cl(e, flow_cl, corr_cl):
    """update.py:89-97; flow_cl [B,H,W,4] (2 + 2 zero channels) -> [B,H,W,128] = cat(conv out 126, flow 2)."""
    cor = F.relu(conv_cl(corr_cl, e.convc1))
    cor = F.relu(conv_cl(cor, e.convc2))
    flo = F.relu(conv_cl(flow_cl, e.convf1))
    flo = F.relu(conv_cl(flo, e.convf2))
    out = F.relu(conv_cl(torch.cat([cor, flo], -1), e.conv))          # [B,H,W,128]: channels 126, 127 are zero pads
    return torch.cat([out[..., :126], flow_cl[..., :2]], -1)


def sep_conv_gru_cl(g, h, x):
    """update.py:45-60 on channel-last h [.,128], x [.,256]."""
    for tag in ("1", "2"):
        hx = torch.cat([h, x], -1)
        z = torch.sigmoid(conv_cl(hx, getattr(g, "convz" + tag)))
        r = torch.sigmoid(conv_cl(hx, getattr(g, "convr" + tag)))
        q = torch.tanh(conv_cl(torch.cat([r * h, x], -1), getattr(g, "convq" + tag)))
        h = (1 - z) * h + z * q
    return h


def flow_head_cl(fh, net):
    """update.py:13-14 -> [B,H,W,4] (delta in channels 0, 1)."""
    return conv_cl(F.relu(conv_cl(net, fh.conv1)), fh.conv2)


def update_block_cl(ub, net, inp, corr, flow_cl):
    """update.py:130-141 on channel-last tensors: returns (net, mask or None, delta [B,H,W,4])."""
    motion = motion_encoder_cl(ub.encoder, flow_cl, corr)
    net = sep_conv_gru_cl(ub.gru, net, torch.cat([inp, motion], -1))
    delta = flow_head_cl(ub.flow_head, net)
    mask = None
    if len(ub.mask) > 0:
        mask = 0.25 * conv_cl(F.relu(conv_cl(net, ub.mask[0])), ub.mask[2])
    return net, mask, delta


def simple_cl(wn, x_cl):
    """Simple.forward (interp_weights_est.py:39-47) on channel-last input [B,h,w,132] -> NCHW [B,2,h,w] after final_act."""
    x = x_cl
    for blk in wn.conv:
        x = conv_cl(x, blk[0])
        if len(blk) == 3:
            x = _norm_cl(x, blk[1])
        x = F.relu(x)
    x = conv_cl(x, wn.out)
    return wn.final_act(to_nchw(x, wn.out.out_channels))


def nconv_unet_train(net, data, conf):
    """NConvUNet.forward live path (nconv_modules.py:106-136, SURVEY.md Appendix A.3, rnc/nconv_unet.py) with autograd.
    Parameters that never reach the output (unshared encoder[N]) keep grad None, as in the reference."""
    if not is_fused(net):
        _require_cuda(data, conf, *net.parameters())

        def layer(m, x, c, up=None, last=False):
            return NConv2dFn.apply(x, c, m.weight, m.eps, m.bias, *(up or (None, None)))

        def pool(x, c):
            return NConvPoolFn.apply(x, c, net.data_pooling == "max_pooling")

        return live_chain(net, data.float(), conf.float(), layer, pool)
    x, c = NConv2dFn.apply(data, conf, net.nconv_in.weight, net.nconv_in.eps)
    x, c = NConv2dFn.apply(x, c, net.nconv_x2[0].weight, net.nconv_x2[0].eps)
    x, c = NConv2dFn.apply(torch.cat((x, x), 1), torch.cat((c, c), 1), net.decoder[0].weight, net.decoder[0].eps)
    return NConv2dFn.apply(x, c, net.nconv_out.weight, net.nconv_out.eps)


class NcupChainFn(torch.autograd.Function):
    """Zero-stuffing + the live NConvUNet chain + out_scale (upsampler.py:143-177 after the weights net, nconv_modules.py:106-136)
    as one fused kernel forward (rnc_ncup_train_fwd) and one fused backward (rnc_ncup_bwd):
    (x_lowres, conf) NCHW [B,2,H4,W4], the positive kernels W1 [2,1,5,5], W2 [2,2,5,5], W3 [2,4,3,3], W4 [1,2,1,1]
    -> out NCHW [B,2,4*H4,4*W4], or with want_conf (out, conf_out): the chain's output confidence den4 / sum(W4) of nconv_out
    in the layout of out, without out_scale; out is the same either way.  The same function as the per-layer NConv2dFn chain
    of ncup_upsampler_train, with gradients that are bit-identical from call to call; when the loss does not use conf_out
    they are those of want_conf=False, bit for bit."""

    SHAPES = ((2, 1, 5, 5), (2, 2, 5, 5), (2, 4, 3, 3), (1, 2, 1, 1))

    @staticmethod
    def forward(ctx, x_lowres, conf, w1, w2, w3, w4, out_scale, want_conf=False):
        if x_lowres.dim() != 4 or x_lowres.shape[1] != 2 or conf.shape != x_lowres.shape:
            raise ValueError("NcupChainFn: x_lowres and conf must both be [B,2,H4,W4]")
        if tuple(tuple(w.shape) for w in (w1, w2, w3, w4)) != NcupChainFn.SHAPES:
            raise ValueError(f"NcupChainFn: weights must have shapes {NcupChainFn.SHAPES}")
        _require_cuda(x_lowres)
        x_lowres, conf = x_lowres.detach().float().contiguous(), conf.detach().float().contiguous()
        wts = torch.cat([w.detach().float().reshape(-1) for w in (w1, w2, w3, w4)])
        B, _, H4, W4 = x_lowres.shape
        out = torch.empty(B, 2, 4 * H4, 4 * W4, dtype=torch.float32, device=x_lowres.device)
        cout = torch.empty_like(out) if want_conf else None
        rnc.ncup_train_fwd(x_lowres, conf, wts, B, H4, W4, float(out_scale), out, cout)
        ctx.save_for_backward(x_lowres, conf, wts)
        ctx.out_scale = float(out_scale)
        ctx.set_materialize_grads(False)        # an unused output's gradient stays None: the kernel skips its term
        return (out, cout) if want_conf else out

    @staticmethod
    def backward(ctx, g_out, g_cout=None):
        x_lowres, conf, wts = ctx.saved_tensors
        B, _, H4, W4 = x_lowres.shape
        need_w = any(ctx.needs_input_grad[2:6])
        if g_out is None and g_cout is None:
            return (None,) * 8
        with torch.cuda.device(x_lowres.device):
            g_out = g_out.float().contiguous() if g_out is not None else None
            g_cout = g_cout.float().contiguous() if g_cout is not None else None
            g_x = torch.empty_like(x_lowres) if ctx.needs_input_grad[0] else None
            g_c = torch.empty_like(conf) if ctx.needs_input_grad[1] else None
            g_w = ws = None
            if need_w:
                g_w = torch.empty(224, dtype=torch.float32, device=x_lowres.device)
                nbytes = rnc.ncup_bwd_workspace_bytes(B, H4, W4)
                ws = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=x_lowres.device)
            if g_x is None and g_c is None and g_w is None:
                return (None,) * 8
            rnc.ncup_bwd(x_lowres, conf, wts, B, H4, W4, ctx.out_scale, g_out, g_cout, g_x, g_c, g_w, ws,
                         ws.numel() * 8 if ws is not None else 0)
        gws = [None] * 4
        if g_w is not None:
            off = 0
            for k, shp in enumerate(NcupChainFn.SHAPES):
                n = shp[0] * shp[1] * shp[2] * shp[3]
                gws[k] = g_w[off:off + n].view(shp) if ctx.needs_input_grad[2 + k] else None
                off += n
        return (g_x, g_c, *gws, None, None)


def ncup_chain_autograd(net, x_lowres, conf, out_scale=1.0, want_conf=False):
    """The NConvUNet `net` (live path) on zero-stuffed (x_lowres, conf), times out_scale, through NcupChainFn; want_conf:
    (out, output confidence)."""
    _require_cuda(x_lowres, conf)
    args = (x_lowres, conf, net.nconv_in.weight, net.nconv_x2[0].weight, net.decoder[0].weight, net.nconv_out.weight, out_scale)
    # want_conf goes to apply only when set: a flow-only call passes the chain's seven inputs alone, the arguments that
    # wrappers of NcupChainFn.apply (tests/test_gpu_train_shapes.py) unpack
    return NcupChainFn.apply(*args, True) if want_conf else NcupChainFn.apply(*args)


def ncup_upsampler_frozen(up, x4, gin, out_scale=8.0, want_conf=False):
    """NConvUpsampler.forward (upsampler.py:143-177) for a frozen trunk: x4 NCHW [B,2,H4,W4] and the weights-net input gin
    (CL [B,H4,W4,136] = cat(x4, area-resized guidance), zero channels beyond 130; rnc_ncup_guidance_fwd) are the trunk's
    detached outputs.  The weights net runs on ConvCL (BatchNorm as configured), the chain on NcupChainFn (with want_conf it
    returns (out, confidence))."""
    with torch.cuda.device(x4.device):
        conf = simple_cl(up.weights_est_net, gin)
        return _ncup_chain_train(up.interpolation_net, x4, conf, out_scale, fused=True, want_conf=want_conf)


def _ncup_chain_train(net, x_lowres, conf, out_scale, fused, want_conf=False):
    """NConvUpsampler.forward after the weights net (upsampler.py:150-177) with autograd: zero-stuffing, the NConvUNet `net`,
    out_scale; x_lowres, conf NCHW [B,2,H4,W4] -> [B,2,4*H4,4*W4].  fused: the shipped network runs on NcupChainFn, with
    out_scale applied inside the kernel; otherwise every network runs the per-layer NConv2dFn chain (the full-training path
    keeps it: the fused backward rounds the gradients differently).  want_conf: (out, the network's output confidence in the
    layout of out, without out_scale)."""
    if fused and is_fused(net):
        return ncup_chain_autograd(net, x_lowres, conf, out_scale, want_conf)
    xh, ch = zero_stuff(x_lowres), zero_stuff(conf)
    b, c, oh, ow = xh.shape
    out, cout = nconv_unet_train(net, xh.view(b * c, 1, oh, ow), ch.view(b * c, 1, oh, ow))
    out = out.view(b, c, oh, ow)
    out = out * out_scale if out_scale != 1.0 else out
    return (out, cout.view(b, c, oh, ow)) if want_conf else out


def zero_stuff(x, scale=4):
    """upsampler.py:179-210: zeros [B,C,s*h,s*w] with out[..., s//2::s, s//2::s] = x."""
    b, c, h, w = x.shape
    out = torch.zeros(b, c, h * scale, w * scale, dtype=x.dtype, device=x.device)
    out[:, :, scale // 2::scale, scale // 2::scale] = x
    return out


def ncup_upsampler_train(up, x_lowres, x_guidance, out_scale=1.0, return_confidence=False):
    """NConvUpsampler.forward (upsampler.py:143-177) with autograd: x_lowres NCHW [B,2,h,w], guidance NCHW [B,128,h/2,w/2].
    return_confidence: (out, output confidence [B,2,4h,4w]), both differentiable."""
    _require_cuda(x_lowres, x_guidance)
    with torch.cuda.device(x_lowres.device):
        # the reference's F.interpolate(mode='area') to twice the size: every area window holds one element, so it is the
        # nearest x2 replication, whose backward adds each element's four terms in a fixed order (area's adds them atomically)
        if tuple(x_lowres.shape[2:]) != (2 * x_guidance.shape[2], 2 * x_guidance.shape[3]):
            raise ValueError("ncup_upsampler_train: the guidance must have half the resolution of x_lowres")
        g4 = F.interpolate(x_guidance, scale_factor=2, mode="nearest")
        w4 = simple_cl(up.weights_est_net, to_cl(torch.cat([x_lowres, g4], 1), pad_to=136))     # pitch % 8 == 0: tensor-core layer
        return _ncup_chain_train(up.interpolation_net, x_lowres, w4, out_scale, fused=False, want_conf=return_confidence)


def simple_train(wn, x):
    with torch.cuda.device(x.device):
        return simple_cl(wn, to_cl(x.float()))


def flow_head_train(fh, x):
    with torch.cuda.device(x.device):
        return to_nchw(flow_head_cl(fh, to_cl(x.float())), 2)


def sep_conv_gru_train(g, h, x):
    with torch.cuda.device(h.device):
        return to_nchw(sep_conv_gru_cl(g, to_cl(h.float()), to_cl(x.float())))


def motion_encoder_train(e, flow, corr):
    with torch.cuda.device(flow.device):
        return to_nchw(motion_encoder_cl(e, to_cl(flow.float()), to_cl(corr.float())))


def update_block_train(ub, net, inp, corr, flow):
    """BasicUpdateBlock.forward (update.py:130-141) with autograd, NCHW in / out."""
    with torch.cuda.device(net.device):
        n, m, d = update_block_cl(ub, to_cl(net.float()), to_cl(inp.float()), to_cl(corr.float()), to_cl(flow.float()))
        net_out = to_nchw(n)
        ub.net = net_out
        mask = to_nchw(m) if m is not None else 0.25 * net_out
        return net_out, mask, to_nchw(d, 2)


def convex_upsample_train(flow, mask):
    """raft.py:73-84 (model `raft`), pointwise torch ops: softmax over the 9 neighbours x unfold(8 * flow)."""
    n, _, h, w = flow.shape
    m = torch.softmax(mask.view(n, 1, 9, 8, 8, h, w), dim=2)
    nb = F.unfold(8 * flow, [3, 3], padding=1).view(n, 2, 9, 1, 1, h, w)
    up = torch.sum(m * nb, dim=2).permute(0, 1, 4, 2, 5, 3)
    return up.reshape(n, 2, 8 * h, 8 * w)


def raft_forward_train(model, image1, image2, iters=12, flow_init=None, test_mode=False, return_confidence=False):
    """RAFT.forward with autograd (raft_nc_dbl.py:115-173 / raft.py:87-143): returns the list of `iters` full-resolution
    predictions (or (flow_low, flow_up) in test_mode).  return_confidence (NCUP model): also the NCUP output confidences,
    as (predictions, confidences) or (flow_low, flow_up, confidence_up)."""
    _PACK_CACHE.clear()
    B, _, Him, Wim = image1.shape
    H8, W8 = Him // 8, Wim // 8
    dev = image1.device
    im1 = 2 * (image1.float() / 255.0) - 1.0
    im2 = 2 * (image2.float() / 255.0) - 1.0
    fmaps = encoder_cl(model.fnet, to_cl(torch.cat([im1, im2], 0))).float()       # [2B,H8,W8,256]
    f1, f2 = fmaps[:B].contiguous(), fmaps[B:].contiguous()
    pyr = CorrPyramid.apply(f2, 4)
    cnet = encoder_cl(model.cnet, to_cl(im1))
    net, inp = torch.tanh(cnet[..., :128]), torch.relu(cnet[..., 128:])
    ys, xs = torch.meshgrid(torch.arange(H8, device=dev), torch.arange(W8, device=dev), indexing="ij")
    coords0 = torch.stack([xs, ys], 0).float()[None].repeat(B, 1, 1, 1)
    coords1 = coords0.clone()
    if flow_init is not None:
        coords1 = coords1 + flow_init
    preds, confs = [], []
    ub = model.update_block
    for _ in range(iters):
        coords1 = coords1.detach()                                                  # raft_nc_dbl.py:149
        corr = CorrLookup.apply(f1, pyr, coords1, 4)
        flow = coords1 - coords0
        net, mask, delta = update_block_cl(ub, net, inp, corr, to_cl(flow))
        ub.net = net                                                                # guidance tap (update.py:135), channel-last here
        coords1 = coords1 + to_nchw(delta, 2)
        flow_lr = coords1 - coords0
        if model.ncup:
            x4 = F.interpolate(flow_lr, scale_factor=2, mode="nearest")             # raft_nc_dbl.py:110
            if return_confidence:
                flow_up, conf_up = ncup_upsampler_train(model.upsampler, x4, to_nchw(net), return_confidence=True)
                flow_up = 8 * flow_up                                               # raft_nc_dbl.py:161 (not on the conf)
                confs.append(conf_up)
            else:
                flow_up = 8 * ncup_upsampler_train(model.upsampler, x4, to_nchw(net))   # raft_nc_dbl.py:161
        else:
            flow_up = convex_upsample_train(flow_lr, to_nchw(mask))
        preds.append(flow_up)
    ub.net = to_nchw(net)
    if test_mode:
        return (coords1 - coords0, preds[-1], confs[-1]) if return_confidence else (coords1 - coords0, preds[-1])
    return (preds, confs) if return_confidence else preds


# --------------------------------------------------------------------------------------------- loss / optimiser / step (train.py)

MAX_FLOW = 400


def sequence_loss(flow_preds, flow_gt, valid, gamma=0.8, max_flow=MAX_FLOW):
    """train.py:46-71 — gamma-weighted L1 over the prediction sequence; invalid pixels count in the mean's denominator."""
    n = len(flow_preds)
    mag = torch.sum(flow_gt ** 2, dim=1).sqrt()
    valid = (valid >= 0.5) & (mag < max_flow)
    loss = 0.0
    for i, pred in enumerate(flow_preds):
        loss = loss + gamma ** (n - i - 1) * (valid[:, None] * (pred - flow_gt).abs()).mean()
    epe = torch.sum((flow_preds[-1] - flow_gt) ** 2, dim=1).sqrt().view(-1)[valid.view(-1)]
    metrics = {"epe": epe.mean().item(), "1px": (epe < 1).float().mean().item(), "3px": (epe < 3).float().mean().item(),
               "5px": (epe < 5).float().mean().item()}
    return loss, metrics


def fetch_optimizer(model, lr=2e-5, wdecay=5e-5, epsilon=1e-8, num_steps=100000):
    """train.py:83-99 (the shipped scripts: AdamW + OneCycleLR, linear anneal, pct_start 0.05, no momentum cycling)."""
    opt = torch.optim.AdamW(model.parameters(), lr=lr, weight_decay=wdecay, eps=epsilon)
    sched = torch.optim.lr_scheduler.OneCycleLR(opt, lr, num_steps + 100, pct_start=0.05, cycle_momentum=False, anneal_strategy="linear")
    return opt, sched


def train_step(model, optimizer, scheduler, image1, image2, flow_gt, valid, iters=12, gamma=0.85, clip=1.0, return_metrics=True):
    """One optimisation step exactly as train.py:203-227 without AMP: zero_grad, forward (list of predictions), sequence_loss,
    backward (under DistributedDataParallel: gradient all-reduce overlapped with it), clip_grad_norm_(clip), step."""
    optimizer.zero_grad()
    preds = model(image1, image2, iters=iters)
    loss, metrics = sequence_loss(preds, flow_gt, valid, gamma)
    loss.backward()
    torch.nn.utils.clip_grad_norm_(model.parameters(), clip)
    optimizer.step()
    if scheduler is not None:
        scheduler.step()
    return loss.detach(), (metrics if return_metrics else None)


def has_unused_parameters(model):
    """Does some parameter of `model` never reach the loss?  Only an NConvUNet with unshared encoders has such parameters
    (encoder[N], behind the decoder's index quirk, nconv_modules.py:128-131); every other parameter receives a gradient
    (SURVEY.md Appendix G)."""
    m = getattr(model, "module", model)
    up = getattr(m, "upsampler", None)
    return up is not None and bool(unused_parameters(up.interpolation_net))


def ddp_model(model, device, bucket_cap_mb=8):
    """train.py:169-175 wraps the model in single-process nn.DataParallel; here: one process per GPU, replicas kept in sync by
    DistributedDataParallel's bucketed NCCL all-reduce of the gradients (19.6 MB fp32).  DDP searches for unused parameters
    only when the configuration has some (has_unused_parameters).  The NConv encoder aliases are one Parameter object: DDP
    sees it once."""
    from torch.nn.parallel import DistributedDataParallel as DDP
    return DDP(model.to(device), device_ids=[device.index], bucket_cap_mb=bucket_cap_mb, broadcast_buffers=False,
               gradient_as_bucket_view=True, find_unused_parameters=has_unused_parameters(model))
