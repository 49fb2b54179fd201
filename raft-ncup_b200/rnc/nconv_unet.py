"""NConvUNet (core/nconv_modules.py:25-136) in every configuration the drop-in accepts: its live path, written once over a
layer operation and a pooling operation, and run by the inference seams, by both engines' upsamplers and (with autograd
Functions as the operations) by the training path.

Live path, with N = num_downsampling and x_k the encoder output at level k (resolution 2^-k, floor sizes):
  N = 0:   nconv_in -> nconv_x2 -> nconv_out
  N >= 1:  x_0 = nconv_x2(nconv_in(data)),  x_k = encoder[k](pool(x_{k-1})) for k = 1 .. N-1.
           Decoder i reads x[i+N] of the reference's list (the index quirk at :128-131), so decoder 0 runs on
           cat(x_{N-1}, x_{N-1}) and decoder i >= 1 on cat(nearest-upsampled decoder i-1 output, x_{N-1-i}); then nconv_out.
           The deepest level, pool(x_{N-1}) -> encoder[N], never reaches the output and is not computed.
The decoder's concatenation is a read pattern of rnc_nconv2d_fwd (the "up" source), never a materialised tensor.
"""
import torch

from .native import rnc


def is_fused(net):
    """Does the fused chain of ncup.cu (rnc_ncup_fwd / rnc_ncup_train_fwd / rnc_ncup_bwd) compute this network's output?
    It is built for the configuration every reference script ships: m = 2, one downsampling, filters 5 / 3 / 1, single
    convolutions, no bias (data pooling and encoder sharing only touch the dead level)."""
    return (net.channels, net.num_downsampling, net.filter_sizes, net.use_double_conv, net.use_bias) == \
        (2, 1, (5, 3, 1), False, False)


def unused_parameters(net):
    """Parameters of `net` that never reach its output: encoder[N].weight_p (and bias) when the encoders are unshared."""
    if net.num_downsampling == 0 or net.shared_encoder:
        return []
    return list(net.encoder[net.num_downsampling].parameters())


def live_chain(net, data, conf, layer, pool):
    """Run the live path.  layer(mod, x, c, up=None, last=False) -> (x, c), where up = (x_up, c_up) is the decoder's coarse
    half and last marks nconv_out; pool(x, c) -> (x, c) is downsample_data_conf with the network's data pooling."""
    x, c = layer(net.nconv_in, data, conf)
    for m in net.nconv_x2:
        x, c = layer(m, x, c)
    n = net.num_downsampling
    if n == 0:
        return layer(net.nconv_out, x, c, last=True)
    skips = [(x, c)]
    for k in range(1, n):
        x, c = layer(net.encoder[k], *pool(x, c))
        skips.append((x, c))
    up = skips[-1]
    for i in range(n):
        up = layer(net.decoder[i], *skips[n - 1 - i], up=up)
    return layer(net.nconv_out, *up, last=True)


def _empty(shape, like, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device=like.device)


def nconv_fwd(x, c, weight, bias, eps, up=None, y_scale=1.0, alloc=_empty):
    """One rnc_nconv2d_fwd on the current stream: (x, c) NCHW fp32 contiguous, weight the positive kernel
    [Cout][Cup+Cin][kh][kw], up = optional coarse (x_up, c_up) read through the nearest-index map; alloc(shape, like)
    provides the outputs."""
    N, Cin, H, W = x.shape
    Cout, Ct, kh, kw = weight.shape
    ux, uc = up if up is not None else (None, None)
    Cup, Hup, Wup = (ux.shape[1], ux.shape[2], ux.shape[3]) if up is not None else (0, 0, 0)
    if c.shape != x.shape or Ct != Cin + Cup or (up is not None and (uc.shape != ux.shape or ux.shape[0] != N)):
        raise ValueError("NConv2d: data/conf/weight shapes do not match")
    y, co = alloc((N, Cout, H, W), x), alloc((N, Cout, H, W), x)
    rnc.nconv2d_fwd(x, c, weight, bias, N, Cin, Cout, H, W, kh, kw, eps, ux, uc, Cup, Hup, Wup, float(y_scale), y, co)
    return y, co


def pool_fwd(x, c, max_pool_data, alloc=_empty):
    """rnc_nconv_pool2_fwd: (data, conf) -> (data_ds, conf_ds, idx [2][N][C][H/2][W/2] int32)."""
    N, C, H, W = x.shape
    xo, co = alloc((N, C, H // 2, W // 2), x), alloc((N, C, H // 2, W // 2), x)
    idx = alloc((2, N, C, H // 2, W // 2), x, torch.int32)
    rnc.nconv_pool2_fwd(x, c, N, C, H, W, int(max_pool_data), xo, co, idx)
    return xo, co, idx


class PackedUNet:
    """Positive kernels (softplus_{beta=10}(weight_p), computed once per weight version) and biases of a network's layers,
    on the network's device, keyed by module."""

    def __init__(self, net):
        self.net = net
        self.max_pool_data = net.data_pooling == "max_pooling"
        self.w = {}
        for m in net.modules():
            if hasattr(m, "weight_p") and id(m) not in self.w:
                b = None if m.bias is None else m.bias.detach().float().contiguous()
                self.w[id(m)] = (m.weight.detach().float().contiguous(), b, m.eps)

    def run(self, data, conf, out_scale=1.0, bufs=None):
        """The live path on NCHW fp32 contiguous (data, conf), out_scale folded into nconv_out -> (y, conf_out).  bufs: an
        optional dict that keeps the intermediates between calls (a workspace); the outputs are always new tensors."""
        seq = iter(range(1 << 30))

        def alloc(shape, like, dtype=torch.float32):
            if bufs is None:
                return _empty(shape, like, dtype)
            key = (next(seq), tuple(shape), dtype)
            if key not in bufs:
                bufs[key] = _empty(shape, like, dtype)
            return bufs[key]

        def layer(m, x, c, up=None, last=False):
            w, b, eps = self.w[id(m)]
            return nconv_fwd(x, c, w, b, eps, up, out_scale if last else 1.0, _empty if last else alloc)

        def pool(x, c):
            return pool_fwd(x, c, self.max_pool_data, alloc)[:2]

        return live_chain(self.net, data, conf, layer, pool)
