"""Pure-torch restatement of NConvUNet's general live path (core/nconv_modules.py:25-136) over a state_dict, for every
configuration the drop-in accepts.  TEST INFRASTRUCTURE ONLY: differentiable, and runs in any dtype (fp64 for gradient
checks).

cfg keys: m (channels_multiplier), nds, enc / dec / out (filter sizes), double, shared, pooling ('conf_based' |
'max_pooling'), bias.
"""
import torch
import torch.nn.functional as F

CONFIGS = {
    "paper": dict(m=2, nds=3, enc=5, dec=3, out=1, double=True, shared=True, pooling="conf_based", bias=False),
    "n2_maxpool_bias": dict(m=2, nds=2, enc=5, dec=3, out=1, double=False, shared=True, pooling="max_pooling", bias=True),
    "n2_unshared": dict(m=2, nds=2, enc=5, dec=3, out=1, double=False, shared=False, pooling="conf_based", bias=False),
    "n0_double": dict(m=2, nds=0, enc=5, dec=3, out=1, double=True, shared=True, pooling="conf_based", bias=False),
    "wide": dict(m=4, nds=2, enc=3, dec=5, out=3, double=False, shared=True, pooling="conf_based", bias=False),
    "thin": dict(m=1, nds=2, enc=7, dec=3, out=1, double=False, shared=True, pooling="conf_based", bias=False),
}


def unet_kwargs(cfg):
    """NConvUNet constructor arguments of a configuration."""
    return dict(in_ch=1, channels_multiplier=cfg["m"], num_downsampling=cfg["nds"], encoder_filter_sz=cfg["enc"],
                decoder_filter_sz=cfg["dec"], out_filter_sz=cfg["out"], use_bias=cfg["bias"], data_pooling=cfg["pooling"],
                shared_encoder=cfg["shared"], use_double_conv=cfg["double"])


def args_overrides(cfg):
    """The reference's --interp_net_* flags (core/upsampler.py:17-25) of a configuration."""
    k = unet_kwargs(cfg)
    return {"interp_net_" + a: k[b] for a, b in (
        ("channels_multiplier", "channels_multiplier"), ("num_downsampling", "num_downsampling"),
        ("encoder_filter_sz", "encoder_filter_sz"), ("decoder_filter_sz", "decoder_filter_sz"),
        ("out_filter_sz", "out_filter_sz"), ("use_bias", "use_bias"), ("data_pooling", "data_pooling"),
        ("shared_encoder", "shared_encoder"), ("use_double_conv", "use_double_conv"))}


def nconv(sd, name, data, conf, eps=1e-20):
    """NConv2d.forward (:164-199) with the layer's weight_p (softplus, beta 10) and optional bias."""
    w = F.softplus(sd[name + ".weight_p"], beta=10)
    pad = w.shape[-1] // 2
    den = F.conv2d(conf, w, padding=pad)
    num = F.conv2d(data * conf, w, padding=pad)
    y = num / (den + eps)
    b = sd.get(name + ".bias")
    if b is not None:
        y = y + b.view(1, -1, 1, 1)
    s = w.reshape(w.shape[0], -1).sum(-1).view(1, -1, 1, 1)
    return y, den / s


def pool(data, conf, pooling):
    """downsample_data_conf (:94-104), ds_factor 2."""
    c, idx = F.max_pool2d(conf, 2, 2, return_indices=True)
    c = c / 4
    if pooling == "conf_based":
        d = data.flatten(2).gather(2, idx.flatten(2)).view_as(idx)
    else:
        d = F.max_pool2d(data, 2, 2)
    return d, c


def unet(sd, cfg, data, conf, p=""):
    """NConvUNet.forward on the live path: the deepest level never reaches the output (decoder i reads x[i+N])."""
    def layer(name, x, c):
        return nconv(sd, p + name, x, c)

    x, c = layer("nconv_in", data, conf)
    for j in range(2 if cfg["double"] else 1):
        x, c = layer(f"nconv_x2.{j}", x, c)
    n = cfg["nds"]
    if n == 0:
        return layer("nconv_out", x, c)
    skips = [(x, c)]
    for k in range(1, n):
        x, c = layer("nconv_x2.0" if cfg["shared"] else f"encoder.{k}", *pool(x, c, cfg["pooling"]))   # shared: one layer
        skips.append((x, c))
    ux, uc = skips[-1]
    for i in range(n):
        sx, sc = skips[n - 1 - i]
        ux = F.interpolate(ux, size=sx.shape[2:], mode="nearest")
        uc = F.interpolate(uc, size=sx.shape[2:], mode="nearest")
        ux, uc = layer(f"decoder.{i}", torch.cat((ux, sx), 1), torch.cat((uc, sc), 1))
    return layer("nconv_out", ux, uc)


def live_parameter_names(cfg):
    """named_parameters() names (first alias of shared layers) that receive a gradient."""
    names = ["nconv_in"] + [f"nconv_x2.{j}" for j in range(2 if cfg["double"] else 1)]
    if not cfg["shared"]:
        names += [f"encoder.{k}" for k in range(1, cfg["nds"])]
    names += [f"decoder.{i}" for i in range(cfg["nds"])] + ["nconv_out"]
    out = []
    for n in names:
        out.append(n + ".weight_p")
        if cfg["bias"] and n != "nconv_out":
            out.append(n + ".bias")
    return out
