"""NConvUNet configurations beyond the shipped one, host side: parameters and state_dict keys against the reference's
goldens, the restated oracle against the reference's outputs and gradients, the options that stay unsupported, the argument
checks of the new entry points, and the DDP unused-parameter predicate."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import ROOT, ref_args
from oracle import ncup_oracle as nco
from oracle.make_golden import tensor_sha

CONFIGS = list(nco.CONFIGS)


@pytest.fixture(scope="module")
def ng():
    z = np.load(os.path.join(ROOT, "tests", "golden", "ncup_cfg.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


@pytest.fixture(scope="module")
def nmeta():
    with open(os.path.join(ROOT, "tests", "golden", "ncup_cfg_meta.json")) as f:
        return json.load(f)


def variant_args(cfg):
    a = ref_args()
    for k, v in nco.args_overrides(cfg).items():
        setattr(a, k, v)
    return a


def golden_sd(ng, name):
    p = f"{name}_sd_"
    return {k[len(p):]: v for k, v in ng.items() if k.startswith(p)}


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


@pytest.mark.parametrize("name", CONFIGS)
def test_state_dict_matches_reference(nmeta, name):
    """Seed 1234 -> the reference's keys (incl. encoder.* aliases), shapes and bit-identical values (RNG draw order)."""
    import raft_nc_dbl
    torch.manual_seed(1234)
    sd = raft_nc_dbl.RAFT(variant_args(nco.CONFIGS[name])).state_dict()
    ref = nmeta[f"{name}_state_sha"]
    assert set(sd) == set(ref)
    assert all(list(v.shape) == nmeta[f"{name}_state_shape"][k] for k, v in sd.items())
    assert all(tensor_sha(v) == ref[k] for k, v in sd.items())


@pytest.mark.parametrize("name", CONFIGS)
def test_unet_state_dict_loads_into_the_drop_in(ng, name):
    from nconv_modules import NConvUNet
    torch.manual_seed(4321)
    net = NConvUNet(**nco.unet_kwargs(nco.CONFIGS[name]))
    sd = golden_sd(ng, name)
    assert list(net.state_dict()) == list(sd)
    assert all(torch.equal(v, sd[k]) for k, v in net.state_dict().items())


@pytest.mark.parametrize("inp", ["even", "odd"])
@pytest.mark.parametrize("name", CONFIGS)
def test_oracle_matches_reference_outputs_and_gradients(ng, nmeta, name, inp):
    cfg = nco.CONFIGS[name]
    sd = {k: v.double().requires_grad_(v.is_floating_point()) for k, v in golden_sd(ng, name).items()}
    d = ng[f"in_{inp}_data"].double().requires_grad_(True)
    c = ng[f"in_{inp}_conf"].double().requires_grad_(True)
    xo, co = nco.unet(sd, cfg, d, c)
    assert (xo - ng[f"{name}_{inp}_xout"]).abs().max() < 1e-4
    assert (co - ng[f"{name}_{inp}_cout"]).abs().max() < 1e-6
    g = torch.Generator().manual_seed(5)
    p1 = torch.randn(xo.shape, generator=g).double()
    p2 = torch.randn(co.shape, generator=g).double()
    ((p1 * xo).sum() + (p2 * co).sum()).backward()
    gd, gc = ng[f"{name}_{inp}_gdata"], ng[f"{name}_{inp}_gconf"]
    ok = gd.abs() < 1e6
    assert rel(d.grad[ok], gd[ok]) < 1e-4
    ok = gc.abs() < 1e6
    assert rel(c.grad[ok], gc[ok]) < 1e-4
    live = nco.live_parameter_names(cfg)
    none = nmeta[f"{name}_{inp}_grad_none"]
    for pn in live:
        assert pn not in none
        ref = ng[f"{name}_{inp}_g_{pn}"]
        # a layer's output is invariant to a common scale of its weights, so its weight gradient is a cancellation whose
        # fp32 value (summed over every pixel) carries rounding noise; nconv_out with one input channel: zero in exact arithmetic
        assert (sd[pn].grad - ref).abs().max() < 1e-3 * max(1.0, ref.abs().max().item()), pn


@pytest.mark.parametrize("kwargs,what", [
    (dict(in_ch=2), "in_ch"), (dict(groups=2), "groups"), (dict(pos_fn="Exp"), "pos_fn"),
    (dict(channels_multiplier=5), "channels_multiplier"), (dict(encoder_filter_sz=9), "encoder_filter_sz"),
    (dict(decoder_filter_sz=4), "decoder_filter_sz"), (dict(out_filter_sz=9), "out_filter_sz"),
    (dict(data_pooling="avg"), "data_pooling")])
def test_unsupported_unet_options_name_themselves(kwargs, what):
    from nconv_modules import NConvUNet
    with pytest.raises(NotImplementedError, match=what):
        NConvUNet(**kwargs)


@pytest.mark.parametrize("flag,value,what", [
    ("final_upsampling_use_residuals", True, "use_residuals"), ("final_upsampling_est_on_high_res", True, "est_on_high_res"),
    ("final_upsampling_use_data_for_guidance", False, "use_data_for_guidance"),
    ("final_upsampling_channels_to_batch", False, "channels_to_batch"), ("final_upsampling_scale", 8, "scale"),
    ("weights_est_net", "unet", "weights_est_net")])
def test_unsupported_upsampler_options_name_themselves(flag, value, what):
    import raft_nc_dbl
    a = ref_args()
    setattr(a, flag, value)
    with pytest.raises(NotImplementedError, match=what):
        raft_nc_dbl.RAFT(a)


def test_nconv_bias_draws_like_the_reference():
    """_ConvNd.reset_parameters draws weight then bias; init_parameters redraws both (nconv_modules.py:201-215)."""
    from nconv_modules import NConv2d
    torch.manual_seed(3)
    m = NConv2d(2, 3, (3, 3), bias=True)
    torch.manual_seed(3)
    w = torch.empty(3, 2, 3, 3)
    torch.nn.init.kaiming_uniform_(w, a=5 ** 0.5)
    b = torch.empty(3)
    torch.nn.init.uniform_(b, -1 / 18 ** 0.5, 1 / 18 ** 0.5)
    w.normal_(2, (2.0 / 27) ** 0.5)
    torch.nn.init.uniform_(b, -1 / 18 ** 0.5, 1 / 18 ** 0.5)
    assert torch.equal(m.bias.detach(), b) and torch.equal(m.weight_p.detach(), torch.nn.functional.softplus(w, beta=10))
    assert list(m.state_dict()) == ["bias", "weight_p"]


def test_new_entry_points_reject_bad_arguments():
    """Argument checks return before any launch: no device is touched."""
    from rnc import native
    L = native.lib()
    P = 4096                                                  # any non-null address: nothing is dereferenced
    f = L.rnc_nconv2d_fwd

    def fwd(N=1, Cin=2, Cout=2, H=8, W=8, kh=3, kw=3, Cup=0, Hup=0, Wup=0, data=P, y=P):
        return f(data, P, P, None, N, Cin, Cout, H, W, kh, kw, 1e-20, P, P, Cup, Hup, Wup, 1.0, y, P, None)

    assert fwd(N=0) == -1 and fwd(Cin=0) == -1 and fwd(Cup=2, Hup=0, Wup=4) == -1
    assert fwd(Cin=5, Cup=4, Hup=4, Wup=4) == -3 and fwd(Cout=5) == -3 and fwd(kh=4) == -3 and fwd(kw=9) == -3
    assert fwd(data=None) == -2 and fwd(y=None) == -2
    b = L.rnc_nconv2d_bwd
    ws = L.rnc_nconv2d_bwd_workspace_bytes(2, 4, 4, 4, 16, 16, 7)
    assert ws > 0 and L.rnc_nconv2d_bwd_workspace_bytes(2, 5, 4, 4, 16, 16, 7) == 0

    def bwd(gy=P, wsb=ws, Cin=4, g_bias=None, g_w=P):
        return b(P, P, P, None, P, P, gy, None, 2, Cin, 4, 16, 16, 7, 7, 1e-20, P, P, 4, 8, 8, P, P, P, P, g_w, g_bias,
                 P, wsb, None)

    assert bwd(Cin=5) == -3 and bwd(gy=None) == -2 and bwd(g_bias=P, g_w=None) == -2 and bwd(wsb=ws - 8) == -5
    assert L.rnc_nconv_pool2_fwd(P, P, 1, 2, 1, 8, 0, P, P, P, None) == -1
    assert L.rnc_nconv_pool2_fwd(P, P, 1, 2, 8, 8, 2, P, P, P, None) == -3
    assert L.rnc_nconv_pool2_fwd(P, P, 1, 2, 8, 8, 0, P, P, None, None) == -2
    assert L.rnc_nconv_pool2_bwd(P, P, P, 0, 2, 8, 8, P, P, None) == -1
    assert L.rnc_nconv_pool2_bwd(P, P, P, 1, 2, 8, 8, None, None, None) == -2


@pytest.mark.parametrize("name", CONFIGS + ["shipped"])
def test_ddp_unused_parameter_predicate(nmeta, name):
    import raft_nc_dbl
    from rnc.train import has_unused_parameters
    a = ref_args() if name == "shipped" else variant_args(nco.CONFIGS[name])
    m = raft_nc_dbl.RAFT(a)
    expect = name != "shipped" and bool(nmeta[f"{name}_even_grad_none"])
    assert has_unused_parameters(m) == expect


def test_training_on_cpu_tensors_fails_loudly():
    """A non-shipped NConvUNet on the CPU, called with grad enabled, raises instead of launching on host pointers."""
    from nconv_modules import NConvUNet
    from rnc.native import RncUnavailable
    from rnc.train import NConv2dFn, NConvPoolFn
    net = NConvUNet()                                         # the reference defaults: N = 3, double convolutions
    x, c = torch.rand(1, 1, 16, 16), torch.rand(1, 1, 16, 16)
    with pytest.raises(RncUnavailable):
        net((x, c))
    with pytest.raises(RncUnavailable):
        NConv2dFn.apply(x, c, torch.rand(2, 1, 3, 3, requires_grad=True), 1e-20)
    with pytest.raises(RncUnavailable):
        NConvPoolFn.apply(x.requires_grad_(True), c, False)
