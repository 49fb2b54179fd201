"""Weights-net (Simple) configurations, host side: module structure, state_dict and RNG draws against the reference's, the
options that stay unsupported, argument checks of the dilated entry points, the header mirror, the shipped pack, and (compiled
for sm_90a, no GPU needed) the absence of floating-point atomics from the dilated weight gradient."""
import ctypes
import json
import os
import re
import subprocess

import pytest
import torch

from conftest import ROOT, ref_args

P = 4096                                                  # any non-null, 16-byte aligned address: nothing is dereferenced

with open(os.path.join(ROOT, "tests", "golden", "wnet_cfg_meta.json")) as _f:
    META = json.load(_f)
CONFIGS = META["configs"]


def variant_model(name):
    import raft_nc_dbl
    num_ch, filter_sz, dilation, dataset = CONFIGS[name]
    a = ref_args(dataset)
    a.weights_est_net_num_ch, a.weights_est_net_filter_sz, a.weights_est_net_dilation = num_ch, filter_sz, dilation
    torch.manual_seed(1234)
    return raft_nc_dbl.RAFT(a)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_state_dict_matches_reference(name):
    from oracle.make_golden import tensor_sha
    sd = variant_model(name).state_dict()
    assert {k: list(v.shape) for k, v in sd.items()} == META[f"{name}_state_shape"]
    assert {k: tensor_sha(v) for k, v in sd.items()} == META[f"{name}_state_sha"]


def test_even_filter_sizes_stay_out_of_scope():
    """The reference's padding k // 2 grows an even layer's output by a pixel, and its model fails (golden script)."""
    assert META["even_filter_runs"] is False
    from interp_weights_est import Simple
    with pytest.raises(NotImplementedError, match="filter_sz"):
        Simple([130, 64, 32], 2, [4, 3, 1])


@pytest.mark.parametrize("kwargs,option", [
    (dict(num_ch=[130, 64, 32, 32, 32, 32, 32, 32], filter_sz=[3] * 8), "num_ch"),     # 7 hidden layers
    (dict(num_ch=[130, 257], filter_sz=[3, 1]), "num_ch"),
    (dict(num_ch=[130, 0], filter_sz=[3, 1]), "num_ch"),
    (dict(num_ch=[130, 64], filter_sz=[9, 1]), "filter_sz"),
    (dict(num_ch=[130, 64], filter_sz=[3, 2]), "filter_sz"),
    (dict(num_ch=[130, 64], filter_sz=[3, 1], dilation=[5, 1]), "dilation"),
    (dict(num_ch=[130, 64], filter_sz=[3, 1], dilation=[1, 0]), "dilation"),
])
def test_unsupported_options_raise_and_name_themselves(kwargs, option):
    from interp_weights_est import Simple
    with pytest.raises(NotImplementedError, match=option):
        Simple(out_ch=2, **kwargs)


def test_accepted_bounds_build():
    from interp_weights_est import Simple
    net = Simple([130, 1, 256, 8, 8, 8, 5], 2, [1, 7, 5, 3, 7, 1, 7], dilation=[4, 1, 2, 3, 4, 1, 4], use_bn=True)
    assert net.num_layers == 6 and net.out.dilation == (4, 4) and net.out.padding == (12, 12)
    assert net.conv[1][0].padding == (3, 3) and net.conv[0][0].padding == (0, 0)
    x = torch.randn(1, 130, 9, 11)
    assert Simple([130], 2, [5], dilation=[2]).out.padding == (4, 4)
    with torch.no_grad():
        assert net.eval().out(torch.zeros(1, 5, 9, 11)).shape == (1, 2, 9, 11) and x.shape[-2:] == (9, 11)


def test_umma_desc_mirrors_dil():
    from rnc.native import UmmaConvDesc
    assert UmmaConvDesc._fields_[-1] == ("dil", ctypes.c_int)
    hdr = open(os.path.join(ROOT, "include", "rnc.h")).read()
    body = hdr[hdr.index("const void* in0_hi;"):hdr.index("} rnc_conv_umma_desc;")]
    assert re.findall(r"\bint dil;", body) and body.rstrip().split("\n")[-1].strip().endswith("*/")


def test_dilated_entry_points_reject_bad_arguments():
    from rnc import native
    L = native.lib()
    ws = L.rnc_conv2d_cl_wgrad_dil_workspace_bytes
    assert ws(64, 32, 2, 8, 8, 3, 3, 2) == L.rnc_conv2d_cl_wgrad_workspace_bytes(64, 32, 2, 8, 8, 3, 3, 1) > 0
    assert ws(64, 32, 2, 8, 8, 3, 3, 0) == 0 and ws(64, 32, 2, 8, 8, 3, 3, 9) == 0 and ws(64, 32, 2, 8, 8, 2, 3, 2) == 0
    nb = ws(64, 32, 2, 8, 8, 3, 3, 2)
    f = L.rnc_conv2d_cl_wgrad_dil_det

    def call(dil=2, cin=64, ldx=64, x=P, wsb=nb):
        return f(x, ldx, cin, P, 32, 32, 2, 8, 8, 3, 3, dil, P, 32, P, P, wsb, None)

    assert call(dil=0) == -1 and call(dil=9) == -1 and call(cin=6, ldx=8) == -1 and call(x=None) == -2 and call(wsb=nb - 4) == -5
    d = native.ConvDesc()
    d.in0, d.c0, d.ld0, d.weight, d.bias, d.out, d.ldo = P, 64, 64, P, P, P, 64
    d.B, d.H, d.W, d.cout, d.kh, d.kw, d.epilogue = 1, 8, 8, 64, 3, 3, native.EPI_RELU
    assert L.rnc_conv2d_cl_dil_fwd(ctypes.byref(d), 0, None) == -1 and L.rnc_conv2d_cl_dil_fwd(ctypes.byref(d), 9, None) == -1
    d.epilogue = native.EPI_GRU_Q
    assert L.rnc_conv2d_cl_dil_fwd(ctypes.byref(d), 2, None) == -3
    u = native.UmmaConvDesc()
    u.in0_hi = u.in0_lo = u.w_hi = u.w_lo = u.bias = u.out_f32 = P
    u.c0, u.ld0, u.ktot, u.coutpad, u.ldo_f32 = 64, 64, 9 * 64, 64, 64
    u.B, u.H, u.W, u.cout, u.kh, u.kw, u.epilogue = 1, 8, 8, 64, 3, 3, native.EPI_RELU
    for bad, status in (({"dil": -1}, -1), ({"dil": 9}, -1), ({"dil": 2, "stride": 2}, -3), ({"dil": 2, "add": P, "ldadd": 64}, -3),
                        ({"dil": 2, "epilogue": native.EPI_GRU_Q}, -3), ({"dil": 2, "flags": native.CONV_OUT_BLOCKED}, -3)):
        v = native.UmmaConvDesc.from_buffer_copy(u)
        for k, val in bad.items():
            setattr(v, k, val)
        assert L.rnc_conv2d_umma_fwd(ctypes.byref(v), None) == status, bad


def packs(up):
    """The weights-net packs of upsampler `up` in the exact and the tensor-core format."""
    from rnc.engine import ExactWnet, PackedSimple
    from rnc.engine_umma import UmmaWnet
    return PackedSimple(up.weights_est_net, ExactWnet), PackedSimple(up.weights_est_net, UmmaWnet)


def shapes(layers):
    return [(l.cout, l.k, l.dil) for l in layers]


def test_shipped_layer_list_is_unchanged():
    """The shipped network packs as before: two exact 3x3 layers, the fused 1x1 head (conf_head) and the tensor-core layers
    with segments [132] and [64]."""
    from rnc.synth import build_model
    m = build_model("raft_nc_dbl")
    pk, pkm = packs(m.upsampler)
    assert (pk.cin, shapes(pk.layers)) == (132, [(64, 3, 1), (32, 3, 1)])
    assert pk.layers[0].wt[0].shape == (9, 132, 64) and pk.layers[1].wt[0].shape == (9, 64, 64) and pk.conv_head is None
    assert pk.conf_head[0].shape == (1, 32, 2)
    assert torch.equal(pk.conf_head[0][0], m.upsampler.weights_est_net.out.weight[:, :, 0, 0].t())
    assert [(l.wt.ktot, l.wt.coutpad) for l in pkm.layers] == [(9 * 192, 64), (9 * 64, 32)] and pkm.conv_head is None
    assert pkm.conf_head[0].shape == (1, 32, 2)
    bufs = pkm.buffers(10, "cpu")
    assert [b.ld for b in bufs[:1]] == [64] and bufs[1].shape == (10, 32) and len(bufs) == 2
    assert [b.shape for b in pk.buffers(10, "cpu")] == [(10, 64), (10, 32)]


def test_variant_layer_lists():
    m = variant_model("wide_k").eval()
    pk, pkm = packs(m.upsampler)
    assert shapes(pk.layers) == [(96, 5, 2), (48, 7, 1)] and (pk.conv_head.k, pk.conv_head.dil) == (3, 3)
    assert pk.conf_head is None and pk.conv_head.wt[0].shape == (9, 48, 64)
    assert pkm.layers[1].wt.ktot == 49 * 2 * 64 and pkm.conv_head.wt.ktot == 9 * 64 and len(pkm.buffers(4, "cpu")) == 3
    m = variant_model("head_only").eval()
    pk, pkm = packs(m.upsampler)
    assert pk.layers == [] and (pk.conv_head.k, pk.conv_head.dil) == (5, 2) and pk.conv_head.wt[0].shape == (25, 132, 64)
    assert pkm.conv_head.wt.ktot == 25 * 192 and [b.shape for b in pkm.buffers(4, "cpu")] == [(4, 32)]
    _, narrow = packs(variant_model("narrow").eval().upsampler)      # 1x1 head on the 16-wide layer's 32 columns
    assert narrow.conf_head[0].shape == (1, 32, 2) and narrow.conf_head[0][0, 16:].abs().max() == 0


def test_dilated_wgrad_has_no_float_atomics(tmp_path):
    try:
        from rnc.build import ARCH, nvcc_path
        nvcc = nvcc_path()
    except RuntimeError:
        pytest.skip("nvcc not available")
    csrc = os.path.join(ROOT, "raft-ncup_b200", "csrc")
    obj = tmp_path / "t.o"
    subprocess.run([nvcc, *ARCH, "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-I", os.path.join(ROOT, "include"), "-I", csrc,
                    "-c", os.path.join(csrc, "train_ops.cu"), "-o", str(obj)], check=True, capture_output=True)
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    fn, seen = None, set()
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            continue
        if fn and ("conv_wgrad_kernel" in fn or "wgrad_reduce_kernel" in fn):
            seen.add("reduce" if "reduce" in fn else "wgrad")
            assert not re.search(r"\b(RED|ATOM|ATOMG)\.[A-Z.]*(F32|F64|FADD|ADD\.F)", line), (fn, line)
    assert seen == {"wgrad", "reduce"}
