"""Host-side logic that needs no GPU: state_dict contract, C-ABI surface, weight packing, error behaviour."""
import ctypes
import os
import re

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, build_model, ref_args
from oracle.make_golden import tensor_sha


@pytest.mark.parametrize("name,dataset,key", [("raft_nc_dbl", "sintel", "raft_nc_dbl"),
                                              ("raft_nc_dbl", "kitti", "raft_nc_dbl_kitti"), ("raft", "sintel", "raft")])
def test_state_dict_matches_reference(meta, name, dataset, key):
    """Same seed -> bit-identical parameters, same keys (incl. shared-module aliases and weight_p) as the reference."""
    sd = build_model(name, dataset).state_dict()
    ref = meta[f"state_sha_{key}"]
    assert set(sd) == set(ref)
    assert all(list(v.shape) == meta[f"state_shape_{key}"][k] for k, v in sd.items())
    assert all(tensor_sha(v) == ref[k] for k, v in sd.items())


def test_state_dict_round_trip_with_dataparallel_prefix():
    m = build_model("raft_nc_dbl")
    sd = {"module." + k: v.clone() for k, v in m.state_dict().items()}     # checkpoints carry `module.` (train.py:231)
    m2 = build_model("raft_nc_dbl", seed=1)
    m2.load_state_dict({k[7:]: v for k, v in sd.items()})
    assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), m2.state_dict().values()))
    assert len(m.update_block.mask) == 0 and not any(k.startswith("update_block.mask") for k in m.state_dict())


def test_ctor_writes_args_like_reference():
    a = ref_args()
    a.dropout = 0.5
    build_model("raft")
    import raft
    m = raft.RAFT(a)
    assert (a.corr_levels, a.corr_radius, a.dropout) == (4, 4, 0)          # raft.py:37-42
    assert m.hidden_dim == m.context_dim == 128


def test_small_model_is_rejected_loudly():
    import raft
    a = ref_args()
    a.small = True
    with pytest.raises(NotImplementedError):
        raft.RAFT(a)


def test_cabi_exports_every_declared_symbol():
    from rnc import native
    hdr = open(os.path.join(ROOT, "include", "rnc.h")).read()
    declared = set(re.findall(r"\b(rnc_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"rnc_status", "rnc_epilogue", "rnc_conv_desc"}
    assert declared == set(native.SIGNATURES), declared ^ set(native.SIGNATURES)
    lib = ctypes.CDLL(native.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    L = native.lib()
    assert L.rnc_abi_version() == native.ABI_VERSION
    assert b"sm_90a" in L.rnc_build_info()
    assert L.rnc_status_string(-1) == b"bad shape"
    # pure host helper: pyramid offsets (55x128 -> 27x64 -> 13x32 -> 6x16, floor mode)
    assert L.rnc_pyramid_offset(8, 256, 55, 128, 4) == 8 * 256 * (55 * 128 + 27 * 64 + 13 * 32 + 6 * 16)
    # pure host helper: pixel tiles of a tensor-core layer (sizes the tile-blocked epilogue tensors)
    assert L.rnc_conv_umma_tiles(1, 5, 1, 8, 55, 128, 0) == 8 * 55            # row halo: 128x1 tiles
    assert L.rnc_conv_umma_tiles(5, 1, 1, 8, 55, 128, 0) == 8 * 8 * 7         # column halo: 16x8 tiles
    assert L.rnc_conv_umma_tiles(5, 1, 1, 8, 55, 128, 1) == 8 * 55            # halo sharing off: 128x1 per-tap tiles
    assert L.rnc_conv_umma_tiles(3, 3, 2, 2, 110, 256, 0) == 2 * 110 * 2      # stride 2: per-tap tiles
    assert L.rnc_conv_umma_tiles(3, 3, 1, 1, 16, 32, 0) == 4                  # narrow image: 32x4 tiles
    assert L.rnc_conv_umma_tiles(0, 3, 1, 1, 16, 32, 0) == 0


def test_binding_appends_the_stream_where_the_header_takes_one(monkeypatch):
    """native.rnc appends the current stream to exactly the entry points whose last parameter is the stream, and passes
    every other argument through to the handle native.lib() returns at call time."""
    from rnc import native
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rnc.h")).read(), flags=re.S)
    streamed = {m.group(1) for m in re.finditer(r"\b(rnc_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", hdr)
                if re.search(r"void\s*\*\s*stream\s*$", m.group(2))}
    assert len(streamed) > 40
    got = {}

    class Handle:
        def __getattr__(self, name):
            return lambda *a: got.__setitem__(name, a) or 0

    monkeypatch.setattr(native, "_lib", Handle())
    monkeypatch.setattr(native, "stream", lambda: "stream")
    for name, (_, argtypes) in native.SIGNATURES.items():
        n = len(argtypes) - (name in streamed)
        getattr(native.rnc, name[4:])(*range(n))
        assert got[name] == tuple(range(n)) + (("stream",) if name in streamed else ()), name


def test_binding_raises_naming_the_entry_point(monkeypatch):
    """A failing status raised through native.rnc names the entry point; tensors arrive as their data_ptr(), views with
    their offset, None as NULL."""
    from rnc import native

    class FailingHandle:
        def rnc_status_string(self, status):
            return b"bad shape"

        def rnc_nchw_to_cl(self, *args):
            self.args = args
            return -1

    fake = FailingHandle()
    monkeypatch.setattr(native, "_lib", fake)
    monkeypatch.setattr(native, "stream", lambda: 7)
    x = torch.zeros(4, 8)
    with pytest.raises(ValueError, match="rnc_nchw_to_cl: bad shape"):
        native.rnc.nchw_to_cl(x, 1, 8, 2, 2, x[:, 4:], 8, 0)
    assert fake.args == (x.data_ptr(), 1, 8, 2, 2, x.data_ptr() + 16, 8, 0, 7)
    with pytest.raises(ValueError, match="rnc_nchw_to_cl"):
        native.rnc.nchw_to_cl(None, 1, 8, 2, 2, x, 8, 0)
    assert fake.args[0] is None


def test_conv_desc_layout_matches_header():
    from rnc.native import ConvDesc
    # 4 pointer/int/int groups, then pointers and ints in header order; no implicit reordering
    names = [f[0] for f in ConvDesc._fields_]
    hdr = open(os.path.join(ROOT, "include", "rnc.h")).read()
    body = hdr[hdr.index("typedef struct {"):hdr.index("} rnc_conv_desc;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    order = re.findall(r"\b(in0|c0|ld0|in1|c1|ld1|weight|bias|out|ldo|h|ldh|aux0|ldaux|B|H|W|cout|kh|kw|epilogue)\b", body)
    assert order == names


def test_umma_conv_desc_layout_matches_header():
    """ctypes mirror of rnc_conv_umma_desc: same member names in the same order as include/rnc.h (and the same size as a C
    compiler lays it out: pointers 8-aligned, ints packed)."""
    from rnc.native import UmmaConvDesc
    names = [f[0] for f in UmmaConvDesc._fields_]
    hdr = open(os.path.join(ROOT, "include", "rnc.h")).read()
    end = hdr.index("} rnc_conv_umma_desc;")
    body = hdr[hdr.rindex("typedef struct {", 0, end):end]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    order = []
    for decl in body.split(";"):
        decl = decl.replace("typedef struct {", "").strip()
        if not decl:
            continue
        for part in decl.split(","):
            order.append(re.findall(r"[A-Za-z_][A-Za-z0-9_]*", part)[-1])
    assert order == names
    import ctypes
    expect = 0
    for _, t in UmmaConvDesc._fields_:
        a = ctypes.alignment(t)
        expect = (expect + a - 1) // a * a + ctypes.sizeof(t)
    assert ctypes.sizeof(UmmaConvDesc) == (expect + 7) // 8 * 8


def test_flag_and_epilogue_constants_match_header():
    """rnc.native mirrors the header's enums and flag bits by value (ctypes passes plain ints)."""
    from rnc import native
    hdr = open(os.path.join(ROOT, "include", "rnc.h")).read()
    flags = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+RNC_CONV_([A-Z0-9_]+)\s+(\d+)", hdr)}
    for name in ("NO_HALO", "AUX_BLOCKED", "OUT_BLOCKED", "TF32", "WINDOW"):
        assert getattr(native, "CONV_" + name) == flags[name], name
    epis = {m.group(1): int(m.group(2)) for m in re.finditer(r"RNC_EPI_([A-Z_]+)\s*=\s*(\d+)", hdr)}
    for name in ("LINEAR", "RELU", "SIGMOID", "GRU_ZR", "GRU_Q", "RELU_FLOW", "RELU_ADD_RELU", "TANH_RELU", "FLOW_DELTA"):
        assert getattr(native, "EPI_" + name) == epis[name], name
    assert int(re.search(r"signature change \(now (\d+)\)", hdr).group(1)) == native.ABI_VERSION


def test_cpu_tensors_fail_loudly_no_fallback():
    from rnc.native import RncUnavailable
    m = build_model("raft_nc_dbl")
    im = torch.zeros(1, 3, 128, 256)
    with torch.no_grad(), pytest.raises(RncUnavailable):
        m(im, im, iters=1, test_mode=True)
    from corr import CorrBlock
    with pytest.raises(RncUnavailable):
        CorrBlock(torch.zeros(1, 256, 16, 32), torch.zeros(1, 256, 16, 32))


def test_training_on_cpu_tensors_fails_loudly_too():
    from rnc.native import RncUnavailable
    m = build_model("raft_nc_dbl").train()
    im = torch.zeros(1, 3, 128, 256)
    with pytest.raises(RncUnavailable):                       # the training path has no CPU fallback either
        m(im, im, iters=1)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "raft-ncup_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert "oracle" not in src.replace("# oracle", ""), f


def test_pack_conv_is_an_implicit_gemm_of_the_reference_conv():
    from rnc.engine import pack_conv
    g = torch.Generator().manual_seed(0)
    w = torch.randn(126, 20, 3, 3, generator=g)
    b = torch.randn(126, generator=g)
    x = torch.randn(2, 20, 9, 11, generator=g)
    pw, pb = pack_conv(w, b, cin_pad=20)
    assert pw.shape == (9, 20, 128) and pb.shape == (128,)
    xp = F.pad(x, (1, 1, 1, 1)).permute(0, 2, 3, 1)                      # CL with zero halo
    acc = torch.zeros(2, 9, 11, 128)
    for t in range(9):
        dy, dx = t // 3, t % 3
        acc += xp[:, dy:dy + 9, dx:dx + 11, :] @ pw[t]
    out = (acc + pb)[..., :126].permute(0, 3, 1, 2)
    assert (out - F.conv2d(x, w, b, padding=1)).abs().max() < 1e-4
    assert pw[:, :, 126:].abs().max() == 0 and pb[126:].abs().max() == 0


def test_bn_fold_matches_eval_batchnorm_in_both_formats():
    from rnc.engine import ExactWnet, PackedUpsampler
    from rnc.engine_umma import UmmaWnet
    m = build_model("raft_nc_dbl")
    wn = m.upsampler.weights_est_net
    g = torch.Generator().manual_seed(0)
    for blk in wn.conv:                                                   # make the running stats non-trivial
        blk[1].running_mean.copy_(torch.randn(blk[1].num_features, generator=g) * 0.1)
        blk[1].running_var.copy_(torch.rand(blk[1].num_features, generator=g) + 0.5)
    pu = PackedUpsampler(m.upsampler, ExactWnet)
    g0 = pu.wnet.layers[0].wt
    x = torch.randn(1, 130, 6, 7, generator=g)
    ref = wn.conv[0](x)
    w = g0[0][:, :130, :64].reshape(3, 3, 130, 64).permute(3, 2, 0, 1)
    out = F.relu(F.conv2d(x, w, g0[1][:64], padding=1))
    assert (out - ref).abs().max() < 1e-4
    assert g0[0].shape[1] == 132 and len(pu.nconv_host) == 224
    # the tensor-core pack of the same layer: fp16 hi/lo planes [CoutPad][9 taps * 3 blocks * 64], value (hi + lo) * unscale
    u0 = PackedUpsampler(m.upsampler, UmmaWnet).wnet.layers[0].wt
    w = ((u0.w_hi.float() + u0.w_lo.float()) * u0.unscale).view(u0.coutpad, 9, 192)[:64, :, :130]
    out = F.relu(F.conv2d(x, w.reshape(64, 3, 3, 130).permute(0, 3, 1, 2), u0.bias[:64], padding=1))
    assert (out - ref).abs().max() < 1e-4


def test_input_padder_matches_reference(meta):
    from utils.utils import InputPadder
    assert InputPadder((1, 3, 436, 1024), "sintel")._pad == meta["sintel_pad"]
    assert InputPadder((1, 3, 375, 1242), "kitti")._pad == meta["kitti_pad"]
    x = torch.randn(1, 3, 436, 1024)
    p = InputPadder(x.shape)
    (y,) = p.pad(x)
    assert y.shape[-2:] == (440, 1024) and torch.equal(p.unpad(y), x)
