"""GPU parity of the wgmma (tensor-core) convolution path against fp32 references: the fp16 hi/lo split must stay
fp32-faithful (north star: 1e-3 EPE after 32 recurrent iterations; plain TF32/bf16 operands fail it, SURVEY.md App. D)."""
import pytest
import torch
import torch.nn.functional as F

from conftest import build_model, frames
from oracle import raft_oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def epe(a, b):
    return (a - b).pow(2).sum(1).sqrt().mean().item()


def split(t):
    hi = t.half()
    return hi, (t - hi.float()).half()


@pytest.fixture(scope="module")
def ueng():
    from rnc.engine_umma import UmmaEngine
    return UmmaEngine()


def test_split_roundtrip_is_near_exact():
    from rnc import native
    import ctypes as C
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(1000, 36, generator=g) * torch.logspace(-4, 3, 36)).to(DEV)
    hi = torch.zeros(1000, 40, dtype=torch.float16, device=DEV)
    lo = torch.zeros_like(hi)
    L = native.lib()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    native.check(L.rnc_f32_to_split(C.c_void_p(x.data_ptr()), 36, 36, 1000, C.c_void_p(hi.data_ptr()), C.c_void_p(lo.data_ptr()), 40, 2, s))
    rec = hi[:, 2:38].float() + lo[:, 2:38].float()
    err = (rec - x).abs()
    assert (err <= x.abs() * 2.0 ** -21 + 6e-8).all()                   # 22 significant bits, absolute floor = half subnormal
    assert hi[:, :2].abs().max() == 0 and hi[:, 38:].abs().max() == 0


@pytest.mark.parametrize("cin,cout,kh,kw,act,W", [
    (324, 256, 1, 1, "relu", 21), (256, 192, 3, 3, "relu", 21), (128, 64, 3, 3, "relu", 32), (384, 256, 1, 5, "sigmoid", 21),
    (384, 128, 5, 1, "none", 64), (132, 64, 3, 3, "relu", 21), (64, 32, 3, 3, "relu", 128), (256, 576, 1, 1, "none", 21)])
def test_umma_conv_matches_fp32(ueng, cin, cout, kh, kw, act, W):
    from rnc import native
    from rnc.engine_umma import SplitBuf, UmmaWeights
    g = torch.Generator().manual_seed(cin + cout + W)
    B, H = 2, 13
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    b = torch.randn(cout, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=(kh // 2, kw // 2)).float()
    ref = {"relu": F.relu, "sigmoid": torch.sigmoid, "none": lambda t: t}[act](ref)
    ld = (cin + 7) // 8 * 8
    buf = SplitBuf(B * H * W, ld, DEV)
    x_cl = x.permute(0, 2, 3, 1).reshape(-1, cin).to(DEV)
    hi, lo = split(x_cl)
    buf.hi[:, :cin], buf.lo[:, :cin] = hi, lo
    wt = UmmaWeights(w.to(DEV), b.to(DEV), [cin])
    out = torch.zeros(B * H * W, wt.coutpad, device=DEV)
    epi = {"relu": native.EPI_RELU, "sigmoid": native.EPI_SIGMOID, "none": native.EPI_LINEAR}[act]
    ueng.uconv(B, H, W, buf.ptrs(), cin, ld, wt, epi, out_f32=out.data_ptr(), ldo_f32=wt.coutpad)
    torch.cuda.synchronize()
    got = out[:, :cout].view(B, H, W, cout).permute(0, 3, 1, 2).cpu()
    err = (got - ref).abs().max().item()
    scale = max(1.0, ref.abs().max().item())
    print(f"umma conv {cin}->{cout} {kh}x{kw}: max err {err:.2e} (scale {scale:.2f})")
    assert err < 2e-5 * scale                                             # fp32-class accuracy (TF32 would be ~1e-3)
    # split output of the same conv reproduces the fp32 output
    obuf = SplitBuf(B * H * W, wt.coutpad, DEV)
    ueng.uconv(B, H, W, buf.ptrs(), cin, ld, wt, epi, out_split=obuf.ptrs(), ldo_split=wt.coutpad)
    rec = (obuf.hi.float() + obuf.lo.float())[:, :cout]
    assert (rec - out[:, :cout]).abs().max().item() < 1e-6 * scale + 1e-7


@pytest.mark.parametrize("cout,W", [(64, 150), (96, 40), (128, 21)])
def test_umma_conv_fused_instance_norm_statistics(ueng, cout, W):
    """rnc_conv_umma_desc.stats + rnc_instnorm_finalize == InstanceNorm2d statistics of the layer's output
    (extractor.py:128-129): ragged tiles, several images per CTA, accumulate-and-rezero protocol."""
    import ctypes as C
    from rnc import native
    from rnc.engine_umma import SplitBuf, UmmaWeights
    g = torch.Generator().manual_seed(cout + W)
    B, H, cin = 3, 11, 64
    x = torch.randn(B, cin, H, W, generator=g) + 0.5
    w = torch.randn(cout, cin, 3, 3, generator=g) / 24.0
    b = torch.randn(cout, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    buf = SplitBuf(B * H * W, cin, DEV)
    buf.hi[:], buf.lo[:] = split(x.permute(0, 2, 3, 1).reshape(-1, cin).to(DEV))
    wt = UmmaWeights(w.to(DEV), b.to(DEV), [cin])
    out = torch.zeros(B * H * W, wt.coutpad, device=DEV)
    stats = torch.zeros(B * cout * 2, dtype=torch.float64, device=DEV)
    mr = torch.zeros(B * cout * 2, device=DEV)
    for _ in range(2):                                     # second round checks that finalize left the sums zeroed
        ueng.uconv(B, H, W, buf.ptrs(), cin, cin, wt, native.EPI_LINEAR, out_f32=out.data_ptr(), ldo_f32=wt.coutpad,
                   stats=stats.data_ptr())
        native.check(ueng.L.rnc_instnorm_finalize(C.c_void_p(stats.data_ptr()), B, H * W, cout, 1e-5, C.c_void_p(mr.data_ptr()),
                                                  C.c_void_p(torch.cuda.current_stream().cuda_stream)), "finalize")
        torch.cuda.synchronize()
        assert stats.abs().max().item() == 0.0
        got = mr.view(B, cout, 2).cpu()
        mean = ref.mean(dim=(2, 3))
        rstd = 1.0 / torch.sqrt(ref.var(dim=(2, 3), unbiased=False) + 1e-5)
        assert (got[..., 0] - mean.float()).abs().max() < 2e-5 * max(1.0, mean.abs().max().item())
        assert ((got[..., 1] - rstd.float()) / rstd.float()).abs().max() < 5e-5


def test_flow_head_conv2_as_taps_plus_gather(ueng):
    """FlowHead.conv2 (update.py:10,14) = 1x1 tensor-core layer over the 9 taps + rnc_flow_tap_gather_fwd, with
    `coords1 += delta_flow` (raft_nc_dbl.py:157); borders exercise the zero padding."""
    import ctypes as C
    from rnc import native
    from rnc.engine_umma import SplitBuf, UmmaWeights
    g = torch.Generator().manual_seed(11)
    B, H, W, cin = 2, 9, 37, 256
    x = torch.relu(torch.randn(B, cin, H, W, generator=g))
    w = torch.randn(2, cin, 3, 3, generator=g) / 48.0
    b = torch.randn(2, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1).float()
    buf = SplitBuf(B * H * W, cin, DEV)
    buf.hi[:], buf.lo[:] = split(x.permute(0, 2, 3, 1).reshape(-1, cin).to(DEV))
    wt = UmmaWeights(w.permute(2, 3, 0, 1).reshape(18, cin, 1, 1).to(DEV), None, [cin])
    taps = torch.zeros(B * H * W, 32, device=DEV)
    ueng.uconv(B, H, W, buf.ptrs(), cin, cin, wt, native.EPI_LINEAR, out_f32=taps.data_ptr(), ldo_f32=32)
    coords = torch.randn(B, 2, H, W, generator=g).to(DEV)
    c0 = coords.clone()
    delta = torch.zeros(B, 2, H, W, device=DEV)
    vp = C.c_void_p
    bd = b.to(DEV)
    native.check(ueng.L.rnc_flow_tap_gather_fwd(vp(taps.data_ptr()), 32, vp(bd.data_ptr()), B, H, W, vp(delta.data_ptr()),
                                                vp(coords.data_ptr()), vp(torch.cuda.current_stream().cuda_stream)), "gather")
    torch.cuda.synchronize()
    assert (delta.cpu() - ref).abs().max() < 2e-5 * max(1.0, ref.abs().max().item())
    assert (coords - (c0 + delta)).abs().max().item() < 1e-6
    assert ueng.L.rnc_flow_tap_gather_fwd(vp(taps.data_ptr()), 16, vp(0), B, H, W, None, vp(coords.data_ptr()), None) != 0


@pytest.mark.parametrize("cin,cout,kh,kw,B,H,W", [(128, 256, 3, 3, 3, 9, 128), (384, 128, 5, 1, 1, 17, 40), (64, 64, 3, 3, 2, 13, 150)])
def test_umma_pair_and_single_cta_forms_agree(ueng, cin, cout, kh, kw, B, H, W):
    """The CTA-pair (cta_group::2) form and the single-CTA form (flag RNC_CONV_NO_PAIR = 8) compute the same products in the
    same order per accumulator: bit-identical outputs, including odd tile counts (ghost tile in the last pair) and the
    hoisted-addend epilogue input."""
    from rnc import native
    from rnc.engine_umma import SplitBuf, UmmaWeights
    g = torch.Generator().manual_seed(cin + cout + W)
    x = torch.randn(B * H * W, cin, generator=g).to(DEV)
    buf = SplitBuf(B * H * W, cin, DEV)
    buf.hi[:], buf.lo[:] = split(x)
    wt = UmmaWeights((torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5).to(DEV), torch.randn(cout, generator=g).to(DEV), [cin])
    add = torch.randn(B * H * W, wt.coutpad, generator=g).to(DEV)
    outs = []
    for flags in (0, 8):
        out = torch.zeros(B * H * W, wt.coutpad, device=DEV)
        ueng.uconv(B, H, W, buf.ptrs(), cin, cin, wt, native.EPI_RELU, out_f32=out.data_ptr(), ldo_f32=wt.coutpad,
                   add=add.data_ptr(), ldadd=wt.coutpad, flags=flags)
        torch.cuda.synchronize()
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    # the addend really is added before the activation
    out0 = torch.zeros_like(outs[0])
    ueng.uconv(B, H, W, buf.ptrs(), cin, cin, wt, native.EPI_LINEAR, out_f32=out0.data_ptr(), ldo_f32=wt.coutpad)
    assert (torch.relu(out0 + add)[:, :cout] - outs[0][:, :cout]).abs().max().item() < 1e-5


def test_umma_two_segment_input(ueng):
    # q-gate convolution: input = cat(r*h [128], x [256]) read from two buffers (update.py:49)
    from rnc import native
    from rnc.engine_umma import SplitBuf, UmmaWeights
    g = torch.Generator().manual_seed(3)
    B, H, W = 1, 16, 32
    a, x = torch.randn(B, 128, H, W, generator=g), torch.randn(B, 256, H, W, generator=g)
    w = torch.randn(128, 384, 1, 5, generator=g) / 44.0
    b = torch.randn(128, generator=g)
    ref = F.conv2d(torch.cat([a, x], 1).double(), w.double(), b.double(), padding=(0, 2)).float()
    sa, sx = SplitBuf(B * H * W, 128, DEV), SplitBuf(B * H * W, 384, DEV)
    sa.hi[:], sa.lo[:] = split(a.permute(0, 2, 3, 1).reshape(-1, 128).to(DEV))
    hx, lx = split(x.permute(0, 2, 3, 1).reshape(-1, 256).to(DEV))
    sx.hi[:, 128:], sx.lo[:, 128:] = hx, lx
    wt = UmmaWeights(w.to(DEV), b.to(DEV), [128, 256])
    out = torch.zeros(B * H * W, 128, device=DEV)
    ueng.uconv(B, H, W, sa.ptrs(), 128, 128, wt, native.EPI_LINEAR, in1=sx.ptrs(128), c1=256, ld1=384, out_f32=out.data_ptr(), ldo_f32=128)
    got = out.view(B, H, W, 128).permute(0, 3, 1, 2).cpu()
    assert (got - ref).abs().max() < 2e-5 * ref.abs().max()


@pytest.mark.parametrize("it", [0, 3])
def test_update_block_teacher_forced_umma(gold, it, monkeypatch):
    monkeypatch.setenv("RNC_CONV", "umma")
    m = build_model("raft_nc_dbl").to(DEV)
    flow = gold[f"coords_it{it}"] - orc.coords_grid(1, 16, 32)
    with torch.no_grad():
        net, mask, delta = m.update_block(gold[f"net_in_it{it}"].to(DEV), gold["inp"].to(DEV), gold[f"corr_it{it}"].to(DEV), flow.to(DEV))
    e_net = (net.cpu() - gold[f"net_out_it{it}"]).abs().max().item()
    e_del = (delta.cpu() - gold[f"delta_it{it}"]).abs().max().item()
    print(f"umma update block it{it}: net err {e_net:.2e}, delta err {e_del:.2e}")
    assert e_net < 5e-5 and e_del < 5e-5                                  # same bar as the exact-fp32 path


@pytest.mark.parametrize("mode", ["umma", "ffma"])
@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_end_to_end_cfg1_both_engines(gold, name, mode, monkeypatch):
    monkeypatch.setenv("RNC_CONV", mode)
    m = build_model(name).to(DEV)
    assert m.engine().mode == mode
    im1, im2 = frames(1, 128, 256)
    with torch.no_grad():
        lo, up = m(im1.to(DEV), im2.to(DEV), iters=4, test_mode=True)
    e = epe(up.cpu(), gold[f"{name}_flow_up"])
    print(f"{name}/{mode}: EPE vs reference golden {e:.3e}")
    assert e < 1e-3 and epe(lo.cpu(), gold[f"{name}_flow_low"]) < 1e-4


@pytest.mark.parametrize("mode", ["umma", "ffma"])
def test_sintel_shape_32_iters_both_engines(mode, monkeypatch):
    """1024x436 (pad 440), 32 iterations, B=1 vs the CPU oracle for each convolution engine; the two engines must also
    agree with each other far below the 1e-3 budget."""
    from utils.utils import InputPadder
    monkeypatch.setenv("RNC_CONV", mode)
    m = build_model("raft_nc_dbl").to(DEV)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    im1, im2 = frames(1, 436, 1024)
    p1, p2 = InputPadder(im1.shape, "sintel").pad(im1, im2)
    with torch.no_grad():
        lo, up = m(p1.to(DEV), p2.to(DEV), iters=32, test_mode=True)
    olo, oup, _ = orc.raft_forward(sd, p1, p2, iters=32, model="raft_nc_dbl", upsample_every_iter=False)
    e = epe(up.cpu(), oup)
    print(f"{mode}: EPE flow_up vs oracle {e:.3e} (|flow_up| {oup.abs().mean():.2f})")
    assert e < 1e-3


def test_kitti_shape_24_iters_warm_start():
    """KITTI frames (375x1242 -> 376x1248 with the 'kitti' padder, evaluate.py:125; 47x156 at 1/8: ragged in both tile
    directions), 24 iterations as evaluate.py:117 runs them, with a non-zero flow_init, vs the CPU oracle."""
    from utils.utils import InputPadder
    m = build_model("raft_nc_dbl").to(DEV)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    im1, im2 = frames(1, 375, 1242)
    padder = InputPadder(im1.shape, "kitti")
    p1, p2 = padder.pad(im1, im2)
    assert p1.shape[-2:] == (376, 1248)
    g = torch.Generator().manual_seed(5)
    init = torch.randn(1, 2, 47, 156, generator=g) * 1.5
    with torch.no_grad():
        lo, up = m(p1.to(DEV), p2.to(DEV), iters=24, flow_init=init.to(DEV), test_mode=True)
    olo, oup, _ = orc.raft_forward(sd, p1, p2, iters=24, model="raft_nc_dbl", flow_init=init, upsample_every_iter=False)
    e = epe(up.cpu(), oup)
    print(f"kitti shape: EPE flow_up vs oracle {e:.3e} (|flow_up| {oup.abs().mean():.2f})")
    assert e < 1e-3 and epe(lo.cpu(), olo) < 2e-4
    assert padder.unpad(up).shape[-2:] == (375, 1242)


# ----------------------------------------------------------------------------- tensor-core correlation lookup


def resident_lookup(f1, f2, coords, lookup_mode):
    """Run the engine's per-iteration lookup into the resident split planes; returns ([B,324,H,W] fp32, flags)."""
    from rnc.engine_umma import CORR_LD, UmmaEngine
    eng = UmmaEngine()
    eng.lookup_mode = lookup_mode
    B, D, H, W = f1.shape
    ws = eng.workspace(DEV, B, H, W, False, False)
    eng.fmap_prepare(ws, f1.to(DEV).contiguous(), f2.to(DEV).contiguous(), 4)
    ws.coords1.copy_(coords.to(DEV))
    ws.corr.hi.fill_(7.0)
    ws.corr.lo.fill_(0.0)
    eng.lookup_resident(ws)
    torch.cuda.synchronize()
    out = (ws.corr.hi.float() + ws.corr.lo.float()).view(-1, 4, 88)        # padded per-level layout: 81 taps + 7 zero pads
    assert (out[:, :, 81:] == 0).all() and (ws.corr.lo.view(-1, 4, 88)[:, :, 81:] == 0).all()
    assert (out[:, :, :81] != 7.0).all()                                    # every tap of every pixel was written
    flags = ws.lookup_flags.cpu() if lookup_mode == "umma" else None
    return eng.corr_nchw(ws).cpu(), flags                                   # resident channel order -> reference order


def fp16_tol(f1, f2):
    # |err| of a 256-term dot product of fp16-rounded operands / 16: ~ sqrt(256) * |f1||f2| * 2^-11 * sqrt(2) / 16
    return 6.0 * (256 ** 0.5) * f1.abs().max().item() * f2.abs().max().item() * 2.0 ** -11 / 16 / 4


@pytest.mark.parametrize("it", [0, 3])
def test_umma_lookup_matches_reference_golden(gold, it):
    out, flags = resident_lookup(gold["fmap1"], gold["fmap2"], gold[f"coords_it{it}"], "umma")
    ref = gold[f"corr_it{it}"]
    err = (out - ref).abs()
    print(f"umma lookup it{it}: max err {err.max():.2e} mean {err.mean():.2e} (|ref| max {ref.abs().max():.1f}), fallback tiles {int(flags.sum())}")
    assert flags.sum() == 0
    assert err.max() < fp16_tol(gold["fmap1"], gold["fmap2"]) and err.mean() < 1e-3
    exact, _ = resident_lookup(gold["fmap1"], gold["fmap2"], gold[f"coords_it{it}"], "ffma")
    assert (exact - ref).abs().max() < 1e-4


def test_umma_lookup_full_size_borders_and_fallback():
    g = torch.Generator().manual_seed(33)
    B, H, W = 2, 55, 128
    f1 = torch.randn(B, 256, H, W, generator=g) * 1.5
    f2 = torch.randn(B, 256, H, W, generator=g) * 1.5
    # smooth flow (coherent tiles) pushed across the image borders + one incoherent region -> fallback tiles
    yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    flow = torch.stack([6 * torch.sin(yy / 9) + 0.03 * xx - 3.3, 5 * torch.cos(xx / 17) - 0.05 * yy + 2.7], 0)[None].repeat(B, 1, 1, 1)
    flow[1, :, 20:30, 40:70] += torch.randn(2, 10, 30, generator=g) * 12
    flow[0, :, 0, 0] = torch.tensor([1e9, -1e9])
    co = orc.coords_grid(B, H, W) + flow
    out, flags = resident_lookup(f1, f2, co, "umma")
    exact, _ = resident_lookup(f1, f2, co, "ffma")
    nf = int(flags.sum())
    err = (out - exact).abs()
    print(f"umma lookup 55x128: max err {err.max():.2e} mean {err.mean():.2e}, fallback tiles {nf}/{flags.numel()}")
    assert 0 < nf < flags.numel() // 2
    assert err.max() < fp16_tol(f1, f2) and err.mean() < 1e-3
    # spot check the exact path itself against the oracle on one image
    ref = orc.corr_lookup_direct(f1[:1], f2[:1], co[:1].clamp(-1e6, 1e6))
    assert (exact[:1] - ref).abs().max() < 2e-4


def test_umma_lookup_odd_size(gold):
    out, flags = resident_lookup(gold["odd_f1"], gold["odd_f2"], gold["odd_coords"], "umma")
    err = (out - gold["odd_corr"]).abs()
    print(f"umma lookup 17x21 randn*6: max err {err.max():.2e}, fallback tiles {int(flags.sum())}/{flags.numel()}")
    assert err.max() < fp16_tol(gold["odd_f1"], gold["odd_f2"])
