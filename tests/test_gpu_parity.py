"""GPU parity: every kernel is called through the C ABI (librnc.so) and compared with the CPU oracle and with the golden
fixtures generated from the unmodified reference.  Floating point -> tolerances are stated per test; the end-to-end
bar is the north star's 1e-3 EPE."""
import pytest
import torch
import torch.nn.functional as F

from conftest import build_model, frames
from oracle import raft_oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def epe(a, b):
    return (a - b).pow(2).sum(1).sqrt().mean().item()


@pytest.fixture(scope="module")
def eng():
    from rnc.engine import Engine
    return Engine()


# ----------------------------------------------------------------------------- K2: correlation lookup


def gpu_lookup(f1, f2, coords, layout=0):
    from corr import CorrBlock
    cb = CorrBlock(f1.to(DEV), f2.to(DEV), num_levels=4, radius=4)
    if layout == 0:
        return cb(coords.to(DEV)).cpu()
    ws = cb.ws
    out = torch.full((ws.B * ws.H8 * ws.W8, 328), 7.0, device=DEV)
    cb.engine.lookup(ws, coords.to(DEV).contiguous(), out, 1, 328)
    assert (out[:, 324:] == 7.0).all()                                   # padding channels untouched
    return out[:, :324].view(ws.B, ws.H8, ws.W8, 324).permute(0, 3, 1, 2).cpu()


@pytest.mark.parametrize("it", [0, 3])
def test_lookup_matches_reference_golden(gold, it):
    out = gpu_lookup(gold["fmap1"], gold["fmap2"], gold[f"coords_it{it}"])
    assert out.shape == (1, 324, 16, 32) and out.dtype == torch.float32 and out.is_contiguous()
    assert (out - gold[f"corr_it{it}"]).abs().max() < 1e-4               # reference CorrBlock.__call__ output
    out_cl = gpu_lookup(gold["fmap1"], gold["fmap2"], gold[f"coords_it{it}"], layout=1)
    assert torch.equal(out, out_cl)


def test_lookup_odd_sizes_and_large_motion(gold):
    # 17x21: pooling drops odd rows/cols; randn*6 coords push many windows across the border (zero padding)
    out = gpu_lookup(gold["odd_f1"], gold["odd_f2"], gold["odd_coords"])
    assert (out - gold["odd_corr"]).abs().max() < 1e-4


def test_lookup_incoherent_tile_fallback_and_wild_coords():
    g = torch.Generator().manual_seed(21)
    f1 = torch.randn(2, 256, 40, 72, generator=g) * 1.5
    f2 = torch.randn(2, 256, 40, 72, generator=g) * 1.5
    co = orc.coords_grid(2, 40, 72) + torch.randn(2, 2, 40, 72, generator=g) * 25     # box > 1024 positions -> global path
    co[0, :, 0, 0] = torch.tensor([1e9, -1e9])                            # far outside: all-zero window
    co[1, :, 5, 5] = torch.tensor([-3.5, 41.25])                          # partially outside
    ref = orc.corr_lookup_direct(f1, f2, co.clamp(-1e6, 1e6))
    out = gpu_lookup(f1, f2, co)
    assert (out - ref).abs().max() < 2e-4
    assert out[0, :, 0, 0].abs().max() == 0


def test_lookup_is_linear_in_fmap1_at_full_size():
    # BASELINE cfg 2 shape (55x128, B=2 to keep it quick): size-independent property instead of an oracle run
    g = torch.Generator().manual_seed(5)
    f1a, f1b = torch.randn(2, 256, 55, 128, generator=g), torch.randn(2, 256, 55, 128, generator=g)
    f2 = torch.randn(2, 256, 55, 128, generator=g) * 1.5
    co = orc.coords_grid(2, 55, 128) + torch.randn(2, 2, 55, 128, generator=g) * 4
    oa, ob, oab = gpu_lookup(f1a, f2, co), gpu_lookup(f1b, f2, co), gpu_lookup(2 * f1a - 3 * f1b, f2, co)
    assert (oab - (2 * oa - 3 * ob)).abs().max() < 2e-3
    # integer shift of the centre moves the 9x9 window by one tap: out(c + (1,0))[i] == out(c)[i+1]
    o1 = gpu_lookup(f1a, f2, co + torch.tensor([1.0, 0.0]).view(1, 2, 1, 1)).view(2, 4, 9, 9, 55, 128)
    o0 = oa.view(2, 4, 9, 9, 55, 128)
    assert (o1[:, 0, :-1] - o0[:, 0, 1:]).abs().max() < 1e-4             # level 0 only: deeper levels see a half-pixel shift
    # spot-check 64 random pixels against the oracle restatement
    ref = orc.corr_lookup_direct(f1a[:1, :, :, :], f2[:1], co[:1])
    assert (oa[:1] - ref).abs().max() < 2e-4


# ----------------------------------------------------------------------------- K3: convolutions / update block


@pytest.mark.parametrize("cin,cout,kh,kw,act", [(324, 256, 1, 1, "relu"), (256, 192, 3, 3, "relu"), (128, 64, 3, 3, "relu"),
                                                (384, 256, 1, 5, "sigmoid"), (384, 128, 5, 1, "none"), (132, 64, 3, 3, "relu"),
                                                (64, 32, 3, 3, "relu"), (256, 576, 1, 1, "none")])
def test_generic_conv_matches_torch(eng, cin, cout, kh, kw, act):
    from rnc import native
    from rnc.engine import pack_conv
    g = torch.Generator().manual_seed(cin + cout)
    B, H, W = 2, 13, 21                                                   # M = 546: exercises the M tail
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    b = torch.randn(cout, generator=g)
    ref = F.conv2d(x, w, b, padding=(kh // 2, kw // 2))
    ref = {"relu": F.relu, "sigmoid": torch.sigmoid, "none": lambda t: t}[act](ref)
    x_cl = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    pk = pack_conv(w.to(DEV), b.to(DEV))
    out = torch.zeros(B * H * W, cout, device=DEV)
    epi = {"relu": native.EPI_RELU, "sigmoid": native.EPI_SIGMOID, "none": native.EPI_LINEAR}[act]
    eng.conv(B, H, W, x_cl.data_ptr(), cin, cin, pk, cout, kh, kw, epi, out.data_ptr(), cout)
    got = out.view(B, H, W, cout).permute(0, 3, 1, 2).cpu()
    assert (got - ref).abs().max() < 2e-5 * max(1.0, ref.abs().max().item())


def test_conv_rejects_bad_arguments(eng):
    from rnc.engine import pack_conv
    pk = pack_conv(torch.zeros(64, 6, 3, 3, device=DEV), torch.zeros(64, device=DEV))
    x = torch.zeros(10, 6, device=DEV)
    with pytest.raises(ValueError):
        eng.conv(1, 2, 5, x.data_ptr(), 6, 6, pk, 64, 3, 3, 1, x.data_ptr(), 64)          # Cin % 4 != 0
    with pytest.raises(ValueError):
        eng.conv(1, 2, 5, x.data_ptr(), 8, 8, pk, 64, 2, 3, 1, x.data_ptr(), 64)          # even kernel


@pytest.mark.parametrize("it", [0, 3])
def test_update_block_teacher_forced(gold, it):
    m = build_model("raft_nc_dbl").to(DEV)
    flow = gold[f"coords_it{it}"] - orc.coords_grid(1, 16, 32)
    with torch.no_grad():
        net, mask, delta = m.update_block(gold[f"net_in_it{it}"].to(DEV), gold["inp"].to(DEV), gold[f"corr_it{it}"].to(DEV), flow.to(DEV))
    assert (net.cpu() - gold[f"net_out_it{it}"]).abs().max() < 5e-5       # reference update_block output
    assert (delta.cpu() - gold[f"delta_it{it}"]).abs().max() < 5e-5
    assert torch.equal(m.update_block.net, net)                           # guidance tap (update.py:135)


def test_update_block_with_mask_head(gold, sd_raft):
    m = build_model("raft").to(DEV)
    flow = gold["coords_it3"] - orc.coords_grid(1, 16, 32)
    net_in, inp, corr = gold["net_in_it3"], gold["inp"], gold["corr_it3"]
    rnet, rmask, rdelta = orc.update_block(sd_raft, net_in, inp, corr, flow, with_mask=True)
    with torch.no_grad():
        net, mask, delta = m.update_block(net_in.to(DEV), inp.to(DEV), corr.to(DEV), flow.to(DEV))
    assert (net.cpu() - rnet).abs().max() < 5e-5 and (delta.cpu() - rdelta).abs().max() < 5e-5
    assert mask.shape == (1, 576, 16, 32) and (mask.cpu() - rmask).abs().max() < 5e-5


# ----------------------------------------------------------------------------- K4 / K5: upsamplers


@pytest.mark.parametrize("it", [0, 3])
def test_ncup_teacher_forced(gold, it):
    m = build_model("raft_nc_dbl").to(DEV)
    with torch.no_grad():
        out = m.upsample_flow(gold[f"ncup_in_flow_it{it}"].to(DEV), gold[f"net_out_it{it}"].to(DEV))
    ref = gold[f"ncup_out_it{it}"]                                        # reference RAFT.upsample_flow output
    assert out.shape == ref.shape
    assert (out.cpu() - ref).abs().max() < 5e-5 * max(1.0, ref.abs().max().item())


def test_ncup_fwd_non_multiple_of_tile(sd_ncup):
    # 4*h = 88, 4*w = 104: tiles overhang; random confidences incl. exact zeros exercise the 1e-20 epsilon
    from rnc import native
    from rnc.engine import Engine
    m = build_model("raft_nc_dbl").to(DEV)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, 2, 22, 26, generator=g) * 3
    c = torch.rand(2, 2, 22, 26, generator=g)
    c[c < 0.15] = 0.0
    xh, ch = orc.zero_stuff(x), orc.zero_stuff(c)
    ref, _ = orc.nconv_unet_live(sd_ncup, xh.view(4, 1, 88, 104), ch.view(4, 1, 88, 104))
    eng = m.upsampler.engine()
    pu = eng.packed_upsampler(m.upsampler)
    out = torch.empty(2, 2, 88, 104, device=DEV)
    xd, cd = x.to(DEV), c.to(DEV)
    native.rnc.ncup_fwd(xd, cd, pu.nconv_host, 2, 22, 26, 8.0, out, None)
    assert (out.cpu() - 8 * ref.view(2, 2, 88, 104)).abs().max() < 1e-4


def test_convex_upsampler_matches_reference_golden(gold):
    m = build_model("raft").to(DEV)
    out = m.upsample_flow(gold["convex_flow"].to(DEV), gold["convex_mask"].to(DEV))
    ref = gold["convex_out"]
    assert (out.cpu() - ref).abs().max() < 2e-6 * ref.abs().max()         # values reach ~40 px: 2e-6 relative


# ----------------------------------------------------------------------------- end to end


@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_end_to_end_cfg1_matches_reference_golden(gold, name):
    """BASELINE configs[0]: 256x128 pair, 4 iterations, against the reference's own outputs."""
    m = build_model(name).to(DEV)
    im1, im2 = frames(1, 128, 256)
    with torch.no_grad():
        lo, up = m(im1.to(DEV), im2.to(DEV), iters=4, test_mode=True)
        preds = m(im1.to(DEV), im2.to(DEV), iters=4, test_mode=False)
    assert len(preds) == 4 and preds[0].shape == (1, 2, 128, 256)
    assert epe(lo.cpu(), gold[f"{name}_flow_low"]) < 1e-4
    assert epe(up.cpu(), gold[f"{name}_flow_up"]) < 1e-3                  # north-star tolerance
    assert epe(preds[0].cpu(), gold[f"{name}_pred0"]) < 1e-3
    assert torch.equal(preds[-1], up)


def test_end_to_end_kitti_config_and_warm_start(gold):
    m = build_model("raft_nc_dbl", "kitti").to(DEV)
    im1, im2 = frames(1, 128, 256)
    with torch.no_grad():
        _, up = m(im1.to(DEV), im2.to(DEV), iters=4, test_mode=True)
    assert epe(up.cpu(), gold["raft_nc_dbl_kitti_flow_up"]) < 1e-3
    m = build_model("raft_nc_dbl").to(DEV)
    with torch.no_grad():
        lo, up = m(im1.to(DEV), im2.to(DEV), iters=2, flow_init=gold["warm_flow_init"].to(DEV), test_mode=True)
    assert epe(lo.cpu(), gold["warm_flow_low"]) < 1e-4 and epe(up.cpu(), gold["warm_flow_up"]) < 1e-3


def test_training_mode_builds_an_autograd_graph():
    """train mode + grad enabled -> the training path (rnc/train.py): a list of `iters` predictions that back-propagate."""
    m = build_model("raft_nc_dbl").to(DEV).train()
    m.freeze_bn()
    im1, im2 = frames(1, 128, 160)
    preds = m(im1.to(DEV), im2.to(DEV), iters=2)
    assert len(preds) == 2 and preds[-1].requires_grad and preds[-1].shape == (1, 2, 128, 160)
    preds[-1].abs().mean().backward()
    assert m.update_block.flow_head.conv2.weight.grad is not None and torch.isfinite(m.fnet.conv1.weight.grad).all()


def test_batch_items_are_independent():
    """Inference shards by batch with no exchange (SURVEY.md §8e): a pair's flow does not depend on its batch mates."""
    m = build_model("raft_nc_dbl").to(DEV)
    im1, im2 = frames(3, 128, 256, seed=3)
    with torch.no_grad():
        _, up3 = m(im1.to(DEV), im2.to(DEV), iters=3, test_mode=True)
        _, up1 = m(im1[1:2].to(DEV), im2[1:2].to(DEV), iters=3, test_mode=True)
    assert epe(up3[1:2].cpu(), up1.cpu()) < 1e-4


@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_end_to_end_sintel_shape_32_iters(name):
    """BASELINE configs[2] shape (1024x436 padded to 440, 32 iterations), one pair, vs the CPU oracle: EPE <= 1e-3."""
    from utils.utils import InputPadder
    m = build_model(name).to(DEV)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    im1, im2 = frames(1, 436, 1024)
    pad = InputPadder(im1.shape, "sintel")
    p1, p2 = pad.pad(im1, im2)
    with torch.no_grad():
        lo, up = m(p1.to(DEV), p2.to(DEV), iters=32, test_mode=True)
    olo, oup, _ = orc.raft_forward(sd, p1, p2, iters=32, model=name, upsample_every_iter=False)
    e_lo, e_up = epe(lo.cpu(), olo), epe(up.cpu(), oup)
    print(f"{name}: EPE flow_low {e_lo:.3e}  flow_up {e_up:.3e}  |flow_up| {oup.abs().mean():.2f}")
    assert pad.unpad(up).shape[-2:] == (436, 1024)
    assert e_up < 1e-3 and e_lo < 1e-3 / 8 * 2
