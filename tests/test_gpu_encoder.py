"""Encoders (core/extractor.py) on the tensor-core path: stem kernel, instance norm, and the full fnet/cnet against the
reference's own outputs (tests/golden: fmap1, fmap2, net0, inp of BASELINE configs[0])."""
import pytest
import torch
import torch.nn.functional as F

from conftest import build_model, frames

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("Hin,Win,relu", [(128, 256, 0), (46, 70, 1), (33, 41, 0)])
def test_stem_conv_matches_torch(Hin, Win, relu):
    from rnc import native
    g = torch.Generator().manual_seed(Hin)
    img = torch.rand(2, 3, Hin, Win, generator=g) * 255
    w = torch.randn(64, 3, 7, 7, generator=g) / 12
    b = torch.randn(64, generator=g)
    ref = F.conv2d(2 * (img / 255.0) - 1.0, w, b, stride=2, padding=3)
    if relu:
        ref = F.relu(ref)
    Ho, Wo = ref.shape[-2:]
    out = torch.zeros(2 * Ho * Wo, 64, device=DEV)
    hi = torch.zeros(2 * Ho * Wo, 64, dtype=torch.float16, device=DEV)
    lo = torch.zeros_like(hi)
    wp = w.permute(1, 2, 3, 0).reshape(147, 64).contiguous().to(DEV)
    imgd, bd = img.to(DEV), b.to(DEV)
    native.rnc.stem_conv7x7s2_fwd(imgd, wp, bd, 2, Hin, Win, relu, out, hi, lo)
    got = out.view(2, Ho, Wo, 64).permute(0, 3, 1, 2).cpu()
    assert (got - ref).abs().max() < 2e-5
    assert ((hi.float() + lo.float()) - out).abs().max() < 1e-6


@pytest.mark.parametrize("Hin,Win,inst", [(128, 256, True), (46, 70, False), (33, 41, True), (440, 1024, False)])
def test_window_stem_matches_torch(Hin, Win, inst):
    """The product's stem: image repacked as a zero-padded pixel plane, convolved on the tensor cores through the sliding-window
    tensor map (rnc_conv_umma_desc.win_pitch), with the InstanceNorm sums fused (fnet) or ReLU + split output (cnet), against
    F.conv2d in fp64 (extractor.py:135,171; raft_nc_dbl.py:118-119).  Odd sizes exercise the right / bottom borders."""
    from rnc import native
    from rnc.encoder_umma import EncoderBuffers, EncoderRunner, PackedEncoder
    from rnc.engine import engine_for
    from rnc.modules import BasicEncoder
    torch.manual_seed(Hin + Win)
    N = 2
    enc = BasicEncoder(output_dim=256, norm_fn="instance" if inst else "batch", dropout=0.0).eval()
    with torch.no_grad():
        enc.conv1.weight.mul_(3.0)
        enc.conv1.bias.uniform_(-1, 1)
        if not inst:
            enc.norm1.running_mean.uniform_(-0.2, 0.2)
            enc.norm1.running_var.uniform_(0.5, 2.0)
            enc.norm1.weight.uniform_(0.5, 1.5)
            enc.norm1.bias.uniform_(-0.3, 0.3)
    img = torch.rand(N, 3, Hin, Win) * 255
    with torch.no_grad():
        x = (2 * (img.double() / 255.0) - 1.0)
        y = F.conv2d(x, enc.conv1.weight.double(), enc.conv1.bias.double(), stride=2, padding=3)
        ref = y if inst else F.relu(F.batch_norm(y, enc.norm1.running_mean.double(), enc.norm1.running_var.double(),
                                                 enc.norm1.weight.double(), enc.norm1.bias.double(), False, 0.0, enc.norm1.eps))
    Ho, Wo = ref.shape[-2:]
    eng = engine_for(torch.device(DEV))
    enc = enc.to(DEV)
    pk = PackedEncoder(enc)
    bufs = EncoderBuffers(DEV, N, Hin, Win)
    E = native
    imgd = img.to(DEV)
    native.rnc.stem_window_prep(imgd, N, Hin, Win, bufs.pitch, bufs.img_hi, bufs.img_lo)
    plane = (bufs.img_hi.float() + bufs.img_lo.float())[:N * Hin * bufs.pitch].view(N, Hin, bufs.pitch, 4).cpu()
    want = torch.zeros(N, Hin, bufs.pitch, 4, dtype=torch.float64)
    want[:, :, 3:3 + Win, :3] = x.permute(0, 2, 3, 1)
    assert (plane.double() - want).abs().max() < 1e-6                  # split halves reproduce the normalised image, zero border
    win = dict(stride=2, hin=Hin, win=Wo, win_pitch=4 * bufs.pitch, flags=E.CONV_WINDOW)
    ptrs = (bufs.img_hi.data_ptr(), bufs.img_lo.data_ptr())
    out = torch.zeros(N * Ho * Wo, 64, device=DEV)
    if inst:
        eng.uconv(N, Ho, Wo, ptrs, 64, 8, pk.stem, E.EPI_LINEAR, out_f32=out.data_ptr(), ldo_f32=64, stats=bufs.stats.data_ptr(), **win)
        sums = bufs.stats[:N * 64 * 2].view(N, 64, 2).cpu()
        assert torch.allclose(sums[..., 0], ref.sum((2, 3)), rtol=1e-5, atol=1e-2)
        assert torch.allclose(sums[..., 1], (ref * ref).sum((2, 3)), rtol=1e-5, atol=1e-2)
    else:
        sp_hi = torch.zeros(N * Ho * Wo, 64, dtype=torch.float16, device=DEV)
        sp_lo = torch.zeros_like(sp_hi)
        eng.uconv(N, Ho, Wo, ptrs, 64, 8, pk.stem, E.EPI_RELU, out_f32=out.data_ptr(), ldo_f32=64,
                  out_split=(sp_hi.data_ptr(), sp_lo.data_ptr()), ldo_split=64, **win)
        assert ((sp_hi.float() + sp_lo.float()) - out).abs().max() < 1e-5
    got = out.view(N, Ho, Wo, 64).permute(0, 3, 1, 2).cpu().double()
    assert (got - ref).abs().max() < 3e-5 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("Cc,mode", [(64, 1), (96, 0), (128, 2)])
def test_instance_norm_matches_torch(Cc, mode):
    from rnc import native
    g = torch.Generator().manual_seed(Cc)
    N, Pn = 3, 1000
    x = torch.randn(N, Pn, Cc, generator=g) * 3 + 1.5
    res = torch.randn(N, Pn, Cc, generator=g)
    ref = F.instance_norm(x.permute(0, 2, 1).reshape(N, Cc, Pn, 1)).reshape(N, Cc, Pn).permute(0, 2, 1)
    if mode >= 1:
        ref = F.relu(ref)
    if mode == 2:
        ref = F.relu(res + ref)
    xd, rd = x.to(DEV).contiguous(), res.to(DEV).contiguous()
    stats = torch.empty(N * Cc * 2, dtype=torch.float64, device=DEV)
    mr = torch.empty(N * Cc * 2, device=DEV)
    out = torch.zeros(N, Pn, Cc, device=DEV)
    hi = torch.zeros(N, Pn, Cc, dtype=torch.float16, device=DEV)
    lo = torch.zeros_like(hi)
    native.rnc.instnorm_stats(xd, N, Pn, Cc, 1e-5, stats, mr)
    native.rnc.instnorm_apply(xd, mr, rd, N, Pn, Cc, mode, out, hi, lo)
    assert (out.cpu() - ref).abs().max() < 2e-5
    assert ((hi.float() + lo.float()) - out).abs().max() < 1e-6


def test_encoders_match_reference_golden(gold, monkeypatch):
    """fnet (instance norm) and cnet (batch norm) at 128x256: outputs land in the resident buffers; compare with the
    reference's fmap1 / fmap2 / tanh(net) / relu(inp)."""
    monkeypatch.setenv("RNC_CONV", "umma")
    m = build_model("raft_nc_dbl").to(DEV)
    eng = m.engine()
    im1, im2 = frames(1, 128, 256)
    ws = eng.workspace(DEV, 1, 16, 32, False, True)
    eng.encoder().run(m, ws, im1.to(DEV), im2.to(DEV))
    torch.cuda.synchronize()
    f1 = ws.f1_cl.view(1, 16, 32, 256).permute(0, 3, 1, 2).cpu()
    f2 = ws.f2_pyr[: 16 * 32 * 256].view(1, 16, 32, 256).permute(0, 3, 1, 2).cpu()
    net = ws.h.view(1, 16, 32, 128).permute(0, 3, 1, 2).cpu()
    hx = (ws.hx.hi.float() + ws.hx.lo.float()).view(1, 16, 32, 384).permute(0, 3, 1, 2).cpu()
    e = [(f1 - gold["fmap1"]).abs().max().item(), (f2 - gold["fmap2"]).abs().max().item(),
         (net - gold["net0"]).abs().max().item(), (hx[:, 128:256] - gold["inp"]).abs().max().item()]
    print(f"encoder errs: fmap1 {e[0]:.2e} fmap2 {e[1]:.2e} net {e[2]:.2e} inp {e[3]:.2e} (|fmap| max {gold['fmap1'].abs().max():.1f})")
    assert max(e[:2]) < 2e-5 * gold["fmap1"].abs().max() and e[2] < 1e-4 and e[3] < 2e-5 * max(1.0, gold["inp"].abs().max().item())
    assert (hx[:, :128] - net).abs().max() < 1e-6
