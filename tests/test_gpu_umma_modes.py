"""wgmma convolution: A-staging modes (per-tap / row halo / column halo), stride 2, residual and encoder-head epilogues,
persistent scheduling over many tiles — each against an fp64 torch convolution."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def split(t):
    hi = t.half()
    return hi, (t - hi.float()).half()


@pytest.fixture(scope="module")
def ueng():
    from rnc.engine_umma import UmmaEngine
    return UmmaEngine()


def run_conv(ueng, x, w, b, stride=1, flags=0, epi="none", res=None):
    from rnc import native
    from rnc.engine_umma import SplitBuf, UmmaWeights
    import os
    flags |= int(os.environ.get("RNC_CONV_FLAGS", "0"))
    B, cin, Hin, Win = x.shape
    cout, _, kh, kw = w.shape
    H, W = (Hin + stride - 1) // stride, (Win + stride - 1) // stride
    ld = (cin + 7) // 8 * 8
    buf = SplitBuf(B * Hin * Win, ld, DEV)
    hi, lo = split(x.permute(0, 2, 3, 1).reshape(-1, cin).to(DEV))
    buf.hi[:, :cin], buf.lo[:, :cin] = hi, lo
    wt = UmmaWeights(w.to(DEV), b.to(DEV), [cin])
    out = torch.zeros(B * H * W, wt.coutpad, device=DEV)
    code = {"none": native.EPI_LINEAR, "relu": native.EPI_RELU, "res": native.EPI_RELU_ADD_RELU, "tanh_relu": native.EPI_TANH_RELU}[epi]
    rbuf = None
    if res is not None:
        rbuf = res.permute(0, 2, 3, 1).reshape(-1, cout).contiguous().to(DEV)
    obuf = SplitBuf(B * H * W, wt.coutpad, DEV)
    ueng.uconv(B, H, W, buf.ptrs(), cin, ld, wt, code, out_f32=out.data_ptr(), ldo_f32=wt.coutpad, out_split=obuf.ptrs(),
               ldo_split=wt.coutpad, stride=stride, hin=Hin, win=Win, res=0 if rbuf is None else rbuf.data_ptr(),
               ldres=cout, flags=flags)
    torch.cuda.synchronize()
    o32 = out[:, :cout].view(B, H, W, cout).permute(0, 3, 1, 2).cpu()
    osp = (obuf.hi.float() + obuf.lo.float())[:, :cout].view(B, H, W, cout).permute(0, 3, 1, 2).cpu()
    return o32, osp


def ref_conv(x, w, b, stride=1):
    kh, kw = w.shape[2:]
    return F.conv2d(x.double(), w.double(), b.double(), stride=stride, padding=(kh // 2, kw // 2)).float()


@pytest.mark.parametrize("kh,kw,W,H,cin,cout", [(1, 5, 128, 9, 128, 64), (3, 3, 128, 9, 64, 64), (3, 3, 200, 5, 64, 128),
                                                 (5, 1, 128, 21, 128, 64), (5, 1, 48, 19, 64, 32), (7, 7, 130, 6, 64, 32)])
def test_halo_modes_match_fp64(ueng, kh, kw, W, H, cin, cout):
    """ROWHALO (kw > 1, W > 64) and COLHALO (kw == 1) use row-shifted operand descriptors; they must agree with the
    per-tap mode and with torch."""
    from rnc import native
    g = torch.Generator().manual_seed(kh * 100 + kw * 10 + W)
    x = torch.randn(2, cin, H, W, generator=g)
    w = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    b = torch.randn(cout, generator=g)
    ref = ref_conv(x, w, b)
    halo, _ = run_conv(ueng, x, w, b)
    tap, _ = run_conv(ueng, x, w, b, flags=native.CONV_NO_HALO)
    e_h, e_t = (halo - ref).abs().max().item(), (tap - ref).abs().max().item()
    print(f"{kh}x{kw} W={W}: halo err {e_h:.2e}, per-tap err {e_t:.2e} (scale {ref.abs().max():.2f})")
    assert e_t < 2e-5 * ref.abs().max()
    assert e_h < 2e-5 * ref.abs().max()


@pytest.mark.parametrize("kh,kw,cin,cout,Hin,Win", [(3, 3, 64, 96, 22, 60), (1, 1, 64, 96, 22, 60), (3, 3, 96, 128, 11, 256)])
def test_stride2_matches_fp64(ueng, kh, kw, cin, cout, Hin, Win):
    g = torch.Generator().manual_seed(kh + cin + Win)
    x = torch.randn(2, cin, Hin, Win, generator=g)
    w = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    b = torch.randn(cout, generator=g)
    ref = ref_conv(x, w, b, stride=2)
    out, _ = run_conv(ueng, x, w, b, stride=2)
    assert out.shape == ref.shape
    err = (out - ref).abs().max().item()
    print(f"stride-2 {kh}x{kw} {cin}->{cout}: err {err:.2e}")
    assert err < 2e-5 * ref.abs().max()


def test_residual_and_head_epilogues(ueng):
    g = torch.Generator().manual_seed(77)
    x = torch.randn(2, 64, 12, 140, generator=g)
    w = torch.randn(64, 64, 3, 3, generator=g) / 24.0
    b = torch.randn(64, generator=g)
    res = torch.randn(2, 64, 12, 140, generator=g)
    ref = F.relu(res + F.relu(ref_conv(x, w, b)))
    o32, osp = run_conv(ueng, x, w, b, epi="res", res=res)
    assert (o32 - ref).abs().max() < 2e-5 * ref.abs().max() and (osp - o32).abs().max() < 1e-6 * ref.abs().max() + 1e-7
    # tanh | relu head: first half of the channels tanh (fp32 + split), second half relu (split only)
    c = ref_conv(x, w, b)
    o32, osp = run_conv(ueng, x, w, b, epi="tanh_relu")
    assert (osp[:, :32] - torch.tanh(c[:, :32])).abs().max() < 2e-5
    assert (osp[:, 32:] - F.relu(c[:, 32:])).abs().max() < 2e-5 * c.abs().max()
    assert (o32[:, :32] - torch.tanh(c[:, :32])).abs().max() < 2e-5 and o32[:, 32:].abs().max() == 0


def test_persistent_many_tiles_and_n_tiles(ueng):
    # 3 images x 40 x 256 = 30720 px = 240 tiles > 132 SMs: every CTA loops; Cout 576 = 9 N tiles of 64
    g = torch.Generator().manual_seed(5)
    x = torch.randn(3, 64, 40, 256, generator=g)
    w = torch.randn(576, 64, 1, 1, generator=g) / 8.0
    b = torch.randn(576, generator=g)
    ref = ref_conv(x, w, b)
    out, _ = run_conv(ueng, x, w, b)
    assert (out - ref).abs().max() < 2e-5 * ref.abs().max()
    w3 = torch.randn(64, 64, 3, 3, generator=g) / 24.0
    ref = F.relu(ref_conv(x, w3, b[:64]))
    out, _ = run_conv(ueng, x, w3, b[:64], epi="relu")
    assert (out - ref).abs().max() < 2e-5 * ref.abs().max()
