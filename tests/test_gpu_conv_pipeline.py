"""The tensor-core convolution's warp-specialised pipeline: the epilogue warpgroup works on tile i while the MMA warpgroups
run the K loop of tile i + 1, and one wgmma batch stays in flight across ring stages.  These tests use grids with more
work items than SMs, so every CTA runs several tiles and the accumulator hand-off is exercised in steady state."""
import pytest
import torch

from test_conv_error_model import check_model, conv_split_ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def split(t):
    hi = t.half()
    return hi, (t - hi.float()).half()


@pytest.fixture(scope="module")
def ueng():
    from rnc.engine_umma import UmmaEngine
    return UmmaEngine()


def _layer(cin, cout, kh, kw, B, H, W, seed):
    from rnc.engine_umma import SplitBuf, UmmaWeights
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    b = torch.randn(cout, generator=g)
    buf = SplitBuf(B * H * W, cin, DEV)
    buf.hi[:], buf.lo[:] = split(x.permute(0, 2, 3, 1).reshape(-1, cin).to(DEV))
    wt = UmmaWeights(w.to(DEV), b.to(DEV), [cin])
    return buf, wt, conv_split_ref(x.to(DEV), wt, weight=w)      # the error model of tests/test_conv_error_model.py


# (cin, cout, kh, kw): row-halo 3x3 and 1x5, column-halo 5x1, per-tap 1x1; 32- / 64- / 128-column tiles
SHAPES = [(128, 128, 3, 3), (256, 128, 1, 5), (256, 64, 5, 1), (96, 32, 1, 1), (128, 256, 1, 1)]


@pytest.mark.parametrize("cin,cout,kh,kw", SHAPES)
def test_many_tiles_per_cta_match_fp64(ueng, cin, cout, kh, kw):
    """6 x 30 x 128 outputs: 180 pixel tiles (x column tiles) on 132 SMs, fp32-faithful against an fp64 convolution."""
    from rnc import native
    B, H, W = 6, 30, 128
    buf, wt, ref = _layer(cin, cout, kh, kw, B, H, W, cin + cout + kh)
    out = torch.zeros(B * H * W, wt.coutpad, device=DEV)
    ueng.uconv(B, H, W, buf.ptrs(), cin, cin, wt, native.EPI_RELU, out_f32=out.data_ptr(), ldo_f32=wt.coutpad)
    torch.cuda.synchronize()
    got = out[:, :cout].view(B, H, W, cout).permute(0, 3, 1, 2)
    for against in ("split", "exact"):
        check_model(f"{cin}->{cout} {kh}x{kw} relu", got, ref, against, act=torch.relu)


@pytest.mark.parametrize("cin,cout,kh,kw", SHAPES)
def test_repeated_calls_are_bit_identical(ueng, cin, cout, kh, kw):
    """The hand-off between the MMA and epilogue warpgroups must not make the result depend on timing."""
    from rnc import native
    from rnc.engine_umma import SplitBuf
    B, H, W = 6, 30, 128
    buf, wt, _ = _layer(cin, cout, kh, kw, B, H, W, 7 * cin + cout)
    outs = []
    for _ in range(2):
        o = SplitBuf(B * H * W, wt.coutpad, DEV)
        ueng.uconv(B, H, W, buf.ptrs(), cin, cin, wt, native.EPI_RELU, out_split=o.ptrs(), ldo_split=wt.coutpad)
        torch.cuda.synchronize()
        outs.append(o)
    assert torch.equal(outs[0].hi, outs[1].hi) and torch.equal(outs[0].lo, outs[1].lo)


def test_fused_stats_over_many_tiles(ueng):
    """LINEAR + fused InstanceNorm sums (the epilogue warpgroup's per-lane fp64 accumulators, flushed when the image or
    column tile changes) over several tiles per CTA and per image."""
    from rnc import native
    B, H, W, cin, cout = 5, 24, 160, 64, 96
    buf, wt, ref = _layer(cin, cout, 3, 3, B, H, W, 11)
    out = torch.zeros(B * H * W, wt.coutpad, device=DEV)
    stats = torch.zeros(B, cout, 2, dtype=torch.float64, device=DEV)
    ueng.uconv(B, H, W, buf.ptrs(), cin, cin, wt, native.EPI_LINEAR, out_f32=out.data_ptr(), ldo_f32=wt.coutpad,
               stats=stats.data_ptr())
    torch.cuda.synchronize()
    got = out[:, :cout].view(B, H * W, cout).double()
    for against in ("split", "exact"):
        check_model("fused stats 64->96 3x3", got.permute(0, 2, 1).reshape(B, cout, H, W), ref, against)
    s1, s2 = got.sum(1), (got * got).sum(1)
    assert torch.allclose(stats[..., 0], s1, rtol=1e-6, atol=1e-6 * H * W)
    assert torch.allclose(stats[..., 1], s2, rtol=1e-6, atol=1e-6 * H * W)
