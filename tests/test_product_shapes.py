"""Pointwise comparison helpers for the product-shape kernel tests (tests/test_gpu_product_shapes.py), and their CPU checks.

The GPU tests compare every hot-path kernel with an fp64 reference of the same operation at the shapes the benchmark and the
training runs use.  This file holds what they share and what can be checked without a GPU:
  - compare(): one pointwise comparator with the per-kind tolerances of the existing suite; a failure names the worst image,
    pixel and 128-pixel tile;
  - the tile geometry of the tensor-core convolution (tile_shape / unblock), mirroring csrc/conv_umma.cu, so that the
    tile-blocked z gate and hoisted GRU addends can be read back channel-last;
  - the list of distinct ConvCL signatures of one training step at config 5, derived here from the oracle's graph.
"""
import math

import pytest
import torch
import torch.nn.functional as F

# ----------------------------------------------------------------------------------------------------------- shapes
# id -> (B, H8, W8): the 1/8-resolution grids the kernels run at
SHAPES = {
    "S1": (8, 55, 128),    # Sintel bench, 440x1024: 440 pixel tiles per layer, row halo for 1x5, ragged 16x8 column halo
    "S2": (2, 47, 156),    # KITTI 376x1248: ragged in x (128 + 28) and in y
    "S3": (2, 48, 64),     # training config 5 (384x512): W8 = 64 puts the 1x5 layers on per-tap tiles
    "S4": (3, 8, 12),      # sub-tile images: W8 < 16 (no column halo), each image one partial tile
}

# ----------------------------------------------------------------------------------------------------------- tolerances
# The bound of every comparison is tol * max(1, max|ref|); the tolerances are those the existing kernel tests use.
TOL = {
    "conv": 2e-5,          # one convolution layer, tensor-core (fp16 hi/lo split) or exact fp32 engine (test_gpu_umma.py)
    "lookup_exact": 1e-4,  # exact fp32 / split lookups (test_gpu_umma.py::test_umma_lookup_matches_reference_golden)
    "ncup": 5e-5,          # rnc_ncup_fwd (test_gpu_ncup_variants.py)
    "convex": 2e-6,        # rnc_convex_upsample_fwd
    "move": 2.0 ** -21,    # data movement and hi/lo splits: exact up to the 22-bit split
}


class Mismatch(AssertionError):
    pass


def compare(what, got, ref, tol, floor=0.0, log=print):
    """Pointwise check of a kernel output against its fp64 reference.

    got, ref: [B, C, H, W] tensors (any device / dtype).  Passes when |got - ref| <= tol * max(1, max|ref|) + floor everywhere
    (floor: an absolute allowance for an operand that is itself rounded to fp32, stated by the caller).  Prints, and on failure
    raises with, the worst image, pixel (y, x), channel and 128-pixel tile (pixel index y * W + x in the image, // 128).
    Returns the worst error."""
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} != reference {tuple(ref.shape)}"
    assert got.dim() == 4, f"{what}: expected [B, C, H, W]"
    ref = ref.double()
    err = (got.double().to(ref.device) - ref).abs()
    if not torch.isfinite(got).all():
        err = torch.where(torch.isfinite(got.to(ref.device)), err, torch.full_like(err, math.inf))
    scale = max(1.0, float(ref.abs().max())) if ref.numel() else 1.0
    bound = tol * scale + floor
    B, C, H, W = err.shape
    flat = int(err.reshape(-1).argmax()) if err.numel() else 0
    b, rem = divmod(flat, C * H * W)
    c, rem = divmod(rem, H * W)
    y, x = divmod(rem, W)
    worst = float(err.reshape(-1)[flat]) if err.numel() else 0.0
    nbad = int((err > bound).sum())
    where = f"image {b}, pixel (y={y}, x={x}), channel {c}, tile {(y * W + x) // 128}"
    log(f"  {what:<34s} {B}x{C}x{H}x{W}: max err {worst:.2e} (bound {bound:.2e}) at {where}")
    if nbad:
        tiles = sorted({(int(bb), int(yy * W + xx) // 128) for bb, yy, xx in
                        (err > bound).amax(1).nonzero().tolist()[:4096]})
        raise Mismatch(f"{what}: {nbad} elements exceed {bound:.3e}; worst {worst:.3e} at {where}; "
                       f"bad (image, tile): {tiles[:16]}{' ...' if len(tiles) > 16 else ''}")
    return worst


def cl(t, B, H, W):
    """[B*H*W, C] channel-last -> [B, C, H, W]."""
    return t.reshape(B, H, W, -1).permute(0, 3, 1, 2)


# ----------------------------------------------------------------------------------------------------------- tile geometry
KBM = 128                  # output pixels per tile (csrc/conv_umma.cu, umma::kBM)
NO_HALO = 1                # RNC_CONV_NO_HALO


def tile_shape(kh, kw, H, W, flags=0, stride=1):
    """(TW, TH) of a tensor-core layer's pixel tiles, as tile_shape() in csrc/conv_umma.cu: row halo 128x1 for kw > 1 when
    W > 64, column halo 16x8 for kw == 1 < kh when W >= 16 and H >= 8, otherwise per-tap TW x 128/TW tiles."""
    if stride == 1 and not flags & NO_HALO and kw > 1 and W > 64:
        return 128, 1
    if stride == 1 and not flags & NO_HALO and kw == 1 and kh > 1 and W >= 16 and H >= 8:
        return 16, 8
    tw = 8
    while tw < W and tw < KBM:
        tw <<= 1
    return tw, KBM // tw


def tiles(kh, kw, B, H, W, flags=0):
    tw, th = tile_shape(kh, kw, H, W, flags)
    return B * -(-W // tw) * -(-H // th)


def blocked_index(kh, kw, B, H, W, flags=0):
    """For every pixel p = (b*H + y)*W + x: (tile, row) of its element in the tile-blocked layout (include/rnc.h,
    RNC_CONV_AUX_BLOCKED): element (tile, channel c, row r) at ((tile * ld + c) * 128 + r)."""
    tw, th = tile_shape(kh, kw, H, W, flags)
    tx = -(-W // tw)
    ty = -(-H // th)
    b = torch.arange(B).view(B, 1, 1)
    y = torch.arange(H).view(1, H, 1)
    x = torch.arange(W).view(1, 1, W)
    tile = (b * ty + y // th) * tx + x // tw
    row = (y % th) * tw + x % tw
    return tile.expand(B, H, W).reshape(-1), row.expand(B, H, W).reshape(-1)


def unblock(buf, ld, C, kh, kw, B, H, W, flags=0):
    """Tile-blocked fp32 tensor of a (kh, kw) layer (ld channels per tile) -> channel-last [B*H*W, C]."""
    tile, row = blocked_index(kh, kw, B, H, W, flags)
    tile, row = tile.to(buf.device), row.to(buf.device)
    c = torch.arange(C, device=buf.device)
    idx = (tile[:, None] * ld + c[None, :]) * KBM + row[:, None]
    return buf.reshape(-1)[idx]


# ----------------------------------------------------------------------------------------------------------- ConvCL list
# Distinct ConvCL signatures (cin, cout, kh, kw, stride, dil, B, Hin, Win) of one raft_nc_dbl training step at config 5
# (B = 2, 384x512): fnet on both frames (B = 4) and cnet (B = 2) at 384x512 -> 192x256 -> 96x128 -> 48x64, the update
# block at 48x64 and the weights net Simple at 96x128.
CFG5_CONV_SIGNATURES = sorted(set(
    [(3, 64, 7, 7, 2, 1, n, 384, 512) for n in (4, 2)]
    + [(64, 64, 3, 3, 1, 1, n, 192, 256) for n in (4, 2)]
    + [(64, 96, 3, 3, 2, 1, n, 192, 256) for n in (4, 2)]
    + [(64, 96, 1, 1, 2, 1, n, 192, 256) for n in (4, 2)]
    + [(96, 96, 3, 3, 1, 1, n, 96, 128) for n in (4, 2)]
    + [(96, 128, 3, 3, 2, 1, n, 96, 128) for n in (4, 2)]
    + [(96, 128, 1, 1, 2, 1, n, 96, 128) for n in (4, 2)]
    + [(128, 128, 3, 3, 1, 1, n, 48, 64) for n in (4, 2)]
    + [(128, 256, 1, 1, 1, 1, n, 48, 64) for n in (4, 2)]
    + [(324, 256, 1, 1, 1, 1, 2, 48, 64), (256, 192, 3, 3, 1, 1, 2, 48, 64), (2, 128, 7, 7, 1, 1, 2, 48, 64),
       (128, 64, 3, 3, 1, 1, 2, 48, 64), (256, 126, 3, 3, 1, 1, 2, 48, 64),
       (384, 128, 1, 5, 1, 1, 2, 48, 64), (384, 128, 5, 1, 1, 1, 2, 48, 64),
       (128, 256, 3, 3, 1, 1, 2, 48, 64), (256, 2, 3, 3, 1, 1, 2, 48, 64)]
    + [(130, 64, 3, 3, 1, 1, 2, 96, 128), (64, 32, 3, 3, 1, 1, 2, 96, 128), (32, 2, 1, 1, 1, 1, 2, 96, 128)]))


def _pair(v):
    return v[0] if isinstance(v, (tuple, list)) else int(v)


def conv2d_signature(x, weight, stride=1, dilation=1):
    cout, cin, kh, kw = weight.shape
    return (cin, cout, kh, kw, _pair(stride), _pair(dilation) if max(kh, kw) > 1 else 1, x.shape[0], x.shape[2], x.shape[3])


# ======================================================================================================== CPU tests


def test_compare_rejects_one_wrong_tile_and_names_it():
    """A single 128-pixel tile of one image off by 1e-4 relative fails the comparator, which names that image and tile; the
    untouched tensor passes."""
    B, C, H, W = SHAPES["S1"][0], 8, 55, 128
    g = torch.Generator().manual_seed(0)
    ref = torch.randn(B, C, H, W, generator=g, dtype=torch.float64) * 3
    got = ref.float()
    assert compare("exact", got, ref, TOL["conv"]) < 1e-6
    bad_img, bad_tile = 5, 37                  # tile 37 = pixels 4736..4863 of the image = row 37 (W = 128)
    scale = float(ref.abs().max())
    flat = got[bad_img].reshape(C, H * W)
    flat[:, bad_tile * 128:(bad_tile + 1) * 128] += 1e-4 * scale
    with pytest.raises(Mismatch) as e:
        compare("one corrupt tile", got, ref, TOL["conv"])
    msg = str(e.value)
    assert f"image {bad_img}," in msg and f"tile {bad_tile}" in msg and f"({bad_img}, {bad_tile})" in msg
    # and a ragged KITTI-width image: the last, partial tile of the last row
    B, H, W = SHAPES["S2"]
    ref = torch.randn(B, 2, H, W, generator=g, dtype=torch.float64)
    got = ref.float().clone()
    got[1, 0, H - 1, W - 1] += 1e-4 * max(1.0, float(ref.abs().max()))
    with pytest.raises(Mismatch, match=rf"image 1, pixel \(y={H - 1}, x={W - 1}\), channel 0, tile {(H * W - 1) // 128}"):
        compare("last pixel", got, ref, TOL["conv"])


def test_compare_rejects_nan_and_shape_mismatch():
    ref = torch.zeros(1, 1, 4, 4, dtype=torch.float64)
    got = ref.float().clone()
    got[0, 0, 2, 3] = float("nan")
    with pytest.raises(Mismatch, match=r"pixel \(y=2, x=3\)"):
        compare("nan", got, ref, 1.0)
    with pytest.raises(AssertionError, match="shape"):
        compare("shape", got[:, :, :3], ref, 1.0)


@pytest.mark.parametrize("sid", list(SHAPES))
@pytest.mark.parametrize("kh,kw,flags", [(1, 5, 0), (5, 1, 0), (1, 5, NO_HALO), (5, 1, NO_HALO)])
def test_blocked_layout_round_trip(sid, kh, kw, flags):
    """unblock() inverts the tile-blocked layout: every pixel gets its own (tile, row) slot inside the tile count the buffer is
    sized for (rnc_conv_umma_tiles), ragged tiles included."""
    B, H, W = SHAPES[sid]
    tile, row = blocked_index(kh, kw, B, H, W, flags)
    nt = tiles(kh, kw, B, H, W, flags)
    assert int(tile.max()) < nt and int(row.max()) < KBM
    slot = tile * KBM + row
    assert slot.unique().numel() == B * H * W
    C, ld = 3, 5
    vals = torch.arange(B * H * W * C, dtype=torch.float32).view(-1, C)
    buf = torch.full((nt * ld * KBM,), -1.0)
    c = torch.arange(C)
    buf[((tile[:, None] * ld + c) * KBM + row[:, None]).reshape(-1)] = vals.reshape(-1)
    assert torch.equal(unblock(buf, ld, C, kh, kw, B, H, W, flags), vals)


def test_tile_modes_at_the_product_shapes():
    """The tile modes the GPU tests rely on reaching: row halo at S1/S2 for 1x5, per-tap at S3 (W8 = 64) and S4, column halo
    ragged in y at S1 (55 rows) and in both directions at S2, none at S4 (W8 < 16)."""
    assert tile_shape(1, 5, 55, 128) == (128, 1) and tile_shape(1, 5, 47, 156) == (128, 1)
    assert tile_shape(1, 5, 48, 64) == (64, 2) and tile_shape(1, 5, 8, 12) == (16, 8)
    assert tile_shape(5, 1, 55, 128) == (16, 8) and 55 % 8 and tile_shape(5, 1, 47, 156) == (16, 8) and 156 % 16 and 47 % 8
    assert tile_shape(5, 1, 8, 12) == (16, 8)
    assert tile_shape(1, 5, 55, 128, NO_HALO) == (128, 1) and tile_shape(5, 1, 55, 128, NO_HALO) == (128, 1)
    assert tiles(3, 3, 8, 55, 128) == 440                     # the 440 pixel tiles per layer of the Sintel bench


def test_cfg5_conv_signatures_match_the_oracle_graph(monkeypatch):
    """The written-out ConvCL list equals the distinct conv2d signatures of the oracle's training graph at config 5 (the NConv
    layers are not ConvCL layers and are left out).  The GPU test checks the same list against a real train_step."""
    from oracle import raft_oracle as orc
    from rnc.synth import build_model, frames
    seen = set()
    real = F.conv2d

    def rec(x, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
        seen.add(conv2d_signature(x, weight, stride, dilation))
        return real(x, weight, bias, stride, padding, dilation, groups)

    monkeypatch.setattr(orc.F, "conv2d", rec)
    monkeypatch.setattr(orc, "nconv_unet_live", lambda sd, data, conf, p="": (data, conf))
    sd = {k: v.detach() for k, v in build_model("raft_nc_dbl").state_dict().items()}
    im1, im2 = frames(2, 384, 512)
    with torch.no_grad():
        orc.raft_forward_graph(sd, im1, im2, iters=1, model="raft_nc_dbl")
    assert sorted(seen) == CFG5_CONV_SIGNATURES
