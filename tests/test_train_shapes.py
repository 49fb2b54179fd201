"""Pointwise fp64 references and magnitude-scaled bounds for the training-shape kernel tests (tests/test_gpu_train_shapes.py),
and their CPU checks.

The GPU tests run real training steps at the reference's training crops (train_raft_nc_{things,sintel,kitti}.sh: 3 samples
per GPU at 400x720, 368x768 and 288x960) and compare every call of the training autograd Functions with an fp64 evaluation of
the same operation on the call's own inputs and upstream gradient.  This file holds what they share and what can be checked
without a GPU:
  - T_SHAPES and the launch geometry they reach (mirrored from csrc/nconv2d.cu, csrc/ncup.cu and the pyramid);
  - compare_mag(): |got - ref| <= tol * mag elementwise, where mag is the same fp64 reference evaluated on absolute values,
    so that a wrong border row or a wrong small-magnitude image cannot hide behind the large part of a tensor;
  - compare_tiles(): a per-tile max-relative bound for the fused NCUP chain, whose nonlinearity has no absolute-value scale;
  - the fp64 references with their magnitudes: conv_ref, nconv_ref, lookup_ref, pyramid_ref.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from test_product_shapes import Mismatch

# ----------------------------------------------------------------------------------------------------------- shapes
# id -> (B per GPU, image H, W).  The reference trains with --batch_size 6 on two GPUs: 3 samples per GPU.
T_SHAPES = {
    "T1": (3, 400, 720),   # Things: 1/8 grid 50x90, NCUP input 100x180
    "T2": (3, 368, 768),   # Sintel: 46x96, 92x192
    "T3": (3, 288, 960),   # KITTI: 36x120, 72x240 (sparse valid mask)
    "T1x2": (6, 400, 720),  # all 6 samples on one GPU: the NConv weight-gradient kernel past its own block cap
}

# csrc/nconv2d.cu: kThreads, grid_for()'s cap of 132 * 8 blocks, and bwd_layout()'s weight grid grid_for(pix / 8)
NCONV_THREADS = 256
NCONV_MAX_BLOCKS = 132 * 8
NCONV_GRID_ELEMS = NCONV_MAX_BLOCKS * NCONV_THREADS            # 270,336: larger launches loop (grid-stride)
NCONV_WEIGHT_PIX = 8 * NCONV_GRID_ELEMS                        # 2,162,688: the weight kernel loops beyond this
NCUP_NB = 32                                                   # csrc/ncup.cu: rnc_ncup_bwd's owned output tile side
PYR_LEVELS = 4


def nconv_grid(total):
    """grid_for() of csrc/nconv2d.cu."""
    return max(1, min(NCONV_MAX_BLOCKS, -(-total // NCONV_THREADS)))


def nconv_weight_grid(pix):
    """bwd_layout().gx: the x extent of nconv2d_bwd_weight_kernel's grid."""
    return nconv_grid(pix // 8)


def grid8(sid):
    B, H, W = T_SHAPES[sid]
    return B, H // 8, W // 8


def pyramid_sizes(H8, W8, levels=PYR_LEVELS):
    """Level sizes of the correlation pyramid (2x2 average pooling, floor mode)."""
    return [(H8 >> l, W8 >> l) for l in range(levels)]


def ncup_partial_tiles(sid):
    """(rows, cols) of rnc_ncup_bwd's 32x32 output tiles that are partial (the output is the full-resolution image)."""
    _, H, W = T_SHAPES[sid]
    return H % NCUP_NB != 0, W % NCUP_NB != 0


# ----------------------------------------------------------------------------------------------------------- tolerances
U32 = 2.0 ** -24


def ulp_tol(n, tf32=False):
    """Relative-to-mag tolerance of an fp32 sum of n products: 16 * 2^-24 * sqrt(n) (random-walk growth of the rounding errors
    with headroom); the TF32 hi/lo route drops the lo*lo product and rounds lo to TF32, ~2^-21 per product: + 2^-19."""
    return 16 * U32 * math.sqrt(max(n, 1)) + (2.0 ** -19 if tf32 else 0.0)


def _where(err, B, C, H, W, flat):
    b, rem = divmod(flat, C * H * W)
    c, rem = divmod(rem, H * W)
    y, x = divmod(rem, W)
    return b, c, y, x, f"image {b}, pixel (y={y}, x={x}), channel {c}, tile {(y * W + x) // 128}"


def _as4d(t):
    if t.dim() == 4:
        return t
    return t.reshape(1, -1, 1, 1)


def compare_mag(what, got, ref, mag, tol, floor=0.0, log=print):
    """Elementwise |got - ref| <= tol * mag + floor, with mag >= |each term| summed (the fp64 reference on absolute values);
    floor: a scalar or an elementwise absolute allowance.

    got, ref, mag: tensors of one shape ([B, C, H, W]; other ranks are checked as one row of channels).  NaN or Inf in got fails.
    Prints, and on failure raises with, the worst element's image, pixel, channel and 128-pixel tile, and the bad (image, tile)
    pairs.  Returns the worst err / bound."""
    assert got.shape == ref.shape == mag.shape, f"{what}: shapes {tuple(got.shape)}, {tuple(ref.shape)}, {tuple(mag.shape)}"
    ref = _as4d(ref.double())
    got = _as4d(got.to(ref.device).double())
    mag = _as4d(mag.to(ref.device).double())
    err = (got - ref).abs()
    err = torch.where(torch.isfinite(got), err, torch.full_like(err, math.inf))
    if torch.is_tensor(floor):
        floor = _as4d(floor.to(ref.device).double())
    bound = tol * mag + floor
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)      # bound 0 (a zero sum): only an exact result passes
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, math.inf), ratio)   # inf / inf: a non-finite operand
    B, C, H, W = err.shape
    if not err.numel():
        return 0.0
    flat = int(ratio.reshape(-1).argmax())
    worst = float(ratio.reshape(-1)[flat])
    *_, where = _where(err, B, C, H, W, flat)
    log(f"  {what:<44s} {B}x{C}x{H}x{W}: worst err/bound {worst:.2e} (err {float(err.reshape(-1)[flat]):.2e}, "
        f"|ref| {abs(float(ref.reshape(-1)[flat])):.2e}, mag {float(mag.reshape(-1)[flat]):.2e}) at {where}")
    bad = ratio > 1
    if bool(bad.any()):
        nbad = int(bad.sum())
        tiles = sorted({(int(bb), int(yy * W + xx) // 128) for bb, yy, xx in bad.amax(1).nonzero().tolist()[:4096]})
        raise Mismatch(f"{what}: {nbad} elements exceed tol * mag (tol {tol:.2e}); worst err/bound {worst:.3e} at {where}; "
                       f"bad (image, tile): {tiles[:16]}{' ...' if len(tiles) > 16 else ''}")
    return worst


def compare_tiles(what, got, ref, tile, tol, big=1e6, log=print):
    """Per-tile bound: |got - ref| <= tol * max_tile |ref| over the positions with |ref| < big, for tile x tile tiles of the
    last two dimensions of [B, C, H, W] tensors (ragged last tiles included).  Returns the worst err / bound."""
    assert got.shape == ref.shape and got.dim() == 4, f"{what}: shapes {tuple(got.shape)}, {tuple(ref.shape)}"
    ref = ref.double()
    got = got.to(ref.device).double()
    ok = torch.isfinite(ref) & (ref.abs() < big)
    r = torch.where(ok, ref, torch.zeros_like(ref))
    err = torch.where(ok, (got - r).abs(), torch.zeros_like(r))
    err = torch.where(ok & ~torch.isfinite(got), torch.full_like(err, math.inf), err)
    B, C, H, W = ref.shape
    ty, tx = -(-H // tile), -(-W // tile)
    rp = F.pad(r.abs(), (0, tx * tile - W, 0, ty * tile - H))
    scale = rp.view(B, C, ty, tile, tx, tile).amax((3, 5))                               # [B, C, ty, tx]
    bound = tol * scale.repeat_interleave(tile, 2).repeat_interleave(tile, 3)[:, :, :H, :W]
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, math.inf), ratio)
    flat = int(ratio.reshape(-1).argmax())
    worst = float(ratio.reshape(-1)[flat])
    b, c, y, x, _ = _where(err, B, C, H, W, flat)
    where = f"image {b}, channel {c}, pixel (y={y}, x={x}), {tile}x{tile} tile ({y // tile}, {x // tile})"
    log(f"  {what:<44s} {B}x{C}x{H}x{W}: worst err/bound {worst:.2e} at {where}")
    bad = ratio > 1
    if bool(bad.any()):
        tl = sorted({(int(bb), int(yy) // tile, int(xx) // tile) for bb, yy, xx in bad.amax(1).nonzero().tolist()[:4096]})
        raise Mismatch(f"{what}: {int(bad.sum())} elements exceed {tol:.1e} * max_tile|ref|; worst err/bound {worst:.3e} at "
                       f"{where}; bad (image, tile row, tile col): {tl[:16]}{' ...' if len(tl) > 16 else ''}")
    return worst


# ----------------------------------------------------------------------------------------------------------- fp64 references
# Every reference takes the call's recorded fp32 tensors (any device) and returns {name: (ref, mag, n)}: the fp64 value, the
# same evaluation on absolute values, and the number of products summed per element (for ulp_tol).

def conv_ref(x, w, b, gy, stride=1, dil=1, grads=("dx", "dw", "db")):
    """conv2d with zero padding (k // 2) * dil.  x [B, Cin, H, W], w [Cout, Cin, kh, kw], b [Cout] or None, gy the upstream
    gradient of y (or None).  y, dx, dw, db."""
    cout, cin, kh, kw = w.shape
    pad = ((kh // 2) * dil, (kw // 2) * dil)

    def ev(x_, w_, b_, g_):
        leaves = [x_.detach().double().requires_grad_("dx" in grads), w_.detach().double().requires_grad_("dw" in grads)]
        leaves.append(None if b_ is None else b_.detach().double().requires_grad_("db" in grads))
        with torch.enable_grad():
            y = F.conv2d(leaves[0], leaves[1], leaves[2], stride, pad, dil)
            want = [t for t in leaves if t is not None and t.requires_grad]
            gs = torch.autograd.grad(y, want, g_.double()) if g_ is not None and want else [None] * len(want)
        out = {"y": y.detach()}
        k = 0
        for name, t in zip(("dx", "dw", "db"), leaves):
            if t is not None and t.requires_grad:
                out[name], k = gs[k], k + 1
        return out

    ref = ev(x, w, b, gy)
    mag = ev(x.abs(), w.abs(), None if b is None else b.abs(), None if gy is None else gy.abs())
    Bn, _, Ho, Wo = ref["y"].shape
    n = {"y": cin * kh * kw + 1, "dx": cout * kh * kw, "dw": Bn * Ho * Wo, "db": Bn * Ho * Wo}
    return {k: (ref[k], mag[k], n[k]) for k in ref if gy is not None or k == "y"}


def _nconv_num_den(x, c, w, ux, uc):
    H, W = x.shape[-2:]
    if ux is not None:
        x = torch.cat([F.interpolate(ux, size=(H, W), mode="nearest"), x], 1)
        c = torch.cat([F.interpolate(uc, size=(H, W), mode="nearest"), c], 1)
    pad = (w.shape[-2] // 2, w.shape[-1] // 2)
    return F.conv2d(x * c, w, padding=pad), F.conv2d(c, w, padding=pad)


def nconv_ref(x, c, w, bias, eps, ux, uc, gy, gc, want=("g_data", "g_conf", "g_w", "g_b", "g_ux", "g_uc")):
    """NConv2d (nconv_modules.py:164-199) with the decoder's nearest-upsampled coarse source ux / uc as the first input channels
    (the formula of test_gpu_ncup_variants.py::test_nconv_layer_up_source_and_bias_match_fp64): y, conf_out and the gradients
    named in `want` for the upstream (gy, gc).

    Magnitudes (the kernel's own a/b form with absolute values, D = den + eps, yq = y - bias):
      y      (sum |x| c w + |yq| den) / D + |bias|        conf_out   den / s
      |a| = |gy| / D,   |b| = |gy| mag_yq / D + |gc| / s
      g_data c sum w |a|;   g_conf sum w (|a||x| + |b|);   g_w sum_p (|a||x| c + |b| c) + sum_p |gc| den / s^2;   g_b sum |gy|.
    |b| takes mag_yq = (sum |x| c w + |yq| den) / D rather than |yq|: the kernel forms b from its own fp32 y, whose error scales
    with mag_yq, and where the quotient cancels |yq| alone would understate it."""
    dd = [None if t is None else t.detach().double() for t in (x, c, w, bias, ux, uc)]
    x, c, w, bias, ux, uc = dd
    Cout = w.shape[0]
    names = ("g_data", "g_conf", "g_w", "g_b", "g_ux", "g_uc")
    leaves = [None if t is None else t.clone().requires_grad_(k in want) for t, k in zip((x, c, w, bias, ux, uc), names)]
    with torch.enable_grad():
        num, den = _nconv_num_den(leaves[0], leaves[1], leaves[2], leaves[4], leaves[5])
        s = leaves[2].reshape(Cout, -1).sum(-1).view(1, -1, 1, 1)
        y = num / (den + eps)
        if leaves[3] is not None:
            y = y + leaves[3].view(1, -1, 1, 1)
        co = den / s
        req = [t for t in leaves if t is not None and t.requires_grad]
        gy_ = torch.zeros_like(y) if gy is None else gy.double()
        gc_ = torch.zeros_like(co) if gc is None else gc.double()
        gs = torch.autograd.grad([y, co], req, [gy_, gc_], allow_unused=True) if req else []
    out = {"y": y.detach(), "conf": co.detach()}
    j = 0
    for t, k in zip(leaves, names):
        if t is not None and t.requires_grad:
            g, j = gs[j], j + 1
            out[k] = torch.zeros_like(t) if g is None else g
    # magnitudes
    Ct, kh, kw = w.shape[1:]
    with torch.no_grad():
        num, den = num.detach(), den.detach()
        s = s.detach()
        D = den + eps
        yq = num / D
        num_abs, _ = _nconv_num_den(x.abs(), c, w, None if ux is None else ux.abs(), uc)
        mag_yq = (num_abs + yq.abs() * den) / D
        mag = {"y": mag_yq + (0 if bias is None else bias.abs().view(1, -1, 1, 1)), "conf": den / s}
        a_abs = gy_.abs() / D
        b_abs = gy_.abs() * mag_yq / D + gc_.abs() / s
    ml = [t if t is None else t.clone().requires_grad_(True) for t in (x.abs(), c, w, None, None if ux is None else ux.abs(), uc)]
    with torch.enable_grad():
        n1, d1 = _nconv_num_den(ml[0], ml[1], ml[2], ml[4], ml[5])
        lx = [ml[0]] + ([ml[4]] if ux is not None else [])
        g_x = torch.autograd.grad((a_abs * n1).sum(), lx, retain_graph=True)
        lc = [ml[1], ml[2]] + ([ml[5]] if uc is not None else [])
        g_c = torch.autograd.grad((a_abs * n1 + b_abs * d1).sum(), lc)
    corr = ((gc_.abs() * den).sum((0, 2, 3)) / s.view(-1) ** 2).view(Cout, 1, 1, 1)
    mag.update({"g_data": g_x[0], "g_conf": g_c[0], "g_w": g_c[1] + corr, "g_b": gy_.abs().sum((0, 2, 3))})
    if ux is not None:
        mag.update({"g_ux": g_x[1], "g_uc": g_c[2]})
    N, _, H, W = y.shape
    pre = 1 if ux is None else max(1, math.ceil(H / ux.shape[2]) * math.ceil(W / ux.shape[3]))   # preimage of a coarse pixel
    n = {"y": Ct * kh * kw + 2, "conf": Ct * kh * kw + 1, "g_data": Cout * kh * kw + 1, "g_conf": Cout * kh * kw + 2,
         "g_ux": pre * (Cout * kh * kw + 1), "g_uc": pre * (Cout * kh * kw + 2), "g_w": 2 * N * H * W + 1, "g_b": N * H * W}
    return {k: (v, mag[k], n[k]) for k, v in out.items()}


def lookup_ref(f1, f2_levels, coords, g_out, grads=True, radius=4):
    """CorrLookup (corr.py:23-44) on fmap1 [B, D, H, W] and the pyramid levels of fmap2 [B, D, Hl, Wl]: the reference's bilinear
    sampling (orc.corr_lookup, at the positions themselves, as the kernels sample) of the volumes f1 . f2_l / sqrt(D), and,
    with g_out [B, 324, H, W], d fmap1 and d f2_l.  The magnitude is the same lookup of |f1| . |f2_l| (the bilinear weights are
    non-negative) against |g_out|.

    Each entry also carries an absolute allowance for the one rounding of the sample position: the kernels' fraction
    s - floor(s) is exact except for -1 < s < 0, where s + 1 rounds by up to 2^-25, so each bilinear weight may be off by
    2^-24 there.  The allowance is 2^-24 times the sum of the |values| of the four lattice corners (the same lookup with every
    corner weighted 1, and its adjoint) at the pixels of a level whose centre lies in (-1, 0) in x or y; it is 0 elsewhere."""
    from oracle import raft_oracle as orc
    B, D, H, W = f1.shape
    co = coords.double()

    def ev(a, levels, g, box):
        a = a.detach().double().requires_grad_(grads)
        levels = [t.detach().double().requires_grad_(grads) for t in levels]
        with torch.enable_grad():
            af = a.reshape(B, D, H * W).transpose(1, 2)
            outs = []
            for l, t in enumerate(levels):
                vol = torch.matmul(af, t.reshape(B, D, -1)).view(B * H * W, 1, *t.shape[-2:]) / math.sqrt(D)
                c = co / 2 ** l
                if box:
                    edge = ((c > -1) & (c < 0)).any(1, keepdim=True)
                    outs.append(4 * orc.corr_lookup([vol], torch.floor(c) + 0.5, radius, torch.float64, round_trip=False) * edge)
                else:
                    outs.append(orc.corr_lookup([vol], c, radius, torch.float64, round_trip=False))
            out = torch.cat(outs, 1)
            gs = torch.autograd.grad(out, [a] + levels, g.double()) if grads else None
        return out.detach(), gs

    ref, gr = ev(f1, f2_levels, g_out, False)
    absd = (f1.abs(), [t.abs() for t in f2_levels], None if g_out is None else g_out.abs())
    mag, gm = ev(*absd, False)
    pos, gp = ev(*absd, True)
    res = {"y": (ref, mag, 4 * D, 2.0 ** -24 * pos)}
    if grads:
        taps = (2 * radius + 1) ** 2
        res["g_f1"] = (gr[0], gm[0], 4 * taps * len(f2_levels) * 4, 2.0 ** -24 * gp[0])
        for l in range(len(f2_levels)):
            res[f"g_f2[{l}]"] = (gr[1 + l], gm[1 + l], 4 * min(H * W, (2 * (radius + 1) << l) ** 2), 2.0 ** -24 * gp[1 + l])
    return res


def pyramid_ref(level_grads):
    """Adjoint of the feature pyramid (level l = 2x2 average pool of level l-1): level_grads [B, D, Hl, Wl] per level -> the
    gradient of level 0, and its magnitude (the adjoint of |g|)."""
    def ev(gl):
        f0 = torch.zeros_like(gl[0], dtype=torch.float64).requires_grad_(True)
        with torch.enable_grad():
            lv, tot = f0, 0
            for l, g in enumerate(gl):
                if l:
                    lv = F.avg_pool2d(lv, 2, stride=2)
                tot = tot + (lv * g.double()).sum()
            return torch.autograd.grad(tot, f0)[0]
    return ev(level_grads), ev([g.abs() for g in level_grads]), len(level_grads)


# ======================================================================================================== CPU tests


def test_compare_mag_rejects_a_small_images_border_row():
    """A 1e-5 error (relative to the elements' own magnitude) in one border row of the one small image of a conv-gradient-like
    tensor (its other images 100x larger) fails compare_mag, naming that image and tile; compare() at the conv tolerance
    accepts it.  NaN fails too."""
    from test_product_shapes import TOL, compare
    B, C, H, W = 3, 8, 50, 90
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(C, C, 1, 1, generator=g, dtype=torch.float64)
    gy = torch.randn(B, C, H, W, generator=g, dtype=torch.float64) * 100
    gy[1] *= 0.01                                              # image 1: 100x smaller upstream gradient than the others
    r = conv_ref(x, w, None, gy)
    ref, mag, n = r["dx"]
    got = ref.float()
    tol = ulp_tol(n)
    assert compare_mag("exact", got, ref, mag, tol) < 1
    bad = got.clone()
    bad[1, :, H - 1, :] += (1e-5 * mag[1, :, H - 1, :]).float()
    compare("dx (norm-scaled)", bad, ref, TOL["conv"])       # hidden behind the large images
    with pytest.raises(Mismatch) as e:
        compare_mag("dx", bad, ref, mag, tol)
    tile = ((H - 1) * W) // 128
    assert "image 1," in str(e.value) and f"(1, {tile})" in str(e.value)
    nan = got.clone()
    nan[2, 3, 7, 11] = float("nan")
    with pytest.raises(Mismatch, match=r"image 2, pixel \(y=7, x=11\), channel 3"):
        compare_mag("nan", nan, ref, mag, tol)


def test_compare_mag_rejects_errors_past_the_first_grid_stride_pass():
    """An error only in elements at flat index >= 270,336 (those a grid-stride kernel writes on its second pass) fails."""
    N, H, W = 6, 400, 720                                      # the NConv planes of T1: 1.73 M elements
    g = torch.Generator().manual_seed(1)
    ref = torch.randn(N, 1, H, W, generator=g, dtype=torch.float64)
    mag = ref.abs() * 2 + 0.1
    got = ref.float()
    assert compare_mag("exact", got, ref, mag, ulp_tol(25)) < 1
    flat = got.view(-1)
    flat[NCONV_GRID_ELEMS::997] *= (1 + 1e-4)
    with pytest.raises(Mismatch) as e:
        compare_mag("second pass", got, ref, mag, ulp_tol(25))
    import re
    b, y, x = map(int, re.search(r"image (\d+), pixel \(y=(\d+), x=(\d+)\)", str(e.value)).groups())
    assert (b * H + y) * W + x >= NCONV_GRID_ELEMS


def test_compare_tiles_names_a_wrong_tile_beside_large_ones():
    g = torch.Generator().manual_seed(2)
    ref = torch.randn(2, 2, 400, 720, generator=g, dtype=torch.float64)
    ref[:, :, :384] *= 1000                                    # the last tile row (16 rows, partial) is 1000x smaller
    got = ref.clone()
    assert compare_tiles("exact", got, ref, NCUP_NB, 1e-4) == 0
    got[1, 0, 390, 700:720] += 3e-4 * float(ref[1, 0, 384:, 704:].abs().max())
    with pytest.raises(Mismatch, match=r"image 1, channel 0, pixel \(y=390.*tile \(12, 2[12]\)"):
        compare_tiles("partial tile", got, ref, NCUP_NB, 1e-4)


def test_training_shapes_reach_the_intended_launch_geometry():
    """The facts the GPU cases rely on: NConv launches past the grid-stride cap at every T shape (N = 2B zero-stuffed
    full-resolution planes), the weight-gradient kernel past its own cap only at T1x2, rnc_ncup_bwd partial tiles at T1 (both
    axes) and T2 (rows) but not T3, and the odd pyramid levels."""
    for sid in ("T1", "T2", "T3", "T1x2"):
        B, H, W = T_SHAPES[sid]
        pix = 2 * B * H * W
        assert pix > NCONV_GRID_ELEMS and nconv_grid(pix) == NCONV_MAX_BLOCKS, sid
        assert -(-pix // (NCONV_MAX_BLOCKS * NCONV_THREADS)) >= 6, sid          # at least 6 grid-stride passes
        past = pix > NCONV_WEIGHT_PIX
        assert past == (sid == "T1x2"), sid
        assert (nconv_weight_grid(pix) == NCONV_MAX_BLOCKS) == past
    assert NCONV_GRID_ELEMS == 270336 and NCONV_WEIGHT_PIX == 2162688
    assert 2 * 3 * 400 * 720 == 1728000 and 2 * 6 * 400 * 720 == 3456000
    assert ncup_partial_tiles("T1") == (True, True)
    assert ncup_partial_tiles("T2") == (True, False)
    assert ncup_partial_tiles("T3") == (False, False)
    assert pyramid_sizes(*grid8("T1")[1:]) == [(50, 90), (25, 45), (12, 22), (6, 11)]
    assert pyramid_sizes(*grid8("T2")[1:]) == [(46, 96), (23, 48), (11, 24), (5, 12)]
    assert pyramid_sizes(*grid8("T3")[1:]) == [(36, 120), (18, 60), (9, 30), (4, 15)]
    for sid, odd in (("T1", {1, 3}), ("T2", {1, 2, 3}), ("T3", {2, 3})):
        sizes = pyramid_sizes(*grid8(sid)[1:])
        assert {l for l, (h, w) in enumerate(sizes) if h % 2 or w % 2} == odd, sid


def test_mag_helpers_equal_brute_force_sums():
    """conv_ref's and nconv_ref's magnitudes equal a brute-force fp64 sum of |terms| on a tiny case (the pyramid adjoint and the
    lookup use the same abs-evaluation of a linear map, checked through the conv)."""
    g = torch.Generator().manual_seed(3)
    B, Ci, Co, H, W = 2, 3, 2, 5, 6
    x = torch.randn(B, Ci, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Co, Ci, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(Co, generator=g, dtype=torch.float64)
    gy = torch.randn(B, Co, H, W, generator=g, dtype=torch.float64)
    r = conv_ref(x, w, b, gy)
    xp = F.pad(x, (1, 1, 1, 1))
    my, mdx, mdw = torch.zeros(B, Co, H, W, dtype=torch.float64), torch.zeros(B, Ci, H + 2, W + 2, dtype=torch.float64), \
        torch.zeros(Co, Ci, 3, 3, dtype=torch.float64)
    for n in range(B):
        for o in range(Co):
            for yy in range(H):
                for xx in range(W):
                    my[n, o, yy, xx] += abs(b[o])
                    for i in range(Ci):
                        for ky in range(3):
                            for kx in range(3):
                                t = abs(xp[n, i, yy + ky, xx + kx] * w[o, i, ky, kx])
                                my[n, o, yy, xx] += t
                                mdx[n, i, yy + ky, xx + kx] += abs(gy[n, o, yy, xx] * w[o, i, ky, kx])
                                mdw[o, i, ky, kx] += abs(gy[n, o, yy, xx] * xp[n, i, yy + ky, xx + kx])
    assert torch.allclose(r["y"][1], my, rtol=1e-12, atol=0)
    assert torch.allclose(r["dx"][1], mdx[:, :, 1:-1, 1:-1], rtol=1e-12, atol=0)
    assert torch.allclose(r["dw"][1], mdw, rtol=1e-12, atol=0)
    assert torch.allclose(r["db"][1], gy.abs().sum((0, 2, 3)), rtol=1e-12, atol=0)

    # NConv with an up source and bias: 1 coarse + 1 full-resolution channel -> 2 outputs, 3x3
    N, H, W, Hu, Wu, eps = 2, 4, 6, 2, 3, 1e-20
    x = torch.randn(N, 1, H, W, generator=g, dtype=torch.float64)
    c = torch.rand(N, 1, H, W, generator=g, dtype=torch.float64)
    ux = torch.randn(N, 1, Hu, Wu, generator=g, dtype=torch.float64)
    uc = torch.rand(N, 1, Hu, Wu, generator=g, dtype=torch.float64)
    w = torch.rand(2, 2, 3, 3, generator=g, dtype=torch.float64) + 0.1
    bias = torch.randn(2, generator=g, dtype=torch.float64)
    gy = torch.randn(N, 2, H, W, generator=g, dtype=torch.float64)
    gc = torch.randn(N, 2, H, W, generator=g, dtype=torch.float64)
    r = nconv_ref(x, c, w, bias, eps, ux, uc, gy, gc)
    X = torch.cat([ux.repeat_interleave(2, 2).repeat_interleave(2, 3), x], 1)
    Cc = torch.cat([uc.repeat_interleave(2, 2).repeat_interleave(2, 3), c], 1)
    Xp, Cp = F.pad(X, (1, 1, 1, 1)), F.pad(Cc, (1, 1, 1, 1))
    s = w.reshape(2, -1).sum(-1)
    den = torch.zeros(N, 2, H, W, dtype=torch.float64)
    num_abs = torch.zeros_like(den)
    num = torch.zeros_like(den)
    for n in range(N):
        for o in range(2):
            for yy in range(H):
                for xx in range(W):
                    for i in range(2):
                        for ky in range(3):
                            for kx in range(3):
                                den[n, o, yy, xx] += Cp[n, i, yy + ky, xx + kx] * w[o, i, ky, kx]
                                num[n, o, yy, xx] += Xp[n, i, yy + ky, xx + kx] * Cp[n, i, yy + ky, xx + kx] * w[o, i, ky, kx]
                                num_abs[n, o, yy, xx] += abs(Xp[n, i, yy + ky, xx + kx]) * Cp[n, i, yy + ky, xx + kx] * w[o, i, ky, kx]
    D = den + eps
    yq = num / D
    mag_yq = (num_abs + yq.abs() * den) / D
    assert torch.allclose(r["y"][0], yq + bias.view(1, -1, 1, 1), rtol=1e-12)
    assert torch.allclose(r["y"][1], mag_yq + bias.abs().view(1, -1, 1, 1), rtol=1e-12)
    a = gy.abs() / D
    bb = gy.abs() * mag_yq / D + gc.abs() / s.view(1, -1, 1, 1)
    A = torch.zeros(N, 2, H + 2, W + 2, dtype=torch.float64)
    Bm = torch.zeros_like(A)
    gw = torch.zeros(2, 2, 3, 3, dtype=torch.float64)
    for n in range(N):
        for o in range(2):
            for yy in range(H):
                for xx in range(W):
                    for i in range(2):
                        for ky in range(3):
                            for kx in range(3):
                                A[n, i, yy + ky, xx + kx] += a[n, o, yy, xx] * w[o, i, ky, kx]
                                Bm[n, i, yy + ky, xx + kx] += bb[n, o, yy, xx] * w[o, i, ky, kx]
                                gw[o, i, ky, kx] += (a[n, o, yy, xx] * abs(Xp[n, i, yy + ky, xx + kx])
                                                     + bb[n, o, yy, xx]) * Cp[n, i, yy + ky, xx + kx]
    A, Bm = A[:, :, 1:-1, 1:-1], Bm[:, :, 1:-1, 1:-1]
    gw += ((gc.abs() * den).sum((0, 2, 3)) / s ** 2).view(2, 1, 1, 1)
    assert torch.allclose(r["g_data"][1], Cc[:, 1:] * A[:, 1:], rtol=1e-12)
    assert torch.allclose(r["g_conf"][1], X[:, 1:].abs() * A[:, 1:] + Bm[:, 1:], rtol=1e-12)
    pool = lambda t: t.view(N, 1, Hu, 2, Wu, 2).sum((3, 5))              # noqa: E731  (the nearest x2 preimage)
    assert torch.allclose(r["g_ux"][1], pool(Cc[:, :1] * A[:, :1]), rtol=1e-12)
    assert torch.allclose(r["g_uc"][1], pool(X[:, :1].abs() * A[:, :1] + Bm[:, :1]), rtol=1e-12)
    assert torch.allclose(r["g_w"][1], gw, rtol=1e-12)
    assert torch.allclose(r["g_b"][1], gy.abs().sum((0, 2, 3)), rtol=1e-12)
    # and the references themselves: NConv's gradients against autograd's (finite differences would be too coarse)
    assert torch.allclose(r["conf"][0], den / s.view(1, -1, 1, 1), rtol=1e-12)


def test_lookup_and_pyramid_references_on_a_tiny_case():
    """lookup_ref equals the direct lookup (corr_lookup_direct, pooled features) and its magnitude bounds |ref|; pyramid_ref's
    adjoint satisfies <adj(g), f> = sum_l <g_l, pool^l(f)>."""
    from oracle import raft_oracle as orc
    g = torch.Generator().manual_seed(4)
    B, D, H, W = 1, 8, 17, 19
    f1 = torch.randn(B, D, H, W, generator=g, dtype=torch.float64)
    f2 = torch.randn(B, D, H, W, generator=g, dtype=torch.float64)
    levels = [f2]
    for _ in range(3):
        levels.append(F.avg_pool2d(levels[-1], 2, stride=2))
    coords = orc.coords_grid(B, H, W).double() + torch.randn(B, 2, H, W, generator=g, dtype=torch.float64) * 3
    gout = torch.randn(B, 324, H, W, generator=g, dtype=torch.float64)
    r = lookup_ref(f1, levels, coords, gout)
    assert torch.allclose(r["y"][0], orc.corr_lookup_direct(f1, f2, coords), rtol=1e-10, atol=1e-12)
    for k, (ref, mag, n, pos) in r.items():
        assert (ref.abs() <= mag * (1 + 1e-12) + 1e-300).all() and (pos >= 0).all(), k
    gl = [torch.randn(l.shape, generator=g, dtype=torch.float64) for l in levels]
    adj, mag, n = pyramid_ref(gl)
    lhs = (adj * f2).sum()
    rhs = sum((a * b).sum() for a, b in zip(gl, levels))
    assert abs(float(lhs - rhs)) < 1e-10 * float(rhs.abs() + 1) and n == 4 and (adj.abs() <= mag * (1 + 1e-12)).all()
