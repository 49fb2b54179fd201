"""An fp64 model of the tensor-core correlation lookup's arithmetic (csrc/corr_lookup_umma.cu), host restatements of its unit
records and schedule, and the elementwise bounds that follow.  tests/test_gpu_lookup_error_model.py holds the kernel to them.

What the kernel computes, per (tile of 8x16 pixels, pyramid level) unit:
  - tensor-core units: the 10x10 lattice dot products of fmap1 against fmap2^l, both rounded once to fp16 (the f1h / f2h
    buffers of UmmaEngine), on wgmma m64nNk16.f32.f16.f16 (products of halves exact, fp32 accumulation over K = 256 in 16
    steps); the epilogue of lookup_level_rows blends the lattice bilinearly with the 1/sqrt(256) = 1/16 scale folded into the
    x weights, and splits the result into hi/lo halves;
  - units whose windows do not fit the fixed boxes (flagged in the workspace): exact_unit, the same lookup in fp32 from the
    unrounded fp32 operands.
Precondition: |features| <= 65504 (beyond, the halves are inf).  The output is a hi/lo pair of halves: up to 65504 it keeps
22 bits, beyond 131008 both halves saturate (split_bound then allows the whole excess, so such outputs test nothing).

lookup_split_ref() evaluates the first in fp64.  Bounds:
  - tensor-core units, against lookup_split_ref:
        |got - ref| <= C_A * 16 * 2^-24 * mag_a + C_E * 2^-24 * gabs + split_bound(ref) + pos
    (C_A: the accumulation constant the convolution model measured for the same instruction, tests/test_conv_error_model.py;
    C_E: the epilogue's roundings, see C_E; gabs: the blend of the |lattice values|; pos: the rounded fraction at -1 < s < 0);
  - R (rounding_bound): the distance of lookup_split_ref from the fp64 lookup of the fp32 operands, from the fp16 rounding
    rule |f - rn16(f)| <= 2^-11 |f| + 2^-25;
  - flagged units, against the fp64 lookup of the fp32 operands: lookup_ref's fp32 bound (tests/test_train_shapes.py,
    ulp_tol(4 D) * mag + pos) plus split_bound for the hi/lo output.
"""
import math
from typing import NamedTuple, Optional

import pytest
import torch
import torch.nn.functional as F

from test_conv_error_model import C_A, U, split_bound, split_emulate
from test_product_shapes import Mismatch
from test_train_shapes import compare_mag, lookup_ref, ulp_tol

D = 256                    # feature channels (kD)
STEPS = D // 16            # K steps of one wgmma m64nNk16
SCALE = 1.0 / 16.0         # 1 / sqrt(D)
LEVELS, RADIUS = 4, 4
NG, NS = 10, 9             # lattice side (kG), taps per side (kS)
TY, TX = 8, 16             # query tile (kTY, kTX)
LVL_STRIDE = 88            # channels per level in the resident row (kLvlStride)
COORD_CLAMP = 1.0e6        # clamp_coord
SUB = 2.0 ** -14           # the exponent a subnormal half (or a zero) carries in the tensor core's alignment

# Epilogue constant: |blend computed - blend of the fp32 lattice values| <= C_E * 2^-24 * gabs (first order).  The longest
# path of a lattice value g to an output o in lookup_level_rows:
#   wx0 = scale - wx1 (wx1 = ax * scale is exact: scale is a power of two; the difference rounds)       1
#   h = wx0 * g0 + wx1 * g1: the product wx0 * g0 and the sum (two roundings; one when contracted to an fma)   2
#   wy0 = 1 - ay                                                                                      1
#   o = wy0 * hprev + ay * h0: the product wy0 * hprev and the sum (two; one when contracted)          2
# Each rounding is relative to its own term, and every term is a nonnegative weight times |g|, so the error of o is at most
# 6 * 2^-24 times the blend of |g|, whether or not the compiler contracts the products into fmas.  The accumulator's own error
# enters the blend with weights that sum to the scale: the C_A term.
C_E = 6.0


# ----------------------------------------------------------------------------------------------------------- kernel constants
def box_w(l):
    return 32 if l == 0 else 24 if l == 1 else 16


def chunk_rows(l):
    return 4 if l <= 1 else 8


def box_h(l):
    return chunk_rows(l) * (6 if l <= 1 else 3)


BOX_KINDS = 4              # TMA boxes of 2, 4, 6, 8 rows per level


def resident_index():
    """Reference channel k = l*81 + i*9 + j -> its position in the resident row, from the kernel's header comment:
    tap (i, j), i < 8 -> j*8 + i;  tap (8, j) -> 72 + j;  81..87 zero pads; level l at l*88."""
    idx = []
    for l in range(LEVELS):
        for i in range(NS):
            for j in range(NS):
                idx.append(l * LVL_STRIDE + (j * 8 + i if i < 8 else 72 + j))
    return torch.tensor(idx, dtype=torch.long)


# ----------------------------------------------------------------------------------------------------------- the model
class LookupRef(NamedTuple):
    ref: torch.Tensor          # fp64 lookup of the given operands  [B, 324, H, W], reference channel order
    mag: torch.Tensor          # the same lookup of |f1| . |f2|
    mag_a: torch.Tensor        # ... with every operand taken at no less than 2^-14 (zero-filled lattice positions too)
    gabs: torch.Tensor         # blend of the |lattice values|
    pos: torch.Tensor          # 2^-24 * sum of the four corners' mag at a level whose sample centre lies in (-1, 0)
    steps: int


def _level_geometry(coords_b, l, Hl, Wl):
    """Sample positions of one image at level l: lattice gather index [P, 100] (a = x offset major, c = y offset minor), its
    in-image mask [P, 10, 10], the bilinear fractions and the (-1, 0) edge mask.  coords are clamped to +-1e6 in their own
    dtype (the kernel's clamp_coord on fp32) and the fractions are exact in fp64."""
    c = coords_b.clamp(-COORD_CLAMP, COORD_CLAMP).double() / 2 ** l
    cx, cy = c[0].reshape(-1), c[1].reshape(-1)
    fx, fy = torch.floor(cx), torch.floor(cy)
    ax, ay = cx - fx, cy - fy
    dev = coords_b.device
    off = torch.arange(NG, device=dev, dtype=torch.float64)
    xi = (fx - RADIUS)[:, None, None] + off[None, :, None]
    yi = (fy - RADIUS)[:, None, None] + off[None, None, :]
    ok = (xi >= 0) & (xi <= Wl - 1) & (yi >= 0) & (yi <= Hl - 1)
    idx = (yi.clamp(0, Hl - 1) * Wl + xi.clamp(0, Wl - 1)).long().reshape(cx.shape[0], -1)
    edge = ((cx > -1) & (cx < 0)) | ((cy > -1) & (cy < 0))
    return idx, ok, ax, ay, edge


def _blend(g, ax, ay):
    """[P, 10 (x), 10 (y)] lattice -> [P, 81] taps (i*9 + j) with the exact bilinear weights."""
    ax, ay = ax[:, None, None], ay[:, None, None]
    return ((1 - ax) * (1 - ay) * g[:, :-1, :-1] + ax * (1 - ay) * g[:, 1:, :-1] + (1 - ax) * ay * g[:, :-1, 1:]
            + ax * ay * g[:, 1:, 1:]).reshape(g.shape[0], -1)


def _lattice(vol, idx, ok, fill=0.0):
    g = vol.gather(1, idx).view(ok.shape)
    fill = fill[:, None, None] if torch.is_tensor(fill) else fill
    return torch.where(ok, g, fill)


def _to_nchw(rows, H, W):
    return rows.view(H, W, -1).permute(2, 0, 1)


def lookup_split_ref(f1h, f2h_levels, coords):
    """fp64 evaluation of what the tensor-core units compute: the lattice dot products of the given operands (the kernel's
    halves: their products are exact), times 1/16, blended with the bilinear weights of the fp32 coordinates.  f1h
    [B, D, H, W], f2h_levels [B, D, Hl, Wl] per level (any float dtype, any device), coords [B, 2, H, W] fp32.  Evaluated one
    image at a time.  Returns a LookupRef."""
    B, _, H, W = f1h.shape
    outs = {k: torch.zeros(B, LEVELS * NS * NS, H, W, dtype=torch.float64, device=f1h.device)
            for k in ("ref", "mag", "mag_a", "gabs", "pos")}
    nu = lambda t: t.abs().clamp_min(SUB)                 # noqa: E731
    for b in range(B):
        a = f1h[b].reshape(D, H * W).t().double()
        for l, f2 in enumerate(f2h_levels):
            Hl, Wl = f2.shape[-2:]
            m = f2[b].reshape(D, Hl * Wl).double()
            idx, ok, ax, ay, edge = _level_geometry(coords[b], l, Hl, Wl)
            g = _lattice((a @ m) * SCALE, idx, ok)
            gm = _lattice((a.abs() @ m.abs()) * SCALE, idx, ok)
            ga = _lattice((nu(a) @ nu(m)) * SCALE, idx, ok, nu(a).sum(1) * SUB * SCALE)
            corners = gm[:, :-1, :-1] + gm[:, 1:, :-1] + gm[:, :-1, 1:] + gm[:, 1:, 1:]
            ch = slice(l * NS * NS, (l + 1) * NS * NS)
            outs["ref"][b, ch] = _to_nchw(_blend(g, ax, ay), H, W)
            outs["mag"][b, ch] = _to_nchw(_blend(gm, ax, ay), H, W)
            outs["mag_a"][b, ch] = _to_nchw(_blend(ga, ax, ay), H, W)
            outs["gabs"][b, ch] = _to_nchw(_blend(g.abs(), ax, ay), H, W)
            outs["pos"][b, ch] = _to_nchw(2.0 ** -24 * corners.reshape(H * W, -1) * edge[:, None], H, W)
    return LookupRef(steps=STEPS, **outs)


def rounding_bound(f1, f2_levels, coords):
    """R: bound on |lookup of the fp32 operands - lookup_split_ref of their halves|, from the rounding rule
    |f - rn16(f)| <= d(f) = 2^-11 |f| + 2^-25 (|f| <= 65504; the floor is half the smallest subnormal):
        f1 f2 - h1 h2 = f1 (f2 - h2) + (f1 - h1) h2,   |h2| <= |f2| + d2
        R = lookup of (|f1| d2 + d1 |f2| + d1 d2), times (1 + 2^-20), plus 2 D 2^-53 mag for the two fp64 evaluations."""
    B, _, H, W = f1.shape
    out = torch.zeros(B, LEVELS * NS * NS, H, W, dtype=torch.float64, device=f1.device)
    d = lambda t: 2.0 ** -11 * t.abs() + 2.0 ** -25       # noqa: E731
    for b in range(B):
        a = f1[b].reshape(D, H * W).t().double()
        for l, f2 in enumerate(f2_levels):
            Hl, Wl = f2.shape[-2:]
            m = f2[b].reshape(D, Hl * Wl).double()
            idx, ok, ax, ay, _ = _level_geometry(coords[b], l, Hl, Wl)
            r = (a.abs() @ d(m) + d(a) @ m.abs() + d(a) @ d(m)) * SCALE
            mag = (a.abs() @ m.abs()) * SCALE
            lat = _lattice(r * (1 + 2.0 ** -20) + 2 * D * 2.0 ** -53 * mag, idx, ok)
            out[b, l * NS * NS:(l + 1) * NS * NS] = _to_nchw(_blend(lat, ax, ay), H, W)
    return out


def exact_ref(f1, f2_levels, coords):
    """lookup_ref's "y" entry (fp64 lookup of the fp32 operands, its magnitude, its fp32 tolerance and position allowance),
    one image at a time: (ref, mag, tol, pos)."""
    parts = [lookup_ref(f1[b:b + 1], [t[b:b + 1] for t in f2_levels], coords[b:b + 1], None, grads=False)["y"]
             for b in range(f1.shape[0])]
    ref, mag, pos = (torch.cat([p[k] for p in parts]) for k in (0, 1, 3))
    return ref, mag, ulp_tol(parts[0][2]), pos


def tc_floor(s):
    """Everything of the tensor-core bound but its C_A term."""
    return C_E * U * s.gabs * (1 + 2.0 ** -20) + split_bound(s.ref) + s.pos


def unit_mask(flags, B, H, W):
    """[tiles * 4] int flags (tile-major, 4 levels) -> bool [B, 324, H, W]: the outputs of flagged units."""
    tx, ty = -(-W // TX), -(-H // TY)
    f = flags.reshape(B, ty, tx, LEVELS).bool()
    f = f.repeat_interleave(TY, 1).repeat_interleave(TX, 2)[:, :H, :W]           # [B, H, W, 4]
    return f.permute(0, 3, 1, 2).repeat_interleave(NS * NS, 1)


def judge_lookup(what, got, flags, s, x, log=print):
    """A lookup output [B, 324, H, W] (reference channel order) against the model: units not flagged by the tensor-core bound
    against s = lookup_split_ref of the halves, flagged units by the fp32 bound against x = exact_ref of the fp32 operands.
    Raises Mismatch naming the worst element.  Returns (worst err/bound of the tensor-core units, of the flagged units)."""
    B, _, H, W = got.shape
    got = got.to(s.ref.device).double()
    fb = unit_mask(flags.to(s.ref.device), B, H, W)
    xref, xmag, xtol, xpos = x
    tc = compare_mag(f"{what} [tensor cores]", torch.where(fb, s.ref, got), s.ref, s.mag_a, C_A * STEPS * U, tc_floor(s),
                     log=log)
    ex = compare_mag(f"{what} [exact units]", torch.where(fb, got, xref), xref, xmag, xtol, xpos + split_bound(xref),
                     log=log) if bool(fb.any()) else 0.0
    return tc, ex


def level_report(got, flags, s):
    """Per level, over the tensor-core units: (worst err / bound, the C_A they need), the latter like the convolution model's
    a_ratio: (|got - ref| - tc_floor)^+ / (16 * 2^-24 * mag_a)."""
    B, _, H, W = got.shape
    got = got.to(s.ref.device).double()
    tc = ~unit_mask(flags.to(s.ref.device), B, H, W)
    err = (got - s.ref).abs()
    fl = tc_floor(s)
    bound = C_A * STEPS * U * s.mag_a + fl
    ratio = torch.where(tc & (err > 0), err / bound, torch.zeros_like(err))
    over = (err - fl).clamp_min(0)
    need = torch.where(tc & (over > 0), over / (STEPS * U * s.mag_a).clamp_min(1e-300), torch.zeros_like(err))
    return [(float(ratio[:, l * 81:(l + 1) * 81].max()), float(need[:, l * 81:(l + 1) * 81].max())) for l in range(LEVELS)]


# ----------------------------------------------------------------------------------------------------------- host restatements
def pyramid_levels(f2_pyr, B, H, W):
    """The engine's flat pyramid (level l: [B][H>>l][W>>l][D] channel-last, levels back to back) -> NCHW views per level."""
    out, off = [], 0
    for l in range(LEVELS):
        Hl, Wl = H >> l, W >> l
        n = B * Hl * Wl * D
        out.append(f2_pyr.reshape(-1)[off:off + n].view(B, Hl, Wl, D).permute(0, 3, 1, 2))
        off += n
    return out


class Records(NamedTuple):
    bx0: torch.Tensor          # [ntiles, 4] union box origin (0 when no window is live)
    by0: torch.Tensor
    nrows: torch.Tensor        # box rows loaded: even, <= box_h, 0 when no window is live
    ov: torch.Tensor           # the union box does not fit: the unit is flagged and recomputed exactly
    uw: torch.Tensor           # union box width and height in level positions (0 when no window is live)
    uh: torch.Tensor
    ix0: torch.Tensor          # [ntiles, 4, 128] window origins of the tile's pixels
    iy0: torch.Tensor
    live: torch.Tensor         # [ntiles, 4, 128] pixel inside the frame with a window not fully outside the level image
    valid: torch.Tensor        # [ntiles, 128] pixel inside the frame


def unit_records(coords, H, W):
    """The producer's per-(tile, level) record (make_rec with window_origin and clamp_coord), for coords [B, 2, H, W] fp32.
    Tile t = b * tiles_per_image + ty * tiles_x + tx, pixel ml = 16 * row + column of the 8x16 tile."""
    B = coords.shape[0]
    tyn, txn = -(-H // TY), -(-W // TX)
    c = coords.detach().cpu().float().clamp(-COORD_CLAMP, COORD_CLAMP)
    pad = (0, txn * TX - W, 0, tyn * TY - H)
    c = F.pad(c, pad)
    valid = F.pad(torch.ones(B, 1, H, W, dtype=torch.bool), pad)
    tiles = lambda t: t.view(B, t.shape[1], tyn, TY, txn, TX).permute(0, 2, 4, 1, 3, 5).reshape(B * tyn * txn, t.shape[1], 128)  # noqa: E731
    c, valid = tiles(c), tiles(valid)[:, 0]
    fields = {k: [] for k in Records._fields if k != "valid"}
    big = 1 << 40
    for l in range(LEVELS):
        Hl, Wl = H >> l, W >> l
        ix0 = torch.floor(c[:, 0] * (1.0 / (1 << l))).long() - RADIUS
        iy0 = torch.floor(c[:, 1] * (1.0 / (1 << l))).long() - RADIUS
        live = valid & ~((ix0 + NG - 1 < 0) | (ix0 > Wl - 1) | (iy0 + NG - 1 < 0) | (iy0 > Hl - 1))
        lx0 = torch.where(live, ix0, big).amin(1)
        ly0 = torch.where(live, iy0, big).amin(1)
        lx1 = torch.where(live, ix0 + NG - 1, -big).amax(1)
        ly1 = torch.where(live, iy0 + NG - 1, -big).amax(1)
        anyl = live.any(1)
        zero = torch.zeros_like(lx0)
        fields["ov"].append(anyl & ((lx1 - lx0 + 1 > box_w(l)) | (ly1 - ly0 + 1 > box_h(l))))
        fields["uw"].append(torch.where(anyl, lx1 - lx0 + 1, zero))
        fields["uh"].append(torch.where(anyl, ly1 - ly0 + 1, zero))
        fields["bx0"].append(torch.where(anyl, lx0, zero))
        fields["by0"].append(torch.where(anyl, ly0, zero))
        fields["nrows"].append(torch.where(anyl, ((ly1 - ly0 + 2) & ~1).clamp_max(box_h(l)), zero))
        fields["ix0"].append(ix0)
        fields["iy0"].append(iy0)
        fields["live"].append(live)
    return Records(valid=valid, **{k: torch.stack(v, 1) for k, v in fields.items()})


def chunks(l, nrows):
    """The chunks of a unit that runs on the tensor cores: [(rows, N = rows * box_w, TMA box kind)]."""
    cr, out, c = chunk_rows(l), [], 0
    while c * cr < nrows:
        rows = min(cr, nrows - c * cr)
        out.append((rows, rows * box_w(l), rows // 2 - 1))
        c += 1
    return out


def grid_size(ntiles, sms):
    """rnc_corr_lookup_umma_fwd's persistent grid: one CTA per SM, fewer when there are fewer units."""
    return min(ntiles * LEVELS, sms)


def unit_at(k, cta, G, ntiles, mode=2):
    """unit_at() of the kernel: the k-th unit of CTA cta as (tile-major, level, tile), or None."""
    full = 0 if mode == 0 else -(-ntiles // G) if mode == 1 else ntiles // G
    if k < full * LEVELS:
        tile = (k // LEVELS) * G + cta
        return (True, k % LEVELS, tile) if tile < ntiles else None
    if mode == 1:
        return None
    kk, done = k - full * LEVELS, full * G
    rem = ntiles - done
    g = kk * G + (G - 1 - cta if kk & 1 else cta)
    if g >= rem * LEVELS:
        return None
    l = g // rem
    return False, l, done + g - l * rem


def unit_rounds(ntiles, G, mode=2):
    if mode == 1:
        return -(-ntiles // G) * LEVELS
    full = 0 if mode == 0 else ntiles // G
    return full * LEVELS + -(-((ntiles - full * G) * LEVELS) // G)


def unit_schedule(ntiles, sms, mode=2):
    """Every unit's (CTA, round, tile-major) under the kernel's schedule: dict (tile, level) -> (cta, k, tm).  Asserts that
    every unit runs exactly once."""
    G = grid_size(ntiles, sms)
    out = {}
    for cta in range(G):
        for k in range(unit_rounds(ntiles, G, mode)):
            u = unit_at(k, cta, G, ntiles, mode)
            if u is not None:
                tm, l, tile = u
                assert (tile, l) not in out, f"unit (tile {tile}, level {l}) scheduled twice"
                out[(tile, l)] = (cta, k, tm)
    assert len(out) == ntiles * LEVELS, f"{ntiles * LEVELS - len(out)} units never scheduled"
    return out


def coverage(B, H, W, coords, sms):
    """The kernel paths a launch reaches, as a set of class tuples (see test_coverage_guard)."""
    rec = unit_records(coords, H, W)
    ntiles = rec.ov.shape[0]
    sched = unit_schedule(ntiles, sms)
    seen = set()
    for (tile, l), (_, _, tm) in sched.items():
        ov, nrows = bool(rec.ov[tile, l]), int(rec.nrows[tile, l])
        skip = ov or nrows == 0
        seen.add(("tile-major" if tm else "level-major",))
        if ov:
            seen.add(("overflow", l))
        if nrows == 0:
            seen.add(("no rows", l))
        if tm and skip:
            seen.add(("tile-major skip", l))
        uw, uh = int(rec.uw[tile, l]), int(rec.uh[tile, l])
        if (uw, uh) == (box_w(l), box_h(l)):
            seen.add(("union", l, "box_w x box_h"))
        if (uw, uh) == (box_w(l) + 1, box_h(l)):
            seen.add(("union", l, "box_w + 1 x box_h"))
        if (uw, uh) == (box_w(l), box_h(l) + 1):
            seen.add(("union", l, "box_w x box_h + 1"))
        if not skip:
            seen.add(("union height", l, uh))
            for rows, n, kind in chunks(l, nrows):
                seen.add(("chunk", l, rows))
                seen.add(("N", n))
                seen.add(("box kind", l, kind))
    for l in range(LEVELS):
        Hl, Wl = H >> l, W >> l
        live, ix0, iy0 = rec.live[:, l], rec.ix0[:, l], rec.iy0[:, l]
        for name, m in (("left", ix0 < 0), ("right", ix0 + NG - 1 > Wl - 1), ("top", iy0 < 0),
                        ("bottom", iy0 + NG - 1 > Hl - 1)):
            if bool((live & m).any()):
                seen.add(("partly outside", l, name))
        if bool((rec.valid & ~live).any()):
            seen.add(("fully outside", l))
    if H % TY:
        seen.add(("ragged rows",))
    if W % TX:
        seen.add(("ragged columns",))
    if H >> 3 == 1:
        seen.add(("smallest", "H"))
    if W >> 3 == 1:
        seen.add(("smallest", "W"))
    return seen


def required_coverage():
    req = {("tile-major",), ("level-major",), ("ragged rows",), ("ragged columns",), ("smallest", "H"), ("smallest", "W"),
           ("tile-major skip", 0), ("tile-major skip", LEVELS - 1)}
    for l in range(LEVELS):
        req |= {("overflow", l), ("no rows", l), ("fully outside", l)}
        req |= {("chunk", l, r) for r in range(2, chunk_rows(l) + 1, 2)}
        req |= {("box kind", l, r // 2 - 1) for r in range(2, chunk_rows(l) + 1, 2)}
        req |= {("partly outside", l, side) for side in ("left", "right", "top", "bottom")}
        req |= {("union", l, k) for k in ("box_w x box_h", "box_w + 1 x box_h", "box_w x box_h + 1")}
        req |= {("union height", l, h) for h in range(NG, box_h(l) + 1)}          # tensor-core units: nrows 10 .. box_h
    req |= {("N", n) for n in (32, 48, 64, 96, 128)}
    return req


# ----------------------------------------------------------------------------------------------------------- stimuli (CPU)
def smooth_features(B, H, W, seed, scale=1.5, low=(6, 8)):
    """Bicubic-upsampled Gaussian noise per channel, times scale."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, *low, generator=g)
    return (F.interpolate(x, size=(H, W), mode="bicubic", align_corners=False) * scale).float()


def pyramid(f2, levels=LEVELS):
    """2x2 average pools of the fp32 features, in fp32 (as rnc_fmap_pyramid)."""
    out = [f2.float()]
    for _ in range(levels - 1):
        out.append(F.avg_pool2d(out[-1], 2, stride=2))
    return out


def smooth_coords(B, H, W, amp=2.0, seed=0):
    from oracle import raft_oracle as orc
    yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    flow = torch.stack([amp * torch.sin(yy / 7 + seed) + 0.02 * xx - 0.6, amp * torch.cos(xx / 9 + seed) - 0.03 * yy + 0.4])
    return (orc.coords_grid(B, H, W) + flow[None]).float()


def halves(f1, levels):
    return f1.half(), [t.half() for t in levels]


# ----------------------------------------------------------------------------------------------------------- CPU tests
def test_resident_order_matches_the_engine():
    from rnc.engine_umma import CORR_LS, corr_resident_index
    assert CORR_LS == LVL_STRIDE
    assert torch.equal(resident_index(), corr_resident_index())


def test_model_equals_lookup_ref_on_unrounded_operands():
    """lookup_split_ref on fp64 operands is the oracle-based lookup_ref (corr.py's bilinear sampling of the volume), its
    magnitude and position allowance included, with windows across every border, fully outside, and at +-1e6."""
    B, H, W = 2, 13, 19
    g = torch.Generator().manual_seed(1)
    f1 = torch.randn(B, D, H, W, generator=g)
    lv = pyramid(torch.randn(B, D, H, W, generator=g))
    co = smooth_coords(B, H, W, amp=6.0) + torch.randn(B, 2, H, W, generator=g) * 2
    co[0, :, 0, :4] = torch.tensor([[-0.25, -0.75, 3.0, -1e6], [2.0, -0.5, -0.125, 1e6]])
    co[1, :, 3, 3] = torch.tensor([1e9, -1e9])
    s = lookup_split_ref(f1.double(), [t.double() for t in lv], co)
    r = lookup_ref(f1, lv, co.clamp(-1e6, 1e6), None, grads=False)["y"]
    for name, a, b in (("ref", s.ref, r[0]), ("mag", s.mag, r[1]), ("pos", s.pos, r[3])):
        assert torch.allclose(a, b, rtol=1e-12, atol=1e-12), name
    assert float(s.pos.max()) > 0 and (s.gabs <= s.mag * (1 + 1e-12)).all() and (s.mag <= s.mag_a).all()


def test_rounding_part_holds_on_subnormal_halves_and_large_operands():
    """|lookup of the fp32 operands - lookup_split_ref of their halves| <= R, with operands from fp16 subnormals (2^-26 ..
    2^-14) to 6e4, random signs; R is not vacuous (within 2^10 of the worst error)."""
    B, H, W = 1, 16, 24
    g = torch.Generator().manual_seed(2)
    e1 = torch.linspace(-26, 15.8, D).view(1, D, 1, 1)
    e2 = torch.linspace(-26, 15.8, W).view(1, 1, 1, W)
    sgn = lambda: torch.where(torch.rand(B, D, H, W, generator=g) < 0.5, -1.0, 1.0)      # noqa: E731
    f1 = (2.0 ** e1 * (0.75 + 0.5 * torch.rand(B, D, H, W, generator=g)) * sgn()).clamp(-6e4, 6e4).float()
    f2 = (2.0 ** e2 * (0.75 + 0.5 * torch.rand(B, D, H, W, generator=g)) * sgn()).clamp(-6e4, 6e4).float()
    f1[0, -1, :2, :2], f2[0, :2, 0, -1] = 6e4, -6e4
    lv = pyramid(f2)
    assert float(f1.abs().max()) == 6e4 and float(f2.abs().max()) == 6e4
    h1, h2 = halves(f1, lv)
    assert bool(((h1 != 0) & (h1.abs() < SUB)).any()) and bool(((h2[0] != 0) & (h2[0].abs() < SUB)).any())
    co = smooth_coords(B, H, W, amp=3.0)
    s = lookup_split_ref(h1, h2, co)
    x = lookup_split_ref(f1.double(), [t.double() for t in lv], co)
    R = rounding_bound(f1, lv, co)
    err = (x.ref - s.ref).abs()
    ratio = float(torch.where(err == 0, torch.zeros_like(err), err / R).max())
    print(f"rounding part: worst |exact - split| / R {ratio:.3e}, max err {float(err.max()):.2e}")
    assert ratio <= 1.0 and ratio > 2.0 ** -10


def emulate(s):
    """The kernel's output if it computed lookup_split_ref exactly: fp32, then split into hi + lo."""
    hi, lo = split_emulate(s.ref.float())
    return hi.double() + lo.double()


def flat_bound(f1, f2):
    """The single per-launch tolerance the lookup was held to before this model: 6 * 16 * max|f1| max|f2| 2^-11 / 64."""
    return 6.0 * 16 * float(f1.abs().max()) * float(f2.abs().max()) * 2.0 ** -11 / 64


@pytest.fixture(scope="module")
def smooth_case():
    B, H, W = 1, 47, 64
    f1, f2 = smooth_features(B, H, W, 11), smooth_features(B, H, W, 12)
    lv = pyramid(f2)
    co = smooth_coords(B, H, W)
    h1, h2 = halves(f1, lv)
    s = lookup_split_ref(h1, h2, co)
    x = exact_ref(f1, lv, co)
    flags = torch.zeros(-(-H // TY) * -(-W // TX) * LEVELS, dtype=torch.int32)
    return f1, f2, lv, co, h1, h2, s, x, flags


def _level(t, l, src):
    out = t.clone()
    out[:, l * 81:(l + 1) * 81] = src[:, l * 81:(l + 1) * 81]
    return out


def test_comparator_rejects_what_the_flat_bound_accepts(smooth_case):
    """Faults applied to the emulated output of smooth 256-channel features at 47x64: each stays within the flat bound
    (against the fp64 lookup of the fp32 operands) and each fails the model."""
    f1, f2, lv, co, h1, h2, s, x, flags = smooth_case
    got = emulate(s)
    judge_lookup("emulated", got, flags, s, x)                 # the fault-free emulation passes
    flat = flat_bound(f1, f2)
    # the fractions rounded to fp16 (level 0); the second row of the y blend dropped (its weight moved to the first) where
    # ay < 1/64 and the window lies inside the level-0 image (at a border the dropped row would be a zero row)
    fl = torch.floor(co)
    frac16 = _level(got, 0, emulate(lookup_split_ref(h1, h2, fl + (co - fl).half().double())))
    ay = co[:, 1:] - fl[:, 1:]
    H, W = co.shape[-2:]
    drop_px = (ay < 1 / 64) & (fl[:, :1] >= 4) & (fl[:, :1] <= W - 6) & (fl[:, 1:] >= 4) & (fl[:, 1:] <= H - 6)
    co_drop = torch.where(torch.cat([torch.zeros_like(drop_px), drop_px], 1), fl, co).double()
    drop = _level(got, 0, emulate(lookup_split_ref(h1, h2, co_drop)))
    assert bool(drop_px.any())
    # a one-lattice shift at level 3, on a nearly uniform fmap2 (1.5 randn per channel + 0.002 x smooth noise), at the taps
    # whose corners lie inside the level-3 image before and after the shift
    B, H, W = co.shape[0], H, W
    f2u = 1.5 * torch.randn(1, D, 1, 1, generator=torch.Generator().manual_seed(3)) + 0.002 * f2
    lvu = pyramid(f2u)
    _, lvuh = halves(f1, lvu)
    su, xu = lookup_split_ref(h1, lvuh, co), exact_ref(f1, lvu, co)
    inner = lambda o: (o[:, :-1, :-1] & o[:, 1:, :-1] & o[:, :-1, 1:] & o[:, 1:, 1:]).reshape(-1, 81)     # noqa: E731
    Hl, Wl = lvu[3].shape[-2:]
    m = (inner(_level_geometry(co[0], 3, Hl, Wl)[1]) & inner(_level_geometry(co[0] + 8.0, 3, Hl, Wl)[1])).t().view(1, 81, H, W)
    gotu = emulate(su)
    shifted = emulate(lookup_split_ref(h1, lvuh, co + 8.0))
    shift = gotu.clone()
    shift[:, 243:] = torch.where(m, shifted[:, 243:], gotu[:, 243:])
    assert int(m.sum()) > 1000
    flat_u = flat_bound(f1, f2u)
    for name, bad, sr, xr, fb in (("fractions rounded to fp16", frac16, s, x, flat),
                                  ("y row dropped where ay < 1/64", drop, s, x, flat),
                                  ("one-lattice shift at level 3", shift, su, xu, flat_u)):
        err = float((bad - xr[0]).abs().max())
        assert err <= fb, f"{name}: the flat bound rejects it already ({err:.2e} > {fb:.2e})"
        with pytest.raises(Mismatch) as e:
            judge_lookup(name, bad, flags, sr, xr)
        print(f"{name}: accepted by the flat bound (max err {err:.2e} <= {fb:.2e}), rejected by the model: {e.value}")


def test_comparator_rejects_a_fallback_unit_computed_from_halves(smooth_case):
    """A flagged unit whose outputs are the lookup of the halves (what a fallback that read f1h / f2h would write): within
    the flat bound, outside the fp32 bound of the flagged units."""
    f1, f2, lv, co, h1, h2, s, x, flags = smooth_case
    got = emulate(s)
    fl = flags.clone().view(-1, LEVELS)
    fl[5, 0] = fl[9, 2] = 1                             # two units now belong to the exact path
    with pytest.raises(Mismatch, match="exact units") as e:
        judge_lookup("fallback from halves", got, fl.view(-1), s, x)
    err = float((got - x[0]).abs().max())
    assert err <= flat_bound(f1, f2)
    print(f"fallback from halves: accepted by the flat bound (max err {err:.2e} <= {flat_bound(f1, f2):.2e}), rejected by "
          f"the model: {e.value}")
    # the same units with the exact values pass
    ok = torch.where(unit_mask(fl.view(-1), *got.shape[:1], *got.shape[2:]), emulate(s._replace(ref=x[0])), got)
    judge_lookup("fallback exact", ok, fl.view(-1), s, x)


@pytest.mark.parametrize("bad", [math.nan, math.inf, -math.inf])
@pytest.mark.parametrize("flagged", [False, True])
def test_comparator_rejects_non_finite(smooth_case, bad, flagged):
    f1, f2, lv, co, h1, h2, s, x, flags = smooth_case
    fl = flags.clone().view(-1, LEVELS)
    fl[0, 1] = int(flagged)                               # tile 0 (pixels y < 8, x < 16), level 1
    got = torch.where(unit_mask(fl.view(-1), 1, 47, 64), x[0], emulate(s))
    got[0, 81 + 40, 3, 5] = bad
    with pytest.raises(Mismatch, match=r"image 0, pixel \(y=3, x=5\), channel 121"):
        judge_lookup("non-finite", got, fl.view(-1), s, x)


def test_schedule_runs_every_unit_once():
    """unit_schedule asserts it: hybrid order over tile counts below, at and above the grid, for two SM counts; the tile-major
    rounds are the complete rounds of tiles."""
    for sms in (132, 114):
        for ntiles in (1, 4, 24, 33, 56, sms, sms + 1, 2 * sms - 1, 448):
            sch = unit_schedule(ntiles, sms)
            G = grid_size(ntiles, sms)
            tm_tiles = {t for (t, l), (_, _, tm) in sch.items() if tm}
            assert tm_tiles == set(range((ntiles // G) * G))
            # the four levels of a tile-major tile run back to back on one CTA
            for t in tm_tiles:
                ks = [sch[(t, l)] for l in range(LEVELS)]
                assert len({c for c, _, _ in ks}) == 1 and [k for _, k, _ in ks] == list(range(ks[0][1], ks[0][1] + 4))


def test_records_on_hand_made_tiles():
    """unit_records on tiles whose union boxes are known: one window, an exact level-0 box, one column more, frame pixels of
    a ragged tile, the +-1e6 clamp."""
    from oracle import raft_oracle as orc
    H, W = 12, 40                                         # tiles 2 x 3, the last column and row ragged
    co = orc.coords_grid(1, H, W).float()
    co[:, :, :8, :16] = torch.tensor([20.5, 5.5]).view(1, 2, 1, 1)          # tile 0: one window at (20, 5)
    xs = torch.arange(16).float()
    co[:, 0, :8, 16:32] = 2.0 + torch.floor(xs * 22 / 15)                    # tile 1: x origins 2 .. 24: width 32
    co[:, 1, :8, 16:32] = 3.0
    co[:, 0, :8, 32:40] = 1e9                                                # tile 2: clamped to 1e6, fully outside
    rec = unit_records(co, H, W)
    assert rec.bx0[0, 0] == 16 and rec.by0[0, 0] == 1 and rec.nrows[0, 0] == 10 and not rec.ov[0, 0]
    assert rec.bx0[0, 1] == 6 and rec.by0[0, 1] == -2 and rec.nrows[0, 1] == 10
    assert rec.bx0[1, 0] == -2 and rec.nrows[1, 0] == 10 and not rec.ov[1, 0]
    assert chunks(0, 10) == [(4, 128, 1), (4, 128, 1), (2, 64, 0)]
    co[:, 0, 0, 31] += 1.0                                                    # one column more than the level-0 box
    assert unit_records(co, H, W).ov[1].tolist() == [True, False, False, False]
    assert rec.nrows[2].tolist() == [0, 0, 0, 0] and int(rec.valid[2].sum()) == 8 * 8
    assert int(rec.valid[5].sum()) == 4 * 8                                  # the corner tile: 4 rows x 8 columns in frame


def test_coverage_guard():
    """The GPU cases of tests/test_gpu_lookup_error_model.py, on the host restatement with 132 SMs, reach every kernel path
    listed in required_coverage(): every (level, chunk rows) pair (so all five N and every box kind a level uses), at each
    level a union of exactly box_w x box_h, one column and one row larger, and every union height from one window (10) to
    box_h on a tensor-core unit (so nrows == box_h: every chunk full), overflow and empty units at each level, tile-major and level-major units, skipped units in tile-major rounds at levels 0 and 3,
    windows partly outside each border and fully outside at each level, ragged tiles and the smallest images."""
    from test_gpu_lookup_error_model import CASES
    seen = set()
    for case in CASES:
        seen |= coverage(case.B, case.H, case.W, case.coords(), 132)
    missing = required_coverage() - seen
    assert not missing, f"no GPU case reaches {sorted(missing)}"
