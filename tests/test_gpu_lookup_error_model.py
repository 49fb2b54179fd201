"""The tensor-core correlation lookup (rnc_corr_lookup_umma_fwd through UmmaEngine.lookup_resident) held to the fp64 model of
its arithmetic in tests/test_lookup_error_model.py.  Every case fills the output planes with NaN (an unwritten tap fails as
non-finite), launches the lookup, and checks: the halves the kernel reads are .half() of the fp32 features bit for bit; the
fallback flags equal the host restatement of the producer's records; the pad channels are zero; every tensor-core unit is
within the model's bound of lookup_split_ref and within R more of the fp64 lookup of the fp32 operands; every flagged unit
within the fp32 bound.  The references are evaluated in fp64 on the device, one image at a time.

Families: feature magnitudes (2^-20 .. 2^15 with subnormal halves, all-positive / cancelling / random signs, smooth and white
features), geometry (union boxes of exactly box_w x box_h and one column or row larger at each level, union heights 10 ..
box_h, sample positions at integers, in (-1, 0) and beyond +-1e6, the smallest images), and schedule (B = 8 at 55x128:
tile-major rounds with skipped units plus a level-major remainder; 4 tiles: fewer units than SMs).  test_coverage_guard of the
CPU file checks that these cases reach every kernel path it lists."""
import math
from typing import Callable, NamedTuple

import pytest
import torch

from test_conv_error_model import C_A, split_bound
from test_lookup_error_model import (D, LEVELS, TX, TY, box_h, box_w, exact_ref, judge_lookup, level_report, lookup_split_ref,
                                     pyramid_levels, rounding_bound, smooth_coords, smooth_features, tc_floor, unit_records,
                                     unit_schedule)
from test_train_shapes import compare_mag

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# ----------------------------------------------------------------------------------------------------------- stimuli
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def white(B, H, W, seed, scale=1.5):
    g = _gen(seed)
    return torch.randn(B, D, H, W, generator=g) * scale, torch.randn(B, D, H, W, generator=g) * scale


def smooth(B, H, W, seed):
    return smooth_features(B, H, W, seed), smooth_features(B, H, W, seed + 1)


def _signed(g, shape, scale):
    mag = scale * (0.75 + 0.5 * torch.rand(shape, generator=g))
    return mag * torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)


def sweep(B, H, W, seed):
    """fmap1 channels log-spaced over 2^-20 .. 2^15, fmap2 columns log-spaced over 2^-20 .. 2^0 (products 2^-40 .. 2^15,
    subnormal halves below 2^-14), random signs.  fmap2 stays below 1 so that the lookup stays inside the hi/lo output's
    range (|out| <= 65504; beyond 131008 both halves saturate and split_bound takes the whole value)."""
    g = _gen(seed)
    f1 = _signed(g, (B, D, H, W), 2.0 ** torch.linspace(-20, 15, D).view(1, D, 1, 1))
    f2 = _signed(g, (B, D, H, W), 2.0 ** torch.linspace(-20, 0, W).view(1, 1, 1, W))
    return f1, f2


def uniform(B, H, W, seed, log2, log2_f2=None):
    g = _gen(seed)
    return _signed(g, (B, D, H, W), 2.0 ** log2), _signed(g, (B, D, H, W), 2.0 ** (log2 if log2_f2 is None else log2_f2))


def signs(B, H, W, seed, kind):
    """"positive": |randn| + 0.1 (every product positive: the worst alignment error); "random": randn; "cancelling":
    positive fmap1 whose second half of channels repeats the first, fmap2 whose second half is minus the first times
    (1 - 1e-3 eps): every dot product cancels to ~1e-3 of its magnitude."""
    g = _gen(seed)
    f1, f2 = torch.randn(B, D, H, W, generator=g), torch.randn(B, D, H, W, generator=g)
    if kind == "random":
        return f1, f2
    f1, f2 = f1.abs() + 0.1, f2.abs() + 0.1
    if kind == "cancelling":
        h = D // 2
        f1[:, h:] = f1[:, :h]
        f2[:, h:] = -f2[:, :h] * (1 - 1e-3 * (2 * torch.rand(B, h, H, W, generator=g) - 1))
    return f1, f2


def tile_coords(B, H, W, spec):
    """Coordinates whose tiles have chosen union boxes: spec(b, tile row, tile column) -> None (identity grid) or
    (level L, Sx, Sy): the tile's level-L window origins span exactly Sx columns and Sy rows, so that its union box is
    Sx + 10 by Sy + 10.  The windows are placed near the tile but shifted where needed so that every one of them overlaps
    the level image (the producer counts only those, so a window fully outside would cut the union): level positions
    -5 .. Wl + 3 (window origins -9 .. Wl - 1).  H, W multiples of the tile."""
    from oracle import raft_oracle as orc
    co = orc.coords_grid(B, H, W)
    px = torch.arange(TX).float()
    py = torch.arange(TY).float()
    for b in range(B):
        for r in range(H // TY):
            for c in range(W // TX):
                s = spec(b, r, c)
                if s is None:
                    continue
                L, sx, sy = s
                Hl, Wl = H >> L, W >> L
                assert sx <= Wl + 8 and sy <= Hl + 8, f"a {sx + 10} x {sy + 10} union does not fit a {Wl} x {Hl} level image"
                xb = min(max((c * TX + TX // 2) // 2 ** L - sx // 2, -5), Wl + 3 - sx)
                yb = min(max((r * TY + TY // 2) // 2 ** L - sy // 2, -5), Hl + 3 - sy)
                co[b, 0, r * TY:(r + 1) * TY, c * TX:(c + 1) * TX] = (2 ** L * (xb + torch.floor(px * sx / (TX - 1)) + 0.5))[None]
                co[b, 1, r * TY:(r + 1) * TY, c * TX:(c + 1) * TX] = (2 ** L * (yb + torch.floor(py * sy / (TY - 1)) + 0.5))[:, None]
    return co.float()


def exact_boxes(B, H, W):
    """Per tile: target level L = t % 4 with a union of exactly box_w x box_h, one column more, or one row more (the last
    two overflow at L)."""
    def spec(b, r, c):
        t = r * (W // TX) + c
        L, v = t % LEVELS, (t // LEVELS) % 3
        return L, box_w(L) - 10 + (v == 1), box_h(L) - 10 + (v == 2)
    return tile_coords(B, H, W, spec)


def union_heights(B, H, W):
    """Per tile: target level t % 4, union height 10 + (t // 4) % 15: every height from one window to box_h at each level."""
    def spec(b, r, c):
        t = r * (W // TX) + c
        return t % LEVELS, t % 3, (t // LEVELS) % 15
    return tile_coords(B, H, W, spec)


def positions(B, H, W):
    """Image 0: integer coordinates; its tile 0 at x and y in (-1, 0) at some level (-0.3, -0.7, -1.3, -2.5, -6: level
    fractions in (-1, 0) at levels 0 .. 3); tiles at +-1e6 and +-1e9 (clamped); the others smooth.  Image 1: a smooth flow
    of amplitude 6 (windows across every border) with a tile 20 px beyond the left border."""
    co = smooth_coords(B, H, W, amp=6.0, seed=1)
    co[0] = torch.round(co[0])
    vals = torch.tensor([-0.3, -0.7, -1.3, -2.5, -6.0, -0.05, -1e-7, 0.0])
    n = TY * TX
    co[0, 0, :TY, :TX] = vals[torch.arange(n) % 8].view(TY, TX)
    co[0, 1, :TY, :TX] = vals[(torch.arange(n) // 8) % 8].view(TY, TX)
    co[0, :, :TY, TX:2 * TX] = torch.tensor([1e6, -1e6]).view(2, 1, 1)
    co[0, :, TY:2 * TY, :TX] = torch.tensor([-1e9, 1e9]).view(2, 1, 1)
    co[0, 0, 2 * TY:3 * TY, TX:2 * TX] = 1.5e6
    if B > 1:
        co[1, 0, TY:2 * TY, :TX] = -20.0
    return co.float()


def schedule_b8(B, H, W):
    """55x128 with B = 8: 448 tiles, 3 tile-major rounds on 132 SMs (tiles 0 .. 395) and 52 tiles' units level-major.  A
    smooth flow with the motion boundary of rnc.synth in images 1 .. 7, and in image 0 (tile-major) and image 7 (tiles
    >= 4: level-major): a tile beyond the right border (levels 0 and 1 without rows, 2 and 3 live), a tile at 1e6 (no
    rows at any level), a tile split between both borders (every level overflows), a tile spread over 30 px (levels 0 .. 2
    overflow, level 3 fits)."""
    from rnc.synth import motion_boundary_flow_init
    co = smooth_coords(B, H, W, amp=3.0, seed=2)
    co[1:] += motion_boundary_flow_init(B - 1, H, W)
    xs = torch.arange(TX).float()
    for b, (r, c) in ((0, (0, 0)), (7, (2, 2))):
        sl = lambda dr, dc: (slice((r + dr) * TY, (r + dr + 1) * TY), slice((c + dc) * TX, (c + dc + 1) * TX))  # noqa: E731
        y, x = sl(0, 0)
        co[b, 0, y, x] = W + 12.0
        y, x = sl(0, 1)
        co[b, :, y, x] = 1e6
        y, x = sl(1, 0)
        co[b, 0, y, x] = torch.where(xs < 8, 0.0, W - 1.0)[None]
        y, x = sl(1, 1)
        co[b, 0, y, x] = (x.start + 2.0 * xs)[None]
    return co.float()


class Case(NamedTuple):
    name: str
    family: str
    B: int
    H: int
    W: int
    feats: Callable            # () -> (fmap1, fmap2) fp32 [B, 256, H, W]
    coords: Callable           # () -> [B, 2, H, W] fp32


def _case(name, family, B, H, W, feats, coords=None):
    return Case(name, family, B, H, W, lambda: feats(B, H, W), coords and (lambda: coords(B, H, W)) or
                (lambda: smooth_coords(B, H, W)))


CASES = [
    _case("sweep 2^-20..2^15", "magnitude", 1, 24, 40, lambda B, H, W: sweep(B, H, W, 1)),
    _case("fmap1 2^-20 (subnormal halves), fmap2 2^10", "magnitude", 1, 16, 48, lambda B, H, W: uniform(B, H, W, 2, -20, 10)),
    _case("fmap1 2^10, fmap2 2^-20 (subnormal halves)", "magnitude", 1, 16, 48, lambda B, H, W: uniform(B, H, W, 17, 10, -20)),
    _case("fmap1 2^-12, fmap2 2^6", "magnitude", 1, 16, 48, lambda B, H, W: uniform(B, H, W, 3, -12, 6)),
    _case("fmap1 2^15, fmap2 2^-4", "magnitude", 1, 16, 48, lambda B, H, W: uniform(B, H, W, 4, 15, -4)),
    _case("positive", "signs", 1, 32, 48, lambda B, H, W: signs(B, H, W, 5, "positive")),
    _case("cancelling", "signs", 1, 32, 48, lambda B, H, W: signs(B, H, W, 6, "cancelling")),
    _case("random", "signs", 1, 32, 48, lambda B, H, W: signs(B, H, W, 7, "random")),
    _case("smooth x1.5 47x64", "smooth/white", 1, 47, 64, lambda B, H, W: smooth(B, H, W, 8)),
    _case("white x1.5 55x128", "smooth/white", 1, 55, 128, lambda B, H, W: white(B, H, W, 9)),
    _case("exact boxes, +1 column, +1 row", "geometry", 1, 64, 128, lambda B, H, W: white(B, H, W, 10), exact_boxes),
    _case("union heights 10..24", "geometry", 1, 64, 128, lambda B, H, W: white(B, H, W, 11), union_heights),
    _case("positions: integers, (-1, 0), +-1e6", "geometry", 2, 40, 56, lambda B, H, W: white(B, H, W, 12), positions),
    _case("smallest 8x8", "geometry", 2, 8, 8, lambda B, H, W: white(B, H, W, 13)),
    _case("smallest 15x150", "geometry", 1, 15, 150, lambda B, H, W: white(B, H, W, 14)),
    _case("B=8 55x128", "schedule", 8, 55, 128, lambda B, H, W: white(B, H, W, 15), schedule_b8),
    _case("4 tiles", "schedule", 1, 16, 32, lambda B, H, W: white(B, H, W, 16)),
]


# ----------------------------------------------------------------------------------------------------------- the launch
@pytest.fixture(scope="module")
def ueng():
    from rnc.engine_umma import UmmaEngine
    eng = UmmaEngine()
    assert eng.lookup_mode == "umma"
    return eng


@pytest.fixture(scope="module")
def report():
    rows = []
    yield rows
    print(f"\n  tensor-core lookup vs its model on {torch.cuda.get_device_name(0)}: worst err/bound and the C_A needed "
          f"(C_A = {C_A}) per level, over the tensor-core units")
    print(f"  {'family':<13s} {'case':<38s} " + " ".join(f"{'L' + str(l) + ' err/bd  C_A':>17s}" for l in range(LEVELS))
          + "  flagged  exact err/bd")
    for fam, name, lv, nf, nu, ex in rows:
        print(f"  {fam:<13s} {name:<38s} " + " ".join(f"{r:8.3f} {c:8.3f}" for r, c in lv) + f"  {nf:4d}/{nu:<4d} {ex:8.3f}")
    by = {}
    for fam, _, lv, *_ in rows:
        by.setdefault(fam, []).append(max(c for _, c in lv))
    print("  C_A needed per family: " + ", ".join(f"{f} {max(v):.3f}" for f, v in by.items()))


def lookup_launch(eng, f1, f2, coords):
    """fmap_prepare + lookup_resident with both output planes and the flags pre-filled with NaN / 7.  Returns the workspace
    and the output [B, 324, H, W] (hi + lo, reference channel order)."""
    B, _, H, W = f1.shape
    ws = eng.workspace(torch.device(DEV), B, H, W, False, False)
    eng.fmap_prepare(ws, f1.to(DEV).contiguous(), f2.to(DEV).contiguous(), LEVELS)
    ws.coords1.copy_(coords.to(DEV))
    ws.corr.hi.fill_(math.nan)
    ws.corr.lo.fill_(math.nan)
    ws.lookup_flags.fill_(7)
    eng.lookup_resident(ws)
    torch.cuda.synchronize()
    return ws, eng.corr_nchw(ws)


def check_launch(what, ws, got, coords, golden=None, log=print):
    """Every check of one launch against the model (see the module docstring).  golden: an fp32 lookup of the same features
    by the reference ([B, 324, H, W], sampled at the positions themselves); the output must lie within the model's bound of
    the fp64 lookup (R included) plus the fp32 bound of the golden's own distance from it.  Returns (level_report, flags,
    R-check worst, exact-unit worst)."""
    B, H, W = ws.B, ws.H8, ws.W8
    hi, lo = ws.corr.hi.view(-1, LEVELS, 88), ws.corr.lo.view(-1, LEVELS, 88)
    assert (hi[:, :, 81:].view(torch.int16) == 0).all() and (lo[:, :, 81:].view(torch.int16) == 0).all(), \
        f"{what}: pad channels not zero"
    assert torch.equal(ws.f1h, ws.f1_cl.reshape(-1).half()) and torch.equal(ws.f2h, ws.f2_pyr.half()), \
        f"{what}: the halves are not .half() of the fp32 features"
    flags = ws.lookup_flags.cpu()
    want = unit_records(coords, H, W).ov.int().reshape(-1)
    bad = (flags != want).nonzero().view(-1).tolist()
    assert not bad, f"{what}: fallback flags differ from the records at units (tile, level) " \
                    f"{[(u // LEVELS, u % LEVELS) for u in bad[:16]]}: kernel {flags[bad[:16]].tolist()}, host {want[bad[:16]].tolist()}"
    f1 = ws.f1_cl.view(B, H, W, D).permute(0, 3, 1, 2)
    f1h = ws.f1h.view(B, H, W, D).permute(0, 3, 1, 2)
    lv, lvh = pyramid_levels(ws.f2_pyr, B, H, W), pyramid_levels(ws.f2h, B, H, W)
    co = coords.to(DEV)
    s = lookup_split_ref(f1h, lvh, co)
    x = exact_ref(f1, lv, co)
    _, ex = judge_lookup(what, got, flags, s, x, log=log)
    # the tensor-core units against the fp64 lookup of the fp32 operands: the model's bound plus R
    from test_lookup_error_model import STEPS, U, unit_mask
    fb = unit_mask(flags.to(DEV), B, H, W)
    floor = tc_floor(s) + rounding_bound(f1, lv, co)
    wr = compare_mag(f"{what} [tensor cores vs fp32 operands]", torch.where(fb, x[0], got.double()), x[0], s.mag_a,
                     C_A * STEPS * U, floor, log=log)
    if golden is not None:
        xref, xmag, xtol, xpos = x
        fp32 = xtol * xmag + xpos
        bound = torch.where(fb, fp32 + split_bound(xref), C_A * STEPS * U * s.mag_a + floor) + fp32
        compare_mag(f"{what} [vs the reference's output]", got, golden.to(DEV), bound, 1.0, log=log)
    return level_report(got, flags, s), flags, wr, ex


def umma_lookup_model(what, f1, f2, coords, golden=None):
    """One tensor-core lookup of fmap1 / fmap2 [B, 256, H, W] at coords [B, 2, H, W], held to the model by check_launch
    (and to the reference's output golden, when given).  Returns the output [B, 324, H, W] and the fallback flags, on the
    CPU."""
    from rnc.engine_umma import UmmaEngine
    eng = UmmaEngine()
    eng.lookup_mode = "umma"
    co = coords.float()
    ws, got = lookup_launch(eng, f1.float(), f2.float(), co)
    check_launch(what, ws, got, co, golden)
    return got.cpu(), ws.lookup_flags.cpu()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_lookup_against_model(ueng, report, case):
    f1, f2 = case.feats()
    co = case.coords()
    assert float(f1.abs().max()) <= 65504 and float(f2.abs().max()) <= 65504, "the model's precondition"
    ws, got = lookup_launch(ueng, f1, f2, co)
    lv, flags, wr, ex = check_launch(case.name, ws, got, co)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ntiles = flags.numel() // LEVELS
    sched = unit_schedule(ntiles, sms)
    tm = sum(1 for v in sched.values() if v[2])
    print(f"  {case.name}: {int(flags.sum())}/{flags.numel()} units flagged, {tm} tile-major units on {sms} SMs, "
          f"tensor cores vs fp32 operands worst err/bound {wr:.3f}")
    report.append((case.family, case.name, lv, int(flags.sum()), flags.numel(), ex))
