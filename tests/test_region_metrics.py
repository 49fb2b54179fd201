"""Per-region validation metrics on the host: the exact boundary distance transform against scipy and a hand-worked square,
the region partials against an independent numpy restatement of the definitions, summarize_regions on hand-built partials,
validate(regions=True) with stub models (its old keys unchanged, KITTI's fl_all equal to f1, gloo at world sizes 2 and 3
equal to world 1), the argument errors, and the C entry points' declarations, argument checks and register use."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from test_consistency import BidiStub
from test_flow_metrics import ROOT, CSRC, Stub, edge_case, run_ranks, stub_samples

NONE = 2 ** 31 - 1


def scipy_dist2(lab):
    """rint(distance_transform_edt(~boundary)^2) of one bool [H,W] label map; None without a boundary pixel."""
    ndimage = pytest.importorskip("scipy.ndimage")
    H, W = lab.shape
    bnd = np.zeros_like(lab)
    for dy, dx in ((1, 0), (-1, 0), (0, 1), (0, -1)):
        for y in range(H):
            for x in range(W):
                if 0 <= y + dy < H and 0 <= x + dx < W and lab[y + dy, x + dx] != lab[y, x]:
                    bnd[y, x] = True
    if not bnd.any():
        return None
    return np.rint(ndimage.distance_transform_edt(~bnd) ** 2).astype(np.int64)


def check_dist2(occ):
    from rnc.metrics import boundary_dist2
    got = boundary_dist2(occ)
    assert got.dtype == torch.int32 and got.shape == occ.shape
    for b in range(occ.shape[0]):
        want = scipy_dist2((occ[b] >= 0.5).numpy())
        if want is None:
            assert (got[b] == NONE).all()
        else:
            assert np.array_equal(got[b].numpy().astype(np.int64), want), b


@pytest.mark.parametrize("B,H,W,p", [(3, 17, 23, 0.5), (2, 31, 40, 0.03), (1, 64, 48, 0.002), (4, 1, 1, 0.5),
                                     (3, 1, 19, 0.4), (3, 21, 1, 0.4), (2, 9, 13, 0.0)])
def test_host_dist2_equals_scipy(B, H, W, p):
    g = np.random.default_rng(B * 1000 + H * W)
    check_dist2(torch.from_numpy((g.random((B, H, W)) < p).astype(np.float32)))


def test_host_dist2_without_a_boundary_is_the_sentinel():
    from rnc.metrics import DIST2_NONE, boundary_dist2
    assert DIST2_NONE == NONE
    for occ in (torch.ones(2, 5, 7), torch.zeros(1, 5, 7), torch.ones(1, 1, 1), torch.full((1, 3, 4), 0.5)):
        assert (boundary_dist2(occ) == NONE).all()
    mixed = torch.stack([torch.ones(6, 8), torch.zeros(6, 8)])
    mixed[0, 2, 3] = 0                                       # a boundary in image 0 only: image 1 keeps the sentinel
    d = boundary_dist2(mixed)
    assert (d[1] == NONE).all() and d[0, 2, 3] == 0 and d[0, 0, 0] == 8     # to (2, 2)


def test_host_dist2_of_a_hand_drawn_square():
    """A 3x3 occluded square in a 7x7 image: the boundary is the square's 8 outer pixels and the 12 clear pixels that touch
    its sides (not the 4 diagonal corners); the centre is 1 from it, the image corners 5 (1 + 2^2)."""
    from rnc.metrics import boundary_dist2
    occ = torch.zeros(1, 7, 7)
    occ[0, 2:5, 2:5] = 1
    want = [[5, 2, 1, 1, 1, 2, 5],
            [2, 1, 0, 0, 0, 1, 2],
            [1, 0, 0, 0, 0, 0, 1],
            [1, 0, 0, 1, 0, 0, 1],
            [1, 0, 0, 0, 0, 0, 1],
            [2, 1, 0, 0, 0, 1, 2],
            [5, 2, 1, 1, 1, 2, 5]]
    assert boundary_dist2(occ)[0].tolist() == want
    assert boundary_dist2(occ.flip(2))[0].tolist() == want
    # the bin edges: a single boundary pixel at (0, 0) of a 1x200 row puts x in d0-10 up to x = 9, d10-60 from 10
    row = torch.zeros(1, 1, 200)
    row[0, 0, 0] = 1
    d = boundary_dist2(row)[0, 0]
    assert d[:2].tolist() == [0, 0] and d[11].item() == 100 and d[61].item() == 3600 and d[141].item() == 19600


# ----------------------------------------------------------------------------- region partials


def numpy_regions(flow, gt, valid, occ=None, noc=None, fg=None):
    """The region definitions restated in numpy float32, pixel by pixel with explicit masks: per image and per cell (Sintel:
    16*occluded + 4*d + s, KITTI: 2*(not noc) + fg) the counts (valid, epe < 1, < 3, < 5, outliers) and the fp64 EPE sum."""
    f, g = flow.numpy().astype(np.float32), gt.numpy().astype(np.float32)
    d = f - g
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        epe = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1])
        mag = np.sqrt(g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1])
        out = (epe > np.float32(3)) & (epe / mag > np.float32(0.05))
    val = np.ones(epe.shape, bool) if valid is None else valid.numpy() >= 0.5
    B = f.shape[0]
    if occ is not None:
        o = occ.numpy() >= 0.5
        d2 = np.full(epe.shape, np.inf)
        for b in range(B):
            s = scipy_dist2(o[b])
            if s is not None:
                d2[b] = s
        dbin = [d2 < 100, (d2 >= 100) & (d2 < 3600), (d2 >= 3600) & (d2 < 19600), d2 >= 19600]
        sbin = [mag < 10, (mag >= 10) & (mag < 40), mag >= 40, np.isnan(mag)]
        masks = [(o if occl else ~o) & dbin[i] & sbin[j] for occl in (False, True) for i in range(4) for j in range(4)]
    else:
        n = noc.numpy() >= 0.5
        fgm = np.zeros(epe.shape, bool) if fg is None else fg.numpy() >= 0.5
        masks = [(n if inside else ~n) & (fgm if f_ else ~fgm) for inside in (True, False) for f_ in (False, True)]
    counts = np.zeros((B, len(masks), 5), np.int64)
    sums = np.zeros((B, len(masks)))
    for c, m in enumerate(masks):
        m = m & val
        for b in range(B):
            mb, e = m[b], epe[b]
            counts[b, c] = [mb.sum(), (mb & (e < 1)).sum(), (mb & (e < 3)).sum(), (mb & (e < 5)).sum(), (mb & out[b]).sum()]
            sums[b, c] = e[mb].astype(np.float64).sum()
    return counts, sums


def region_batch(B, H, W, seed, speed=20.0):
    g = torch.Generator().manual_seed(seed)
    gt = torch.randn(B, 2, H, W, generator=g) * speed
    flow = gt + torch.randn(B, 2, H, W, generator=g) * 3
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    occ = torch.stack([((yy - H * (0.3 + 0.1 * b)) ** 2 + (xx - W / 2) ** 2 < (H / 4) ** 2).float() for b in range(B)])
    occ = torch.maximum(occ, (torch.rand(B, H, W, generator=g) > 0.995).float())
    valid = (torch.rand(B, H, W, generator=g) > 0.2).float()
    return flow, gt, valid, occ


def assert_partials_equal(p, counts, sums):
    assert p.counts.dtype == torch.int64 and p.epe_sum.dtype == torch.float64
    assert np.array_equal(p.counts.numpy(), counts)
    np.testing.assert_allclose(p.epe_sum.numpy(), sums, rtol=1e-12, atol=0)


@pytest.mark.parametrize("with_valid", [False, True])
def test_host_sintel_partials_equal_numpy(with_valid):
    from rnc.metrics import host_partials, host_region_partials
    flow, gt, valid, occ = region_batch(3, 300, 170, seed=1)
    valid = valid if with_valid else None
    p = host_region_partials(flow, gt, valid, occ=occ)
    assert p.counts.shape == (3, 32, 5)
    counts, sums = numpy_regions(flow, gt, valid, occ=occ)
    assert_partials_equal(p, counts, sums)
    assert (counts[:, [c for c in range(32) if (c >> 2) & 3 == 2], 0] > 0).any()     # the d60-140 bin is populated
    assert (counts[:, [c for c in range(32) if c & 3 == 2], 0] > 0).any()            # and s40+
    assert torch.equal(p.counts.sum(1), host_partials(flow, gt, valid).counts)


def test_host_kitti_partials_equal_numpy():
    from rnc.metrics import host_partials, host_region_partials
    flow, gt, valid, occ = region_batch(2, 40, 90, seed=2)
    noc = (torch.rand(2, 40, 90, generator=torch.Generator().manual_seed(3)) > 0.3).float()
    for fg in (occ, None):
        p = host_region_partials(flow, gt, valid, noc=noc, fg=fg)
        assert p.counts.shape == (2, 4, 5) and p.fg.tolist() == [fg is not None] * 2
        assert_partials_equal(p, *numpy_regions(flow, gt, valid, noc=noc, fg=fg))
        assert torch.equal(p.counts.sum(1), host_partials(flow, gt, valid).counts)


def test_host_partials_at_the_edges():
    """test_flow_metrics.edge_case's thresholds, zero-magnitude ground truth and invalid image, and NaN and inf."""
    from rnc.metrics import host_partials, host_region_partials
    flow, gt, valid = edge_case()
    flow[0, 0, 2, 5] = float("nan")
    gt[0, 1, 3, 0] = float("nan")
    flow[0, 1, 3, 1] = float("inf")
    occ = torch.zeros(2, 4, 6)
    occ[0, :, 3:] = 1
    p = host_region_partials(flow, gt, valid, occ=occ)
    assert_partials_equal(p, *numpy_regions(flow, gt, valid, occ=occ))
    assert torch.equal(p.counts.sum(1), host_partials(flow, gt, valid).counts)
    assert p.counts[0, :, 0].sum() == 23 and p.counts[1].sum() == 0
    assert p.counts[0, [3, 7, 11, 15, 19, 23, 27, 31], 0].sum() == 1                # the NaN magnitude: no speed bin
    k = host_region_partials(flow, gt, valid, noc=1 - occ, fg=occ)
    assert_partials_equal(k, *numpy_regions(flow, gt, valid, noc=1 - occ, fg=occ))


def test_summarize_regions_hand_built():
    from rnc.metrics import RegionPartials, summarize_regions
    counts = torch.zeros(2, 32, 5, dtype=torch.int64)
    sums = torch.zeros(2, 32, dtype=torch.float64)
    counts[0, 0], sums[0, 0] = torch.tensor([4, 1, 2, 3, 0]), 10.0          # matched, d0-10, s0-10
    counts[0, 17], sums[0, 17] = torch.tensor([2, 0, 0, 1, 1]), 9.0         # unmatched, d0-10, s10-40
    counts[1, 6], sums[1, 6] = torch.tensor([6, 0, 0, 0, 6]), 60.0          # matched, d10-60, s40+
    counts[1, 31], sums[1, 31] = torch.tensor([1, 0, 0, 0, 1]), float("nan")  # unmatched, no d-bin, no s-bin
    r = summarize_regions(RegionPartials(counts, sums, torch.zeros(2, dtype=torch.bool)))
    assert list(r) == ["epe_matched", "epe_unmatched", "epe_d0-10", "epe_d10-60", "epe_d60-140", "epe_s0-10", "epe_s10-40",
                       "epe_s40+", "region_pixels"]
    assert r["epe_matched"] == 70.0 / 10 and math.isnan(r["epe_unmatched"])
    assert r["epe_d0-10"] == 19.0 / 6 and r["epe_d10-60"] == 10.0 and math.isnan(r["epe_d60-140"])
    assert r["epe_s0-10"] == 2.5 and r["epe_s10-40"] == 4.5 and r["epe_s40+"] == 10.0
    assert r["region_pixels"] == {"matched": 10, "unmatched": 3, "d0-10": 6, "d10-60": 6, "d60-140": 0, "s0-10": 4,
                                  "s10-40": 2, "s40+": 6}
    kc = torch.zeros(2, 4, 5, dtype=torch.int64)
    kc[0, 0, [0, 4]] = torch.tensor([10, 1])        # noc, background
    kc[0, 3, [0, 4]] = torch.tensor([5, 5])         # occluded, foreground
    kc[1, 2, [0, 4]] = torch.tensor([5, 2])         # occluded, background
    ks = torch.zeros(2, 4, dtype=torch.float64)
    k = summarize_regions(RegionPartials(kc, ks, torch.ones(2, dtype=torch.bool)))
    assert k == {"fl_all": 100 * 8 / 20, "fl_bg": 100 * 3 / 15, "fl_fg": 100.0, "fl_all_noc": 10.0, "fl_bg_noc": 10.0,
                 "fl_fg_noc": k["fl_fg_noc"], "region_pixels": {"all": 20, "bg": 15, "fg": 5, "all_noc": 10, "bg_noc": 10,
                                                                "fg_noc": 0}}
    assert math.isnan(k["fl_fg_noc"])
    part = summarize_regions(RegionPartials(kc, ks, torch.tensor([True, False])))
    assert list(part) == ["fl_all", "fl_all_noc", "region_pixels"] and part["region_pixels"] == {"all": 20, "all_noc": 10}
    with pytest.raises(ValueError, match="cells"):
        summarize_regions(RegionPartials(kc[:, :3], ks[:, :3], torch.ones(2, dtype=torch.bool)))


# ----------------------------------------------------------------------------- validate(regions=True)


def region_samples(sparse, fg_every=True):
    """stub_samples with region masks: Sintel-style an occluded disc plus speckle, KITTI-style noc and fg (one sample
    without fg unless fg_every)."""
    g = torch.Generator().manual_seed(11 + sparse)
    out = []
    for k, s in enumerate(stub_samples(sparse)):
        h, w = s[0].shape[-2:]
        if sparse:
            m = {"noc": (torch.rand(h, w, generator=g) > 0.3).float(), "fg": (torch.rand(h, w, generator=g) > 0.6).float()}
            if not fg_every and k == 6:
                del m["fg"]
        else:
            yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
            m = {"occ": torch.maximum(((yy - k) ** 2 + (xx - 15) ** 2 < 30).float(),
                                      (torch.rand(h, w, generator=g) > 0.97).float())}
        out.append((s[0], s[1], s[2], s[3] if sparse else None, m))
    return out


def same(got, want):
    """Dicts equal bit for bit, NaN equal to NaN."""
    assert got.keys() == want.keys()
    for k in want:
        assert got[k] == want[k] or (isinstance(want[k], float) and math.isnan(want[k]) and math.isnan(got[k])), k
    return True


def host_regions_of(model, samples):
    """summarize_regions of the host region partials of the stub's flows, image by image."""
    from rnc.metrics import cat_regions, host_region_partials, summarize_regions
    parts = []
    for s in samples:
        flow = model(s[0][None], s[1][None])[1]
        masks = {k: v[None] for k, v in s[4].items()}
        parts.append(host_region_partials(flow, s[2][None], None if s[3] is None else s[3][None], **masks))
    return summarize_regions(cat_regions(parts))


@pytest.mark.parametrize("sparse", [False, True])
def test_validate_regions_keeps_the_old_keys_and_equals_the_host(sparse):
    from rnc.harness import validate
    mode = "kitti" if sparse else "sintel"
    samples = region_samples(sparse)
    plain = validate(Stub(), [s[:4] for s in samples], iters=1, mode=mode, batch_size=3, device="cpu")
    want = host_regions_of(Stub(), samples)
    for bs in (1, 3, 8):
        res = validate(Stub(), samples, iters=1, mode=mode, batch_size=bs, device="cpu", regions=True)
        assert {k: res[k] for k in plain} == plain                              # the old keys, bit for bit
        assert same({k: res[k] for k in res if k not in plain}, want)
    if sparse:
        assert res["fl_all"] == res["f1"] and set(res["region_pixels"]) == {"all", "bg", "fg", "all_noc", "bg_noc", "fg_noc"}
        part = validate(Stub(), region_samples(True, fg_every=False), iters=1, mode=mode, device="cpu", regions=True)
        assert "fl_fg" not in part and part["fl_all"] == res["fl_all"] and part["fl_all_noc"] == res["fl_all_noc"]
    else:
        assert all(res["region_pixels"][k] > 0 for k in ("matched", "unmatched", "d0-10", "d10-60", "s0-10", "s10-40"))


def test_validate_regions_with_consistency_scores_the_occlusions():
    from rnc.harness import validate
    from rnc.metrics import host_fb_consistency, summarize_occlusion
    samples = region_samples(False)
    m = BidiStub()
    rows = []
    for s in samples:
        a, b = s[0][None], s[1][None]
        occ_fw = host_fb_consistency(m(a, b)[1], m(b, a)[1])[0][0]
        p, t = occ_fw != 0, s[4]["occ"] >= 0.5
        rows.append([int((p & t).sum()), int(p.sum()), int(t.sum())])
    want = summarize_occlusion(torch.tensor(rows))
    assert 0 < want["occ_precision"] < 1 and 0 < want["occ_recall"] <= 1
    plain = validate(m, [s[:4] for s in samples], iters=1, batch_size=4, device="cpu", consistency=True)
    res = validate(m, samples, iters=1, batch_size=4, device="cpu", consistency=True, regions=True)
    assert {k: res[k] for k in plain} == plain
    assert {k: res[k] for k in ("occ_precision", "occ_recall", "occ_f1")} == want
    assert same({k: res[k] for k in res if k.startswith("epe_") or k == "region_pixels"}, host_regions_of(m, samples))
    kitti = validate(m, region_samples(True), iters=1, batch_size=4, device="cpu", consistency=True, regions=True)
    assert "fl_all" in kitti and not any(k.startswith("occ_") for k in kitti)


def test_validate_regions_argument_errors_name_the_sample():
    from rnc.harness import validate
    sintel, kitti = region_samples(False), region_samples(True)
    with pytest.raises(ValueError, match="sample 2 has 3 items"):
        validate(Stub(), sintel[:2] + [sintel[2][:3]], device="cpu", regions=True)
    with pytest.raises(ValueError, match="sample 1 is Kitti-style but sample 0 is Sintel-style"):
        validate(Stub(), [sintel[0], kitti[1]], device="cpu", regions=True)
    bad = sintel[3][:4] + ({"occ": torch.zeros(5, 5)},)
    with pytest.raises(ValueError, match=r"sample 3's occ mask is \(5, 5\), expected \[H,W\] = \(20, 30\)"):
        validate(Stub(), sintel[:3] + [bad], device="cpu", regions=True)
    for masks in ({"occ": sintel[0][4]["occ"], "noc": sintel[0][4]["occ"]}, {"fg": sintel[0][4]["occ"]}, "occ"):
        with pytest.raises(ValueError, match="sample 0's fifth item"):
            validate(Stub(), [sintel[0][:4] + (masks,)], device="cpu", regions=True)
    # regions=False is unchanged: a fifth item is ignored, as before
    assert validate(Stub(), sintel, device="cpu") == validate(Stub(), stub_samples(False), device="cpu")


def test_region_partials_argument_errors():
    from rnc.metrics import boundary_dist2, region_partials
    flow, gt, valid, occ = region_batch(2, 8, 9, seed=4)
    with pytest.raises(ValueError, match="not both or neither"):
        region_partials(flow, gt, valid)
    with pytest.raises(ValueError, match="not both or neither"):
        region_partials(flow, gt, valid, occ=occ, noc=occ)
    with pytest.raises(ValueError, match="fg goes with noc"):
        region_partials(flow, gt, valid, occ=occ, fg=occ)
    with pytest.raises(ValueError, match=r"expected occ \[B,H,W\]"):
        region_partials(flow, gt, valid, occ=occ[:, :7])
    with pytest.raises(ValueError, match=r"expected fg \[B,H,W\]"):
        region_partials(flow, gt, valid, noc=occ, fg=occ[0])
    with pytest.raises(ValueError, match="boundary_dist2"):
        boundary_dist2(occ[0, 0])


def _gloo_worker(rank, world, port, sparse, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from rnc.harness import validate
        m = BidiStub()
        res = validate(m, region_samples(sparse, fg_every=False), iters=1, batch_size=3, device="cpu", regions=True,
                       consistency=True)
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,sparse", [(2, True), (3, False), (2, False)])
def test_validate_regions_gloo_equals_world_1(world, sparse):
    from rnc.harness import validate
    want = validate(BidiStub(), region_samples(sparse, fg_every=False), iters=1, batch_size=3, device="cpu", regions=True,
                    consistency=True)
    assert "region_pixels" in want
    for got in run_ranks(_gloo_worker, world, sparse):
        assert same(got, want)                              # bit for bit, on every rank


# ----------------------------------------------------------------------------- C ABI


def test_entry_points_declared_and_bound():
    from rnc import native
    with open(os.path.join(ROOT, "include", "rnc.h")) as f:
        hdr = f.read()
    declared = set(re.findall(r"\b(rnc_\w+)\s*\(", hdr))
    for n in ("rnc_boundary_dist2", "rnc_region_metrics", "rnc_region_metrics_workspace_bytes"):
        assert n in declared and n in native.SIGNATURES, n
    defs = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(RNC_\w+)\s+(\d+)", hdr)}
    assert defs["RNC_DIST2_NONE"] == native.DIST2_NONE == NONE
    assert (defs["RNC_REGIONS_SINTEL"], defs["RNC_REGIONS_KITTI"]) == (native.REGIONS_SINTEL, native.REGIONS_KITTI)
    assert native.REGION_CELLS == {native.REGIONS_SINTEL: defs["RNC_REGION_CELLS_SINTEL"],
                                   native.REGIONS_KITTI: defs["RNC_REGION_CELLS_KITTI"]} == {0: 32, 1: 4}


def test_entry_points_reject_bad_arguments():
    from rnc import native
    L = native.lib()
    P = 1 << 20   # never dereferenced: every check fails on the host before a launch
    n0 = L.rnc_launch_count()

    def dist2(B=2, H=436, W=1024, occ=P, d2=P):
        return L.rnc_boundary_dist2(occ, H * W, W, 1, B, H, W, d2, None)

    assert dist2(B=0) == -1 and dist2(H=0) == -1 and dist2(W=-1) == -1 and dist2(B=65536) == -1
    assert dist2(H=4097) == -1 and dist2(W=4097) == -1
    assert dist2(occ=0) == -2 and dist2(d2=0) == -2 and dist2(occ=P + 2) == -2 and dist2(d2=P + 1) == -2
    ws = L.rnc_region_metrics_workspace_bytes(0, 3, 436, 1024)
    assert ws == 3 * 218 * 32 * 32 and L.rnc_region_metrics_workspace_bytes(1, 3, 436, 1024) == 3 * 218 * 4 * 32
    assert L.rnc_region_metrics_workspace_bytes(2, 3, 4, 5) == 0 and L.rnc_region_metrics_workspace_bytes(-1, 3, 4, 5) == 0
    assert L.rnc_region_metrics_workspace_bytes(0, 0, 4, 5) == 0 and L.rnc_region_metrics_workspace_bytes(0, 1, 1 << 15, 1 << 15) == 0

    def call(kind=0, B=3, H=436, W=1024, flow=P, gt=P, valid=P, mask=P, d2=P, fg=0, counts=P, sums=P, wsp=P, wsb=ws):
        return L.rnc_region_metrics(kind, flow, 40, 20, 5, 1, gt, 40, 20, 5, 1, valid, 20, 5, 1, mask, 20, 5, 1, d2, fg, 20, 5,
                                    1, B, H, W, counts, sums, wsp, wsb, None)

    assert call(kind=2) == -3 and call(kind=-1) == -3
    assert call(B=0) == -1 and call(H=0) == -1 and call(W=-1) == -1 and call(B=65536) == -1 and call(H=1 << 15, W=1 << 15) == -1
    assert call(flow=0) == -2 and call(gt=0) == -2 and call(mask=0) == -2 and call(counts=0) == -2 and call(sums=0) == -2
    assert call(wsp=0) == -2 and call(d2=0) == -2 and call(fg=P) == -2                 # Sintel: d2 required, no fg
    assert call(kind=1, d2=P) == -2                                                      # KITTI: no d2
    assert call(flow=P + 2) == -2 and call(valid=P + 2) == -2 and call(mask=P + 1) == -2 and call(d2=P + 2) == -2
    assert call(kind=1, d2=0, fg=P + 2) == -2 and call(counts=P + 4) == -2 and call(wsp=P + 8) == -2
    assert call(wsb=ws - 1) == -5 and call(kind=1, d2=0, wsb=ws // 8 - 1) == -5
    assert L.rnc_launch_count() == n0


def test_region_metrics_cu_does_not_spill(tmp_path):
    from rnc.build import ARCH, nvcc_path
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-c", os.path.join(CSRC, "region_metrics.cu"), "-o", str(tmp_path / "r.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    kernels = re.findall(r"Function properties for \S*\d((?:dist2|region)_[a-z0-9_]+_kernel)", log)
    assert sorted(kernels) == ["dist2_column_kernel", "dist2_row_kernel", "region_part_kernel", "region_reduce_kernel"], kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 4 and all(a == "0" and b == "0" for a, b in spills), spills
