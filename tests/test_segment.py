"""Label propagation on the host (rnc.segment.host_propagate_step, the kernel's reference) against hand-built fields and
analytic motions, the DAVIS counts and statistics against hand-computed cases, the argument checks of the propagation, the
counts and the harness, validate_segmentation under gloo, the C entry points' error codes and declarations, and a compile of
segment.cu for sm_90a."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from rnc import native
from rnc.segment import (COUNT_FG_MATCH, COUNT_GT_MATCH, COUNT_INTER, COUNT_N_FG, COUNT_N_GT, COUNT_UNION,
                         contour_accuracy, decay_bins, host_propagate, host_propagate_step, host_segmentation_counts,
                         propagate, propagate_step, region_similarity, seg2bmap, segmentation_counts, statistics,
                         summarize_segmentation, tolerance)
from rnc.synth import shift_sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def step_inputs(H, W, dx=0.0, dy=0.0):
    """One video's step inputs: labels 0, G = (dx, dy) everywhere, nothing occluded."""
    L = torch.zeros(1, H, W, dtype=torch.uint8)
    G = torch.empty(1, 2, H, W)
    G[:, 0], G[:, 1] = dx, dy
    return L, G, torch.zeros(1, H, W, dtype=torch.uint8)


def square(H, W, y0, x0, side, label=1):
    L = torch.zeros(H, W, dtype=torch.uint8)
    L[y0:y0 + side, x0:x0 + side] = label
    return L


# ----------------------------------------------------------------------------------------------------------- propagation


@pytest.mark.parametrize("dy,dx", [(3, 4), (1, 2), (0, 5)])
def test_the_true_flows_of_a_shift_sequence_give_the_shifted_masks(dy, dx):
    T, H, W, side, y0, x0 = 7, 40, 64, 8, 6, 5
    seq = shift_sequence(T, H, W, seed=3, dy=dy, dx=dx)
    assert torch.equal(seq[1][:, dy:, dx:], seq[0][:, :H - dy, :W - dx])     # content moves by (dx, dy) a frame
    G = torch.empty(1, T - 1, 2, H, W)
    G[:, :, 0], G[:, :, 1] = -dx, -dy                                       # frame k+1 -> k
    occ = torch.zeros(1, T - 1, H, W, dtype=torch.uint8)
    first = (square(H, W, y0, x0, side, 3) + square(H, W, 20, 30, 5, 7))[None]
    got = host_propagate(first, G, occ)
    assert got.shape == (1, T, H, W) and got.dtype == torch.uint8
    for t in range(T):
        want = square(H, W, y0 + t * dy, x0 + t * dx, side, 3) + square(H, W, 20 + t * dy, 30 + t * dx, 5, 7)
        assert torch.equal(got[0, t], want), t
    assert torch.equal(propagate(first, G, occ), got)                       # CPU tensors take the host path
    # the first rows and columns' sources leave the frame: unmatched, filled from the background next to them
    gt = got[0]
    s = summarize_segmentation([host_segmentation_counts(got[0, 1:-1], gt[1:-1], 7)])
    assert s["J-Mean"] == 1.0 and s["F-Mean"] == 1.0 and s["J&F-Mean"] == 1.0 and s["objects"] == 7


def vote(L, x, y, ux, uy):
    """The label pixel (x, y) of the next frame gets from L through the flow (ux, uy) there."""
    H, W = L.shape
    _, G, occ = step_inputs(H, W)
    G[0, 0, y, x], G[0, 1, y, x] = ux, uy
    return int(host_propagate_step(L[None], G, occ)[0, y, x])


def test_a_fractional_target_takes_the_heavier_label_and_the_smaller_on_a_tie():
    L = torch.zeros(4, 8, dtype=torch.uint8)
    L[:, 3], L[:, 4] = 5, 2
    assert vote(L, 1, 1, 2.5, 0.0) == 2                                     # 0.5 each: the smaller label
    L[:, 3], L[:, 4] = 2, 5
    assert vote(L, 1, 1, 2.5, 0.0) == 2
    assert vote(L, 1, 1, 2.75, 0.0) == 5                                    # 0.25 against 0.75
    assert vote(L, 1, 1, 2.25, 0.5) == 2                                    # rows do not change the columns' weights
    # p' = (3.25, 1.5): taps (1,3), (1,4), (2,3), (2,4) weigh 0.375, 0.125, 0.375, 0.125
    L[2, 3] = 9                                                             # 2 and 9 0.375 each, 5 0.25: the smaller
    assert vote(L, 1, 1, 2.25, 0.5) == 2
    L[1, 4] = 9                                                             # 9 gathers 0.125 + 0.375 against 2's 0.375
    assert vote(L, 1, 1, 2.25, 0.5) == 9


def test_a_target_exactly_on_the_last_row_or_column_is_matched():
    L = torch.arange(20, dtype=torch.uint8).reshape(4, 5) + 1
    assert vote(L, 0, 0, 4.0, 3.0) == int(L[3, 4])                          # p' = (W-1, H-1)
    assert vote(L, 1, 2, 3.0, 1.0) == int(L[3, 4])
    assert vote(L, 0, 1, 4.0, 0.0) == int(L[1, 4])
    # just outside: unmatched, so the pixel takes its nearest matched pixel's label, its left neighbour's own (zero flow)
    assert vote(L, 2, 1, 2.0 + 2 ** -20, 0.0) == int(L[1, 1])


@pytest.mark.parametrize("why", ["occluded", "nan", "inf", "-inf"])
def test_an_unmatched_pixel_takes_the_nearest_matched_label_ties_to_the_column_then_the_row(why):
    H, W, y, x = 7, 9, 3, 4
    L = torch.arange(H * W, dtype=torch.uint8).reshape(H, W) + 1
    _, G, occ = step_inputs(H, W)                                           # zero flow: a matched pixel keeps its label

    def unmatch(yy, xx):
        if why == "occluded":
            occ[0, yy, xx] = 1
        else:
            G[0, 1, yy, xx] = float(why)
    unmatch(y, x)                                                           # four neighbours at distance 1: the left one
    assert int(host_propagate_step(L[None], G, occ)[0, y, x]) == int(L[y, x - 1])
    unmatch(y, x - 1)                                                       # up, down and right: column x, then the upper
    got = host_propagate_step(L[None], G, occ)[0]
    assert int(got[y, x]) == int(L[y - 1, x]) and int(got[y, x - 1]) == int(L[y, x - 2])
    expect = L.clone()
    expect[y, x], expect[y, x - 1] = L[y - 1, x], L[y, x - 2]
    assert torch.equal(got, expect)                                         # every matched pixel keeps its own label


def test_a_frame_without_a_matched_pixel_is_all_background():
    L = square(6, 8, 1, 1, 3, 4)[None]
    _, G, occ = step_inputs(6, 8)
    assert torch.equal(host_propagate_step(L, G, torch.ones_like(occ)), torch.zeros_like(L))
    assert torch.equal(host_propagate_step(L, G, occ), L)
    assert torch.equal(host_propagate_step(L, torch.full_like(G, float("nan")), occ), torch.zeros_like(L))
    assert torch.equal(host_propagate_step(L, G + 100, occ), torch.zeros_like(L))       # every target leaves the frame


def test_the_strip_a_moving_square_uncovers_is_filled_by_the_rule():
    H, W, y0, x0, side, d = 12, 20, 4, 6, 4, 2
    L = square(H, W, y0, x0, side)[None]                                    # frame k: the square at columns 6..9
    _, G, occ = step_inputs(H, W)
    rows = slice(y0, y0 + side)
    G[0, 0, rows, x0 + d:x0 + d + side] = -d                                # frame k+1: at columns 8..11, background static
    occ[0, rows, x0:x0 + d] = 1                                             # columns 6, 7: hidden in frame k
    got = host_propagate_step(L, G, occ)[0]
    want = square(H, W, y0, x0 + d, side)
    # column 6: the background at column 5 is at distance 1 and the smallest column.  Column 7: on rows 5 and 6 the square
    # at column 8 is the only pixel at distance 1; on rows 4 and 7 the background above or below ties with it at distance
    # 1 and has the smaller column.
    want[5:7, x0 + 1] = 1
    assert torch.equal(got, want), got[y0 - 1:y0 + side + 1, x0 - 1:x0 + side + d + 1]
    # without the masks the static background's zero flow would pull the old square into the strip
    naive = host_propagate_step(L, G, torch.zeros_like(occ))[0]
    assert naive[rows, x0:x0 + d].eq(1).all()


def test_propagate_chains_the_steps_on_strided_views():
    V, T, H, W = 2, 4, 9, 11
    g = torch.Generator().manual_seed(0)
    big = torch.randn(V, T - 1, 3, H, W + 2, generator=g) * 2
    G = big[:, :, 1:, :, 1:W + 1]                                           # strided in every dimension
    occ = (torch.rand(V, T - 1, H, W, generator=g) < 0.2).to(torch.uint8)
    first = torch.randint(0, 255, (V, H, W), generator=g, dtype=torch.uint8)
    got = propagate(first, G, occ)
    k_by_k = [first]
    for k in range(T - 1):
        k_by_k.append(propagate_step(k_by_k[-1], G[:, k].contiguous(), occ[:, k]))
    assert torch.equal(got, torch.stack(k_by_k, 1))
    assert torch.equal(host_propagate(first.long(), G, occ.bool()), got)


# ----------------------------------------------------------------------------------------------------------- metrics


def cells(b):
    return sorted(map(tuple, np.argwhere(b).tolist()))


def test_seg2bmap_on_hand_computed_masks():
    H, W = 4, 5

    def one(y, x):
        s = np.zeros((H, W), bool)
        s[y, x] = True
        return seg2bmap(s)
    assert cells(one(1, 1)) == [(0, 0), (0, 1), (1, 0), (1, 1)]
    assert cells(one(H - 1, 2)) == [(2, 1), (2, 2), (3, 1), (3, 2)]            # last row: s ^ e only
    assert cells(one(1, W - 1)) == [(0, 3), (0, 4), (1, 3), (1, 4)]            # last column: s ^ so only
    assert cells(one(H - 1, W - 1)) == [(2, 3), (2, 4), (3, 3)]                # the bottom-right pixel is never a boundary
    assert not seg2bmap(np.ones((H, W), bool)).any()
    assert not seg2bmap(np.zeros((H, W), bool)).any()
    s = np.zeros((H, W), bool)
    s[1:3, 1:4] = True
    want = np.zeros((H, W), bool)
    want[0:3, 0:4] = True
    want[1, 1:3] = False                                                    # the inside of the block
    assert (seg2bmap(s) == want).all()
    assert (seg2bmap(np.stack([s, s]))[1] == want).all()                    # batched


def counts_of(pred, gt, K=1):
    return host_segmentation_counts(torch.as_tensor(pred, dtype=torch.uint8)[None],
                                    torch.as_tensor(gt, dtype=torch.uint8)[None], K)[0]


def test_the_four_boundary_cases_an_empty_union_and_void_pixels():
    H, W = 12, 16
    obj = square(H, W, 3, 4, 5).numpy()
    none = np.zeros((H, W), np.uint8)
    c = counts_of(none, obj).tolist()[0]                                    # (n_fg, n_gt) = (0, > 0): P = 1, R = 0
    assert c[COUNT_N_FG] == 0 and c[COUNT_N_GT] > 0 and contour_accuracy(c) == 0.0 and region_similarity(c) == 0.0
    c = counts_of(obj, none).tolist()[0]                                    # (> 0, 0): P = 0, R = 1
    assert c[COUNT_N_GT] == 0 and c[COUNT_N_FG] > 0 and contour_accuracy(c) == 0.0
    c = counts_of(none, none).tolist()[0]                                   # (0, 0): P = R = 1, and J = 1
    assert c == [0] * 6 and contour_accuracy(c) == 1.0 and region_similarity(c) == 1.0
    c = counts_of(obj, obj).tolist()[0]
    assert c[COUNT_INTER] == c[COUNT_UNION] == 25 and c[COUNT_FG_MATCH] == c[COUNT_N_FG] == c[COUNT_N_GT] == 20
    assert contour_accuracy(c) == 1.0 and region_similarity(c) == 1.0
    assert contour_accuracy([1, 2, 4, 8, 0, 0]) == 0.0                      # P + R = 0
    assert math.isclose(contour_accuracy([1, 2, 4, 8, 1, 6]), 2 * 0.25 * 0.75 / (0.25 + 0.75))
    void = obj * 255                                                        # the prediction lies only on void pixels
    c = counts_of(obj, void).tolist()[0]
    assert c == [0] * 6 and region_similarity(c) == 1.0 and contour_accuracy(c) == 1.0
    half = void.copy()
    half[:, :6] = 0                                                         # void on columns 6.. of the square only
    gt = square(H, W, 3, 4, 2).numpy()                                      # columns 4, 5 rows 3, 4
    c = counts_of(obj, np.maximum(half, gt)).tolist()[0]
    assert c[COUNT_INTER] == 4 and c[COUNT_UNION] == 10                     # M: columns 4, 5 of the square's 5 rows


def test_the_boundary_tolerance():
    assert tolerance(480, 854) == 8 and tolerance(1080, 1920) == 18 and tolerance(40, 60) == 1
    H, W = 40, 60                                                           # r = 1
    for shift, matched in ((0, True), (1, True), (2, False)):
        pred, gt = np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8)
        pred[5:30, 10:20] = 1
        gt[5:30, 10 + shift:20 + shift] = 1
        c = counts_of(pred, gt).tolist()[0]
        if matched:
            assert c[COUNT_FG_MATCH] == c[COUNT_N_FG] and c[COUNT_GT_MATCH] == c[COUNT_N_GT], (shift, c)
        else:                                                               # only the top and bottom rows still meet
            assert c[COUNT_FG_MATCH] < c[COUNT_N_FG] and c[COUNT_GT_MATCH] < c[COUNT_N_GT], (shift, c)
    pred, gt = np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8)       # two points: distance^2 = 1 + 1 > r^2
    pred[10, 10], gt[11, 11] = 1, 1
    c = counts_of(pred, gt).tolist()[0]
    assert c[COUNT_N_FG] == 4 and c[COUNT_N_GT] == 4
    assert c[COUNT_FG_MATCH] == 3 and c[COUNT_GT_MATCH] == 3                # every boundary pixel but the far corner


def test_the_decay_bins_by_hand():
    want = {1: [(0, 1), (0, 1), (0, 1), (0, 1)], 2: [(0, 1), (0, 2), (1, 2), (1, 2)], 3: [(0, 2), (1, 2), (1, 3), (2, 3)],
            4: [(0, 2), (1, 3), (2, 3), (2, 4)], 5: [(0, 2), (1, 3), (2, 4), (3, 5)], 6: [(0, 2), (1, 4), (3, 5), (4, 6)],
            7: [(0, 3), (2, 4), (3, 6), (5, 7)], 8: [(0, 3), (2, 5), (4, 6), (5, 8)], 9: [(0, 3), (2, 5), (4, 7), (6, 9)],
            10: [(0, 3), (2, 6), (5, 8), (7, 10)]}
    for n, bins in want.items():
        assert decay_bins(n) == bins, n
    m, o, d = statistics([1.0, 0.8, 0.6, 0.4, 0.2])
    assert math.isclose(m, 0.6) and o == 0.6 and math.isclose(d, 0.9 - 0.3)
    assert statistics([0.7]) == (0.7, 1.0, 0.0)


def test_summaries_average_per_object_then_over_objects():
    def frame(*objs):                                                       # (inter, union) per object, F = 1
        return [[i, u, 4, 4, 4, 4] for i, u in objs]
    a = [frame((1, 2), (4, 4)), frame((1, 4), (4, 4)), frame((3, 4), (0, 4))]      # video 1: two objects, three frames
    b = [frame((2, 2))]                                                     # video 2: one object, one frame
    s = summarize_segmentation([torch.tensor(a), b])
    j = [(0.5 + 0.25 + 0.75) / 3, (1 + 1 + 0) / 3, 1.0]
    assert s["objects"] == 3 and s["videos"] == 2
    assert math.isclose(s["J-Mean"], sum(j) / 3)
    assert math.isclose(s["J-Recall"], (1 / 3 + 2 / 3 + 1) / 3)
    # decay of 3 frames: bin 0 = v[0:2], bin 3 = v[2:3]
    assert math.isclose(s["J-Decay"], ((0.375 - 0.75) + (1 - 0) + 0) / 3)
    assert s["F-Mean"] == 1.0 and s["F-Recall"] == 1.0 and s["F-Decay"] == 0.0
    assert math.isclose(s["J&F-Mean"], (s["J-Mean"] + 1.0) / 2)
    assert math.isnan(summarize_segmentation([])["J-Mean"])


def test_segmentation_counts_on_the_cpu_is_the_host():
    g = torch.Generator().manual_seed(5)
    gt = torch.randint(0, 4, (3, 20, 30), generator=g, dtype=torch.uint8)
    gt[:, :3] = 255
    pred = torch.randint(0, 4, (3, 20, 30), generator=g, dtype=torch.uint8)
    got = segmentation_counts(pred, gt, 3)
    assert got.shape == (3, 3, native.SEGMENT_COUNTS) and got.dtype == torch.int64
    assert torch.equal(got, host_segmentation_counts(pred, gt, 3))
    assert segmentation_counts(pred, gt, 0).shape == (3, 0, native.SEGMENT_COUNTS)


def test_argument_errors_raise_before_any_launch():
    L, G, occ = step_inputs(6, 9)
    with pytest.raises(ValueError, match="flow_bw"):
        propagate_step(L, G[..., :8], occ)
    with pytest.raises(ValueError, match="occ_bw"):
        propagate_step(L, G, occ[:, 1:])
    with pytest.raises(ValueError, match="labels"):
        propagate_step(L[0], G, occ)
    with pytest.raises(ValueError, match="one device"):
        propagate_step(L, G.to("meta"), occ)
    bad = L.clone()
    bad[0, 2, 2] = 255
    with pytest.raises(ValueError, match="0..254"):
        propagate_step(bad, G, occ)
    with pytest.raises(ValueError, match="integer labels"):
        propagate_step(L.float(), G, occ)
    wide = step_inputs(1, 4097)
    with pytest.raises(ValueError, match="4096"):
        propagate_step(*wide)
    Gs, Os = G[:, None].repeat(1, 3, 1, 1, 1), occ[:, None].repeat(1, 3, 1, 1)
    with pytest.raises(ValueError, match="T >= 2"):
        propagate(L, Gs[:, :0], Os[:, :0])
    with pytest.raises(ValueError, match="flow_bw"):
        propagate(L, Gs[:, :, :1], Os)
    with pytest.raises(ValueError, match="occ_bw"):
        propagate(L, Gs, Os[:, :2])
    with pytest.raises(ValueError, match="0..254"):
        propagate(bad, Gs, Os)
    with pytest.raises(ValueError, match="one device"):
        propagate(L, Gs, Os.to("meta"))
    with pytest.raises(ValueError, match="one \\[N,H,W\\] shape"):
        segmentation_counts(L, L[:, 1:], 1)
    with pytest.raises(ValueError, match="object count"):
        segmentation_counts(L, L, 255)
    with pytest.raises(ValueError, match="one device"):
        segmentation_counts(L, L.to("meta"), 1)
    with pytest.raises(ValueError, match="4096"):
        segmentation_counts(wide[0], wide[0], 1)


def test_propagate_masks_and_validate_segmentation_check_their_arguments():
    from rnc.harness import propagate_masks, validate_segmentation
    from rnc.synth import build_model
    m = build_model("raft")
    seqs = [[torch.zeros(3, 16, 16)] * 3]
    first = [torch.zeros(16, 16, dtype=torch.uint8)]
    with pytest.raises(ValueError, match="inference only"):
        propagate_masks(m, seqs, first)
    with torch.no_grad():
        with pytest.raises(ValueError, match="1 videos but 2 first-frame"):
            propagate_masks(m, seqs, first * 2)
        with pytest.raises(ValueError, match="T >= 2"):
            propagate_masks(m, [seqs[0][:1]], first)
        with pytest.raises(ValueError, match="expected first labels"):
            propagate_masks(m, seqs, [first[0][:8]])
        with pytest.raises(ValueError, match="0..254"):
            propagate_masks(m, seqs, [first[0] + 255])
        assert propagate_masks(m, [], []) == []
        with pytest.raises(ValueError, match="T >= 3"):
            validate_segmentation(m, [seqs[0][:2]], [torch.zeros(2, 16, 16, dtype=torch.uint8)])
        with pytest.raises(ValueError, match="expected ground truth"):
            validate_segmentation(m, seqs, [torch.zeros(2, 16, 16, dtype=torch.uint8)])
        with pytest.raises(ValueError, match="ground-truth label sets"):
            validate_segmentation(m, seqs, [])


# ----------------------------------------------------------------------------- validate_segmentation under torch.distributed


class _InferenceModel:
    def _needs_grad(self):
        return False


def _stub_bidirectional(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                        alpha1=0.01, alpha2=0.5):
    """run_sequences_bidirectional's yields in its step order, on the CPU: backward flows from the frames' first channels,
    masks from a threshold on the third; one frame size per call, as the real one requires."""
    from rnc.harness import sequence_schedule
    assert len({tuple(f.shape) for s in sequences for f in s}) == 1
    for step in sequence_schedule([len(s) for s in sequences], batch_size):
        for c in step:
            if not c.idle:
                a, b = sequences[c.seq][c.pair], sequences[c.seq][c.pair + 1]
                yield c.seq, c.pair, {"flow_up_bw": (a[:2] - b[:2]) / 32, "occ_bw": (b[2] > 220).to(torch.uint8)}


def segmentation_split():
    """Seven videos of 3 to 7 frames in two frame sizes, with moving squares as the ground truth and some void pixels."""
    seqs, gts = [], []
    for k, (n, H, W) in enumerate(((5, 12, 20), (3, 16, 14), (7, 12, 20), (4, 16, 14), (3, 12, 20), (6, 16, 14),
                                   (4, 12, 20))):
        seqs.append(shift_sequence(n, H, W, seed=k, dy=1, dx=k % 3))
        gt = torch.zeros(n, H, W, dtype=torch.uint8)
        for t in range(n):
            gt[t, 2 + t // 2:7 + t // 2, 1 + t:6 + t] = 1
            if k % 2:
                gt[t, 8:11, 3 + (t + k) % 4:7 + (t + k) % 4] = 2 + k // 3
            gt[t, -1, :3] = 255
        gts.append(gt)
    return seqs, gts


def _segmentation_worker(rank, world, port, q):
    import torch.distributed as dist
    from rnc import harness
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        harness.run_sequences_bidirectional = _stub_bidirectional
        q.put((rank, harness.validate_segmentation(_InferenceModel(), *segmentation_split(), batch_size=2, device="cpu")))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_validate_segmentation_gloo_equals_world_1(world, monkeypatch):
    from test_flow_metrics import run_ranks
    from rnc import harness
    monkeypatch.setattr(harness, "run_sequences_bidirectional", _stub_bidirectional)
    seqs, gts = segmentation_split()
    want = harness.validate_segmentation(_InferenceModel(), seqs, gts, batch_size=2, device="cpu")
    counts = []                                         # per video, as the host defines it
    for seq, gt in zip(seqs, gts):
        r = [x[2] for x in _stub_bidirectional(None, [seq])]
        first = torch.where(gt[0] == 255, 0, gt[0])
        pred = host_propagate(first[None], torch.stack([p["flow_up_bw"] for p in r])[None],
                              torch.stack([p["occ_bw"] for p in r])[None])[0]
        counts.append(host_segmentation_counts(pred[1:-1], gt[1:-1], int(first.max())))
    assert want == summarize_segmentation(counts) and want["videos"] == len(seqs) and want["objects"] == 12
    assert 0 < want["J-Mean"] < 1
    for got in run_ranks(_segmentation_worker, world):
        assert got == want                              # bit for bit, on every rank


# ----------------------------------------------------------------------------- C ABI


_CTYPE = {"long long": native.C.c_longlong, "int": native.C.c_int, "size_t": native.C.c_size_t, "float": native.C.c_float}
NAMES = ("rnc_propagate_labels_workspace_bytes", "rnc_propagate_labels", "rnc_segmentation_counts_workspace_bytes",
         "rnc_segmentation_counts")


def test_declarations_match_the_binding():
    with open(os.path.join(ROOT, "include", "rnc.h")) as f:
        header = f.read()
    assert f"#define RNC_SEGMENT_COUNTS {native.SEGMENT_COUNTS}" in header
    for name in NAMES:
        m = re.search(r"\n(int|size_t) " + name + r"\(([^;]*)\);", header)
        assert m, name
        args = [a.strip() for a in m.group(2).replace("\n", " ").split(",")]
        want = [native.C.c_void_p if "*" in a else _CTYPE[a.rsplit(" ", 1)[0].replace("const ", "")] for a in args]
        res, argtypes = native.SIGNATURES[name]
        assert argtypes == want, name
        assert res is (native.C.c_int if m.group(1) == "int" else native.C.c_size_t), name


def test_entry_points_return_their_error_codes():
    L = native.lib()
    P = 1 << 20                                         # never dereferenced: every check fails on the host before a launch
    n0 = L.rnc_launch_count()
    ws = L.rnc_propagate_labels_workspace_bytes(3, 40, 60)
    assert ws == 3 * 40 * 60 * 4
    for bad in ((0, 4, 4), (65536, 4, 4), (1, 0, 4), (1, 4, 4097)):
        assert L.rnc_propagate_labels_workspace_bytes(*bad) == 0, bad

    def prop(V=3, H=40, W=60, lab=P, flow=P, occ=P, out=P, wsp=P, wsb=ws):
        return L.rnc_propagate_labels(lab, 1, 1, 1, flow, 1, 1, 1, 1, occ, 1, 1, 1, V, H, W, out, 1, 1, 1, wsp, wsb, None)

    for bad in (dict(V=0), dict(V=65536), dict(H=0), dict(W=4097), dict(H=-1)):
        assert prop(**bad) == -1, bad
    for bad in (dict(lab=0), dict(flow=0), dict(occ=0), dict(out=0), dict(wsp=0), dict(flow=P + 2), dict(wsp=P + 8)):
        assert prop(**bad) == -2, bad
    assert prop(wsb=ws - 1) == -5
    cws = L.rnc_segmentation_counts_workspace_bytes(10, 3, 40, 60)
    assert cws == 2 * 10 * 3 * 40 * 60 * 4 + 10 * 3 * 2 * 24
    for bad in ((0, 1, 4, 4), (1, 0, 4, 4), (1, 255, 4, 4), (32768, 1, 4, 4), (1, 1, 4097, 4)):
        assert L.rnc_segmentation_counts_workspace_bytes(*bad) == 0, bad

    def cnt(N=10, K=3, H=40, W=60, pred=P, gt=P, counts=P, wsp=P, wsb=cws):
        return L.rnc_segmentation_counts(pred, 1, 1, 1, gt, 1, 1, 1, N, K, H, W, counts, wsp, wsb, None)

    for bad in (dict(N=0), dict(K=0), dict(K=255), dict(N=20000, K=2), dict(H=0), dict(W=4097)):
        assert cnt(**bad) == -1, bad
    for bad in (dict(pred=0), dict(gt=0), dict(counts=0), dict(wsp=0), dict(counts=P + 4), dict(wsp=P + 8)):
        assert cnt(**bad) == -2, bad
    assert cnt(wsb=cws - 1) == -5
    assert L.rnc_launch_count() == n0


def test_segment_cu_has_no_atomics_and_does_not_spill(tmp_path):
    from rnc.build import ARCH, CSRC, nvcc_path
    cubin = str(tmp_path / "s.cubin")
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-cubin", os.path.join(CSRC, "segment.cu"), "-o", cubin]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    kernels = re.findall(r"Function properties for \S*?\d((?:vote|dist2_column|dist2_row|cta_partials|image_reduce)_kernel)",
                         log)
    assert sorted(kernels) == sorted(["vote_kernel", "dist2_column_kernel", "dist2_column_kernel", "dist2_row_kernel",
                                      "dist2_row_kernel", "cta_partials_kernel", "image_reduce_kernel"]), kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 7 and all(a == "0" and b == "0" for a, b in spills), spills
    assert re.findall(r"(\d+) bytes stack frame", log) == ["0"] * 7
    cuobjdump = os.path.join(os.path.dirname(nvcc_path()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    assert "FFMA" not in sass.split("vote_kernel", 1)[1].split("Function :", 1)[0]       # every operation rounded once
    assert not re.search(r"\b(ATOM|ATOMS|ATOMG|RED)\b", sass)
