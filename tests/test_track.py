"""Point tracking on the host (rnc.track.host_track, the kernel's reference) against the rule's stated properties and against
analytic trajectories, the TAP-Vid counts against a numpy transcription of their definitions, the argument checks of track,
track_metrics and track_points, the C entry points' error codes and declarations, and a compile of track.cu for sm_90a."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from rnc import native
from rnc.track import (COUNT_EVALUATED, COUNT_FP, COUNT_GT_VISIBLE, COUNT_OCC_AGREE, COUNT_TP, COUNT_WITHIN, THRESHOLDS,
                       grid_queries, host_track, host_track_metrics, summarize_tracking, track, track_metrics)
from rnc.synth import shift_sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def fields(T, H, W, dx=0.0, dy=0.0, bx=None, by=None):
    """One video's stacked inputs: F = (dx, dy) and G = (bx, by) (default -F) everywhere, no occlusion."""
    F = torch.empty(1, T - 1, 2, H, W)
    F[:, :, 0], F[:, :, 1] = dx, dy
    G = torch.empty(1, T - 1, 2, H, W)
    G[:, :, 0], G[:, :, 1] = -dx if bx is None else bx, -dy if by is None else by
    occ = torch.zeros(1, T - 1, H, W, dtype=torch.uint8)
    return F, G, occ, occ.clone()


def Q(*qs):
    return torch.tensor([qs], dtype=torch.float32)


def test_constant_translation_gives_exact_positions():
    T, H, W, dx, dy = 6, 20, 30, 2.0, 1.0
    q = Q((0, 3, 4), (2, 10, 7), (5, 20, 12), (3, 15.25, 8.5))
    tracks, vis = host_track(*fields(T, H, W, dx, dy), q)
    assert tracks.shape == (1, 4, T, 2) and tracks.dtype == torch.float32 and vis.dtype == torch.uint8
    for n, (t0, x, y) in enumerate(q[0].tolist()):
        for t in range(T):
            assert tracks[0, n, t].tolist() == [x + (t - t0) * dx, y + (t - t0) * dy], (n, t)
    assert (vis == 1).all()


def test_a_point_that_leaves_the_frame_is_lost_and_keeps_advancing():
    T, H, W = 6, 5, 10
    tracks, vis = host_track(*fields(T, H, W, 3.0, 0.0), Q((0, 2, 1), (5, 9, 2)))
    assert tracks[0, 0, :, 0].tolist() == [2, 5, 8, 11, 14, 17]          # the clamped samples still give u = 3
    assert vis[0, 0].tolist() == [1, 1, 1, 0, 0, 0]
    assert tracks[0, 1, :, 0].tolist() == [-6, -3, 0, 3, 6, 9]           # backward from frame 5
    assert vis[0, 1].tolist() == [0, 0, 1, 1, 1, 1]


def test_an_occluded_pixel_loses_the_point_at_the_next_frame():
    T, H, W = 6, 8, 16
    F, G, occ, occ_bw = fields(T, H, W, 1.0, 0.0)
    occ[0, 2, 3, 4] = 1                                                  # the point sits at (4, 3) in frame 2
    tracks, vis = host_track(F, G, occ, occ_bw, Q((0, 2, 3)))
    assert vis[0, 0].tolist() == [1, 1, 1, 0, 0, 0]
    assert tracks[0, 0, :, 0].tolist() == [2, 3, 4, 5, 6, 7]
    occ_bw[0, 2, 3, 4] = 1                                               # a mask of the other direction: no effect
    assert torch.equal(host_track(F, G, torch.zeros_like(occ), occ_bw, Q((0, 2, 3)))[1], torch.ones(1, 1, T, dtype=torch.uint8))


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_a_non_finite_flow_holds_the_position_and_loses_the_point(bad):
    T, H, W = 5, 8, 16
    F, G, occ, occ_bw = fields(T, H, W, 1.0, 1.0)
    F[0, 1, 1, 2, 3] = bad                                               # the y component at (3, 2), the position in frame 1
    tracks, vis = host_track(F, G, occ, occ_bw, Q((0, 2, 1)))
    assert tracks[0, 0].tolist() == [[2, 1], [3, 2], [3, 2], [4, 3], [5, 4]]
    assert vis[0, 0].tolist() == [1, 1, 0, 0, 0]


def test_a_middle_query_tracks_backward_through_the_backward_flows_and_masks():
    T, H, W = 7, 12, 20
    F, G, occ, occ_bw = fields(T, H, W, 1.0, 0.0, bx=0.0, by=-1.0)       # backward flow unrelated to the forward one
    occ[:] = 1                                                           # forward: lost at the next frame
    occ_bw[0, 1, 5, 8] = 1                                               # frame 2, where the backward walk is at (8, 5)
    tracks, vis = host_track(F, G, occ, occ_bw, Q((3, 8, 6)))
    assert tracks[0, 0].tolist() == [[8, 3], [8, 4], [8, 5], [8, 6], [9, 6], [10, 6], [11, 6]]
    assert vis[0, 0].tolist() == [0, 0, 1, 1, 0, 0, 0]


def test_a_query_on_the_border_samples_clamped_taps():
    T, H, W = 2, 4, 6
    F, G, occ, occ_bw = fields(T, H, W)
    g = torch.Generator().manual_seed(0)
    F[0, 0] = torch.randint(-3, 1, (2, H, W), generator=g).float()      # moves left and up: stays in the frame
    G[0, 0] = -F[0, 0]
    tracks, _ = host_track(F, G, occ, occ_bw, Q((0, W - 1, H - 1), (0, W - 1, 0.5), (0, 0, H - 1)))
    f = F[0, 0]
    assert tracks[0, 0, 1].tolist() == [W - 1 + f[0, H - 1, W - 1].item(), H - 1 + f[1, H - 1, W - 1].item()]
    # x = W-1: both x taps are column W-1 (the right one clamped, weight 0); y = 0.5: rows 0 and 1 weighted 0.5 each
    assert tracks[0, 1, 1, 0].item() == W - 1 + 0.5 * (f[0, 0, W - 1] + f[0, 1, W - 1]).item()
    assert tracks[0, 2, 1].tolist() == [f[0, H - 1, 0].item(), H - 1 + f[1, H - 1, 0].item()]


@pytest.mark.parametrize("x,occluded,visible", [(2.5, 2, 0), (2.5, 3, 1), (3.5, 4, 0), (3.5, 3, 1), (1.5, 2, 0)])
def test_the_mask_is_read_at_rint_with_ties_to_even(x, occluded, visible):
    F, G, occ, occ_bw = fields(2, 3, 8)
    occ[0, 0, 1, occluded] = 1
    assert host_track(F, G, occ, occ_bw, Q((0, x, 1)))[1][0, 0].tolist() == [1, visible]


def shift_truth(T, H, W, dx, dy):
    """The true inputs of a shift_sequence video: F = (dx, dy), G = -F, occ_k where p + F leaves the frame, occ_bw_k where
    p - F does."""
    F, G, occ, occ_bw = fields(T, H, W, float(dx), float(dy))
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    out = lambda x, y: ((x < 0) | (x > W - 1) | (y < 0) | (y > H - 1)).to(torch.uint8)      # noqa: E731
    occ[:] = out(xs + dx, ys + dy)
    occ_bw[:] = out(xs - dx, ys - dy)
    return F, G, occ, occ_bw


@pytest.mark.parametrize("dy,dx", [(3, 4), (-2, 5), (1, -3)])
def test_the_true_flows_of_a_shift_sequence_give_the_true_trajectories(dy, dx):
    T, H, W = 8, 24, 40
    seq = shift_sequence(T, H, W, seed=2, dy=abs(dy), dx=abs(dx))
    if dy > 0 and dx > 0:                                                # the flow really is (dx, dy)
        assert torch.equal(seq[1][:, dy:, dx:], seq[0][:, :H - dy, :W - dx])
    inputs = shift_truth(T, H, W, dx, dy)
    g = torch.Generator().manual_seed(dy * 10 + dx)
    N = 200
    q = torch.stack([torch.randint(0, T, (N,), generator=g).float(), torch.randint(0, W, (N,), generator=g).float(),
                     torch.randint(0, H, (N,), generator=g).float()], -1)[None]
    tracks, vis = host_track(*inputs, q)
    t = torch.arange(T).float()
    gx = q[0, :, 1:2] + (t - q[0, :, :1]) * dx
    gy = q[0, :, 2:3] + (t - q[0, :, :1]) * dy
    gt = torch.stack([gx, gy], -1)[None]
    gvis = ((gx >= 0) & (gx <= W - 1) & (gy >= 0) & (gy <= H - 1)).to(torch.uint8)[None]
    assert torch.equal(tracks, gt) and torch.equal(vis, gvis)
    assert 0 < int(gvis.sum()) < gvis.numel()                            # some points do leave
    s = summarize_tracking(host_track_metrics(tracks, vis, gt, gvis, q, H, W))
    assert s["occlusion_accuracy"] == 1.0 and s["average_pts_within_thresh"] == 1.0 and s["average_jaccard"] == 1.0


def test_points_behind_a_moving_square_are_lost_when_it_covers_them():
    T, H, W, side, y0, x0, d = 8, 20, 48, 6, 7, 2, 4
    F, G, occ, occ_bw = fields(T, H, W)
    rows = slice(y0, y0 + side)
    for k in range(T - 1):
        a, b = x0 + k * d, x0 + (k + 1) * d                              # the square's left column at frames k and k + 1
        F[0, k, 0, rows, a:a + side] = d
        G[0, k, 0, rows, b:b + side] = -d
        cover = torch.zeros(H, W, dtype=torch.bool)
        cover[rows, b:b + side] = True
        here = torch.zeros(H, W, dtype=torch.bool)
        here[rows, a:a + side] = True
        occ[0, k] = (cover & ~here).to(torch.uint8)                      # background frame k+1 hides
        occ_bw[0, k] = (here & ~cover).to(torch.uint8)                   # background frame k showed
    xs = list(range(x0 + side, 40))
    q = Q(*[(0, x, y0 + 2) for x in xs], (0, x0 + 1, y0 + 1), (0, 45, 2))
    tracks, vis = host_track(F, G, occ, occ_bw, q)
    for n, x in enumerate(xs):
        c = next((t for t in range(1, T) if x0 + t * d <= x < x0 + t * d + side), None)    # first frame the square covers x
        want = [1] * T if c is None else [1] * c + [0] * (T - c)
        assert vis[0, n].tolist() == want, (x, c)
        still = T if c is None else c + 1                                # then the square carries it along
        assert (tracks[0, n, :still] == torch.tensor([float(x), y0 + 2.0])).all(), (x, c)
    on = len(xs)
    assert tracks[0, on, :, 0].tolist() == [x0 + 1 + t * d for t in range(T)] and (vis[0, on] == 1).all()
    assert (vis[0, on + 1] == 1).all()


def metrics_numpy(tr, vis, gt, gvis, q, H, W):
    """TAP-Vid's counts written directly in numpy float32 (one rounding per operation, no FMA)."""
    f = np.float32
    tr, gt = tr.numpy().astype(f), gt.numpy().astype(f)
    scale = np.array([W, H], dtype=f)
    d = (tr * f(256)) / scale - (gt * f(256)) / scale
    d2 = d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]
    pv, gv = vis.numpy() != 0, gvis.numpy() != 0
    V, N, T = pv.shape
    ev = np.ones((V, N, T), bool)
    for v in range(V):
        for n in range(N):
            ev[v, n, int(q[v, n, 0])] = False
    out = np.zeros((V, native.TRACK_COUNTS), np.int64)
    for v in range(V):
        e = ev[v]
        out[v, COUNT_EVALUATED] = e.sum()
        out[v, COUNT_OCC_AGREE] = (e & (pv[v] == gv[v])).sum()
        out[v, COUNT_GT_VISIBLE] = (e & gv[v]).sum()
        for j, delta in enumerate(THRESHOLDS):
            w = d2[v] < f(delta * delta)
            out[v, COUNT_WITHIN + j] = (e & w & gv[v]).sum()
            out[v, COUNT_TP + j] = (e & w & gv[v] & pv[v]).sum()
            out[v, COUNT_FP + j] = (e & pv[v] & (~gv[v] | ~w)).sum()
    return torch.from_numpy(out)


def random_tracks(V, N, T, H, W, seed):
    """Predictions near the ground truth with offsets of exactly delta (in 256x256 units when H = W = 256) mixed in."""
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(V, N, T, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0])
    off = torch.randn(V, N, T, 2, generator=g) * 6
    ties = torch.rand(V, N, T, generator=g) < 0.3
    delta = torch.tensor(THRESHOLDS, dtype=torch.float32)[torch.randint(0, 5, (V, N, T), generator=g)]
    off[..., 0] = torch.where(ties, delta, off[..., 0])
    off[..., 1] = torch.where(ties, 0.0, off[..., 1])
    gt = torch.where(ties[..., None], torch.round(gt), gt)
    tr = gt + off
    tr[0, 0, 1] = float("nan")
    vis = (torch.rand(V, N, T, generator=g) < 0.7).to(torch.uint8)
    gvis = torch.rand(V, N, T, generator=g) < 0.6
    q = torch.stack([torch.randint(0, T, (V, N), generator=g).float(), torch.zeros(V, N), torch.zeros(V, N)], -1)
    return tr, vis, gt, gvis, q


@pytest.mark.parametrize("H,W", [(256, 256), (436, 1024), (37, 23)])
def test_host_track_metrics_equal_the_numpy_transcription(H, W):
    tr, vis, gt, gvis, q = random_tracks(3, 40, 9, H, W, seed=H)
    got = host_track_metrics(tr, vis, gt, gvis, q, H, W)
    assert torch.equal(got, metrics_numpy(tr, vis, gt, gvis, q, H, W))
    assert torch.equal(track_metrics(tr, vis, gt, gvis, q, H, W), got)          # CPU tensors take the host path
    assert (got[:, COUNT_EVALUATED] == 40 * 8).all()
    if H == W == 256:                                                   # a tie at exactly delta is not within
        tie = host_track_metrics(torch.tensor([[[[3.0, 5.0], [6.0, 5.0]]]]), torch.ones(1, 1, 2, dtype=torch.uint8),
                                 torch.tensor([[[[3.0, 5.0], [2.0, 5.0]]]]), torch.ones(1, 1, 2, dtype=torch.uint8),
                                 Q((0, 3, 5)), H, W)[0]
        assert tie[COUNT_WITHIN:COUNT_WITHIN + 5].tolist() == [0, 0, 0, 1, 1]     # distance 4: within 8 and 16 only


def test_summarize_tracking_averages_per_video_then_over_videos():
    c = torch.zeros(2, native.TRACK_COUNTS, dtype=torch.int64)
    c[0, :3] = torch.tensor([10, 9, 8])
    c[0, COUNT_WITHIN:COUNT_WITHIN + 5] = torch.tensor([0, 2, 4, 6, 8])
    c[0, COUNT_TP:COUNT_TP + 5] = torch.tensor([0, 2, 4, 6, 8])
    c[0, COUNT_FP:COUNT_FP + 5] = torch.tensor([8, 6, 4, 2, 0])
    c[1, :3] = torch.tensor([4, 2, 4])
    c[1, COUNT_WITHIN:COUNT_WITHIN + 5] = 4
    c[1, COUNT_TP:COUNT_TP + 5] = 2
    s = summarize_tracking(c)
    assert s["videos"] == 2
    assert math.isclose(s["occlusion_accuracy"], (0.9 + 0.5) / 2)
    assert math.isclose(s["pts_within_2"], (2 / 8 + 1) / 2)
    assert math.isclose(s["average_pts_within_thresh"], (0.5 + 1) / 2)
    assert math.isclose(s["jaccard_1"], (0 / 16 + 0.5) / 2) and math.isclose(s["jaccard_16"], (8 / 8 + 0.5) / 2)
    assert math.isclose(s["average_jaccard"], ((0 / 16 + 2 / 14 + 4 / 12 + 6 / 10 + 8 / 8) / 5 + 0.5) / 2)
    assert summarize_tracking([list(r) for r in c.tolist()]) == s
    assert math.isnan(summarize_tracking([])["average_jaccard"])


def test_grid_queries_cover_the_frame_in_row_major_order():
    q = grid_queries(5, 7, 3, stride=2)
    assert q.shape == (12, 3) and q.dtype == torch.float32
    assert q[:5].tolist() == [[3, 0, 0], [3, 2, 0], [3, 4, 0], [3, 6, 0], [3, 0, 2]]
    assert torch.equal(grid_queries(4, 6, 0)[:, 1:], torch.stack(torch.meshgrid(torch.arange(6.0), torch.arange(4.0),
                                                                                 indexing="xy"), -1).reshape(-1, 2))
    with pytest.raises(ValueError):
        grid_queries(4, 4, 0, stride=0)


def test_argument_errors_raise_before_any_launch():
    T, H, W = 4, 6, 9
    F, G, o, ob = fields(T, H, W)
    for bad in ((1.5, 2, 2), (-1, 2, 2), (T, 2, 2), (float("nan"), 2, 2)):
        with pytest.raises(ValueError, match="t must be an integer"):
            track(F, G, o, ob, Q(bad))
    for bad in ((0, -0.1, 2), (0, W - 1 + 0.01, 2), (0, 2, H), (0, 2, -1e-6), (0, float("nan"), 1), (0, 1, float("inf"))):
        with pytest.raises(ValueError, match="must lie in"):
            track(F, G, o, ob, Q(bad))
    ok = Q((0, 1, 1))
    with pytest.raises(ValueError, match="T >= 2"):
        track(F[:, :0], G[:, :0], o[:, :0], ob[:, :0], ok)
    with pytest.raises(ValueError, match="flow_bw"):
        track(F, G[..., :5], o, ob, ok)
    with pytest.raises(ValueError, match="flow and flow_bw"):
        track(F[0], G[0], o, ob, ok)
    with pytest.raises(ValueError, match="occ_bw"):
        track(F, G, o, ob[:, :2], ok)
    with pytest.raises(ValueError, match="expected occ "):
        track(F, G, o[..., 1:], ob, ok)
    with pytest.raises(ValueError, match="queries"):
        track(F, G, o, ob, ok[0])
    with pytest.raises(ValueError, match="queries"):
        track(F, G, o, ob, torch.zeros(2, 1, 3))
    with pytest.raises(ValueError, match="queries"):
        track(F, G, o, ob, torch.zeros(1, 1, 2))
    with pytest.raises(ValueError, match="one device"):
        track(F, G.to("meta"), o, ob, ok)
    tr, vis = host_track(F, G, o, ob, ok)
    with pytest.raises(ValueError, match="tracks and gt_tracks"):
        track_metrics(tr, vis, tr[:, :, :2], vis, ok, H, W)
    with pytest.raises(ValueError, match="gt_visible"):
        track_metrics(tr, vis, tr, vis[..., :2], ok, H, W)
    with pytest.raises(ValueError, match="queries"):
        track_metrics(tr, vis, tr, vis, ok[:, :, :2], H, W)
    with pytest.raises(ValueError, match="t must be an integer"):
        track_metrics(tr, vis, tr, vis, Q((T, 1, 1)), H, W)


def test_track_points_checks_its_arguments():
    from rnc.harness import track_points
    from rnc.synth import build_model
    m = build_model("raft")
    seqs = [[torch.zeros(3, 16, 16)] * 3]
    with pytest.raises(ValueError, match="inference only"):
        track_points(m, seqs, [Q((0, 1, 1))[0]])
    with torch.no_grad():
        with pytest.raises(ValueError, match="1 videos but 2 query sets"):
            track_points(m, seqs, [Q((0, 1, 1))[0]] * 2)
        with pytest.raises(ValueError, match="T >= 2"):
            track_points(m, [[torch.zeros(3, 16, 16)]], [Q((0, 1, 1))[0]])
        with pytest.raises(ValueError, match="t must be an integer"):
            track_points(m, seqs, [Q((3, 1, 1))[0]])
        with pytest.raises(ValueError, match="must lie in"):
            track_points(m, seqs, [Q((0, 16, 1))[0]])
        assert track_points(m, [], []) == []


# ----------------------------------------------------------------------------- validate_tracking under torch.distributed


class _InferenceModel:
    def _needs_grad(self):
        return False


def _stub_bidirectional(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                        alpha1=0.01, alpha2=0.5):
    """run_sequences_bidirectional's yields in its step order, on the CPU: flows from the frames' first channels, masks from
    a threshold on the third."""
    from rnc.harness import sequence_schedule
    for step in sequence_schedule([len(s) for s in sequences], batch_size):
        for c in step:
            if not c.idle:
                a, b = sequences[c.seq][c.pair], sequences[c.seq][c.pair + 1]
                yield c.seq, c.pair, {"flow_up": (b[:2] - a[:2]) / 64, "flow_up_bw": (a[1:] - b[1:]) / 64,
                                      "occ": (a[2] > 230).to(torch.uint8), "occ_bw": (b[2] > 230).to(torch.uint8)}


def tracking_split():
    """Six videos of 2 to 7 frames with 5 to 40 queries each, and a perturbed ground truth."""
    H, W = 12, 20
    seqs, qs, gts, gvs = [], [], [], []
    for k, (n, N) in enumerate(((5, 12), (2, 5), (7, 40), (3, 9), (6, 17), (4, 30))):
        seqs.append(shift_sequence(n, H, W, seed=k, dy=k % 3, dx=2))
        g = torch.Generator().manual_seed(k)
        qs.append(torch.stack([torch.randint(0, n, (N,), generator=g).float(), torch.rand(N, generator=g) * (W - 1),
                               torch.rand(N, generator=g) * (H - 1)], -1))
        gts.append(torch.rand(N, n, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0]))
        gvs.append(torch.rand(N, n, generator=g) < 0.8)
    return seqs, qs, gts, gvs


def _tracking_worker(rank, world, port, q):
    import torch.distributed as dist
    from rnc import harness
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        harness.run_sequences_bidirectional = _stub_bidirectional
        q.put((rank, harness.validate_tracking(_InferenceModel(), *tracking_split(), batch_size=2, device="cpu")))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_validate_tracking_gloo_equals_world_1(world, monkeypatch):
    from test_flow_metrics import run_ranks
    from rnc import harness
    monkeypatch.setattr(harness, "run_sequences_bidirectional", _stub_bidirectional)
    seqs, qs, gts, gvs = tracking_split()
    want = harness.validate_tracking(_InferenceModel(), seqs, qs, gts, gvs, batch_size=2, device="cpu")
    counts = []                                         # per video, as the host defines it
    for seq, q, gt, gv in zip(seqs, qs, gts, gvs):
        r = [x[2] for x in _stub_bidirectional(None, [seq])]
        stack = [torch.stack([p[name] for p in r])[None] for name in ("flow_up", "flow_up_bw", "occ", "occ_bw")]
        tr, vis = host_track(*stack, q[None])
        counts.append(host_track_metrics(tr, vis, gt[None], gv[None], q[None], 12, 20)[0])
    assert want == summarize_tracking(torch.stack(counts)) and want["videos"] == len(seqs)
    for got in run_ranks(_tracking_worker, world):
        assert got == want                              # bit for bit, on every rank


# ----------------------------------------------------------------------------- C ABI


_CTYPE = {"long long": native.C.c_longlong, "int": native.C.c_int, "size_t": native.C.c_size_t, "float": native.C.c_float}


def test_declarations_match_the_binding():
    with open(os.path.join(ROOT, "include", "rnc.h")) as f:
        header = f.read()
    assert f"#define RNC_TRACK_THRESHOLDS {native.TRACK_THRESHOLDS}" in header
    assert f"#define RNC_TRACK_COUNTS {native.TRACK_COUNTS}" in header
    for name in ("rnc_track", "rnc_track_metrics_workspace_bytes", "rnc_track_metrics"):
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

    def tr(V=2, N=100, T=5, H=40, W=60, flow=P, bw=P, occ=P, ob=P, q=P, tracks=P, vis=P):
        s5, s4 = (1, 1, 1, 1, 1), (1, 1, 1, 1)
        return L.rnc_track(flow, *s5, bw, *s5, occ, *s4, ob, *s4, q, V, N, T, H, W, tracks, vis, None)

    for bad in (dict(V=0), dict(V=65536), dict(N=0), dict(T=1), dict(H=0), dict(W=-1), dict(W=(1 << 24) + 1),
                dict(N=1 << 28, T=4)):
        assert tr(**bad) == -1, bad
    for bad in (dict(flow=0), dict(bw=0), dict(occ=0), dict(ob=0), dict(q=0), dict(tracks=0), dict(vis=0),
                dict(flow=P + 2), dict(q=P + 1), dict(tracks=P + 4)):
        assert tr(**bad) == -2, bad
    ws = L.rnc_track_metrics_workspace_bytes(3, 1000, 50)
    assert ws == 3 * 25 * 72 and L.rnc_track_metrics_workspace_bytes(0, 5, 5) == 0
    assert L.rnc_track_metrics_workspace_bytes(1, 5, 1) == 0 and L.rnc_track_metrics_workspace_bytes(1, 1 << 28, 4) == 0

    def met(V=3, N=1000, T=50, H=40, W=60, a=P, b=P, c=P, d=P, q=P, counts=P, wsp=P, wsb=ws):
        return L.rnc_track_metrics(a, b, c, d, q, V, N, T, H, W, counts, wsp, wsb, None)

    for bad in (dict(V=0), dict(T=1), dict(N=0), dict(H=0), dict(W=0)):
        assert met(**bad) == -1, bad
    for bad in (dict(a=0), dict(b=0), dict(c=0), dict(d=0), dict(q=0), dict(counts=0), dict(wsp=0), dict(a=P + 4),
                dict(c=P + 4), dict(counts=P + 4), dict(wsp=P + 8)):
        assert met(**bad) == -2, bad
    assert met(wsb=ws - 1) == -5
    assert L.rnc_launch_count() == n0


def test_track_cu_has_no_atomics_and_does_not_spill(tmp_path):
    from rnc.build import ARCH, CSRC, nvcc_path
    cubin = str(tmp_path / "t.cubin")
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-cubin", os.path.join(CSRC, "track.cu"), "-o", cubin]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    kernels = re.findall(r"Function properties for \S*?\d((?:track|cta_partials|image_reduce)_kernel)", log)
    assert sorted(kernels) == ["cta_partials_kernel", "image_reduce_kernel", "track_kernel"], kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 3 and all(a == "0" and b == "0" for a, b in spills), spills
    assert re.findall(r"(\d+) bytes stack frame", log) == ["0"] * 3
    cuobjdump = os.path.join(os.path.dirname(nvcc_path()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    assert "FFMA" not in sass.split("track_kernel", 1)[1].split("Function :", 1)[0]      # every operation rounded once
    assert not re.search(r"\b(ATOM|ATOMS|ATOMG|RED)\b", sass)
