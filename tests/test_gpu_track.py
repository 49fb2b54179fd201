"""Point tracking on the GPU (rnc_track, rnc_track_metrics): the kernels against the host oracle bit for bit, batch
independence and repeatability, and track_points and validate_tracking against run_sequences_bidirectional's outputs tracked
and scored on the host."""
import pytest
import torch
import torch.nn.functional as F

from conftest import build_model
from rnc.harness import run_sequences_bidirectional, track_points, validate_tracking
from rnc.synth import shift_sequence
from rnc.track import grid_queries, host_track, host_track_metrics, summarize_tracking, track, track_metrics

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def random_video(V, T, H, W, seed, scale=4.0, special=True):
    """Smooth random flows (bilinear-upsampled noise) with NaN and inf entries, random masks, queries in every frame."""
    g = torch.Generator().manual_seed(seed)

    def smooth():
        low = torch.randn(V * (T - 1), 2, max(H // 8, 2), max(W // 8, 2), generator=g) * scale
        return F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False).view(V, T - 1, 2, H, W)
    flow, flow_bw = smooth(), smooth()
    if special:
        flow[0, 0, 0, 3:6, 4:9] = float("nan")
        flow[-1, T // 2, 1, H // 2, :] = float("inf")
        flow_bw[0, T - 2, 0, :, W // 3] = -float("inf")
        flow_bw[-1, 0, 1, 1, 1] = float("nan")
    occ = (torch.rand(V, T - 1, H, W, generator=g) < 0.05).to(torch.uint8)
    occ_bw = (torch.rand(V, T - 1, H, W, generator=g) < 0.05).to(torch.uint8)
    N = 6 * T
    q = torch.stack([torch.arange(N).remainder(T).float().expand(V, N), torch.rand(V, N, generator=g) * (W - 1),
                     torch.rand(V, N, generator=g) * (H - 1)], -1)
    q[:, :T, 1:] = torch.round(q[:, :T, 1:])                    # some on pixel centres
    q[0, 0, 1:] = torch.tensor([W - 1.0, H - 1.0])              # a corner
    return flow, flow_bw, occ, occ_bw, q


def same(a, b):
    return a.shape == b.shape and bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def test_track_equals_the_host_oracle_on_random_fields():
    cpu = random_video(3, 7, 23, 37, seed=1)
    tracks, vis = track(*(t.to(DEV) for t in cpu))
    want_t, want_v = host_track(*cpu)
    assert same(tracks.cpu(), want_t) and torch.equal(vis.cpu(), want_v)
    assert 0 < int(vis.sum()) < vis.numel()


def test_track_reads_strided_inputs():
    V, T, H, W = 2, 5, 30, 44
    flow, flow_bw, occ, occ_bw, q = random_video(V, T, H, W, seed=2)
    big = torch.zeros(V, T - 1, 3, H + 3, W + 5)
    big[:, :, 1:, 2:H + 2, 3:W + 3] = flow
    fv = big.to(DEV)[:, :, 1:, 2:H + 2, 3:W + 3]                # strided in every dimension but x
    ov = occ.to(DEV).transpose(-1, -2).contiguous().transpose(-1, -2)       # an x-major mask
    got = track(fv, flow_bw.to(DEV), ov, occ_bw.to(DEV), q.to(DEV))
    assert not fv.is_contiguous() and not ov.is_contiguous()
    want = host_track(flow, flow_bw, occ, occ_bw, q)
    assert same(got[0].cpu(), want[0]) and torch.equal(got[1].cpu(), want[1])


def test_dense_tracking_at_sintel_size_equals_the_host_oracle():
    T, H, W = 12, 436, 1024
    flow, flow_bw, occ, occ_bw, _ = random_video(1, T, H, W, seed=3, scale=12.0)
    q = grid_queries(H, W, 0, stride=4)[None]
    tracks, vis = track(flow.to(DEV), flow_bw.to(DEV), occ.to(DEV), occ_bw.to(DEV), q.to(DEV))
    want_t, want_v = host_track(flow, flow_bw, occ, occ_bw, q)
    assert same(tracks.cpu(), want_t) and torch.equal(vis.cpu(), want_v)
    q5 = grid_queries(H, W, 5, stride=4)[None]                  # a middle frame: both directions
    tracks, vis = track(flow.to(DEV), flow_bw.to(DEV), occ.to(DEV), occ_bw.to(DEV), q5.to(DEV))
    want_t, want_v = host_track(flow, flow_bw, occ, occ_bw, q5)
    assert same(tracks.cpu(), want_t) and torch.equal(vis.cpu(), want_v)


def test_a_video_is_the_same_alone_or_in_a_batch_and_from_call_to_call():
    dev = [t.to(DEV) for t in random_video(5, 9, 40, 64, seed=4)]
    full = track(*dev)
    again = track(*dev)
    assert torch.equal(full[1], again[1]) and same(full[0], again[0])
    one = track(*(t[3:4] for t in dev))
    assert same(one[0][0], full[0][3]) and torch.equal(one[1][0], full[1][3])


@pytest.mark.parametrize("V", [1, 5])
def test_track_metrics_counts_equal_the_host(V):
    H, W, T = 48, 80, 10
    cpu = random_video(V, T, H, W, seed=5 + V)
    tracks, vis = host_track(*cpu)
    q = cpu[4]
    g = torch.Generator().manual_seed(V)
    gt = tracks + torch.randn(tracks.shape, generator=g) * 0.6
    gt[..., 1] = torch.where(torch.rand(gt.shape[:3], generator=g) < 0.2, tracks[..., 1] + 0.5, gt[..., 1])   # ties
    gvis = (torch.rand(vis.shape, generator=g) < 0.8).to(torch.uint8)
    want = host_track_metrics(tracks, vis, gt, gvis, q, H, W)
    got = track_metrics(*(t.to(DEV) for t in (tracks, vis, gt, gvis, q)), H, W)
    assert torch.equal(got.cpu(), want)
    if V == 5:
        one = track_metrics(*(t[2:3].to(DEV) for t in (tracks, vis, gt, gvis, q)), H, W)
        assert torch.equal(one[0], got[2])


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


H, W, ITERS = 64, 128, 6


def videos():
    seqs = [[f.to(DEV) for f in shift_sequence(n, H, W, seed=s, dy=1, dx=2)] for s, n in enumerate((5, 3))]
    g = torch.Generator().manual_seed(11)
    qs = [grid_queries(H, W, 0, stride=8),
          torch.stack([torch.randint(0, 3, (40,), generator=g).float(), torch.rand(40, generator=g) * (W - 1),
                       torch.rand(40, generator=g) * (H - 1)], -1)]
    return seqs, qs


def host_tracks(m, seqs, qs, warm_start):
    """run_sequences_bidirectional's outputs collected per video, then host_track of each video alone."""
    got = {}
    for s, k, r in run_sequences_bidirectional(m, seqs, ITERS, warm_start=warm_start, batch_size=2, device=DEV):
        got[s, k] = {name: r[name].cpu() for name in ("flow_up", "flow_up_bw", "occ", "occ_bw")}
    out = []
    for s, q in enumerate(qs):
        stack = [torch.stack([got[s, k][name] for k in range(len(seqs[s]) - 1)])[None]
                 for name in ("flow_up", "flow_up_bw", "occ", "occ_bw")]
        tr, vis = host_track(*stack, q[None])
        out.append((tr[0], vis[0]))
    return out


@pytest.mark.parametrize("warm_start", [False, True])
def test_track_points_is_the_sequence_pass_then_host_track(warm_start, monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft_nc_dbl").to(DEV)
    seqs, qs = videos()
    with torch.no_grad():
        got = track_points(m, seqs, qs, ITERS, warm_start=warm_start, batch_size=2, device=DEV)
        want = host_tracks(m, seqs, qs, warm_start)
    assert len(got) == 2
    for (tr, vis), (wt, wv), seq, q in zip(got, want, seqs, qs):
        assert tr.shape == (q.shape[0], len(seq), 2) and vis.shape == (q.shape[0], len(seq))
        assert tr.is_cuda and same(tr.cpu(), wt) and torch.equal(vis.cpu(), wv)


def test_validate_tracking_equals_the_host_counts(monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft").to(DEV)
    seqs, qs = videos()
    gts, gvs = [], []
    for seq, q in zip(seqs, qs):                                # the true motion of shift_sequence: (2, 1) per frame
        t = torch.arange(len(seq)).float()
        gx = q[:, 1:2] + (t - q[:, :1]) * 2
        gy = q[:, 2:3] + (t - q[:, :1])
        gts.append(torch.stack([gx, gy], -1))
        gvs.append((gx <= W - 1) & (gy <= H - 1) & (gx >= 0) & (gy >= 0))
    res = validate_tracking(m, seqs, qs, gts, gvs, ITERS, batch_size=2, device=DEV)
    with torch.no_grad():
        mine = host_tracks(m, seqs, qs, False)
    counts = torch.cat([host_track_metrics(tr[None], vis[None], gt[None], gv[None], q[None], H, W)
                        for (tr, vis), gt, gv, q in zip(mine, gts, gvs, qs)])
    assert res == summarize_tracking(counts) and res["videos"] == 2
    print(res)
