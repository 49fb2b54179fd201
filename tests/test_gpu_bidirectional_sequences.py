"""Bidirectional sequence inference on the GPU (rnc.harness.run_sequences_bidirectional): five sequences of 2, 3, 4, 6 and 7
frames at 128x256 in three slots, so that slots restart and go idle, give per pair what bidirectional_flow gives one pair
at a time with the two warm-start rules, on both models, both encoder routes, cold and warm; the forward rows are
run_sequences' flows; every frame is encoded once."""
import pytest
import torch

from conftest import build_model
from rnc.harness import bidirectional_flow, bidirectional_warm_start, run_sequences, run_sequences_bidirectional, \
    sequence_schedule
from rnc.metrics import fb_consistency
from rnc.synth import frames, shift_sequence
from utils.utils import forward_interpolate

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LENS = [2, 3, 4, 6, 7]
H, W, B, ITERS = 128, 256, 3, 12
KEYS = ("flow_low", "flow_up", "flow_low_bw", "flow_up_bw", "occ", "occ_bw", "fb_err", "fb_err_bw")
FLOWS = ("flow_low", "flow_up", "flow_low_bw", "flow_up_bw")


def random_sequences():
    return [[frames(1, H, W, seed=100 * s + t)[0][0].to(DEV) for t in range(n)] for s, n in enumerate(LENS)]


def shift_sequences():
    return [[f.to(DEV) for f in shift_sequence(n, H, W, seed=s)] for s, n in enumerate(LENS)]


def sequenced(m, seqs, warm, conf=False, between=None):
    got = {}
    for s, p, r in run_sequences_bidirectional(m, seqs, ITERS, warm_start=warm, batch_size=B, device=DEV,
                                               return_confidence=conf):
        assert (s, p) not in got
        assert r["flow_up"].shape == r["flow_up_bw"].shape == (2, H, W) and r["occ"].shape == (H, W)
        assert r["flow_low"].shape == (2, H // 8, W // 8) and all(v.is_cuda for v in r.values())
        got[(s, p)] = r
        if between is not None:
            between()
    return got


def pairwise(m, seqs, warm, conf=False):
    """The one-pair-at-a-time loop: bidirectional_flow per pair, warm-started from the previous pair's low-resolution flows
    by forward_interpolate (forward) and -forward_interpolate(-b) (backward)."""
    want = {}
    for s, seq in enumerate(seqs):
        prev = None
        for k in range(len(seq) - 1):
            fi = None
            if warm and prev is not None:
                fi = (forward_interpolate(prev["flow_low"]), -forward_interpolate(-prev["flow_low_bw"]))
            prev = bidirectional_flow(m, seq[k][None], seq[k + 1][None], ITERS, flow_init=fi, return_confidence=conf)
            want[(s, k)] = {key: v[0] for key, v in prev.items()}
    return want


def worst_epe(got, want):
    return max((got[k][key] - want[k][key]).pow(2).sum(0).sqrt().mean().item() for k in want for key in FLOWS)


@pytest.fixture(autouse=True)
def inference():
    """run_sequences_bidirectional and bidirectional_flow are inference only: they raise with grad enabled."""
    with torch.no_grad():
        yield


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def test_two_direction_warm_start_equals_the_oracle():
    from oracle import raft_oracle as orc
    g = torch.Generator().manual_seed(11)
    nb = 3
    f = torch.randn(2 * nb, 2, 40, 64, generator=g) * 5
    out = bidirectional_warm_start(f.to(DEV)).cpu()
    for j in range(nb):
        assert torch.equal(out[j], orc.forward_interpolate(f[j])), j
        assert torch.equal(out[nb + j], -orc.forward_interpolate(-f[nb + j])), nb + j
    assert torch.equal(out[:nb], forward_interpolate(f[:nb].to(DEV)).cpu())


@pytest.mark.parametrize("warm", [False, True])
@pytest.mark.parametrize("name,conf", [("raft_nc_dbl", False), ("raft_nc_dbl", True), ("raft", False)])
def test_bit_identical_to_the_pairwise_loop_with_the_exact_lookup(name, conf, warm, monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model(name).to(DEV)
    seqs = shift_sequences() if warm else random_sequences()
    got, want = sequenced(m, seqs, warm, conf), pairwise(m, seqs, warm, conf)
    assert got.keys() == want.keys()
    keys = KEYS + (("confidence", "confidence_bw") if conf else ())
    for k in want:
        assert set(got[k]) == set(keys)
    bad = [(k, key) for k in want for key in keys if not torch.equal(got[k][key], want[k][key])]
    assert not bad, f"{len(bad)} of {len(want) * len(keys)} results differ, worst flow EPE {worst_epe(got, want):.3e}: {bad}"
    fw = {(s, p): f for s, p, f in run_sequences(m, seqs, ITERS, warm_start=warm, batch_size=B, device=DEV)}
    assert fw.keys() == got.keys()
    assert all(torch.equal(fw[k], got[k]["flow_up"]) for k in fw)


@pytest.mark.parametrize("warm", [False, True])
@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_default_mode_matches_the_pairwise_loop(name, warm):
    m = build_model(name).to(DEV)
    seqs = shift_sequences() if warm else random_sequences()
    got, want = sequenced(m, seqs, warm), pairwise(m, seqs, warm)
    e = worst_epe(got, want)
    print(f"{name} warm={warm}: worst EPE vs the pairwise loop {e:.2e}")
    assert e <= (1e-3 if warm else 1e-4)


@pytest.mark.parametrize("warm", [False, True])
def test_torch_encoder_route_matches_the_pairwise_loop(warm, monkeypatch):
    monkeypatch.setenv("RNC_ENCODER", "cudnn")
    m = build_model("raft_nc_dbl").to(DEV)
    seqs = shift_sequences() if warm else random_sequences()
    got, want = sequenced(m, seqs, warm), pairwise(m, seqs, warm)
    e = worst_epe(got, want)
    print(f"cudnn encoders warm={warm}: worst EPE vs the pairwise loop {e:.2e}")
    assert e <= (1e-3 if warm else 1e-4)


def test_masks_are_fb_consistency_of_the_yielded_flows():
    m = build_model("raft_nc_dbl").to(DEV)
    n = 0
    for _, _, r in run_sequences_bidirectional(m, shift_sequences(), ITERS, warm_start=True, batch_size=B, device=DEV,
                                               alpha1=0.02, alpha2=0.7):
        want = fb_consistency(r["flow_up"][None], r["flow_up_bw"][None], 0.02, 0.7)
        for key, w in zip(("occ", "occ_bw", "fb_err", "fb_err_bw"), want):
            assert torch.equal(r[key], w[0]), key
        n += 1
    assert n == sum(LENS) - len(LENS)


def test_other_forwards_between_steps_change_nothing(monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model("raft_nc_dbl").to(DEV)
    seqs = shift_sequences()
    x1, x2 = (x.to(DEV) for x in frames(B, H, W, seed=9))

    def other():
        m(x1, x2, iters=ITERS, test_mode=True)
        bidirectional_flow(m, x1, x2, ITERS)                 # the same 2B-slot shape as the generator's workspace
    want = sequenced(m, seqs, True)
    got = sequenced(m, seqs, True, between=other)
    bad = [(k, key) for k in want for key in KEYS if not torch.equal(got[k][key], want[k][key])]
    assert not bad, bad


def test_encoders_run_on_each_new_frame_once(monkeypatch):
    from rnc.encoder_umma import EncoderRunner
    m = build_model("raft_nc_dbl").to(DEV)
    if m.engine().mode != "umma":
        pytest.skip("tensor-core encoders only")
    images = {"instance": 0, "batch": 0}
    trunk = EncoderRunner._trunk

    def counted(self, pk, bufs, image, N, Hin, Win):
        assert image.shape[0] == N
        images[pk.kind] += N
        return trunk(self, pk, bufs, image, N, Hin, Win)

    monkeypatch.setattr(EncoderRunner, "_trunk", counted)
    n = sum(1 for _ in run_sequences_bidirectional(m, random_sequences(), iters=2, batch_size=B, device=DEV))
    steps = sequence_schedule(LENS, B)
    idle = sum(c.idle for step in steps for c in step)
    assert n == sum(LENS) - len(LENS)
    # fnet and cnet each see every frame once, plus frame 2 of each idle slot-step (an idle slot recomputes its last pair)
    assert images == {"instance": sum(LENS) + idle, "batch": sum(LENS) + idle}, images


def test_model_on_another_device_raises():
    m = build_model("raft_nc_dbl")
    with pytest.raises(ValueError, match="model parameters are on cpu"):
        next(run_sequences_bidirectional(m, shift_sequences(), ITERS, batch_size=B, device=DEV))
