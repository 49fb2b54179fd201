"""Sequence inference on the GPU (rnc.harness.run_sequences): five sequences of 2, 3, 4, 6 and 7 frames at 128x256 in three
slots, so that slots restart and go idle, give per sequence the flows of run_sequence, with and without warm start, on both
models and on both encoder routes; fnet encodes every frame once."""
import pytest
import torch

from conftest import build_model
from rnc.harness import run_sequence, run_sequences, sequence_schedule
from rnc.synth import frames, shift_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LENS = [2, 3, 4, 6, 7]
H, W, B, ITERS = 128, 256, 3, 12


def random_sequences():
    return [[frames(1, H, W, seed=100 * s + t)[0][0] for t in range(n)] for s, n in enumerate(LENS)]


def shift_sequences():
    return [shift_sequence(n, H, W, seed=s) for s, n in enumerate(LENS)]


def both(m, seqs, warm):
    """(run_sequences' flows by (seq, pair), run_sequence's)."""
    got = {}
    for s, p, flow in run_sequences(m, seqs, iters=ITERS, warm_start=warm, batch_size=B, device=DEV):
        assert flow.is_cuda and flow.shape == (2, H, W) and (s, p) not in got
        got[(s, p)] = flow.cpu()
    want = {(s, p): f for s, seq in enumerate(seqs) for p, f in enumerate(run_sequence(m, seq, ITERS, warm, device=DEV))}
    assert got.keys() == want.keys()
    return got, want


def worst_epe(got, want):
    return max((got[k] - want[k]).pow(2).sum(0).sqrt().mean().item() for k in want)


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


@pytest.mark.parametrize("warm", [False, True])
@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_bit_identical_to_run_sequence_with_the_exact_lookup(name, warm, monkeypatch, det):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    m = build_model(name).to(DEV)
    got, want = both(m, shift_sequences() if warm else random_sequences(), warm)
    bad = [k for k in want if not torch.equal(got[k], want[k])]
    assert not bad, f"{len(bad)} of {len(want)} pairs differ, worst EPE {worst_epe(got, want):.3e}: {bad}"


@pytest.mark.parametrize("warm", [False, True])
@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_default_mode_matches_run_sequence(name, warm):
    m = build_model(name).to(DEV)
    got, want = both(m, shift_sequences() if warm else random_sequences(), warm)
    e = worst_epe(got, want)
    print(f"{name} warm={warm}: worst EPE vs run_sequence {e:.2e}")
    assert e <= (1e-3 if warm else 1e-4)


@pytest.mark.parametrize("warm", [False, True])
def test_torch_encoder_route_matches_run_sequence(warm, monkeypatch):
    monkeypatch.setenv("RNC_ENCODER", "cudnn")
    m = build_model("raft_nc_dbl").to(DEV)
    got, want = both(m, shift_sequences() if warm else random_sequences(), warm)
    e = worst_epe(got, want)
    print(f"cudnn encoders warm={warm}: worst EPE vs run_sequence {e:.2e}")
    assert e <= (1e-3 if warm else 1e-4)


def test_fnet_encodes_each_frame_once(monkeypatch):
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
    seqs = random_sequences()
    n = sum(1 for _ in run_sequences(m, seqs, iters=2, batch_size=B, device=DEV))
    steps = sequence_schedule(LENS, B)
    idle = sum(c.idle for step in steps for c in step)
    assert n == sum(LENS) - len(LENS)
    # every frame once, plus frame 2 of each idle slot-step (an idle slot recomputes its last pair); cnet on every slot
    assert images["instance"] == sum(LENS) + idle, images
    assert images["batch"] == B * len(steps), images
