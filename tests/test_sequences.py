"""Sequence inference on the host: the slot schedule of rnc.harness.run_sequences and its argument checks."""
import pytest
import torch

from rnc.harness import run_sequences, sequence_schedule
from rnc.synth import shift_sequence

CASES = [
    ([2], 1), ([2], 4), ([1], 3), ([1, 1], 2), ([], 8),
    ([2, 3, 4, 6, 7], 3), ([7, 6, 4, 3, 2], 3), ([2, 3, 4, 6, 7], 8), ([2, 3, 4, 6, 7], 1),
    ([5, 1, 2, 9, 1, 3], 2), ([2] * 9, 4), ([20, 50, 33, 41, 27, 45, 38, 22, 49, 30, 36, 25], 8),
]


def check(lengths, B):
    steps = sequence_schedule(lengths, B)
    live = [s for s, n in enumerate(lengths) if n >= 2]
    nslot = min(B, len(live))
    seen = {}                                   # seq -> pairs in the order they ran
    started = []                                # sequences in the order they started
    last_start = max((t for t, step in enumerate(steps) for c in step if c.restart), default=None)
    for t, step in enumerate(steps):
        assert len(step) == nslot
        for j, c in enumerate(step):
            prev = steps[t - 1][j] if t else None
            if c.idle:
                # an idle slot repeats its previous (seq, pair) and only after the last sequence has started
                assert prev is not None and (c.seq, c.pair) == (prev.seq, prev.pair) and not c.restart
                assert t >= last_start
                continue
            assert c.restart == (c.pair == 0)
            if c.restart:
                started.append(c.seq)
                if len(started) > nslot:        # a sequence after the first B restarts a slot whose sequence just ended
                    assert prev is not None and not prev.idle and prev.pair == lengths[prev.seq] - 2
                else:
                    assert t == 0
            else:
                assert prev is not None and not prev.idle and (prev.seq, prev.pair + 1) == (c.seq, c.pair)
            seen.setdefault(c.seq, []).append(c.pair)
        assert any(not c.idle for c in step)
    assert started == live
    assert seen == {s: list(range(lengths[s] - 1)) for s in live}
    return steps


@pytest.mark.parametrize("lengths,B", CASES)
def test_schedule_runs_every_pair_once_in_order(lengths, B):
    check(lengths, B)


def test_schedule_restarts_and_idle_slots():
    steps = check([2, 3, 4, 6, 7], 3)
    # slots: 0 -> seq 0 (1 pair) then seq 3 (5 pairs); 1 -> seq 1 (2) then seq 4 (6); 2 -> seq 2 (3 pairs), then idle
    assert [(c.seq, c.pair, c.restart, c.idle) for c in steps[1]] == [(3, 0, True, False), (1, 1, False, False), (2, 1, False, False)]
    assert len(steps) == 8
    idle = sum(c.idle for step in steps for c in step)
    assert idle == len(steps) * 3 - (1 + 2 + 3 + 5 + 6)
    assert sequence_schedule([2, 3], 8) and all(len(s) == 2 for s in sequence_schedule([2, 3], 8))
    assert sequence_schedule([1, 0], 4) == []
    with pytest.raises(ValueError):
        sequence_schedule([2], 0)


def test_mismatched_frame_sizes_raise():
    seqs = [[torch.zeros(3, 64, 96)] * 3, [torch.zeros(3, 64, 96), torch.zeros(3, 64, 104)]]
    with pytest.raises(ValueError, match=r"\(3, 64, 96\) and \(3, 64, 104\)"):
        next(run_sequences(None, seqs, device="cpu"))


def test_one_frame_sequences_yield_nothing():
    assert list(run_sequences(None, [[torch.zeros(3, 64, 96)]], device="cpu")) == []


def test_shift_sequence_is_a_translation():
    fr = shift_sequence(4, 40, 56, dy=3, dx=4)
    assert len(fr) == 4 and all(f.shape == (3, 40, 56) for f in fr)
    for a, b in zip(fr[:-1], fr[1:]):
        assert torch.equal(b[:, 3:, 4:], a[:, :-3, :-4])      # content at (y, x) of frame t is at (y + 3, x + 4) of frame t + 1
