"""Slot plans of the encoder stage (rnc.slot_plan) on the host: an interpreter applies each plan to frame labels instead of
tensors, and checks what every slot holds after each call of the pair forward, the bidirectional pass and the two kinds of
sequence step, which images the encoders see, and how often."""
import pytest

from rnc.harness import sequence_schedule
from rnc.slot_plan import CARRY, NEW, SAVED, runs, slot_plan

from test_sequences import CASES


def apply(plan, slots, saved, label):
    """One encoder call on labels.  slots: per slot (f1, f2, ctx) of the last call (None before the first); saved: slot ->
    context saved by the last call; label(frame, row) -> the frame an image is.  Returns the new (slots, saved)."""
    fnet = [label(*e) for e in plan.fnet_in]
    cnet = [label(*e) for e in plan.cnet_in]

    def get(src, j, field, new):
        if src is None:
            return slots[j][field]
        kind, i = src
        if kind == NEW:
            return new[i]
        if kind == CARRY:
            return slots[i][1]
        assert kind == SAVED and i in saved
        return saved[i]
    out = [(get(plan.f1[j], j, 0, fnet), get(plan.f2[j], j, 1, fnet), get(plan.ctx[j], j, 2, cnet))
           for j in range(len(plan.f1))]
    return out, {s: out[s][2] for s in plan.save}


@pytest.mark.parametrize("B", [1, 2, 3, 8])
@pytest.mark.parametrize("bidirectional", [False, True])
def test_pair_and_bidirectional_plans(B, bidirectional):
    plan = slot_plan(B, bidirectional=bidirectional)
    both = [(1, j) for j in range(B)] + [(2, j) for j in range(B)]
    assert plan.fnet_in == both
    assert plan.cnet_in == (both if bidirectional else both[:B])
    assert not plan.save
    slots, _ = apply(plan, [None] * len(plan.f1), {}, lambda f, r: (r, f))
    want = [((j, 1), (j, 2), (j, 1)) for j in range(B)]
    if bidirectional:
        want += [((j, 2), (j, 1), (j, 2)) for j in range(B)]
    assert slots == want


@pytest.mark.parametrize("bidirectional", [False, True])
@pytest.mark.parametrize("lengths,B", CASES)
def test_sequence_step_plans(lengths, B, bidirectional):
    steps = sequence_schedule(lengths, B)
    if not steps:
        return
    B = len(steps[0])
    S = 2 * B if bidirectional else B
    slots, saved = [None] * S, {}
    fnet = cnet = 0
    for t, step in enumerate(steps):
        restart = [j for j, c in enumerate(step) if c.restart]
        carry = [j for j, c in enumerate(step) if not c.restart and not c.idle]
        plan = slot_plan(B, carry, restart, bidirectional)
        new_frames = [(2, j) for j in range(B)] + [(1, j) for j in restart]
        assert plan.fnet_in == new_frames
        assert plan.cnet_in == (new_frames if bidirectional else [(1, j) for j in range(B)])
        assert list(plan.save) == (list(range(B, 2 * B)) if bidirectional else [])
        fnet, cnet = fnet + len(plan.fnet_in), cnet + len(plan.cnet_in)
        before = slots
        slots, saved = apply(plan, slots, saved, lambda f, r: (step[r].seq, step[r].pair + f - 1))
        for j, c in enumerate(step):
            k = (c.seq, c.pair), (c.seq, c.pair + 1)
            assert slots[j] == (k[0], k[1], k[0]), (t, j)
            if bidirectional:
                assert slots[B + j] == (k[1], k[0], k[1]), (t, j)
            if c.idle:
                assert slots[j::B] == before[j::B], (t, j)
        # one head launch per run of restarted slots, never more than one per restarted slot
        assert sum(kind == NEW for _, kind, _, _ in runs(plan.f1[:B])) <= len(restart)
    # every frame once, plus frame 2 of each idle slot-step (an idle slot recomputes its last pair)
    idle = sum(c.idle for step in steps for c in step)
    assert fnet == sum(n for n in lengths if n >= 2) + idle
    assert cnet == (fnet if bidirectional else B * len(steps))


def test_runs():
    srcs = [(NEW, 3), (NEW, 4), None, None, (CARRY, 5), (CARRY, 6), (NEW, 0), (SAVED, 9)]
    assert runs(srcs) == [[0, NEW, 3, 2], [2, None, 2, 2], [4, CARRY, 5, 2], [6, NEW, 0, 1], [7, SAVED, 9, 1]]
    assert runs([(1, 0), (1, 1), (2, 0), (2, 1), (1, 3)]) == [[0, 1, 0, 2], [2, 2, 0, 2], [4, 1, 3, 1]]
