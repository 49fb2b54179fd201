"""Slot plans: which encoded image fills each workspace slot's feature maps and context in one encoder call (host only).

A forward's workspace has S slots, each one pair of frames.  An encoder call runs fnet on the images `fnet_in` and cnet on
`cnet_in`, each entry (frame, row): frame 1 or 2 of batch row `row` of (image1, image2).  For each slot, `f1` (fmap1),
`f2` (level 0 of the fmap2 pyramid) and `ctx` (tanh(net), relu(inp)) name a source:

* (NEW, i): image i of this call's fnet_in (f1, f2) or cnet_in (ctx);
* (CARRY, s): the previous call's f2 of slot s (fnet normalises each image on its own, so a frame's features do not depend
  on the batch it was encoded in);
* (SAVED, s): the context of slot s, saved at the previous call before the GRU overwrote it (slot s is in `save`);
* None: keep the slot's rows as they are (an idle slot repeats its last pair).

`save` is the range of slots whose context is saved for the next call; it is the same at every call of one stage.
"""
from collections import namedtuple

import torch

NEW, CARRY, SAVED = "new", "carry", "saved"

SlotPlan = namedtuple("SlotPlan", "fnet_in cnet_in f1 f2 ctx save")


def slot_plan(B, carry=(), restart=None, bidirectional=False):
    """The plan of one encoder call over B pairs (image1[j], image2[j]).

    restart None: a forward of B new pairs; fnet runs on [image1, image2].  Else one step of sequence inference: slot j's
    frame 1 is the last step's frame 2 for j in `carry`, a new frame for j in `restart`, and idle otherwise; fnet runs on
    [image2, image1 of the restarted slots].  cnet runs on image1.

    bidirectional: 2B slots, slot B + j the backward pair (image2[j], image1[j]).  cnet runs on fnet's images, so each frame's
    context serves the pair that starts at it.  In a sequence step, a carried forward slot's context is its backward slot's
    from the last step, which every step saves."""
    if restart is None:
        fnet_in = [(1, j) for j in range(B)] + [(2, j) for j in range(B)]
        frame1 = [(NEW, j) for j in range(B)]
        frame2 = [(NEW, B + j) for j in range(B)]
    else:
        fnet_in = [(2, j) for j in range(B)] + [(1, j) for j in restart]
        frame1 = [None] * B
        for j in carry:
            frame1[j] = (CARRY, j)
        for r, j in enumerate(restart):
            frame1[j] = (NEW, B + r)
        frame2 = [(NEW, j) for j in range(B)]
    if not bidirectional:
        return SlotPlan(fnet_in, [(1, j) for j in range(B)], frame1, frame2, [(NEW, j) for j in range(B)], range(0))
    ctx = [(SAVED, B + s[1]) if s is not None and s[0] == CARRY else s for s in frame1]
    return SlotPlan(fnet_in, fnet_in, frame1 + frame2, frame2 + frame1, ctx + frame2,
                    range(0) if restart is None else range(B, 2 * B))


def runs(sources):
    """(first slot, kind, first index, count) of each run of consecutive slots whose sources are of one kind with consecutive
    indices: one launch or copy per run.  A kept slot's run has kind None and its own slot as the index.  Also groups
    fnet_in / cnet_in into runs of consecutive rows of one frame (kind = the frame)."""
    out = []
    for j, s in enumerate(sources):
        kind, i = s if s is not None else (None, j)
        if out and out[-1][1] == kind and out[-1][0] + out[-1][3] == j and out[-1][2] + out[-1][3] == i:
            out[-1][3] += 1
        else:
            out.append([j, kind, i, 1])
    return out


def images(frames, entries):
    """The batch of fnet_in / cnet_in `entries` from frames = (image1, image2): one piece per run of consecutive rows."""
    pieces = [frames[f - 1][r:r + k] for _, f, r, k in runs(entries)]
    return (pieces[0] if len(pieces) == 1 else torch.cat(pieces)).contiguous()
