"""Evaluation loops in the shape of the reference's drivers (evaluate.py:111-143 validate_sintel, :146-182
validate_kitti, :25-55 create_sintel_submission with warm start), runnable on any iterable of samples — the datasets
themselves are out of scope (no data offline, SURVEY.md C12), so `bench.py` / the tests feed synthetic pairs.

Differences from the reference, all behaviour-preserving: pairs of equal size are evaluated in batches instead of one at a
time (the model's batch items are independent; frames of a different size — KITTI's vary — start a new batch), and the
warm-start forward interpolation runs on the GPU.  Metrics aggregate as the reference's loops do (rnc.metrics): Sintel-style
(`valid` absent) pools all pixels (evaluate.py:131-137), KITTI-style averages per-image means (evaluate.py:172-179).  Under
torch.distributed every rank takes a share of the samples, sequences or pairs (rnc.dist).
"""
import math
import os
from collections import deque, namedtuple
from concurrent.futures import ThreadPoolExecutor

import torch

from utils import frame_utils
from utils.utils import InputPadder, forward_interpolate

from .restate import check_sides


def _shape_batches(samples, batch_size, regions=False):
    """Consecutive samples of one frame size, batch_size at a time; a new size (KITTI's vary) closes the batch.  With
    regions, samples are _region_sample's 5-tuples and stay as they are."""
    batch = []
    for s in samples:
        if not regions:
            s = tuple(s) if len(s) == 4 else (s[0], s[1], s[2], None)
        if batch and batch[0][0].shape != s[0].shape:
            yield batch
            batch = []
        batch.append(s)
        if len(batch) == batch_size:
            yield batch
            batch = []
    if batch:
        yield batch


_Staged = namedtuple("_Staged", "im1 im2 gt valid sparse ready masks regions")
# a sample's region masks, checked: its index in the split, "sintel" or "kitti", and the masks ({"occ"} or {"noc"[, "fg"]})
_Regions = namedtuple("_Regions", "index kind masks")
_REGION_KEYS = {frozenset({"occ"}): "sintel", frozenset({"noc"}): "kitti", frozenset({"noc", "fg"}): "kitti"}


def _region_samples(samples, world, rank):
    """validate(regions=True)'s samples (this rank's share of the split), each checked and returned as (image1, image2,
    flow_gt, valid, _Regions).  ValueError naming the sample's index in the split when it has no fifth item, the item is not
    one of the dicts {"occ"}, {"noc"}, {"noc", "fg"}, a mask is not [H,W] of the frame's size, or it is of the other style
    than the samples before it."""
    first = None
    for k, s in enumerate(samples):
        i = rank + world * k
        if len(s) != 5:
            raise ValueError(f"validate(regions=True): sample {i} has {len(s)} items; expected (image1, image2, flow_gt, valid, "
                             f"masks) with masks {{'occ': mask}} or {{'noc': mask[, 'fg': mask]}}")
        masks = s[4]
        kind = _REGION_KEYS.get(frozenset(masks)) if isinstance(masks, dict) else None
        if kind is None:
            raise ValueError(f"validate(regions=True): sample {i}'s fifth item must be {{'occ': mask}} or {{'noc': mask[, 'fg': "
                             f"mask]}}, got {sorted(masks) if isinstance(masks, dict) else type(masks).__name__}")
        hw = tuple(s[0].shape[-2:])
        for name, m in masks.items():
            if tuple(m.shape) != hw:
                raise ValueError(f"validate(regions=True): sample {i}'s {name} mask is {tuple(m.shape)}, expected [H,W] = {hw}")
        if first is None:
            first = (i, kind)
        elif kind != first[1]:
            raise ValueError(f"validate(regions=True): sample {i} is {kind.capitalize()}-style but sample {first[0]} is "
                             f"{first[1].capitalize()}-style; one split is one or the other")
        yield (s[0], s[1], s[2], s[3], _Regions(i, kind, masks))


def _stage(batch, dev, copy_stream, regions=False):
    """Enqueue the upload of a batch: each field stacked into a pinned host tensor and copied without blocking on copy_stream,
    so that it overlaps the forward running on the compute stream.  valid is None when no sample has one; a sample without
    one among samples with one counts every pixel valid.  With regions, the region masks travel the same way: occ, or noc
    and fg (fg when a sample of the batch has one; a sample without counts every pixel as background)."""
    sparse = [s[3] is not None for s in batch]
    H, W = batch[0][0].shape[-2:]
    fields = [[s[0] for s in batch], [s[1] for s in batch], [s[2].float() for s in batch]]
    if any(sparse):
        fields.append([torch.ones(H, W) if s[3] is None else s[3].float() for s in batch])
    names = []
    if regions:
        for name in ("occ", "noc", "fg"):
            if any(name in s[4].masks for s in batch):
                names.append(name)
                fields.append([s[4].masks[name].float() if name in s[4].masks else torch.zeros(H, W) for s in batch])
    nv = 4 if any(sparse) else 3
    meta = [s[4] for s in batch] if regions else None
    if dev.type != "cuda":
        host = [torch.stack(f).to(dev) for f in fields]
    else:
        host = []
        for f in fields:
            pinned = torch.empty((len(f),) + tuple(f[0].shape), dtype=f[0].dtype, pin_memory=True)
            torch.stack(f, out=pinned)
            with torch.cuda.stream(copy_stream):          # allocated on copy_stream: its memory is never in use by older work
                host.append(pinned.to(dev, non_blocking=True))
    ready = None
    if dev.type == "cuda":
        ready = torch.cuda.Event()
        ready.record(copy_stream)
    return _Staged(*host[:3], host[3] if nv == 4 else None, sparse, ready, dict(zip(names, host[nv:])), meta)


def bidirectional_flow(model, image1, image2, iters=32, flow_init=None, mode="sintel", return_confidence=False, alpha1=0.01,
                       alpha2=0.5):
    """Flow in both directions of B pairs from one encoder pass, with their forward-backward consistency.  image1, image2:
    [B,3,H,W] (0..255) on the model's device, of any size: they are padded with InputPadder(mode) and the results unpadded.
    flow_init: None or a pair (fw, bw) of low-resolution warm starts, each [B,2,H'/8,W'/8] at the padded size or None.
    Returns a dict of flow_low / flow_up (image1 -> image2), flow_low_bw / flow_up_bw (image2 -> image1), each the flow
    model(...) gives for that order of the frames (flow_low stays at the padded 1/8 resolution, as the forward's), and of
    occ / occ_bw (uint8 [B,H,W]) and fb_err / fb_err_bw (float32 [B,H,W]) of rnc.metrics.fb_consistency(flow_up, flow_up_bw,
    alpha1, alpha2) on the unpadded flows.  return_confidence (NCUP model): also confidence / confidence_bw, the upsampler's
    output confidence unpadded like the flows.  Inference only: with grad enabled on a model that requires grad it raises
    ValueError."""
    from .metrics import fb_consistency
    if image1.dim() != 4 or image1.shape != image2.shape:
        raise ValueError(f"bidirectional_flow: expected two [B,3,H,W] images of one shape, got {tuple(image1.shape)} and "
                         f"{tuple(image2.shape)}")
    B = image1.shape[0]
    padder = InputPadder(image1.shape, mode=mode)
    p1, p2 = padder.pad(image1.float(), image2.float())
    out = model.forward_bidirectional(p1, p2, iters=iters, flow_init=flow_init, return_confidence=return_confidence)
    flow_low, flow_up = out[0], padder.unpad(out[1])
    res = {"flow_low": flow_low[:B], "flow_up": flow_up[:B], "flow_low_bw": flow_low[B:], "flow_up_bw": flow_up[B:]}
    if return_confidence:
        conf = padder.unpad(out[2])
        res["confidence"], res["confidence_bw"] = conf[:B], conf[B:]
    res["occ"], res["occ_bw"], res["fb_err"], res["fb_err_bw"] = fb_consistency(res["flow_up"], res["flow_up_bw"], alpha1, alpha2)
    return res


@torch.no_grad()
def validate(model, samples, iters=32, mode="sintel", batch_size=8, device="cuda", confidence=False, consistency=False,
             regions=False):
    """samples: iterable of (image1 [3,H,W], image2 [3,H,W], flow_gt [2,H,W], valid [H,W] or None).
    Returns the metrics validate_sintel / validate_kitti print: EPE, 1px/3px/5px, and KITTI F1 when `valid` is given
    (rnc.metrics.summarize: Sintel-style pools every pixel, KITTI-style averages the per-image mean EPE).

    On a CUDA device each batch is uploaded through pinned buffers on a side stream while the previous batch computes, its
    metrics are taken on the device (rnc_flow_metrics) and stay there as per-image partials; the host reads them once, at the
    end.  Under torch.distributed with more than one rank, rank r evaluates the samples of index = r (mod world) (a sequence,
    such as the reference's FlowDataset, is indexed, so each rank loads only its own samples), the per-image partials are
    all-gathered, and every rank returns the same dict, bit for bit the single-process one.

    confidence=True (NCUP model) also evaluates the upsampler's output confidence: the forward returns it, unpadded like the
    flow, each pixel is scored by rnc.metrics.confidence_score, and rnc.metrics.sparsification's per-image partials travel
    with the flow metrics'.  The dict gains "sparsification" and "ideal" (100 mean EPEs each, at the removed fractions k/100)
    and "ause" (rnc.metrics.summarize_sparsification); its other keys are those of confidence=False, bit for bit.

    consistency=True evaluates forward-backward consistency as a reliability score: each batch runs the bidirectional pass
    (model.forward_bidirectional), its forward flow is scored as above, and each pixel is ranked by -fb_err of
    rnc.metrics.fb_consistency.  The dict gains "fb_sparsification", "fb_ause" and "ideal" (which depends on the EPE only,
    so one serves both scores).  The forward rows of the bidirectional pass are the flows of model(image1, image2), so the
    other keys are those of consistency=False: bit for bit wherever the forward itself repeats bit for bit (the exact lookup
    under torch.use_deterministic_algorithms), and within its run-to-run spread otherwise.

    regions=True also gives the per-region errors the Sintel and KITTI 2015 benchmarks publish (the definitions are in
    rnc.metrics).  Each sample is then (image1, image2, flow_gt, valid or None, masks), masks {"occ": [H,W]} for a Sintel-style
    split or {"noc": [H,W]} / {"noc": [H,W], "fg": [H,W]} for a KITTI-style one.  The masks travel with valid; per batch
    rnc.metrics.region_partials (rnc_boundary_dist2 and rnc_region_metrics on CUDA) takes per-image partials that stay on the
    device with the others and are gathered with them.  The dict gains rnc.metrics.summarize_regions' keys: epe_matched,
    epe_unmatched, epe_d0-10, epe_d10-60, epe_d60-140, epe_s0-10, epe_s10-40, epe_s40+ (Sintel-style) or fl_all, fl_all_noc
    and, when every sample has fg, fl_bg, fl_fg, fl_bg_noc, fl_fg_noc (KITTI-style), and region_pixels.  With consistency=True
    and a Sintel-style split it also gains occ_precision, occ_recall and occ_f1, which score fb_consistency's occlusion mask
    of the forward flow (rnc.metrics.occlusion_counts) against occ over the valid pixels.  The other keys are those of
    regions=False, bit for bit.  ValueError, naming the sample's index, for a sample without masks, with a mask of the wrong
    shape, or of the other style than the rest of the split."""
    from .dist import gather_strided, strided_items, world_rank
    from .metrics import (Partials, RegionPartials, SparsPartials, cat, confidence_score, fb_consistency, flow_metrics,
                          from_images, images, occlusion_counts, region_partials, sparsification, summarize, summarize_occlusion,
                          summarize_regions, summarize_sparsification)
    model.eval()
    world, rank = world_rank()
    dev = torch.device(device)
    if dev.type == "cuda" and dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    copy_stream = torch.cuda.Stream(dev) if dev.type == "cuda" else None
    # this rank's per-batch partials by name, with the type each concatenates to
    kinds = {"flow": Partials}
    if confidence:
        kinds["confidence"] = SparsPartials
    if consistency:
        kinds["consistency"] = SparsPartials
    if regions:
        kinds["regions"] = RegionPartials
    parts = {name: [] for name in kinds}
    occlusion, sparse, rmeta = [], [], []
    items = strided_items(samples, world, rank)
    batches = _shape_batches(_region_samples(items, world, rank) if regions else items, batch_size, regions)

    def stage_next():
        b = next(batches, None)
        return None if b is None else _stage(b, dev, copy_stream, regions)
    nxt = stage_next()
    while nxt is not None:
        cur = nxt
        if cur.ready is not None:
            compute = torch.cuda.current_stream(dev)
            compute.wait_event(cur.ready)
            for t in (*cur[:4], *cur.masks.values()):
                if t is not None:
                    t.record_stream(compute)
        padder = InputPadder(cur.im1.shape, mode=mode)
        p1, p2 = padder.pad(cur.im1.float(), cur.im2.float())
        B = p1.shape[0]
        if consistency:
            _, flow_pr, *conf = model.forward_bidirectional(p1, p2, iters=iters, return_confidence=confidence)
            flow_bw, flow_pr = padder.unpad(flow_pr[B:]), flow_pr[:B]
            conf = conf[0][:B] if confidence else None
        elif confidence:
            _, flow_pr, conf = model(p1, p2, iters=iters, test_mode=True, return_confidence=True)
        else:
            _, flow_pr = model(p1, p2, iters=iters, test_mode=True)
        flow = padder.unpad(flow_pr)
        parts["flow"].append(flow_metrics(flow, cur.gt, cur.valid))
        if confidence:
            parts["confidence"].append(sparsification(flow, cur.gt, cur.valid, confidence_score(padder.unpad(conf))))
            del conf
        if regions:
            rp = region_partials(flow, cur.gt, cur.valid, **cur.masks)
            parts["regions"].append(rp._replace(fg=torch.tensor(["fg" in r.masks for r in cur.regions])))
            rmeta += cur.regions
        if consistency:
            occ_fw, _, fb_err, _ = fb_consistency(flow, flow_bw)
            parts["consistency"].append(sparsification(flow, cur.gt, cur.valid, -fb_err))
            if regions and "occ" in cur.masks:
                occlusion.append(occlusion_counts(occ_fw, cur.masks["occ"], cur.valid))
            del flow_bw, fb_err, occ_fw
        sparse += cur.sparse
        del cur, p1, p2, flow_pr, flow
        nxt = stage_next()                          # staged while this batch computes
    # one record per image of this rank, {name: value}: its partials, whether it had a valid mask, and with regions its index
    # and style (and, Sintel-style with consistency, its occlusion counts), gathered back into sample order
    local = {name: images(cat(kind, parts[name])) for name, kind in kinds.items()}
    local["sparse"] = sparse
    if regions:
        local["style"] = [(m.index, m.kind) for m in rmeta]
    if occlusion:
        local["occlusion"] = torch.cat(occlusion).cpu().tolist()
    rows = gather_strided([dict(zip(local, r)) for r in zip(*local.values())], world)

    def gathered(name):
        return from_images(kinds[name], [r[name] for r in rows])
    res = summarize(gathered("flow"), "kitti" if any(r["sparse"] for r in rows) else "sintel")
    for name, prefix in (("confidence", ""), ("consistency", "fb_")):
        if name in kinds:
            summ = summarize_sparsification(gathered(name))
            res.update({prefix + "sparsification": summ["sparsification"], "ideal": summ["ideal"], prefix + "ause": summ["ause"]})
    if regions and rows:
        i0, kind0 = rows[0]["style"]
        for i, kind in (r["style"] for r in rows):
            if kind != kind0:
                raise ValueError(f"validate(regions=True): sample {i} is {kind.capitalize()}-style but sample {i0} is "
                                 f"{kind0.capitalize()}-style; one split is one or the other")
        res.update(summarize_regions(gathered("regions")))
        if consistency and kind0 == "sintel":
            res.update(summarize_occlusion(torch.tensor([r["occlusion"] for r in rows], dtype=torch.int64)))
    return res


@torch.no_grad()
def run_sequence(model, frames, iters=32, warm_start=False, mode="sintel", device="cuda"):
    """create_sintel_submission's inner loop (evaluate.py:31-44): consecutive frame pairs of one sequence, optionally
    warm-starting each pair from the forward-interpolated low-resolution flow of the previous one.  Returns the list of
    unpadded [2,H,W] flows (CPU)."""
    model.eval()
    flows, flow_prev = [], None
    for f1, f2 in zip(frames[:-1], frames[1:]):
        im1, im2 = f1[None].to(device).float(), f2[None].to(device).float()
        padder = InputPadder(im1.shape, mode=mode)
        p1, p2 = padder.pad(im1, im2)
        flow_low, flow_pr = model(p1, p2, iters=iters, flow_init=flow_prev, test_mode=True)
        flows.append(padder.unpad(flow_pr[0]).cpu())
        if warm_start:
            flow_prev = forward_interpolate(flow_low[0])[None]
    return flows


SlotStep = namedtuple("SlotStep", "seq pair restart idle")


def sequence_schedule(lengths, batch_size):
    """Slot schedule of run_sequences for sequences of `lengths` frames: min(batch_size, number of sequences with a pair)
    slots run in lockstep, one pair each per step.  Returns one list per step of each slot's SlotStep(seq, pair, restart,
    idle): pair k of sequence seq is frames (k, k + 1); restart marks pair 0 (the slot's frame 1 is new, not the previous
    step's frame 2); an idle slot has no sequence left and repeats its previous (seq, pair), whose result is dropped.  A slot
    whose sequence ends takes the next sequence not yet started, in order; sequences of fewer than two frames are skipped."""
    if batch_size < 1:
        raise ValueError(f"batch_size must be >= 1, got {batch_size}")
    pending = deque(s for s, n in enumerate(lengths) if n >= 2)
    cur = [SlotStep(pending.popleft(), 0, True, False) for _ in range(min(batch_size, len(pending)))]
    steps = []
    while any(not c.idle for c in cur):
        steps.append(list(cur))
        for j, c in enumerate(cur):
            if c.idle:
                continue
            if c.pair + 2 < lengths[c.seq]:
                cur[j] = SlotStep(c.seq, c.pair + 1, False, False)
            elif pending:
                cur[j] = SlotStep(pending.popleft(), 0, True, False)
            else:
                cur[j] = c._replace(restart=False, idle=True)
    return steps


def _stack(frames, device, padder):
    x = torch.stack(frames)
    if x.device.type == "cpu" and torch.device(device).type == "cuda":
        x = x.pin_memory()
    return padder.pad(x.to(device, non_blocking=True).float())[0]


def _sequence_setup(sequences, batch_size, mode, model, return_confidence):
    """The argument checks and the schedule shared by run_sequences and run_sequences_bidirectional: ValueError for frames
    of more than one [3,H,W] size and for return_confidence on the convex model.  Returns (sequence_schedule's steps, the
    InputPadder of the frame size), or ([], None) when no sequence has a pair."""
    sizes = [tuple(f.shape) for seq in sequences for f in seq]
    for s in sizes:
        if len(s) != 3 or s != sizes[0]:
            raise ValueError(f"all frames of one call must have the same [3,H,W] size: got {sizes[0]} and {s}")
    if return_confidence and not model.ncup:
        raise ValueError("return_confidence: the convex-upsampling RAFT has no NCUP upsampler and so no output confidence")
    steps = sequence_schedule([len(seq) for seq in sequences], batch_size)
    return steps, (InputPadder(sizes[0], mode=mode) if steps else None)


def _step_images(sequences, step, device, padder):
    """Frames 1 and 2 of every slot of one step, padded, on the device."""
    return (_stack([sequences[c.seq][c.pair] for c in step], device, padder),
            _stack([sequences[c.seq][c.pair + 1] for c in step], device, padder))


def _sequence_engine(model, im1):
    """(device, engine) of a sequence generator's first step; ValueError when the model is on another device."""
    from .engine import _require_cuda, engine_for, module_device
    dev = _require_cuda(im1)
    if module_device(model) != dev:
        raise ValueError(f"model parameters are on {module_device(model)} but device is {dev}")
    return dev, engine_for(dev)


def _sequence_workspace(eng, model, dev, slots, im1):
    """A sequence generator's own workspace of `slots` slots: the features carried from step to step live in it, so the
    caller may run other forwards of the same shape between two steps."""
    pk = eng.packed_update(model.update_block)
    return eng.WS(dev, slots, im1.shape[2] // 8, im1.shape[3] // 8, pk.has_mask, model.ncup)


@torch.no_grad()
def run_sequences(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                  return_confidence=False):
    """create_sintel_submission (evaluate.py:23-55) over many sequences at batch throughput.  sequences: list of frame lists,
    every frame [3,H,W] of one size.  Yields (seq_index, pair_index, flow): the unpadded [2,H,W] flow_up of every pair, on
    the device; per sequence the flows equal run_sequence(model, seq, iters, warm_start, mode)'s.  return_confidence (NCUP
    model): yields (seq_index, pair_index, flow, confidence), the upsampler's output confidence unpadded like the flow.

    Slots run in lockstep (sequence_schedule).  Each step encodes only new frames: a continuing slot's frame 1 is its last
    frame 2, whose fnet features are handed over on the device (rnc.slot_plan).  With warm_start, a slot starts from
    forward_interpolate of its own previous low-resolution flow, and from zero (a cold start) at pair 0.  The steps run
    eagerly and never wait for the host; the caller moves or writes the flows."""
    steps, padder = _sequence_setup(sequences, batch_size, mode, model, return_confidence)
    if not steps:
        return
    for step, _, flow_up, conf in _sequence_steps(model, sequences, steps, padder, iters, warm_start, device,
                                                  return_confidence, False):
        for j, c in enumerate(step):
            if not c.idle:
                if return_confidence:
                    yield c.seq, c.pair, padder.unpad(flow_up[j]), padder.unpad(conf[j])
                else:
                    yield c.seq, c.pair, padder.unpad(flow_up[j])


@torch.no_grad()
def _sequence_steps(model, sequences, steps, padder, iters, warm_start, device, return_confidence, bidirectional):
    """The step loop of run_sequences (B slots) and, with bidirectional, of run_sequences_bidirectional (2B slots, slot
    B + j the backward pair of slot j).  Yields (step, flow_low, flow_up, confidence or None) of each step, every slot,
    padded.  A step is _forward_eager with the step's slot plan on the generator's own workspace; with warm_start the next
    step starts from this one's flow_low (forward_interpolate, or bidirectional_warm_start), a restarted slot from zero."""
    from .engine import _Timed
    from .model import EncoderStage
    from .slot_plan import slot_plan
    model.eval()
    stage = EncoderStage(model)
    B = len(steps[0])
    ws = fi = zero = None
    for step in steps:
        im1, im2 = _step_images(sequences, step, device, padder)
        if ws is None:
            dev, eng = _sequence_engine(model, im1)
        restart = [j for j, c in enumerate(step) if c.restart]
        stage.plan = slot_plan(B, [j for j, c in enumerate(step) if not c.restart and not c.idle], restart, bidirectional)
        with torch.cuda.device(dev), eng.lock:
            if ws is None:
                ws = _sequence_workspace(eng, model, dev, (2 if bidirectional else 1) * B, im1)
            for j in restart if fi is not None else ():
                fi[j::B].copy_(zero)        # rows j (and B + j): a cold start, coords0 + 0.0 is exactly coords0
            flow_low, flow_up, *conf = model._forward_eager(eng, im1, im2, iters, fi, True, encode=stage, ws=ws,
                                                            return_confidence=return_confidence)
            if warm_start:
                with _Timed(eng, "warm_start"):
                    fi = bidirectional_warm_start(flow_low) if bidirectional else forward_interpolate(flow_low)
                if zero is None:
                    zero = torch.zeros_like(fi[0::B])
        yield step, flow_low, flow_up, (conf[0] if return_confidence else None)


def bidirectional_warm_start(flow_low):
    """Warm starts of the next step of bidirectional sequence inference, both directions in one launch
    (rnc_forward_interpolate_bidir_fwd).  flow_low: [2B,2,H,W] on a CUDA device, rows [0, B) forward flows f_{k->k+1},
    rows [B, 2B) backward flows b_{k+1->k}.  Row j of the result is forward_interpolate(f) (the reference's warm start);
    row B + j assumes constant velocity backwards: the point at x in frame k+1 is at x - b(x) in frame k+2 and its backward
    flow there is b(x), so each sample moves to x - b(x) and carries b(x), with forward_interpolate's validity test,
    nearest-sample rule and fill 0.  As an identity it is -forward_interpolate(-b), bit for bit."""
    from .engine import _require_cuda
    from .native import rnc
    dev = _require_cuda(flow_low)
    if flow_low.dim() != 4 or flow_low.shape[0] % 2 or flow_low.shape[1] != 2:
        raise ValueError(f"bidirectional_warm_start: expected [2B,2,H,W], got {tuple(flow_low.shape)}")
    f = flow_low.detach().float().contiguous()
    N, _, H, W = f.shape
    out = torch.empty_like(f)
    with torch.cuda.device(dev):
        rnc.forward_interpolate_bidir_fwd(f, N // 2, H, W, out)
    return out


def run_sequences_bidirectional(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                                return_confidence=False, alpha1=0.01, alpha2=0.5):
    """Forward and backward flow, with forward-backward occlusion masks, for every consecutive frame pair of many
    sequences, each frame encoded once.  sequences: list of frame lists, every frame [3,H,W] of one size.  Yields
    (seq_index, pair_index, result) for pair k = frames (k, k + 1) of every sequence; result has bidirectional_flow's keys
    (flow_low, flow_up, flow_low_bw, flow_up_bw, occ, occ_bw, fb_err, fb_err_bw, and with return_confidence (NCUP model)
    confidence, confidence_bw), each that pair's slice without the batch dimension, on the device, unpadded as
    bidirectional_flow's.  Cold, pair k's result is bidirectional_flow(model, f_k[None], f_{k+1}[None], iters, mode=mode)'s.
    With warm_start, pair k > 0 starts from bidirectional_warm_start of pair k - 1's flow_low and flow_low_bw (the forward
    rule of run_sequences, and its mirror for the backward flow); pair 0 starts cold in both directions.  The forward rows
    are run_sequences(model, sequences, ...)'s flows.

    Slots run in lockstep as in run_sequences (sequence_schedule), on a workspace of 2B slots: slot j holds a sequence's
    forward pair, slot B + j its backward pair.  fnet and cnet encode each new frame once per step: a frame's features
    and context serve the backward pair that starts at it and, one step later, the forward pair that starts at it
    (rnc.slot_plan).  Each step checks consistency on both directions in one launch
    (rnc.metrics.fb_consistency with alpha1, alpha2) and computes both warm starts in one launch; the steps never wait for
    the host.  Inference only: with grad enabled on a model that requires grad it raises ValueError."""
    steps, padder = _sequence_setup(sequences, batch_size, mode, model, return_confidence)
    if not steps:
        return
    _check_inference(model, "run_sequences_bidirectional",
                     " (training through the bidirectional pass is model(..., bidirectional=True))")
    from .metrics import fb_consistency
    B = len(steps[0])
    for step, flow_low, flow_up, conf in _sequence_steps(model, sequences, steps, padder, iters, warm_start, device,
                                                         return_confidence, True):
        up = padder.unpad(flow_up)
        occ, occ_bw, err, err_bw = fb_consistency(up[:B], up[B:], alpha1, alpha2)
        conf = padder.unpad(conf) if return_confidence else None
        for j, c in enumerate(step):
            if c.idle:
                continue
            res = {"flow_low": flow_low[j], "flow_up": up[j], "flow_low_bw": flow_low[B + j], "flow_up_bw": up[B + j],
                   "occ": occ[j], "occ_bw": occ_bw[j], "fb_err": err[j], "fb_err_bw": err_bw[j]}
            if return_confidence:
                res["confidence"], res["confidence_bw"] = conf[j], conf[B + j]
            yield c.seq, c.pair, res


def interpolate_frames(model, frame0, frame1, times=(0.5,), iters=32, mode="sintel", alpha1=0.01, alpha2=0.5):
    """The frames between frame0 and frame1 ([B,3,H,W], 0..255, on the model's device, any size) at each of `times`:
    bidirectional_flow(model, frame0, frame1, iters, mode=mode, alpha1=alpha1, alpha2=alpha2), then rnc.interp.interpolate of
    its unpadded flows and occlusion masks.  Returns float32 [B,T,3,H,W].  Inference only: with grad enabled on a model that
    requires grad it raises ValueError."""
    from .interp import _times, interpolate
    _check_inference(model, "interpolate_frames")
    _times(times)                                   # a bad time raises before the flow pass
    r = bidirectional_flow(model, frame0, frame1, iters, mode=mode, alpha1=alpha1, alpha2=alpha2)
    return interpolate(frame0, frame1, r["flow_up"], r["flow_up_bw"], r["occ"], r["occ_bw"], times)


@torch.no_grad()
def validate_interpolation(model, sequences, iters=32, mode="sintel", batch_size=8, warm_start=False, device="cuda"):
    """Middlebury's interpolation error of a split of videos, which needs no ground-truth flow: for every triplet of frames
    (k, k + 1, k + 2) of every sequence, frame k + 1 is interpolated at t = 0.5 from frames k and k + 2 and scored against the
    real one.  sequences: list of frame lists, every frame [3,H,W] (0..255) of one size.  The pairs (k, k + 2) are the
    consecutive pairs of each sequence's even-indexed and odd-indexed frames, which run_sequences_bidirectional(model, ...,
    iters, warm_start, batch_size, mode, device) runs side by side; each pair's flows and masks go through rnc.interp.interpolate
    and rnc.interp.interpolation_error on the device.  Returns rnc.interp.summarize_interpolation of the per-triplet partials
    in (sequence, k) order: ie, psnr and frames.  Cold, each triplet's partials are those of bidirectional_flow + interpolate +
    interpolation_error of its pair alone; warm, each pair starts from the previous pair of its subsequence.  Either way
    they do not depend on batch_size.  Under torch.distributed rank r takes the sequences of index = r (mod world), the partials are
    all-gathered, and every rank returns the single-process result."""
    from .dist import gather_strided, strided_items, world_rank
    from .interp import interpolate, interpolation_error, summarize_interpolation
    from .metrics import InterpPartials, cat, from_images, images
    world, rank = world_rank()
    mine = list(strided_items(range(len(sequences)), world, rank))
    subs, origin = [], []                           # origin[i]: (sequence index, offset) of subsequence i
    for s in mine:
        for off in (0, 1):
            subs.append(sequences[s][off::2])
            origin.append((s, off))
    parts = {s: [None] * max(len(sequences[s]) - 2, 0) for s in mine}      # per sequence, triplet k's partials
    for i, p, r in run_sequences_bidirectional(model, subs, iters, warm_start=warm_start, batch_size=batch_size, mode=mode,
                                               device=device):
        s, off = origin[i]
        k = off + 2 * p
        seq = sequences[s]
        dev = r["flow_up"].device
        f0, f2, gt = (seq[j][None].to(dev).float() for j in (k, k + 2, k + 1))
        pred = interpolate(f0, f2, r["flow_up"][None], r["flow_up_bw"][None], r["occ"][None], r["occ_bw"][None], (0.5,))
        parts[s][k] = interpolation_error(pred[:, 0], gt)
    every = gather_strided([images(cat(InterpPartials, parts[s])) for s in mine], world)
    return summarize_interpolation(from_images(InterpPartials, [t for seq in every for t in seq]))


def _check_inference(model, what, why=""):
    if model._needs_grad():
        raise ValueError(f"{what} is inference only: call it under torch.no_grad(){why}")


def _check_counts(sequences, what, *lists):
    """Each (noun, items) of lists as a list of items; ValueError unless every one holds one item per video."""
    items = [list(x) for _, x in lists]
    if any(len(x) != len(sequences) for x in items):
        got = [f"{len(x)} {noun}" for (noun, _), x in zip(lists, items)]
        if len(got) > 1:
            got = [", ".join(got[:-1]), got[-1]]
        raise ValueError(f"{what}: {len(sequences)} videos but {' and '.join(got)}")
    return items


def _check_frames(seq, what, need=2, why=""):
    """ValueError for a video of fewer than `need` frames: each application's first check of a video."""
    if len(seq) < need:
        raise ValueError(f"{what}: a video needs T >= {need} frames{why}, got {len(seq)}")


def _by_size(sequences, indices):
    """The indices grouped by their video's frame size, in order of first appearance."""
    groups = {}
    for i in indices:
        groups.setdefault(tuple(sequences[i][0].shape[-2:]), []).append(i)
    return list(groups.values())


class _PairStack(dict):
    """Named results of the flow pass over `sequences`, stacked by add into [V,T-1,...] tensors, T the longest video's frame
    count, allocated at the first pair on its results' device: float32 `flows` padded with 0, uint8 `masks` padded with 1,
    so a shorter video's missing pairs are zero flows occluded in both directions."""

    def __init__(self, sequences, flows, masks=()):
        super().__init__()
        self.pairs = (len(sequences), max((len(seq) for seq in sequences), default=1) - 1)
        self.pads = [(name, 0, torch.float32) for name in flows] + [(name, 1, torch.uint8) for name in masks]

    def add(self, s, k, r):
        for name, pad, dtype in self.pads:
            if name not in self:
                self[name] = torch.full((*self.pairs, *r[name].shape), pad, dtype=dtype, device=r[name].device)
            self[name][s, k].copy_(r[name])


def _pad_videos(videos, pad):
    """Per-video tensors [n_v,...] of one dtype and device stacked into [V,n,...], n the largest n_v, the items past a video's
    n_v set to pad (a number, or a tensor that broadcasts to one item)."""
    out = videos[0].new_empty((len(videos), max(t.shape[0] for t in videos), *videos[0].shape[1:]))
    out[:] = pad
    for v, t in enumerate(videos):
        out[v, :t.shape[0]] = t
    return out


def track_points(model, sequences, queries, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                 alpha1=0.01, alpha2=0.5):
    """Tracks of query points through whole videos (rnc.track's rule: the bidirectional flows chained from each query frame,
    with a visible flag that turns off for good at the first occlusion, non-finite flow or exit from the frame).
    sequences: list of V frame lists, every frame [3,H,W] (0..255) of one size, each video of T_v >= 2 frames; queries: V
    float32 [N_v,3] tensors (or a [V,N,3] tensor) of (t, x, y), t an integer frame index and (x, y) pixel coordinates in the
    frame (rnc.track.grid_queries gives dense queries).  Returns a list of V (tracks float32 [N_v,T_v,2], visible uint8
    [N_v,T_v]) on the device.

    run_sequences_bidirectional(model, sequences, iters, warm_start, batch_size, mode, device, alpha1=alpha1, alpha2=alpha2)
    runs first, and each pair's flow_up, flow_up_bw, occ and occ_bw are copied into stacked device tensors as they are yielded:
    with T the longest video's frame count, V (T - 1) (2 flows x 2 channels x 4 B + 2 masks x 1 B) = 18 V (T - 1) bytes per
    pixel, e.g. 3.2 GB for eight 50-frame videos of 436x1024.  A shorter video's missing pairs are zero flows with every
    pixel occluded; they only extend its tracks past its last frame, and those frames are dropped.  Then rnc.track.track runs
    once over all videos, one launch, so each track is what rnc.track.track gives for its video alone.  ValueError before the
    flow pass for a video of fewer than two frames, a bad query or a query count that does not match the videos.  Inference
    only: with grad enabled on a model that requires grad it raises ValueError."""
    from .track import check_queries, track
    _check_inference(model, "track_points")
    qs, = _check_counts(sequences, "track_points", ("query sets", queries))
    if not sequences:
        return []
    H, W = sequences[0][0].shape[-2:]
    lens = [len(seq) for seq in sequences]
    for T, q in zip(lens, qs):
        if q.dim() != 2:
            raise ValueError(f"track_points: expected each video's queries as [N,3], got {tuple(q.shape)}")
        check_queries(q, T, H, W, "track_points")
    flows = _PairStack(sequences, ("flow_up", "flow_up_bw"), ("occ", "occ_bw"))
    for s, k, r in run_sequences_bidirectional(model, sequences, iters, warm_start=warm_start, batch_size=batch_size,
                                               mode=mode, device=device, alpha1=alpha1, alpha2=alpha2):
        flows.add(s, k, r)
    # (0, 0, 0) pads a video's queries to the largest count; their tracks are dropped
    q = _pad_videos([qv.to(flows["flow_up"].device, torch.float32) for qv in qs], 0)
    tracks, visible = track(flows["flow_up"], flows["flow_up_bw"], flows["occ"], flows["occ_bw"], q)
    return [(tracks[v, :qv.shape[0], :lens[v]], visible[v, :qv.shape[0], :lens[v]]) for v, qv in enumerate(qs)]


@torch.no_grad()
def validate_tracking(model, sequences, queries, gt_tracks, gt_visible, iters=32, warm_start=False, batch_size=8,
                      mode="sintel", device="cuda", alpha1=0.01, alpha2=0.5):
    """TAP-Vid's metrics of track_points on a split of videos: occlusion_accuracy, average_pts_within_thresh (< delta^x_avg),
    average_jaccard, their per-threshold terms and the video count (rnc.track.summarize_tracking).  sequences and queries as
    track_points'; gt_tracks: V [N_v,T_v,2] (x, y) pixel positions; gt_visible: V [N_v,T_v] (non-zero is visible, TAP-Vid's
    `occluded` negated).  Each video's counts come from rnc.track.track_metrics on the device; they are integers, so the
    result does not depend on batch_size or on the order of the videos.  Under torch.distributed rank r takes the videos of
    index = r (mod world), the per-video counts are all-gathered, and every rank returns the single-process result."""
    from .dist import gather_strided, strided_items, world_rank
    from .track import summarize_tracking, track_metrics
    world, rank = world_rank()
    mine = list(strided_items(range(len(sequences)), world, rank))
    _check_counts(sequences, "validate_tracking", ("query sets", queries), ("ground-truth tracks", gt_tracks),
                  ("visibility sets", gt_visible))
    got = track_points(model, [sequences[i] for i in mine], [queries[i] for i in mine], iters, warm_start, batch_size, mode,
                       device, alpha1, alpha2)
    counts = []
    for i, (tr, vis) in zip(mine, got):
        H, W = sequences[i][0].shape[-2:]
        dev = tr.device
        c = track_metrics(tr[None], vis[None], gt_tracks[i][None].to(dev), gt_visible[i][None].to(dev),
                          queries[i][None].to(dev), H, W)
        counts.append(c[0].tolist())
    return summarize_tracking(gather_strided(counts, world))


def propagate_masks(model, sequences, first_labels, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                    alpha1=0.01, alpha2=0.5):
    """The labels of every frame of V videos from those of frame 0 (rnc.segment's rule: each pixel of frame k+1 takes the
    bilinear vote of frame k's labels at the end of its backward flow, or, where that flow is occluded, non-finite or leaves
    the frame, the label of its nearest pixel that has a vote).  sequences: list of V frame lists, every frame [3,H,W]
    (0..255) of one size, each video of T_v >= 2 frames; first_labels: V integer [H,W] label maps of frame 0 (0 background,
    1..254 objects).  Returns a list of V uint8 [T_v,H,W] label tensors on the device.

    run_sequences_bidirectional(model, sequences, iters, warm_start, batch_size, mode, device, alpha1=alpha1, alpha2=alpha2)
    yields each video's pairs in order, and pair k's flow_up_bw and occ_bw step that video's labels from frame k to k + 1 at
    once (rnc.segment.propagate_step's rule, one rnc_propagate_labels call), so no flow is kept: the memory is the labels, one
    byte per pixel per frame.  ValueError before the flow pass for a video of fewer than two frames, first labels of another
    size, a label outside 0..254 or a label-map count that does not match the videos.  Inference only: with grad enabled on
    a model that requires grad it raises ValueError."""
    from . import native
    from .segment import _step, check_labels
    _check_inference(model, "propagate_masks")
    firsts, = _check_counts(sequences, "propagate_masks", ("first-frame label maps", first_labels))
    if not sequences:
        return []
    for seq, first in zip(sequences, firsts):
        _check_frames(seq, "propagate_masks")
        if tuple(first.shape) != tuple(seq[0].shape[-2:]):
            raise ValueError(f"propagate_masks: expected first labels {list(seq[0].shape[-2:])}, got {list(first.shape)}")
        check_sides(*first.shape, "propagate_masks")
        check_labels(first, "propagate_masks")
    out, ws = None, None
    for s, k, r in run_sequences_bidirectional(model, sequences, iters, warm_start=warm_start, batch_size=batch_size,
                                               mode=mode, device=device, alpha1=alpha1, alpha2=alpha2):
        if out is None:
            dev = r["flow_up_bw"].device
            out = [torch.empty(len(seq), *first.shape, dtype=torch.uint8, device=dev) for seq, first in zip(sequences, firsts)]
            for o, first in zip(out, firsts):
                o[0] = first
            if dev.type == "cuda":
                ws = torch.empty(native.rnc.propagate_labels_workspace_bytes(1, *firsts[0].shape), dtype=torch.uint8,
                                 device=dev)
        labels = out[s]
        _step(labels[k][None], r["flow_up_bw"][None], r["occ_bw"][None], labels[k + 1][None], ws)
    return out


@torch.no_grad()
def validate_segmentation(model, sequences, gt_labels, iters=32, warm_start=False, batch_size=8, mode="sintel",
                          device="cuda", alpha1=0.01, alpha2=0.5):
    """DAVIS's semi-supervised J and F of propagate_masks on a split of videos: J&F-Mean, J-Mean, J-Recall, J-Decay, F-Mean,
    F-Recall, F-Decay and the object and video counts (rnc.segment.summarize_segmentation).  sequences: list of V frame
    lists, every frame [3,H,W] (0..255), each video of T_v >= 3 frames and one size (videos may differ in size); gt_labels: V
    integer [T_v,H,W] label maps (0 background, 1..254 objects, 255 void).  Each video starts from its ground truth's frame 0
    with void mapped to 0; its objects are 1..K, K its frame 0's largest non-void label, scored on frames 1..T_v-2 by
    rnc.segment.segmentation_counts on the device.  Videos of one frame size run through one propagate_masks call.  The
    counts are integers, so the result does not depend on batch_size or on the order of the videos.  Under
    torch.distributed rank r takes the videos of index = r (mod world), the per-video counts are all-gathered, and every rank
    returns the single-process result."""
    from .dist import gather_strided, strided_items, world_rank
    from .segment import VOID, segmentation_counts, summarize_segmentation
    world, rank = world_rank()
    _check_counts(sequences, "validate_segmentation", ("ground-truth label sets", gt_labels))
    for seq, gt in zip(sequences, gt_labels):
        _check_frames(seq, "validate_segmentation", 3, " (the first and last are not scored)")
        if tuple(gt.shape) != (len(seq), *seq[0].shape[-2:]):
            raise ValueError(f"validate_segmentation: expected ground truth {[len(seq), *seq[0].shape[-2:]]}, got "
                             f"{list(gt.shape)}")
    mine = list(strided_items(range(len(sequences)), world, rank))
    counts = {}
    for idx in _by_size(sequences, mine):
        firsts = [torch.where(gt_labels[i][0] == VOID, 0, gt_labels[i][0]) for i in idx]
        preds = propagate_masks(model, [sequences[i] for i in idx], firsts, iters, warm_start, batch_size, mode, device,
                                alpha1, alpha2)
        for i, first, pred in zip(idx, firsts, preds):
            K = int(first.max())
            gt = gt_labels[i].to(pred.device)
            counts[i] = segmentation_counts(pred[1:-1], gt[1:-1], K).tolist()
    return summarize_segmentation(gather_strided([counts[i] for i in mine], world))


def inpaint_videos(model, sequences, masks, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                   alpha1=0.01, alpha2=0.5, sweeps=512, max_distance=None):
    """Remove the masked regions of V videos (rnc.inpaint's rule: complete the flows inside the holes, carry each hole pixel
    along them to the nearest frames that see it, fill what no frame sees spatially).  sequences: list of V frame lists,
    every frame [3,H,W] (0..255), each video of T_v >= 2 frames and one size (videos may differ in size); masks: V [T_v,H,W]
    tensors, non-zero where a pixel is to be filled.  Returns a list of V (frames float32 [T_v,3,H,W], source uint8
    [T_v,H,W]) on the device, source being rnc.inpaint's SOURCE_* map.

    The model sees the frames with every hole pixel set to 0, so the result depends only on the known pixels, as an
    inpainting benchmark feeds a corrupted video.  Videos of one frame size run together:
    run_sequences_bidirectional(model, ..., iters, warm_start, batch_size, mode, device) runs first, and each pair's flow_up
    and flow_up_bw are copied into stacked device tensors as they are yielded; a shorter video's missing pairs are zero flows
    occluded in both directions, so no chain enters them.  rnc.inpaint's steps 2-4 then complete the stacked flows in place
    (harmonic_fill with `sweeps`), check them with fb_consistency(alpha1, alpha2), propagate (chains of at most
    max_distance frames; None: no limit) and fill the rest.  With T the longest video's frame count, a size group keeps
    V T (12 B frames + 12 B result + 1 B mask + 1 B source) + V (T - 1) (2 flows x 2 channels x 4 B + 2 masks x 1 B) ~ 44
    V T bytes per pixel, plus at most 1 GiB of fill workspace: e.g. 7.2 GB for eight 50-frame videos of 480x854.
    ValueError before the flow pass for a video of fewer than two frames, a mask of another shape, a side above 4096, a
    mask count that does not match the videos, sweeps < 0 or max_distance < 1.  Inference only: with grad enabled on a
    model that requires grad it raises ValueError."""
    from .inpaint import _check_sweeps, _max_distance, _run
    _check_inference(model, "inpaint_videos")
    masks, = _check_counts(sequences, "inpaint_videos", ("mask sets", masks))
    _check_sweeps(sweeps, "inpaint_videos")
    for seq, m in zip(sequences, masks):
        _check_frames(seq, "inpaint_videos")
        if tuple(m.shape) != (len(seq), *seq[0].shape[-2:]):
            raise ValueError(f"inpaint_videos: expected masks {[len(seq), *seq[0].shape[-2:]]}, got {list(m.shape)}")
        check_sides(*m.shape[-2:], "inpaint_videos")
        _max_distance(max_distance, "inpaint_videos", len(seq))
    out = [None] * len(sequences)
    for idx in _by_size(sequences, range(len(sequences))):
        seqs = [sequences[i] for i in idx]
        holes = [masks[i] != 0 for i in idx]
        seen = [[torch.where(h[t].to(f.device), 0.0, f.float()) for t, f in enumerate(seq)] for seq, h in zip(seqs, holes)]
        flows = _PairStack(seqs, ("flow_up", "flow_up_bw"))
        for s, k, r in run_sequences_bidirectional(model, seen, iters, warm_start=warm_start, batch_size=batch_size,
                                                   mode=mode, device=device, alpha1=alpha1, alpha2=alpha2):
            flows.add(s, k, r)
        dev = flows["flow_up"].device
        frames = _pad_videos([torch.stack([f.to(dev).float() for f in seq]) for seq in seqs], 0)
        hole = _pad_videos([h.to(dev, torch.uint8) for h in holes], 0)
        lens = [len(seq) for seq in seqs]
        res, source = _run(frames, hole, flows["flow_up"], flows["flow_up_bw"], sweeps, max_distance, alpha1, alpha2,
                           lengths=lens)
        for v, i in enumerate(idx):
            out[i] = (res[v, :lens[v]], source[v, :lens[v]])
    return out


@torch.no_grad()
def validate_inpainting(model, sequences, masks, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                        alpha1=0.01, alpha2=0.5, sweeps=512, max_distance=None):
    """PSNR and SSIM of inpaint_videos against the uncorrupted videos: psnr, ssim, and the scored frame and video counts
    (rnc.inpaint.summarize_inpainting).  sequences: the ground-truth videos, as inpaint_videos takes them; masks: V [T_v,H,W]
    hole masks.  Only frames with at least one hole pixel are scored: PSNR from rnc.interp.interpolation_error's fp64
    squared-error sum (100 dB for a frame without error), SSIM from rnc.inpaint.ssim, each averaged over a video's scored
    frames and then over videos.  A frame's partials do not depend on the batch.  Under torch.distributed rank r takes the
    videos of index = r (mod world), the per-frame partials are all-gathered, and every rank returns the single-process
    result."""
    from .dist import gather_strided, strided_items, world_rank
    from .inpaint import ssim, summarize_inpainting
    from .interp import interpolation_error
    world, rank = world_rank()
    _check_counts(sequences, "validate_inpainting", ("mask sets", masks))
    mine = list(strided_items(range(len(sequences)), world, rank))
    got = inpaint_videos(model, [sequences[i] for i in mine], [masks[i] for i in mine], iters, warm_start, batch_size, mode,
                         device, alpha1, alpha2, sweeps, max_distance)
    records = []
    for i, (pred, _) in zip(mine, got):
        dev = pred.device
        scored = (masks[i] != 0).flatten(1).any(1).nonzero().flatten().tolist()
        if not scored:
            records.append([])
            continue
        gt = torch.stack([sequences[i][t].to(dev).float() for t in scored])
        err = interpolation_error(pred[scored], gt)
        s, c = ssim(pred[scored], gt)
        records.append([list(r) for r in zip(err.sq_sum.tolist(), err.count.tolist(), s.tolist(), c.tolist())])
    return summarize_inpainting(gather_strided(records, world))


def _consistent_steps(model, sequences, processed, iters, warm_start, batch_size, mode, device, alpha1, alpha2, lam, alpha,
                      sweeps, what):
    """make_temporally_consistent's loop: yields (video, pair, result, outputs) after each step, outputs being the list of
    V [T_v,C,H,W] results on the device, frame pair + 1 of the video just written."""
    from . import native
    from .temporal import _check_params, temporal_step
    _check_inference(model, what)
    procs, = _check_counts(sequences, what, ("processed videos", processed))
    _check_params(lam, alpha, sweeps, what)
    for seq, p in zip(sequences, procs):
        _check_frames(seq, what)
        if p.dim() != 4 or p.shape[0] != len(seq) or tuple(p.shape[2:]) != tuple(seq[0].shape[-2:]):
            raise ValueError(f"{what}: expected processed frames [{len(seq)},C,{seq[0].shape[-2]},{seq[0].shape[-1]}], got "
                             f"{list(p.shape)}")
        if not 1 <= p.shape[1] <= native.HARMONIC_MAX_CHANNELS:
            raise ValueError(f"{what}: expected 1 to {native.HARMONIC_MAX_CHANNELS} processed channels, got {p.shape[1]}")
        check_sides(*p.shape[-2:], what)
    out, ws = None, {}
    for s, k, r in run_sequences_bidirectional(model, sequences, iters, warm_start=warm_start, batch_size=batch_size,
                                               mode=mode, device=device, alpha1=alpha1, alpha2=alpha2):
        dev = r["flow_up_bw"].device
        if out is None:
            out = [torch.empty(p.shape, dtype=torch.float32, device=dev) for p in procs]
            for o, p in zip(out, procs):
                o[0] = p[0]
        o, seq = out[s], sequences[s]
        C = o.shape[1]
        if dev.type == "cuda" and C not in ws:
            ws[C] = torch.empty(native.rnc.temporal_step_workspace_bytes(1, C, *o.shape[-2:]), dtype=torch.uint8, device=dev)
        i0, i1 = (seq[j].to(dev).float()[None] for j in (k, k + 1))
        temporal_step(o[k][None], procs[s][k + 1].to(dev)[None], i0, i1, r["flow_up_bw"][None], r["occ_bw"][None], lam, alpha,
                      sweeps, out=o[k + 1][None], workspace=ws.get(C))
        yield s, k, r, out


def make_temporally_consistent(model, sequences, processed, iters=32, warm_start=False, batch_size=8, mode="sintel",
                               device="cuda", alpha1=0.01, alpha2=0.5, lam=0.1, alpha=50.0, sweeps=512):
    """Remove the flicker of V videos processed frame by frame (rnc.temporal's rule: each output frame keeps its processed
    frame's gradients and is pulled toward the previous output, warped along the backward flow, where the flow is matched
    and the frames agree).  sequences: list of V original frame lists, every frame [3,H,W] (0..255) of one size, each video
    of T_v >= 2 frames; processed: V tensors [T_v,C,H,W], 1 <= C <= 4, the per-frame results (any range).  Returns a list of
    V float32 [T_v,C,H,W] tensors on the device, frame 0 being the processed frame 0.

    The flows come from the original frames: run_sequences_bidirectional(model, sequences, iters, warm_start, batch_size,
    mode, device, alpha1=alpha1, alpha2=alpha2) yields each video's pairs in order, and pair k's flow_up_bw and occ_bw step
    that video from frame k to k + 1 at once (rnc.temporal.temporal_step with lam, alpha and sweeps, one rnc_temporal_step
    call), so no flow is kept: the memory is the outputs.  ValueError before the flow pass for a video of fewer than two
    frames, processed frames of another shape, a channel count outside 1..4, a side above 4096, a processed-video count that
    does not match the videos or a bad lam, alpha or sweeps.  Inference only: with grad enabled on a model that requires
    grad it raises ValueError."""
    out = []
    for *_, out in _consistent_steps(model, sequences, processed, iters, warm_start, batch_size, mode, device, alpha1, alpha2,
                                     lam, alpha, sweeps, "make_temporally_consistent"):
        pass
    return out if sequences else []


@torch.no_grad()
def validate_temporal_consistency(model, sequences, processed, iters=32, warm_start=False, batch_size=8, mode="sintel",
                                  device="cuda", alpha1=0.01, alpha2=0.5, lam=0.1, alpha=50.0, sweeps=512):
    """The warping error of a split's processed videos and of make_temporally_consistent's outputs, with the outputs'
    fidelity to the processed frames (so that freezing a video does not score well): warping_error_processed,
    warping_error, psnr, ssim, and the frame and video counts (rnc.temporal.summarize_temporal).  sequences and processed as
    make_temporally_consistent's.  Each pair's flows score frame k + 1 of both videos as it is stepped
    (rnc.temporal.warping_error, on the device); psnr (rnc.interp.interpolation_error, 100 dB cap) and ssim (rnc.inpaint.ssim)
    compare O_t with P_t over frames 1..T_v-1 (frame 0 is P_0 by the rule) when C = 3 and the frames are at least 11x11,
    and are NaN otherwise.  The partials are per frame, so the result does not depend on batch_size or on the order of the
    videos.  Under torch.distributed rank r takes the videos of index = r (mod world), the per-frame partials are
    all-gathered, and every rank returns the single-process result."""
    from .dist import gather_strided, strided_items, world_rank
    from .inpaint import SSIM_RADIUS, ssim
    from .interp import interpolation_error
    from .temporal import summarize_temporal, warping_error
    world, rank = world_rank()
    procs, = _check_counts(sequences, "validate_temporal_consistency", ("processed videos", processed))
    mine = list(strided_items(range(len(sequences)), world, rank))
    warp = {i: [None] * (len(sequences[i]) - 1) for i in mine}
    got = None
    for s, k, r, out in _consistent_steps(model, [sequences[i] for i in mine], [procs[i] for i in mine], iters, warm_start,
                                          batch_size, mode, device, alpha1, alpha2, lam, alpha, sweeps,
                                          "validate_temporal_consistency"):
        dev = out[s].device
        g, m = r["flow_up_bw"][None, None], r["occ_bw"][None, None]
        wp = warping_error(procs[mine[s]][k:k + 2].to(dev)[None], g, m)
        wo = warping_error(out[s][k:k + 2][None], g, m)
        warp[mine[s]][k] = (wp[0][0, 0], wo[0][0, 0], wp[1][0, 0])
        got = out
    records = []
    for j, i in enumerate(mine):
        o = got[j]
        p = procs[i].to(o.device).float()
        T, C, H, W = o.shape
        rows = [[float(a), float(b), int(c)] for a, b, c in warp[i]]
        nan = [[math.nan] * 4 for _ in range(T - 1)]
        if C == 3 and min(H, W) >= 2 * SSIM_RADIUS + 1:
            err = interpolation_error(o[1:], p[1:])
            ss, sc = ssim(o[1:], p[1:])
            nan = [list(x) for x in zip(err.sq_sum.tolist(), err.count.tolist(), ss.tolist(), sc.tolist())]
        records.append([a + b for a, b in zip(rows, nan)])
    return summarize_temporal(gather_strided(records, world))


def stabilize_videos(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda", radius=30,
                     sigma=10.0, crop=True, crop_min=0.5, stride=8, hypotheses=256, tau=2.0, refine=4, seed=0, fill=False,
                     sweeps=512, max_distance=None, alpha1=0.01, alpha2=0.5):
    """Stabilize V videos (rnc.stabilize's rule: fit each pair's camera motion to its forward flow by RANSAC, smooth the
    camera path with a Gaussian of sigma frames over +-radius frames, zoom in to crop the uncovered borders, and warp).
    sequences: list of V frame lists, every frame [3,H,W] (0..255) of one size, each video of T_v >= 2 frames.  Returns a
    list of V dicts on the device: frames float32 [T_v,3,H,W], valid uint8 [T_v,H,W] (0 where the output pixel has no input,
    which happens only when the video's alpha is under crop_min or crop=False), motion fp64 [T_v-1,3,3] (A_k, frame k ->
    k+1), transforms fp64 [T_v,3,3] (M_t, input frame t -> output frame t), alpha (fp64 scalar tensor, the closed-form
    crop scale before crop_min applies), and inliers, matched and status int32 [T_v-1] of each pair's fit.

    run_sequences(model, sequences, iters, warm_start, batch_size, mode, device) yields each pair's forward flow, which is
    fitted at once (rnc.stabilize.fit_homographies with stride, hypotheses, tau, refine and seed) and dropped: only its 3x3
    matrix is kept.  The forward flow is enough: RANSAC rejects the pixels a backward check would flag.  Then each video's
    path is smoothed (smooth_path) and its frames warped (warp_frames) on the device.  ValueError before the flow pass for a
    video of fewer than two frames, a side above 4096 or a bad radius, sigma, crop_min, stride, hypotheses, tau, refine,
    seed, sweeps, max_distance, alpha1 or alpha2.  Inference only: with grad enabled on a model that requires grad it raises
    ValueError.

    fill=True fills every pixel with valid = 0 from the neighbouring frames (rnc.stabilize's step 5, the motion inpainting
    of Matsushita et al.), and each dict gains source uint8 [T_v,H,W] (rnc.inpaint's SOURCE_* map, SOURCE_KNOWN where the
    pixel comes from its own frame).  crop and fill are independent: crop=False, fill=True is the full-frame stabilizer;
    crop=True with crop_min above the video's alpha zooms part of the way and fills the rest.  The flow pass is then
    run_sequences_bidirectional(..., alpha1=alpha1, alpha2=alpha2), whose forward flows are run_sequences' bit for bit, so
    motion, transforms, alpha, the fit counts, valid and the pixels with valid != 0 are fill=False's; both flows of every
    pair are kept in stacked device tensors, a shorter video padded as inpaint_videos pads it.  Then
    rnc.stabilize.fill_uncovered(..., sweeps, max_distance, alpha1, alpha2) runs on the stack.  With T the longest video's
    frame count it keeps V T (12 B warped + 12 B filled frames + 1 B valid + 1 B hole + 1 B source) + V (T - 1) (2 flows
    and 2 residuals x 2 channels x 4 B + 2 occlusion masks x 1 B + 2 x 4 B of consistency error while it is checked) ~ 69
    V T bytes per pixel, plus at most 1 GiB of fill workspace: e.g. 11.3 GB for eight 50-frame videos of 480x854 (17.3 GB
    peak measured on that workload with the model, its workspace and the input frames on the device)."""
    from .stabilize import (_check_fill_params, _check_fit_params, _check_path_params, fit_homographies, smooth_path,
                            warp_frames)
    what = "stabilize_videos"
    _check_inference(model, what)
    _check_fit_params(stride, hypotheses, tau, refine, seed, what)
    _check_path_params(radius, sigma, crop_min, what)
    if fill:
        _check_fill_params(sweeps, max_distance, alpha1, alpha2, what)
    for seq in sequences:
        _check_frames(seq, what)
        check_sides(*seq[0].shape[-2:], what)
    from . import native
    fits = [[None] * (len(seq) - 1) for seq in sequences]
    ws = None
    flows = _PairStack(sequences, ("flow_up", "flow_up_bw")) if fill else None
    kw = dict(warm_start=warm_start, batch_size=batch_size, mode=mode, device=device)
    if fill:
        pairs = run_sequences_bidirectional(model, sequences, iters, alpha1=alpha1, alpha2=alpha2, **kw)
    else:
        pairs = ((s, k, {"flow_up": flow}) for s, k, flow in run_sequences(model, sequences, iters, **kw))
    for s, k, r in pairs:
        flow = r["flow_up"]
        if flow.is_cuda and ws is None:
            H, W = flow.shape[-2:]
            ws = torch.empty(native.rnc.homography_fit_workspace_bytes(1, H, W, stride, hypotheses), dtype=torch.uint8,
                             device=flow.device)
        fits[s][k] = fit_homographies(flow[None], stride, hypotheses, tau, refine, seed, workspace=ws)
        if fill:
            flows.add(s, k, r)
    out = []
    for seq, fit in zip(sequences, fits):
        A, inl, mat, st = (torch.cat([f[j] for f in fit]) for j in range(4))
        dev = A.device
        H, W = seq[0].shape[-2:]
        M, Minv, alpha = smooth_path(A[None], H, W, radius, sigma, crop, crop_min)
        frames, valid = warp_frames(torch.stack([f.to(dev).float() for f in seq]), Minv[0])
        out.append({"frames": frames, "valid": valid, "motion": A, "transforms": M[0], "alpha": alpha[0], "inliers": inl,
                    "matched": mat, "status": st})
        if fill:
            out[-1]["transforms_inv"] = Minv[0]
    if fill and out:
        _fill_stabilized(out, flows, sweeps, max_distance, alpha1, alpha2)
    return out


def _fill_stabilized(out, flows, sweeps, max_distance, alpha1, alpha2):
    """stabilize_videos' fill: the results stacked and padded (zero frames without holes, identity motion and maps, and
    _fill's padding pairs occluded in both directions), filled, and written back into each dict with its source map."""
    from .stabilize import _fill
    lens = [r["frames"].shape[0] for r in out]
    eye = torch.eye(3, dtype=torch.float64, device=out[0]["frames"].device)
    frames = _pad_videos([r["frames"] for r in out], 0)
    valid = _pad_videos([r["valid"] for r in out], 1)
    motion, maps = (_pad_videos([r[key] for r in out], eye) for key in ("motion", "transforms"))
    maps_inv = _pad_videos([r.pop("transforms_inv") for r in out], eye)
    res, source = _fill(frames, valid, flows["flow_up"], flows["flow_up_bw"], motion, maps, maps_inv, sweeps, max_distance,
                        alpha1, alpha2, lengths=lens)
    for v, r in enumerate(out):
        r["frames"], r["source"] = res[v, :lens[v]], source[v, :lens[v]]


@torch.no_grad()
def validate_stabilization(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda", radius=30,
                           sigma=10.0, crop=True, crop_min=0.5, stride=8, hypotheses=256, tau=2.0, refine=4, seed=0, fill=False,
                           sweeps=512, max_distance=None, alpha1=0.01, alpha2=0.5):
    """The standard stabilization scores of stabilize_videos' output beside the input's (Liu et al. 2013; ITF of Matsushita
    et al. 2006), from the known maps rather than re-estimated features (rnc.stabilize.stabilization_metrics, on the host in
    fp64): cropping, distortion, stability_translation, stability_rotation and stability of the output, and the input's
    input_stability_*; itf and input_itf, each the mean over a video's consecutive frame pairs of their PSNR
    (rnc.interp.interpolation_error's partials on the device, rnc.inpaint.psnr's 100 dB cap), then over videos; frames and
    videos, their numbers (rnc.stabilize.summarize_stabilization).  Arguments as stabilize_videos'.  With fill=True two
    scores are added, each the mean over a video's frames and then over videos: filled, the share of output pixels not
    taken from their own frame (source != SOURCE_KNOWN), and filled_spatial, the share filled spatially (SOURCE_SPATIAL).
    Under torch.distributed rank r takes the videos of index = r (mod world), the per-video records are all-gathered, and
    every rank returns the single-process result."""
    from .dist import gather_strided, strided_items, world_rank
    from .inpaint import SOURCE_KNOWN, SOURCE_SPATIAL
    from .interp import interpolation_error
    from .stabilize import stabilization_metrics, summarize_stabilization
    world, rank = world_rank()
    mine = [sequences[i] for i in strided_items(range(len(sequences)), world, rank)]
    res = stabilize_videos(model, mine, iters, warm_start, batch_size, mode, device, radius, sigma, crop, crop_min, stride,
                           hypotheses, tau, refine, seed, fill, sweeps, max_distance, alpha1, alpha2)
    records = []
    for seq, r in zip(mine, res):
        out = r["frames"]
        inp = torch.stack([f.to(out.device).float() for f in seq])
        rows = [interpolation_error(v[1:], v[:-1]) for v in (out, inp)]
        rec = (stabilization_metrics(r["motion"], r["transforms"]),
               *[list(zip(e.sq_sum.tolist(), e.count.tolist())) for e in rows])
        if fill:                                         # per frame: pixels, filled pixels, spatially filled pixels
            src = r["source"].flatten(1)
            rec += ([[src.shape[1], a, b] for a, b in zip((src != SOURCE_KNOWN).sum(1).tolist(),
                                                          (src == SOURCE_SPATIAL).sum(1).tolist())],)
        records.append(rec)
    records = gather_strided(records, world)
    summary = summarize_stabilization([r[:3] for r in records])
    if fill:
        n = len(records)
        for j, key in ((1, "filled"), (2, "filled_spatial")):
            summary[key] = sum(sum(f[j] / f[0] for f in r[3]) / len(r[3]) for r in records) / n if n else math.nan
    return summary


def size_batches(items, batch_size, key):
    """Batches of create_kitti_submission: the items of one key(item) (a frame size) in order of appearance, batch_size at a
    time.  A batch is yielded as soon as it is full, the partial batches at the end in order of their size's first
    appearance, so that at most batch_size items of each size are held at once."""
    if batch_size < 1:
        raise ValueError(f"batch_size must be >= 1, got {batch_size}")
    open_batches = {}
    for it in items:
        b = open_batches.setdefault(key(it), [])
        b.append(it)
        if len(b) == batch_size:
            yield open_batches.pop(key(it))
    yield from open_batches.values()


class _SubmissionWriter:
    """Writes each step's flows, and with write_png their colour coding, to files on a thread pool while the next step
    computes.  step() colour-codes the step's flows in one rnc.viz launch and enqueues their copies to pinned host buffers;
    the pool's threads wait for those copies and encode the files (cv2.imwrite and file writes release the GIL).  The pool
    has a thread per core this process may run on, and at most MAX_STEPS steps are in flight, so host memory stays
    bounded.  Leaving the context waits for every file; a writer thread's exception is raised there or from step()."""
    MAX_STEPS = 2

    def __init__(self):
        cores = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else os.cpu_count()
        self.pool = ThreadPoolExecutor(max_workers=max(1, cores or 1), thread_name_prefix="rnc-submission")
        self.inflight = deque()

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc, tb):
        try:
            if exc_type is None:
                while self.inflight:
                    self._retire()
        finally:
            for futs in self.inflight:
                for f in futs:
                    f.cancel()
            self.pool.shutdown(wait=True)

    def _retire(self):
        for f in self.inflight.popleft():
            f.result()

    def step(self, flows, files, write_flow):
        """flows: [n,2,H,W] (any strides); files: n (flow path, png path or None); write_flow(path, [H,W,2] float32)."""
        png = None
        if any(p is not None for _, p in files):
            from .viz import flow_to_image
            png = _to_host(flow_to_image(flows))
        flo = _to_host(flows.permute(0, 2, 3, 1))
        done = None
        if flows.is_cuda:
            done = torch.cuda.Event()
            done.record(torch.cuda.current_stream(flows.device))
        for f, p in files:
            os.makedirs(os.path.dirname(f) or ".", exist_ok=True)
            if p is not None:
                os.makedirs(os.path.dirname(p) or ".", exist_ok=True)
        self.inflight.append([self.pool.submit(_write_pair, done, write_flow, f, flo[j], p, None if p is None else png[j])
                              for j, (f, p) in enumerate(files)])
        while len(self.inflight) > self.MAX_STEPS:
            self._retire()


def _to_host(x):
    """Enqueue a copy of x into a contiguous (pinned, for a CUDA x) host tensor."""
    x = x.contiguous()
    if not x.is_cuda:
        return x.clone()
    return torch.empty(x.shape, dtype=x.dtype, pin_memory=True).copy_(x, non_blocking=True)


def _write_pair(done, write_flow, flo_path, flo, png_path, png):
    if done is not None:
        done.synchronize()
    write_flow(flo_path, flo.numpy())
    if png_path is not None:
        import cv2
        if not cv2.imwrite(png_path, png.numpy()):
            raise OSError(f"cv2.imwrite could not write {png_path}")


def _model_device(model):
    from .engine import module_device
    return module_device(model) or torch.device("cuda", torch.cuda.current_device())


@torch.no_grad()
def create_sintel_submission(model, sequences, iters=32, warm_start=False, output_path="sintel_submission", write_png=False,
                             batch_size=8):
    """create_sintel_submission (evaluate.py:23-55) on run_sequences.  sequences: iterable of (dstype, scene, frames), frames
    a list of [3,H,W] images of one size for all sequences.  Writes output_path/dstype/scene/frame%04d.flo for pair k (frames
    k, k + 1) with k + 1 in the name, and with write_png its colour coding (rnc.viz, as utils.flow_viz) to
    output_path + "_png"/dstype/scene/frame%04d.png.  Files are written on a thread pool while the next step computes;
    returns when all are written.  Under torch.distributed each rank runs whole sequences, assigned longest-first by pair count
    (rnc.dist.greedy_assignment), and no rank returns before every rank's files are written."""
    from .dist import barrier, greedy_assignment, world_rank
    seqs = list(sequences)
    world, rank = world_rank()
    if world > 1:
        owner = greedy_assignment([max(len(f) - 1, 0) for _, _, f in seqs], world)
        seqs = [s for s, r in zip(seqs, owner) if r == rank]
    try:
        frames = [f for _, _, f in seqs]
        steps = sequence_schedule([len(f) for f in frames], batch_size)
        flows = run_sequences(model, frames, iters=iters, warm_start=warm_start, batch_size=batch_size,
                              device=_model_device(model))
        with _SubmissionWriter() as w:
            for step in steps:
                got = [next(flows) for c in step if not c.idle]
                files = []
                for s, k, _ in got:
                    dstype, scene, _ = seqs[s]
                    name = "frame%04d" % (k + 1)
                    files.append((os.path.join(output_path, dstype, scene, name + ".flo"),
                                  os.path.join(output_path + "_png", dstype, scene, name + ".png") if write_png else None))
                w.step(torch.stack([f for _, _, f in got]), files, frame_utils.writeFlow)
    finally:
        barrier()


@torch.no_grad()
def create_kitti_submission(model, pairs, iters=24, output_path="kitti_submission", write_png=False, batch_size=8):
    """create_kitti_submission (evaluate.py:58-87) in batches.  pairs: iterable of (frame_id, image1 [3,H,W], image2), of any
    mix of sizes; pairs of one size run together, batch_size at a time (size_batches), padded as InputPadder(mode="kitti").
    Writes output_path/frame_id (frame_utils.writeFlowKITTI) and with write_png output_path + "_png"/(frame_id + ".png").
    Files are written on a thread pool while the next batch computes; returns when all are written.  Under torch.distributed
    rank r runs the pairs of index = r (mod world), and no rank returns before every rank's files are written."""
    from .dist import barrier, strided_items, world_rank
    model.eval()
    device = _model_device(model)
    world, rank = world_rank()
    try:
        with _SubmissionWriter() as w:
            for batch in size_batches(strided_items(pairs, world, rank), batch_size, key=lambda p: tuple(p[1].shape)):
                padder = InputPadder(batch[0][1].shape, mode="kitti")
                im1 = _stack([p[1] for p in batch], device, padder)
                im2 = _stack([p[2] for p in batch], device, padder)
                _, flow_pr = model(im1, im2, iters=iters, test_mode=True)
                files = [(os.path.join(output_path, fid), os.path.join(output_path + "_png", fid + ".png") if write_png else None)
                         for fid, _, _ in batch]
                w.step(padder.unpad(flow_pr), files, frame_utils.writeFlowKITTI)
    finally:
        barrier()


def load_checkpoint(model, state):
    """Checkpoints are saved from an nn.DataParallel wrapper (train.py:231): strip the `module.` prefix when present, then
    load strictly (evaluate.py:252-257 loads into the wrapper instead)."""
    if isinstance(state, str):
        state = torch.load(state, map_location="cpu")
    state = {(k[7:] if k.startswith("module.") else k): v for k, v in state.items()}
    return model.load_state_dict(state)
