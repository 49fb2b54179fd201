"""Evaluation loops in the shape of the reference's drivers (evaluate.py:111-143 validate_sintel, :146-182
validate_kitti, :25-55 create_sintel_submission with warm start), runnable on any iterable of samples — the datasets
themselves are out of scope (no data offline, SURVEY.md C12), so `bench.py` / the tests feed synthetic pairs.

Differences from the reference, all behaviour-preserving: pairs of equal size are evaluated in batches instead of one at a
time (the model's batch items are independent; frames of a different size — KITTI's vary — start a new batch), and the
warm-start forward interpolation runs on the GPU.  Metrics aggregate exactly as the reference's loops do: Sintel-style
(`valid` absent) pools all pixels (evaluate.py:131-137), KITTI-style averages per-image means (evaluate.py:172-179).
"""
from collections import deque, namedtuple

import numpy as np
import torch

from utils.utils import InputPadder, forward_interpolate


@torch.no_grad()
def validate(model, samples, iters=32, mode="sintel", batch_size=8, device="cuda"):
    """samples: iterable of (image1 [3,H,W], image2 [3,H,W], flow_gt [2,H,W], valid [H,W] or None).
    Returns the metrics validate_sintel / validate_kitti print: EPE, 1px/3px/5px, and KITTI F1 when `valid` is given."""
    model.eval()
    epe_all, f1_all, batch = [], [], []
    epe_img = []                                            # KITTI: per-image mean EPE (evaluate.py:172)

    def flush():
        if not batch:
            return
        im1 = torch.stack([b[0] for b in batch]).to(device).float()
        im2 = torch.stack([b[1] for b in batch]).to(device).float()
        padder = InputPadder(im1.shape, mode=mode)
        p1, p2 = padder.pad(im1, im2)
        _, flow_pr = model(p1, p2, iters=iters, test_mode=True)
        flow = padder.unpad(flow_pr).cpu()
        for k, (_, _, gt, valid) in enumerate(batch):
            epe = torch.sum((flow[k] - gt) ** 2, dim=0).sqrt()
            if valid is None:
                epe_all.append(epe.view(-1).numpy())
            else:                                           # evaluate.py:163-171
                mag = torch.sum(gt ** 2, dim=0).sqrt().view(-1)
                val = valid.view(-1) >= 0.5
                e = epe.view(-1)
                out = ((e > 3.0) & ((e / mag) > 0.05)).float()
                epe_img.append(e[val].mean().item())
                epe_all.append(e[val].numpy())
                f1_all.append(out[val].numpy())
        batch.clear()

    for s in samples:
        s = s if len(s) == 4 else (s[0], s[1], s[2], None)
        if batch and batch[0][0].shape != s[0].shape:       # frame sizes differ (KITTI): close the batch
            flush()
        batch.append(s)
        if len(batch) == batch_size:
            flush()
    flush()
    e = np.concatenate(epe_all)
    res = {"epe": float(np.mean(e)), "1px": float(np.mean(e < 1)), "3px": float(np.mean(e < 3)), "5px": float(np.mean(e < 5))}
    if f1_all:
        res["epe"] = float(np.mean(epe_img))                # evaluate.py:178: mean of the per-image means
        res["f1"] = float(100 * np.mean(np.concatenate(f1_all)))   # evaluate.py:175,179: pooled over all valid pixels
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


@torch.no_grad()
def run_sequences(model, sequences, iters=32, warm_start=False, batch_size=8, mode="sintel", device="cuda",
                  return_confidence=False):
    """create_sintel_submission (evaluate.py:23-55) over many sequences at batch throughput.  sequences: list of frame lists,
    every frame [3,H,W] of one size.  Yields (seq_index, pair_index, flow): the unpadded [2,H,W] flow_up of every pair, on
    the device; per sequence the flows equal run_sequence(model, seq, iters, warm_start, mode)'s.  return_confidence (NCUP
    model): yields (seq_index, pair_index, flow, confidence), the upsampler's output confidence unpadded like the flow.

    Slots run in lockstep (sequence_schedule).  Each step encodes only new frames: a continuing slot's frame 1 is its last
    frame 2, whose fnet features are handed over on the device (rnc.model.SequenceStage).  With warm_start, a slot starts
    from forward_interpolate of its own previous low-resolution flow, and from zero (a cold start) at pair 0.  The steps
    run eagerly and never wait for the host; the caller moves or writes the flows."""
    sizes = [tuple(f.shape) for seq in sequences for f in seq]
    for s in sizes:
        if len(s) != 3 or s != sizes[0]:
            raise ValueError(f"all frames of one call must have the same [3,H,W] size: got {sizes[0]} and {s}")
    if return_confidence and not model.ncup:
        raise ValueError("return_confidence: the convex-upsampling RAFT has no NCUP upsampler and so no output confidence")
    steps = sequence_schedule([len(seq) for seq in sequences], batch_size)
    if not steps:
        return
    from .engine import _require_cuda, engine_for, module_device
    from .model import SequenceStage
    model.eval()
    padder = InputPadder(sizes[0], mode=mode)
    stage = SequenceStage(model)
    ws = fi = zero = None
    for step in steps:
        im1 = _stack([sequences[c.seq][c.pair] for c in step], device, padder)
        im2 = _stack([sequences[c.seq][c.pair + 1] for c in step], device, padder)
        if ws is None:
            dev = _require_cuda(im1)
            if module_device(model) != dev:
                raise ValueError(f"model parameters are on {module_device(model)} but device is {dev}")
            eng = engine_for(dev)
        stage.restart = [j for j, c in enumerate(step) if c.restart]
        stage.carry = [j for j, c in enumerate(step) if not c.restart and not c.idle]
        with torch.cuda.device(dev), eng.lock:
            if ws is None:
                # this generator's own workspace: the features carried from step to step live in it, so the caller may run
                # other forwards of the same shape between two steps
                pk = eng.packed_update(model.update_block)
                ws = eng.WS(dev, len(step), im1.shape[2] // 8, im1.shape[3] // 8, pk.has_mask, model.ncup)
            for j in stage.restart if fi is not None else ():
                fi[j].copy_(zero)           # cold start: coords0 + 0.0 is exactly coords0, as with flow_init=None
            flow_low, flow_up, *conf = model._forward_eager(eng, im1, im2, iters, fi, True, encode=stage, ws=ws,
                                                            return_confidence=return_confidence)
            if warm_start:
                fi = forward_interpolate(flow_low)
                if zero is None:
                    zero = torch.zeros_like(fi[0])
        for j, c in enumerate(step):
            if not c.idle:
                if return_confidence:
                    yield c.seq, c.pair, padder.unpad(flow_up[j]), padder.unpad(conf[0][j])
                else:
                    yield c.seq, c.pair, padder.unpad(flow_up[j])


def load_checkpoint(model, state):
    """Checkpoints are saved from an nn.DataParallel wrapper (train.py:231): strip the `module.` prefix when present, then
    load strictly (evaluate.py:252-257 loads into the wrapper instead)."""
    if isinstance(state, str):
        state = torch.load(state, map_location="cpu")
    state = {(k[7:] if k.startswith("module.") else k): v for k, v in state.items()}
    return model.load_state_dict(state)
