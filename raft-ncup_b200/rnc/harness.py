"""Evaluation loops in the shape of the reference's drivers (evaluate.py:111-143 validate_sintel, :146-182
validate_kitti, :25-55 create_sintel_submission with warm start), runnable on any iterable of samples — the datasets
themselves are out of scope (no data offline, SURVEY.md C12), so `bench.py` / the tests feed synthetic pairs.

Differences from the reference, all behaviour-preserving: pairs of equal size are evaluated in batches instead of one at a
time (the model's batch items are independent; frames of a different size — KITTI's vary — start a new batch), and the
warm-start forward interpolation runs on the GPU.  Metrics aggregate exactly as the reference's loops do: Sintel-style
(`valid` absent) pools all pixels (evaluate.py:131-137), KITTI-style averages per-image means (evaluate.py:172-179).
"""
import os
from collections import deque, namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from utils import frame_utils
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
    returns when all are written."""
    seqs = list(sequences)
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


@torch.no_grad()
def create_kitti_submission(model, pairs, iters=24, output_path="kitti_submission", write_png=False, batch_size=8):
    """create_kitti_submission (evaluate.py:58-87) in batches.  pairs: iterable of (frame_id, image1 [3,H,W], image2), of any
    mix of sizes; pairs of one size run together, batch_size at a time (size_batches), padded as InputPadder(mode="kitti").
    Writes output_path/frame_id (frame_utils.writeFlowKITTI) and with write_png output_path + "_png"/(frame_id + ".png").
    Files are written on a thread pool while the next batch computes; returns when all are written."""
    model.eval()
    device = _model_device(model)
    with _SubmissionWriter() as w:
        for batch in size_batches(pairs, batch_size, key=lambda p: tuple(p[1].shape)):
            padder = InputPadder(batch[0][1].shape, mode="kitti")
            im1 = _stack([p[1] for p in batch], device, padder)
            im2 = _stack([p[2] for p in batch], device, padder)
            _, flow_pr = model(im1, im2, iters=iters, test_mode=True)
            files = [(os.path.join(output_path, fid), os.path.join(output_path + "_png", fid + ".png") if write_png else None)
                     for fid, _, _ in batch]
            w.step(padder.unpad(flow_pr), files, frame_utils.writeFlowKITTI)


def load_checkpoint(model, state):
    """Checkpoints are saved from an nn.DataParallel wrapper (train.py:231): strip the `module.` prefix when present, then
    load strictly (evaluate.py:252-257 loads into the wrapper instead)."""
    if isinstance(state, str):
        state = torch.load(state, map_location="cpu")
    state = {(k[7:] if k.startswith("module.") else k): v for k, v in state.items()}
    return model.load_state_dict(state)
