"""Validation throughput: rnc.harness.validate against the host-metrics loop it replaces and against the batched forward alone,
plus the metrics kernel's own time.

    python tools/validate_bench.py [--pairs N] [--out DIR]
    torchrun --nproc_per_node G tools/validate_bench.py      (adds the scaling of validate over G GPUs)

Samples are synthetic Sintel-size pairs (436x1024, rnc.synth.frames, a random ground truth) held as CPU tensors, as a
DataLoader delivers them; raft_nc_dbl, B = 8, 32 iterations.  Prints one JSON line per measurement, each with the card name
and power limit read in the same run:
  kernel     rnc.metrics.flow_metrics at B = 8 on the unpadded view of a 440-row batch, without and with a valid mask: CUDA
             events around each of 50 launches, median and range;
  validate   pairs/s of validate(batch_size=8), of the previous loop (restated below: blocking pageable uploads, every flow
             copied to the host, the EPE and the thresholds computed there), and of the batched forward on inputs already
             padded on the device (the ceiling), with the largest relative difference of the two loops' metrics;
  scaling    under torchrun: pairs/s of validate over all ranks (the slowest rank's clock) and the single-rank figure.
Each pass is one host clock around the whole call, ended by a device synchronise; every shape is warmed up first.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-ncup_b200")]

ITERS, B, H, W = 32, 8, 436, 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def emit(line, out):
    print(json.dumps(line), flush=True)
    if out:
        with open(os.path.join(out, "validate_bench.jsonl"), "a") as f:
            f.write(json.dumps(line) + "\n")


@torch.no_grad()
def host_metrics_loop(model, samples, iters, batch_size, device):
    """validate() as it was before the metrics moved to the device (Sintel-style samples only)."""
    from utils.utils import InputPadder
    epe_all = []
    for k in range(0, len(samples), batch_size):
        batch = samples[k:k + batch_size]
        im1 = torch.stack([b[0] for b in batch]).to(device).float()
        im2 = torch.stack([b[1] for b in batch]).to(device).float()
        padder = InputPadder(im1.shape)
        p1, p2 = padder.pad(im1, im2)
        _, flow_pr = model(p1, p2, iters=iters, test_mode=True)
        flow = padder.unpad(flow_pr).cpu()
        for j, (_, _, gt) in enumerate(batch):
            epe_all.append(torch.sum((flow[j] - gt) ** 2, dim=0).sqrt().view(-1).numpy())
    e = np.concatenate(epe_all)
    return {"epe": float(np.mean(e)), "1px": float(np.mean(e < 1)), "3px": float(np.mean(e < 3)), "5px": float(np.mean(e < 5))}


def clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=48)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("validate_bench needs a CUDA device")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
        dist.init_process_group("nccl")
    rank = dist.get_rank() if world > 1 else 0
    dev = torch.device("cuda", torch.cuda.current_device())
    out = args.out if rank == 0 else None
    if out:
        os.makedirs(out, exist_ok=True)
    from rnc.harness import validate
    from rnc.metrics import flow_metrics
    from rnc.synth import build_model, frames
    from utils.utils import InputPadder

    cd = card()
    m = build_model("raft_nc_dbl").to(dev)
    im1, im2 = frames(args.pairs, H, W, seed=1)
    g = torch.Generator().manual_seed(2)
    samples = [(im1[i], im2[i], torch.randn(2, H, W, generator=g) * 4) for i in range(args.pairs)]
    del im1, im2

    if world > 1:
        validate(m, samples[:B], iters=ITERS, batch_size=B, device=dev)          # warm-up
        t0 = time.perf_counter()
        validate(m, samples, iters=ITERS, batch_size=B, device=dev)
        torch.cuda.synchronize()
        t = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if rank == 0:
            t1, _ = clock(lambda: validate_one(m, samples))
            emit({"card": cd, "what": "scaling", "world": world, "pairs": args.pairs, "iters": ITERS, "batch_size": B,
                  "pairs_per_s": round(args.pairs / t.item(), 2), "one_rank_pairs_per_s": round(args.pairs / t1, 2)}, out)
        dist.barrier()
        dist.destroy_process_group()
        return

    # kernel
    padder = InputPadder((3, H, W))
    flow_up = torch.randn(B, 2, H + 4, W, device=dev) * 6
    flow = padder.unpad(flow_up)
    gt = torch.randn(B, 2, H, W, device=dev) * 6
    valid = (torch.rand(B, H, W, device=dev) > 0.5).float()
    for v, name in ((None, "dense"), (valid, "valid")):
        for _ in range(5):
            flow_metrics(flow, gt, v)
        ms = []
        for _ in range(50):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            flow_metrics(flow, gt, v)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        emit({"card": cd, "what": "kernel", "mask": name, "B": B, "size": f"{H}x{W}", "ms_median": round(statistics.median(ms), 4),
              "ms_min": round(min(ms), 4), "ms_max": round(max(ms), 4)}, out)
    del flow_up, flow, gt, valid

    # validate, the host-metrics loop, and the forward alone
    validate(m, samples[:B], iters=ITERS, batch_size=B, device=dev)
    host_metrics_loop(m, samples[:B], ITERS, B, dev)
    tn, new = clock(lambda: validate(m, samples, iters=ITERS, batch_size=B, device=dev))
    to, old = clock(lambda: host_metrics_loop(m, samples, ITERS, B, dev))
    resident = []
    for k in range(0, args.pairs, B):
        p = InputPadder((3, H, W))
        resident.append(p.pad(torch.stack([s[0] for s in samples[k:k + B]]).to(dev),
                              torch.stack([s[1] for s in samples[k:k + B]]).to(dev)))

    def forwards():
        with torch.no_grad():
            for p1, p2 in resident:
                m(p1, p2, iters=ITERS, test_mode=True)
    forwards()
    tf, _ = clock(forwards)
    diff = max(abs(new[k] - old[k]) / max(abs(old[k]), 1e-30) for k in old)
    emit({"card": cd, "what": "validate", "pairs": args.pairs, "size": f"{H}x{W}", "iters": ITERS, "batch_size": B,
          "validate_pairs_per_s": round(args.pairs / tn, 2), "host_metrics_loop_pairs_per_s": round(args.pairs / to, 2),
          "resident_forward_pairs_per_s": round(args.pairs / tf, 2), "max_rel_metric_diff": diff, "metrics": new}, out)


def validate_one(m, samples):
    """validate on this rank alone, the process group left aside."""
    from rnc import dist as rdist
    from rnc.harness import validate
    keep = rdist.world_rank
    rdist.world_rank = lambda: (1, 0)
    try:
        return validate(m, samples, iters=ITERS, batch_size=B)
    finally:
        rdist.world_rank = keep


if __name__ == "__main__":
    main()
