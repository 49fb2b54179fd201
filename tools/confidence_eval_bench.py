"""Cost of confidence evaluation: rnc_sparsification alone, and validate with and without confidence=True.

    python tools/confidence_eval_bench.py [--pairs N] [--rounds R]

Prints one JSON line, with the card name and power limit read in the same run:
  kernel     rnc.metrics.sparsification at B = 8, 436x1024 (Sintel), on the unpadded views of a padded batch with a valid
             mask: CUDA events around each of 50 launches after 5 warm-up launches; median, range, and pixels/s at the median;
  validate   pairs/s of validate(batch_size=8) on a seeded synthetic split of `pairs` Sintel-size pairs (rnc.synth.frames, a
             random ground truth, held as CPU tensors as a DataLoader delivers them), raft_nc_dbl, 32 iterations, without and
             with confidence=True.  The two run alternately `rounds` times after a warm-up of each; each pass is one host clock
             around the whole call, ended by a device synchronise.  The overhead is the median with-confidence time over the
             median without, in percent.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-ncup_b200")]

ITERS, B, H, W = 32, 8, 436, 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("confidence_eval_bench needs a CUDA device")
    from rnc.harness import validate
    from rnc.metrics import sparsification
    from rnc.synth import build_model, frames
    from utils.utils import InputPadder

    dev = torch.device("cuda", torch.cuda.current_device())
    out = {"card": card()}

    g = torch.Generator(device=dev).manual_seed(0)
    padder = InputPadder((3, H, W))
    flow = padder.unpad(torch.randn(B, 2, H + 4, W, device=dev, generator=g) * 6)
    score = padder.unpad(torch.rand(B, 2, H + 4, W, device=dev, generator=g))[:, 0]
    gt = torch.randn(B, 2, H, W, device=dev, generator=g) * 6
    valid = (torch.rand(B, H, W, device=dev, generator=g) > 0.1).float()
    for _ in range(5):
        sparsification(flow, gt, valid, score)
    ms = []
    for _ in range(50):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        sparsification(flow, gt, valid, score)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    med = statistics.median(ms)
    out["kernel"] = {"B": B, "size": f"{H}x{W}", "launches": 50, "ms_median": round(med, 4), "ms_min": round(min(ms), 4),
                     "ms_max": round(max(ms), 4), "pixels_per_s": round(B * H * W / (med * 1e-3))}
    del flow, score, gt, valid

    m = build_model("raft_nc_dbl").to(dev)
    im1, im2 = frames(args.pairs, H, W, seed=1)
    gcpu = torch.Generator().manual_seed(2)
    samples = [(im1[i], im2[i], torch.randn(2, H, W, generator=gcpu) * 4) for i in range(args.pairs)]
    del im1, im2
    validate(m, samples[:B], iters=ITERS, batch_size=B, device=dev)
    validate(m, samples[:B], iters=ITERS, batch_size=B, device=dev, confidence=True)
    t_off, t_on = [], []
    for _ in range(args.rounds):
        t, plain = clock(lambda: validate(m, samples, iters=ITERS, batch_size=B, device=dev))
        t_off.append(t)
        t, res = clock(lambda: validate(m, samples, iters=ITERS, batch_size=B, device=dev, confidence=True))
        t_on.append(t)
    off, on = statistics.median(t_off), statistics.median(t_on)
    out["validate"] = {"pairs": args.pairs, "size": f"{H}x{W}", "iters": ITERS, "batch_size": B, "rounds": args.rounds,
                       "pairs_per_s": [round(args.pairs / t, 2) for t in t_off],
                       "confidence_pairs_per_s": [round(args.pairs / t, 2) for t in t_on],
                       "overhead_percent": round(100 * (on - off) / off, 2),
                       "flow_metrics_equal": all(res[k] == plain[k] for k in plain), "ause": res["ause"]}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
