"""Cost of bidirectional inference: bidirectional_flow against two graph-replayed forwards, and rnc_fb_consistency alone.

    python tools/bidirectional_bench.py [--model raft_nc_dbl] [--rounds R] [--reps N]

Prints one JSON line, with the card name and power limit read in the same run:
  pairs/s    B = 8 pairs of 440x1024 frames (rnc.synth.frames, on the device), 32 iterations, flows in both directions:
             (a) model(im1, im2) then model(im2, im1), each replayed from its CUDA graph; (b) rnc.harness.bidirectional_flow
             (one encoder pass, the loop at 2B slots replayed from its graph, then the consistency check on the unpadded
             flows).  After a warm-up of each, `rounds` rounds alternate (a) and (b); each is one host clock around `reps`
             calls, ended by a device synchronise.  Medians and every round are listed; the gain is median (b) over median (a).
  kernel     rnc.metrics.fb_consistency on B = 8 pairs at 436x1024 (Sintel): CUDA events around each of 50 launches after
             5 warm-up launches; median and range, and the bytes a launch must move (two flows read once, the sampled taps
             mostly from cache; occ and err written) over the median.
  equal      the largest EPE between (a) and (b), in each direction.
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

ITERS, B, H, W = 32, 8, 440, 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def clock(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="raft_nc_dbl", choices=["raft_nc_dbl", "raft"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bidirectional_bench needs a CUDA device")
    from rnc.harness import bidirectional_flow
    from rnc.metrics import fb_consistency
    from rnc.synth import build_model, frames

    dev = torch.device("cuda", torch.cuda.current_device())
    out = {"card": card(), "model": args.model, "B": B, "H": H, "W": W, "iters": ITERS}
    m = build_model(args.model).to(dev).eval()
    im1, im2 = (t.to(dev) for t in frames(B, H, W, seed=3))

    def two():
        a = m(im1, im2, iters=ITERS, test_mode=True)
        b = m(im2, im1, iters=ITERS, test_mode=True)
        return a[1], b[1]

    def bidi():
        r = bidirectional_flow(m, im1, im2, iters=ITERS)
        return r["flow_up"], r["flow_up_bw"]

    with torch.no_grad():
        for _ in range(3):                       # eager, capture, replay
            fa, fb = two()
            ga, gb = bidi()
        out["equal_epe"] = [(x - y).pow(2).sum(1).sqrt().max().item() for x, y in ((fa, ga), (fb, gb))]
        ta, tb = [], []
        for _ in range(args.rounds):
            ta.append(B * args.reps / clock(two, args.reps)[0])
            tb.append(B * args.reps / clock(bidi, args.reps)[0])
    out["two_forwards_pairs_s"] = {"median": statistics.median(ta), "rounds": ta}
    out["bidirectional_pairs_s"] = {"median": statistics.median(tb), "rounds": tb}
    out["gain"] = statistics.median(tb) / statistics.median(ta)

    g = torch.Generator(device=dev).manual_seed(0)
    kh = 436
    f = torch.randn(B, 2, kh, W, device=dev, generator=g) * 8
    b = -f + torch.randn(B, 2, kh, W, device=dev, generator=g)
    for _ in range(5):
        fb_consistency(f, b)
    times = []
    for _ in range(50):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fb_consistency(f, b)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    med = statistics.median(times)
    nbytes = 2 * (2 * B * kh * W * 4) + 2 * B * kh * W * (1 + 4)
    out["kernel_ms"] = {"median": med, "min": min(times), "max": max(times), "GB_s": nbytes / med / 1e6}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
