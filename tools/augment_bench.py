"""GPU augmentation cost: one batch of B = 6 things-shaped samples (540x960 -> 400x720, FlowAugmentor(-0.4, 0.8)).

    python tools/augment_bench.py [--reps 20]

Prints, with the card name and power limit: the host draws and packing, the packed host-to-device copy and the four
kernels, each timed with CUDA events (medians over --reps batches); and, when a copy of the original project is present under
oracle/_ref/core, the reference augmentor's CPU time per sample on this host (one thread, cv2.setNumThreads(1)).
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "raft-ncup_b200"))
from oracle.make_golden_aug import make_inputs   # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--B", type=int, default=6)
    a = ap.parse_args()
    from rnc import augment
    crop, H, W = [400, 720], 540, 960
    aug = augment.FlowAugmentor(crop, -0.4, 0.8, do_flip=True)
    samples = []
    for i in range(a.B):
        im1, im2, fl, _ = make_inputs(H, W, 1000 + i, False, False)
        samples.append((torch.from_numpy(im1).permute(2, 0, 1).float(), torch.from_numpy(im2).permute(2, 0, 1).float(),
                        torch.from_numpy(fl).permute(2, 0, 1).float(), None))
    dev = torch.device("cuda:0")
    np.random.seed(0)
    torch.manual_seed(0)
    for _ in range(3):
        aug.batch(samples, dev)
    torch.cuda.synchronize()
    host, copy, kern, total = [], [], [], []
    for _ in range(a.reps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        t0 = time.perf_counter()
        descs, buf = aug._pack(*aug._draw_batch(samples))
        t1 = time.perf_counter()
        ev[0].record()
        d = buf.to(dev, non_blocking=True)
        ev[1].record()
        aug._launch(descs, d)
        ev[2].record()
        torch.cuda.synchronize()
        total.append((time.perf_counter() - t0) * 1e3)
        host.append((t1 - t0) * 1e3)
        copy.append(ev[0].elapsed_time(ev[1]))
        kern.append(ev[1].elapsed_time(ev[2]))
    name, pl = card()
    mb = sum(s[0].numel() * 2 + s[2].numel() * 4 for s in samples) / 1e6
    med = statistics.median
    print(f"card: {name}, power limit {pl}")
    print(f"B = {a.B} things samples {H}x{W} -> {crop[0]}x{crop[1]}, packed upload {mb:.1f} MB, medians of {a.reps}:")
    print(f"  host draws + packing {med(host):.3f} ms")
    print(f"  host-to-device copy  {med(copy):.3f} ms")
    print(f"  kernels (4 + memset) {med(kern):.3f} ms")
    print(f"  batch() wall time    {med(total):.3f} ms (host draws, packing, copy, kernels, synchronised)")
    ref = os.path.join(ROOT, "oracle", "_ref", "core")
    if os.path.exists(os.path.join(ref, "utils", "augmentor.py")):
        try:
            import cv2
            sys.path.insert(0, ref)
            from utils.augmentor import FlowAugmentor as RefAug
            cv2.setNumThreads(1)
            torch.set_num_threads(1)
            r = RefAug(crop, -0.4, 0.8, do_flip=True)
            im1, im2, fl, _ = make_inputs(H, W, 1000, False, False)
            t0 = time.perf_counter()
            n = 10
            for _ in range(n):
                r(im1.copy(), im2.copy(), fl.copy())
            print(f"  reference augmentor on this host's CPU: {(time.perf_counter() - t0) / n * 1e3:.1f} ms / sample "
                  "(1 thread)")
        except ImportError as e:
            print(f"  reference augmentor: not run ({e})")
    else:
        print("  reference augmentor: oracle/_ref/core absent, not run")


if __name__ == "__main__":
    main()
