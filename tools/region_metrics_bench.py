"""Cost of the per-region validation metrics: validate with and without regions=True, and the two kernels alone.

    python tools/region_metrics_bench.py [--model raft_nc_dbl] [--rounds R] [--images N]

Prints one JSON line, with the card name and power limit read in the same run:
  validate  N synthetic Sintel-style samples (436x1024, rnc.synth.frames, ground truth and an occluded disc per sample) in
            batches of B = 8, 32 iterations: after a warm-up of each, `rounds` rounds alternate regions=False and
            regions=True; each is one host clock around a validate call (which ends by reading its results to the host).
            Medians and every round are listed; the overhead is median(regions) / median(plain) - 1.
  kernels   rnc_boundary_dist2 and rnc_region_metrics (through rnc.metrics.boundary_dist2 and region_partials, Sintel-style)
            on B = 8 images of 436x1024: CUDA events around each of 50 launches after 5 warm-up launches; median and range.
            region_partials includes its own boundary_dist2, so kernels.regions_ms less kernels.dist2_ms is the metrics pass.
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def disc(h, w, cy, cx, r):
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    return (((yy - cy) ** 2 + (xx - cx) ** 2) < r * r).float()


def samples(n):
    from rnc.synth import frames
    im1, im2 = frames(n, H, W, seed=3)
    g = torch.Generator().manual_seed(4)
    out = []
    for i in range(n):
        gt = torch.randn(2, H, W, generator=g) * 8
        out.append((im1[i].cpu(), im2[i].cpu(), gt, None, {"occ": disc(H, W, H / 2, 150 + 60 * (i % 12), 60 + 5 * (i % 7))}))
    return out


def events(fn, n=50, warm=5):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return {"median_ms": round(statistics.median(ts), 4), "min_ms": round(min(ts), 4), "max_ms": round(max(ts), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="raft_nc_dbl", choices=["raft_nc_dbl", "raft"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("region_metrics_bench needs a CUDA device")
    from rnc.harness import validate
    from rnc.metrics import boundary_dist2, region_partials
    from rnc.synth import build_model

    dev = torch.device("cuda", torch.cuda.current_device())
    out = {"card": card(), "model": args.model, "B": B, "H": H, "W": W, "iters": ITERS, "images": args.images}
    model = build_model(args.model).to(dev)
    data = samples(args.images)
    plain_data = [s[:4] for s in data]

    def run(regions):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = validate(model, data if regions else plain_data, iters=ITERS, batch_size=B, regions=regions)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, res

    run(False)
    run(True)
    plain, reg = [], []
    for _ in range(args.rounds):
        plain.append(run(False)[0])
        t, res = run(True)
        reg.append(t)
    mp, mr = statistics.median(plain), statistics.median(reg)
    out["validate"] = {"plain_s": [round(t, 3) for t in plain], "regions_s": [round(t, 3) for t in reg],
                       "plain_median_s": round(mp, 3), "regions_median_s": round(mr, 3),
                       "overhead_pct": round(100 * (mr / mp - 1), 2), "pairs_per_s_plain": round(args.images / mp, 2),
                       "pairs_per_s_regions": round(args.images / mr, 2),
                       "epe_matched": res["epe_matched"], "epe_unmatched": res["epe_unmatched"]}

    g = torch.Generator(device=dev).manual_seed(5)
    gt = torch.randn(B, 2, H, W, device=dev, generator=g) * 8
    flow = gt + torch.randn(B, 2, H, W, device=dev, generator=g)
    occ = torch.stack([s[4]["occ"] for s in data[:B]]).to(dev)
    out["kernels"] = {"dist2_ms": events(lambda: boundary_dist2(occ)),
                      "regions_ms": events(lambda: region_partials(flow, gt, None, occ=occ))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
