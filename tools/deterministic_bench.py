"""Cost of deterministic mode (torch.use_deterministic_algorithms(True)) on the training path.

    python tools/deterministic_bench.py [--reps 9] [--out DIR]

Times the cfg-5 step (B = 2, 384x512, 12 iterations, train_step with frozen BatchNorm) in the default and the deterministic
mode, alternating the two modes, on two models: raft_nc_dbl with a trainable trunk (full training through
raft_forward_train) and raft_nc_dbl built with --freeze_raft (the frozen-trunk route).  Each sample is the median of three
consecutive steps.  Then times the one operation whose kernel changes with the mode, the correlation-lookup backward, atomic
form against deterministic form, at cfg 5 and at the bench shape (B = 8, 440x1024).  Prints one JSON line with the card name
and power limit beside the numbers (medians over --reps samples with their range, milliseconds).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-ncup_b200")]

DEV = "cuda:0"
B, H, W, ITERS = 2, 384, 512, 12
OP_SHAPES = {"cfg5": (2, 384, 512), "bench": (8, 440, 1024)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn, n):
    """Median of n event-timed calls of fn (ms); one untimed call first."""
    fn()
    out = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def set_mode(det):
    torch.use_deterministic_algorithms(det, warn_only=False)


def step_models():
    import raft_nc_dbl
    from rnc.synth import build_model, ref_args
    full = build_model("raft_nc_dbl").to(DEV).train()
    full.freeze_bn()
    torch.manual_seed(1234)
    a = ref_args()
    a.freeze_raft = True
    frozen = raft_nc_dbl.RAFT(a).to(DEV).train()
    frozen.freeze_bn()
    return {"full": full, "frozen": frozen}


def bench_steps(reps):
    from rnc.synth import frames
    from rnc.train import fetch_optimizer, train_step
    im1, im2 = (t.to(DEV) for t in frames(B, H, W))
    g = torch.Generator().manual_seed(3)
    gt = (torch.randn(B, 2, H, W, generator=g) * 4).to(DEV)
    valid = torch.ones(B, H, W, device=DEV)
    res = {}
    for route, m in step_models().items():
        opt, sched = fetch_optimizer(m, lr=1e-6, num_steps=1000)

        def step():
            train_step(m, opt, sched, im1, im2, gt, valid, iters=ITERS, return_metrics=False)
        times = {False: [], True: []}
        for det in (False, True):                               # warm both modes
            set_mode(det)
            step()
        for _ in range(reps):
            for det in (False, True):
                set_mode(det)
                times[det].append(timed(step, 3))
        set_mode(False)
        res[route] = {"default_ms": statistics.median(times[False]), "deterministic_ms": statistics.median(times[True]),
                      "default_range": [min(times[False]), max(times[False])],
                      "deterministic_range": [min(times[True]), max(times[True])]}
    return res


def bench_ops(reps, B, H, W):
    from rnc.native import rnc
    res = {}
    H8, W8 = H // 8, W // 8
    f1 = torch.randn(B, H8, W8, 256, device=DEV)
    pyr = torch.randn(rnc.pyramid_offset(B, 256, H8, W8, 4), device=DEV)
    ys, xs = torch.meshgrid(torch.arange(H8, device=DEV), torch.arange(W8, device=DEV), indexing="ij")
    coords = (torch.stack([xs, ys]).float()[None] + 4 * torch.randn(B, 2, H8, W8, device=DEV)).contiguous()
    g_out = torch.randn(B, H8, W8, 324, device=DEV)
    g1, g2 = torch.empty_like(f1), torch.empty_like(pyr)
    ws = torch.empty(rnc.corr_lookup_bwd_workspace_bytes(B, H8, W8, 4) // 4 + 4, device=DEV)
    args = (f1, pyr, coords, g_out, 324, B, 256, H8, W8, 4, 4, g1, g2)

    def atomic():
        g2.zero_()
        rnc.corr_lookup_bwd(*args)

    def det():
        rnc.corr_lookup_bwd_det(*args, ws, ws.numel() * 4)
    res["lookup_bwd"] = alternate(atomic, det, reps)
    return res


def alternate(a, b, reps, inner=20):
    ta, tb = [], []
    for _ in range(reps):
        ta.append(timed(lambda: [a() for _ in range(inner)], 1) / inner)
        tb.append(timed(lambda: [b() for _ in range(inner)], 1) / inner)
    return {"atomic_ms": statistics.median(ta), "deterministic_ms": statistics.median(tb),
            "atomic_range": [min(ta), max(ta)], "deterministic_range": [min(tb), max(tb)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/deterministic_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("deterministic_bench.py measures on a GPU; none is visible")
    torch.backends.cudnn.benchmark = False
    ops = {tag: bench_ops(args.reps, *shape) for tag, shape in OP_SHAPES.items()}
    line = {"card": card(), "shape": [B, H, W], "iters": ITERS, "ops": ops, "steps": bench_steps(args.reps)}
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "deterministic_bench.json"), "w") as f:
            f.write(json.dumps(line, indent=1))


if __name__ == "__main__":
    main()
