"""Step time and memory of unsupervised fine-tuning (rnc.train.unsupervised_step) beside supervised training (train_step).

    python tools/unsupervised_bench.py [--steps 5] [--warmup 2]

Model raft_nc_dbl, train mode, freeze_bn(); cfg 5 per GPU: B = 2, 384x512, 12 iterations; AdamW + OneCycle.
(a) steps, one variant after the other, on two models (one full, one built with freeze_raft):
  full_supervised / full_unsupervised      train_step / unsupervised_step through the full-training route
  frozen_supervised / frozen_unsupervised  the same on the frozen-trunk route (only the upsampler trains)
  unsupervised_step runs the bidirectional forward, so its forward and backward carry 2B = 4 rows.
(b) the loss terms alone, sum_i gamma^(11-i) (C_i + 2 Sm_i) over 12 predictions of 2B rows with one fixed mask, forward and
  backward: fused (census_loss, smoothness_loss on csrc/photometric.cu) against host (host_census_loss, host_smoothness_loss in
  fp32 torch on the same GPU), with the relative difference of the two losses.
Medians of CUDA events after warm-up; peak memory is torch.cuda.max_memory_allocated over each variant's timed calls, in MB.
Prints one JSON line with the device name and its power limit (read-only query).  Writes nothing to the tree."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-ncup_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def measure(fn, warmup, steps, dev):
    """(median ms, peak MB over the timed calls, last result)."""
    for _ in range(warmup):
        r = fn()
    torch.cuda.synchronize(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    times = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn()
        e1.record()
        torch.cuda.synchronize(dev)
        times.append(e0.elapsed_time(e1))
    return statistics.median(times), torch.cuda.max_memory_allocated(dev) / 2 ** 20, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--height", type=int, default=384)
    ap.add_argument("--width", type=int, default=512)
    ap.add_argument("--iters", type=int, default=12)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unsupervised_bench needs a GPU")
    from rnc.synth import build_model, frames, ref_args
    from rnc.train import fetch_optimizer, train_step, unsupervised_step
    from rnc.unsupervised import census_loss, host_census_loss, host_smoothness_loss, smoothness_loss

    dev = torch.device("cuda:0")
    B, H, W, n = args.batch, args.height, args.width, args.iters
    full = build_model("raft_nc_dbl").to(dev).train()
    import raft_nc_dbl
    torch.manual_seed(1234)
    a = ref_args("sintel")
    a.freeze_raft = True
    frozen = raft_nc_dbl.RAFT(a).to(dev)
    for m in (full, frozen):
        m.train()
        m.freeze_bn()
    im1, im2 = (t.to(dev) for t in frames(B, H, W, seed=31))
    g = torch.Generator().manual_seed(32)
    gt = (torch.randn(B, 2, H, W, generator=g) * 5).to(dev)
    valid = (torch.rand(B, H, W, generator=g) > 0.1).float().to(dev)
    res = {}
    for route, m in (("full", full), ("frozen", frozen)):
        opt, sched = fetch_optimizer(m, lr=1e-5, num_steps=100000)
        for kind, step in (("supervised", lambda: train_step(m, opt, sched, im1, im2, gt, valid, iters=n)),
                           ("unsupervised", lambda: unsupervised_step(m, opt, sched, im1, im2, iters=n))):
            ms, mb, (loss, _) = measure(step, args.warmup, args.steps, dev)
            res[f"{route}_{kind}_step_ms"] = round(ms, 2)
            res[f"{route}_{kind}_peak_mb"] = round(mb)
            res[f"{route}_{kind}_loss"] = float(loss)

    # (b) the loss terms alone over n predictions of 2B rows
    src, tgt = torch.cat([im1, im2]), torch.cat([im2, im1])
    preds = [(torch.randn(2 * B, 2, H, W, generator=g) * 3).to(dev).requires_grad_() for _ in range(n)]
    mask = (torch.rand(2 * B, H, W, generator=g) < 0.9).to(dev)

    def terms(census, smooth):
        def run():
            loss = 0.0
            for i, p in enumerate(preds):
                loss = loss + 0.85 ** (n - 1 - i) * (census(src, tgt, p, mask) + 2.0 * smooth(src, p))
            loss.backward()
            return loss.detach()
        return run

    del full, frozen, m, opt, sched
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated(dev) / 2 ** 20
    for kind, fn in (("fused", terms(census_loss, smoothness_loss)), ("host", terms(host_census_loss, host_smoothness_loss))):
        ms, mb, loss = measure(fn, args.warmup, args.steps, dev)
        res[f"loss_{kind}_ms"] = round(ms, 3)
        res[f"loss_{kind}_peak_mb"] = round(mb - base)
        res[f"loss_{kind}"] = float(loss)
        for p in preds:
            p.grad = None
    res["loss_rel_diff"] = abs(res["loss_fused"] - res["loss_host"]) / abs(res["loss_host"])
    print(json.dumps({"metric": "unsupervised_step_ms", "shape": [B, H, W], "iters": n, "steps": args.steps,
                      "warmup": args.warmup, **res, "device": torch.cuda.get_device_name(dev),
                      "power_limit_w": power_limit_w()}))


if __name__ == "__main__":
    main()
