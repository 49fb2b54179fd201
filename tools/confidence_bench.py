"""Cost of returning the NCUP output confidence.

    python tools/confidence_bench.py [--reps 200] [--steps 10] [--warmup 3]

  kernel   rnc_ncup_fwd with conf_out NULL against non-NULL at the benchmark shape (B = 8, H4 x W4 = 110 x 256: 440x1024 outputs),
           alternating call by call, CUDA events around each call; the confidence adds one division and one 4-byte store per
           output pixel.
  frozen   a cfg-5 frozen-trunk fine-tuning step (raft_nc_dbl with freeze_raft, train mode, freeze_bn(); B = 2, 384x512,
           12 iterations; forward, sequence_loss, backward, AdamW step) without and with return_confidence, alternating step
           by step; with the confidence the step adds sum(0.01 * conf) per prediction to the loss, so its backward runs the
           confidence adjoint (NcupChainFn with want_conf / rnc_ncup_bwd given g_conf_out).
Medians after warm-up.  Prints one JSON line with the device name and its power limit (read-only query).  Writes nothing to
the tree."""
import argparse
import ctypes
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
import torch.nn.functional as F  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def kernel_bench(reps, warmup):
    from rnc.native import rnc
    B, H4, W4 = 8, 110, 256
    g = torch.Generator().manual_seed(3)
    dev = torch.device("cuda:0")
    x = (5 * torch.randn(B, 2, H4, W4, generator=g)).to(dev)
    c = torch.rand(B, 2, H4, W4, generator=g).to(dev)
    w = torch.cat([F.softplus(0.3 * torch.randn(n, generator=g), beta=10) for n in (50, 100, 72, 2)])
    hw = (ctypes.c_float * 224)(*w.tolist())
    out, out2, conf = (torch.empty(B, 2, 4 * H4, 4 * W4, device=dev) for _ in range(3))
    plain = lambda: rnc.ncup_fwd(x, c, hw, B, H4, W4, 8.0, out, None)          # noqa: E731
    with_conf = lambda: rnc.ncup_fwd(x, c, hw, B, H4, W4, 8.0, out2, conf)     # noqa: E731
    t = {"plain": [], "conf": []}
    for i in range(warmup + reps):
        a, b = timed(plain), timed(with_conf)
        if i >= warmup:
            t["plain"].append(a)
            t["conf"].append(b)
    assert torch.equal(out, out2)
    return {k: statistics.median(v) for k, v in t.items()}


def frozen_bench(steps, warmup, B=2, H=384, W=512, iters=12):
    from rnc.synth import build_model, frames, ref_args
    from rnc.train import fetch_optimizer, sequence_loss
    dev = torch.device("cuda:0")
    build_model("raft_nc_dbl")
    import raft_nc_dbl
    torch.manual_seed(1234)
    a = ref_args("sintel")
    a.freeze_raft = True
    m = raft_nc_dbl.RAFT(a).to(dev).train()
    m.freeze_bn()
    opt, _ = fetch_optimizer(m, lr=1e-6, num_steps=10 ** 6)
    im1, im2 = (t.to(dev) for t in frames(B, H, W, seed=9))
    g = torch.Generator().manual_seed(10)
    gt = (5 * torch.randn(B, 2, H, W, generator=g)).to(dev)
    valid = torch.ones(B, H, W, device=dev)

    def step(conf):
        opt.zero_grad(set_to_none=True)
        if conf:
            preds, confs = m(im1, im2, iters=iters, return_confidence=True)
            loss = sequence_loss(preds, gt, valid, gamma=0.85)[0] + sum(0.01 * c.sum() for c in confs)
        else:
            loss = sequence_loss(m(im1, im2, iters=iters), gt, valid, gamma=0.85)[0]
        loss.backward()
        opt.step()

    t = {"plain": [], "conf": []}
    for i in range(warmup + steps):
        a_ms, b_ms = timed(lambda: step(False)), timed(lambda: step(True))
        if i >= warmup:
            t["plain"].append(a_ms)
            t["conf"].append(b_ms)
    return {k: statistics.median(v) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("confidence_bench needs a GPU")
    k = kernel_bench(args.reps, max(args.warmup, 10))
    f = frozen_bench(args.steps, args.warmup)
    res = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
           "ncup_fwd_ms": round(k["plain"], 4), "ncup_fwd_conf_ms": round(k["conf"], 4),
           "kernel_overhead_pct": round(100 * (k["conf"] / k["plain"] - 1), 2),
           "frozen_step_ms": round(f["plain"], 2), "frozen_step_conf_ms": round(f["conf"], 2),
           "frozen_overhead_pct": round(100 * (f["conf"] / f["plain"] - 1), 2)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
