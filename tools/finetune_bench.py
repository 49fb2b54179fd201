"""Step time of fine-tuning the NCUP upsampler on a frozen RAFT trunk (the reference's --freeze_raft, train.py:295).

    python tools/finetune_bench.py [--steps 10] [--warmup 3]

Model raft_nc_dbl built with freeze_raft, train mode, freeze_bn(); cfg 5 per GPU: B = 2, 384x512, 12 iterations; each step is
rnc.train.train_step (AdamW + OneCycle).  In one process, alternating step by step on the same model and optimiser:
  frozen   the model's own forward, which routes a frozen trunk to the inference engine (rnc.model.frozen_trunk)
  exact    rnc.train.raft_forward_train, the full-training path (exact CUDA-core kernels for the trunk too)
plus the NCUP chain alone (zero-stuffing + the four normalized convolutions, forward + backward) on the same inputs:
  fused    NcupChainFn (rnc_ncup_train_fwd / rnc_ncup_bwd)
  layers   the per-layer NConv2dFn chain of ncup_upsampler_train
CUDA events after warm-up, medians.  Prints one JSON line with the device name and its power limit (read-only query).
Writes nothing to the tree."""
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


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), r


class _ExactPath:
    """The model seen through raft_forward_train (what a frozen-trunk model ran before it had its own route)."""

    def __init__(self, model):
        self.model = model

    def __call__(self, image1, image2, iters=12):
        from rnc.train import raft_forward_train
        with torch.cuda.device(image1.device):
            return raft_forward_train(self.model, image1, image2, iters)

    def parameters(self):
        return self.model.parameters()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--height", type=int, default=384)
    ap.add_argument("--width", type=int, default=512)
    ap.add_argument("--iters", type=int, default=12)
    args = ap.parse_args()
    from rnc.model import frozen_trunk
    from rnc.synth import build_model, frames, ref_args
    from rnc.train import fetch_optimizer, ncup_chain_autograd, nconv_unet_train, train_step, zero_stuff

    dev = torch.device("cuda:0")
    B, H, W = args.batch, args.height, args.width
    build_model("raft_nc_dbl")
    import raft_nc_dbl
    torch.manual_seed(1234)
    a = ref_args("sintel")
    a.freeze_raft = True
    model = raft_nc_dbl.RAFT(a).to(dev).train()
    model.freeze_bn()
    im1, im2 = (t.to(dev) for t in frames(B, H, W, seed=31))
    g = torch.Generator().manual_seed(32)
    gt = (torch.randn(B, 2, H, W, generator=g) * 5).to(dev)
    valid = (torch.rand(B, H, W, generator=g) > 0.1).float().to(dev)
    assert frozen_trunk(model, im1, im2)
    opt, sched = fetch_optimizer(model, lr=1e-5, num_steps=100000)
    paths = {"frozen": model, "exact": _ExactPath(model)}
    ms = {k: [] for k in paths}
    loss = {}
    for i in range(args.warmup + args.steps):
        order = ("frozen", "exact") if i % 2 == 0 else ("exact", "frozen")
        for k in order:
            t, (l, _) = timed(lambda: train_step(paths[k], opt, sched, im1, im2, gt, valid, iters=args.iters, return_metrics=False))
            loss[k] = float(l)
            if i >= args.warmup:
                ms[k].append(t)

    # the NCUP chain alone, forward + backward, on one iteration's inputs at 1/4 resolution
    net = model.upsampler.interpolation_net
    H4, W4 = H // 4, W // 4
    x4 = (5 * torch.randn(B, 2, H4, W4, generator=g)).to(dev)
    conf = torch.rand(B, 2, H4, W4, generator=g).to(dev)
    gout = torch.randn(B, 2, H, W, generator=g).to(dev)

    def fused():
        x, c = x4.clone().requires_grad_(True), conf.clone().requires_grad_(True)
        ncup_chain_autograd(net, x, c, 8.0).backward(gout)

    def layers():
        x, c = x4.clone().requires_grad_(True), conf.clone().requires_grad_(True)
        xh, ch = zero_stuff(x), zero_stuff(c)
        b, C, oh, ow = xh.shape
        y, _ = nconv_unet_train(net, xh.view(b * C, 1, oh, ow), ch.view(b * C, 1, oh, ow))
        (8.0 * y.view(b, C, oh, ow)).backward(gout)

    chain = {"fused": [], "layers": []}
    for i in range(args.warmup + args.steps):
        for k, fn in (("fused", fused), ("layers", layers)):
            t, _ = timed(fn)
            if i >= args.warmup:
                chain[k].append(t)
    med = {k: statistics.median(v) for k, v in ms.items()}
    cmed = {k: statistics.median(v) for k, v in chain.items()}
    print(json.dumps({
        "metric": "finetune_step_ms", "shape": [B, H, W], "iters": args.iters, "steps": args.steps, "warmup": args.warmup,
        "frozen_step_ms": round(med["frozen"], 2), "exact_step_ms": round(med["exact"], 2),
        "speedup": round(med["exact"] / med["frozen"], 2),
        "chain_fused_ms": round(cmed["fused"], 3), "chain_per_layer_ms": round(cmed["layers"], 3),
        "loss_frozen": loss["frozen"], "loss_exact": loss["exact"],
        "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w()}))


if __name__ == "__main__":
    main()
