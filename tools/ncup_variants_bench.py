"""Time NConvUNet configurations: the shipped one (fused rnc_ncup_fwd / NcupChainFn) against the per-level chain of
rnc/nconv_unet.py for `paper` (N = 3, double convolutions) and `wide` (m = 4, filters 3 / 5 / 3).

    python tools/ncup_variants_bench.py [--reps 20] [--steps 5]

Per configuration, one JSON line:
  upsampler_ms   NConvUpsampler.forward under no_grad at the bench shape (B = 8, 440x1024 images: x_lowres [8,2,110,256],
                 guidance [8,128,55,128]), one call, median over --reps
  frozen_step_ms train_step of raft_nc_dbl with --freeze_raft at cfg 5 (tools/finetune_bench.py: B = 2, 384x512, 12
                 iterations), median over --steps
  ref_upsampler_ms the reference's eager NConvUpsampler (oracle/_ref/core) on the same inputs, when oracle/_ref is present
Writes nothing but stdout.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-ncup_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

from finetune_bench import power_limit_w, timed  # noqa: E402

CONFIGS = {
    "shipped": {},
    "paper": dict(interp_net_channels_multiplier=2, interp_net_num_downsampling=3, interp_net_use_double_conv=True),
    "wide": dict(interp_net_channels_multiplier=4, interp_net_num_downsampling=2, interp_net_encoder_filter_sz=3,
                 interp_net_decoder_filter_sz=5, interp_net_out_filter_sz=3),
}


def model_args(name):
    from rnc.synth import ref_args
    a = ref_args()
    for k, v in CONFIGS[name].items():
        setattr(a, k, v)
    return a


def reference_upsampler(args, dev):
    """The original project's get_upsampler (oracle/_ref/core), seeded like the drop-in, or None when it is absent."""
    core = os.path.join(ROOT, "oracle", "_ref", "core")
    if not os.path.exists(os.path.join(core, "upsampler.py")):
        return None
    import importlib.util
    saved = {k: sys.modules.pop(k) for k in ("upsampler", "nconv_modules", "interp_weights_est") if k in sys.modules}
    sys.path.insert(0, core)
    try:
        spec = importlib.util.spec_from_file_location("ref_upsampler", os.path.join(core, "upsampler.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        torch.manual_seed(0)
        return mod.get_upsampler(2, 128, args).to(dev).eval()
    finally:
        sys.path.remove(core)
        for k in ("upsampler", "nconv_modules", "interp_weights_est"):
            sys.modules.pop(k, None)
        sys.modules.update(saved)


def median_ms(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    return statistics.median(timed(fn)[0] for _ in range(reps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ncup_variants_bench needs a GPU")
    import raft_nc_dbl
    from rnc.synth import frames
    from rnc.train import fetch_optimizer, train_step
    dev = torch.device("cuda:0")
    card, plim = torch.cuda.get_device_name(0), power_limit_w()
    g = torch.Generator().manual_seed(0)
    x4 = (torch.randn(8, 2, 110, 256, generator=g) * 4).to(dev)
    guid = torch.randn(8, 128, 55, 128, generator=g).to(dev)
    im1, im2 = (t.to(dev) for t in frames(2, 384, 512))
    gt = (torch.randn(2, 2, 384, 512, generator=g) * 5).to(dev)
    valid = torch.ones(2, 384, 512, device=dev)
    for name in CONFIGS:
        a = model_args(name)
        torch.manual_seed(1234)
        m = raft_nc_dbl.RAFT(a).to(dev).eval()
        with torch.no_grad():
            up_ms = median_ms(lambda: m.upsampler(x4, guid), args.reps, args.warmup)
        ref = reference_upsampler(a, dev)
        ref_ms = None
        if ref is not None:
            with torch.no_grad():
                ref_ms = median_ms(lambda: ref(x4, guid), args.reps, args.warmup)
        a.freeze_raft = True
        torch.manual_seed(1234)
        mf = raft_nc_dbl.RAFT(a).to(dev)
        mf.train()
        mf.freeze_bn()
        opt, sched = fetch_optimizer(mf, lr=1e-5, num_steps=args.steps + args.warmup + 1)

        def step():
            return train_step(mf, opt, sched, im1, im2, gt, valid, iters=12, return_metrics=False)

        step_ms = median_ms(step, args.steps, args.warmup)
        print(json.dumps({"config": name, "upsampler_ms": round(up_ms, 3), "frozen_step_ms": round(step_ms, 2),
                          "ref_upsampler_ms": None if ref_ms is None else round(ref_ms, 3), "gpu": card,
                          "power_limit_w": plim}), flush=True)
        del m, mf, ref, opt
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
