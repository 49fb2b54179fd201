"""Time weights-net (Simple) configurations of the NCUP upsampler: the shipped [64, 32] / [3, 3, 1] network against the
configurations of oracle/make_golden_wnet.py (dilated layers, a deeper net, 5x5 / 7x7 filters with a dilated 3x3 head, a
narrow net, a head-only net).

    python tools/wnet_variants_bench.py [--reps 20]

Per configuration, one JSON line: upsampler_ms, NConvUpsampler.forward under no_grad at the bench shape (B = 8, 440x1024
images: x_lowres [8,2,110,256], guidance [8,128,55,128]), one call, median and range over --reps; ref_upsampler_ms, the same
for the reference's eager upsampler (oracle/_ref/core) when present.  Writes nothing but stdout.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-ncup_b200"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

from finetune_bench import power_limit_w, timed  # noqa: E402
from ncup_variants_bench import reference_upsampler  # noqa: E402
from oracle.make_golden_wnet import CONFIGS  # noqa: E402


def model_args(name):
    from rnc.synth import ref_args
    if name == "shipped":
        return ref_args()
    num_ch, filter_sz, dilation, dataset = CONFIGS[name]
    a = ref_args(dataset)
    a.weights_est_net_num_ch, a.weights_est_net_filter_sz, a.weights_est_net_dilation = list(num_ch), list(filter_sz), list(dilation)
    return a


def times_ms(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    return [timed(fn)[0] for _ in range(reps)]


def summary(ts):
    return {"median": round(statistics.median(ts), 3), "min": round(min(ts), 3), "max": round(max(ts), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wnet_variants_bench needs a GPU")
    import raft_nc_dbl
    dev = torch.device("cuda:0")
    card, plim = torch.cuda.get_device_name(0), power_limit_w()
    g = torch.Generator().manual_seed(0)
    x4 = (torch.randn(8, 2, 110, 256, generator=g) * 4).to(dev)
    guid = torch.randn(8, 128, 55, 128, generator=g).to(dev)
    for name in ["shipped", *CONFIGS]:
        a = model_args(name)
        torch.manual_seed(1234)
        m = raft_nc_dbl.RAFT(a).to(dev).eval()
        with torch.no_grad():
            up = times_ms(lambda: m.upsampler(x4, guid), args.reps, args.warmup)
        ref = reference_upsampler(a, dev)
        ref_t = None
        if ref is not None:
            with torch.no_grad():
                ref_t = summary(times_ms(lambda: ref(x4, guid), args.reps, args.warmup))
        print(json.dumps({"config": name, "upsampler_ms": summary(up), "ref_upsampler_ms": ref_t, "gpu": card,
                          "power_limit_w": plim}), flush=True)
        del m, ref
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
