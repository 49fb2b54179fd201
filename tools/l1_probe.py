"""Encoder layer-1 convolution (64 -> 64, 3x3, 16 images of 220x512) under developer variants: where does the time go?"""
import os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "raft-ncup_b200")):
    sys.path.insert(0, p)
from rnc import native
from rnc.engine_umma import UmmaEngine, SplitBuf, UmmaWeights
eng = UmmaEngine(); dev = "cuda:0"
N, H, W = int(os.environ.get("N", 16)), 220, 512
g = torch.Generator().manual_seed(0)
buf = SplitBuf(N * H * W, 64, dev); buf.hi.normal_(); buf.lo.normal_(0, 1e-3)
wt = UmmaWeights(torch.randn(64, 64, 3, 3, generator=g).to(dev) / 40, torch.zeros(64, device=dev), [64])
out32 = torch.empty(N * H * W, 64, device=dev)
outs = SplitBuf(N * H * W, 64, dev)
stats = torch.zeros(N * 64 * 2, dtype=torch.float64, device=dev)
E = native
variants = {
    "linear+stats f32": dict(epi=E.EPI_LINEAR, out_f32=out32.data_ptr(), ldo_f32=64, stats=stats.data_ptr()),
    "linear f32": dict(epi=E.EPI_LINEAR, out_f32=out32.data_ptr(), ldo_f32=64),
    "relu split": dict(epi=E.EPI_RELU, out_split=outs.ptrs(), ldo_split=64),
    "relu split, no halo": dict(epi=E.EPI_RELU, out_split=outs.ptrs(), ldo_split=64, flags=E.CONV_NO_HALO),
}
for name, kw in variants.items():
    epi = kw.pop("epi")
    def run():
        eng.uconv(N, H, W, buf.ptrs(), 64, 64, wt, epi, **kw)
    for _ in range(3):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        run()
    e1.record(); torch.cuda.synchronize()
    print(f"{name:32s} {e0.elapsed_time(e1) / 10 * 1e3:7.1f} us", flush=True)
