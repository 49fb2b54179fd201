"""Diagnostic: where do a B=8 forward and eight B=1 forwards diverge?  EPE(B=8 vs B=1) per engine mode and iteration count."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-ncup_b200")]
from rnc.synth import build_model, frames  # noqa: E402
from utils.utils import InputPadder  # noqa: E402


def epe(a, b):
    return (a - b).pow(2).sum(1).sqrt().mean().item()


im1, im2 = frames(8, 436, 1024)
p1, p2 = InputPadder(im1.shape, "sintel").pad(im1, im2)
p1, p2 = p1.cuda(), p2.cuda()
for env in ({}, {"RNC_LOOKUP": "ffma"}, {"RNC_ENCODER": "cudnn"}, {"RNC_CONV": "ffma"}):
    for k in ("RNC_LOOKUP", "RNC_CONV", "RNC_ENCODER"):
        os.environ.pop(k, None)
    os.environ.update(env)
    m = build_model("raft_nc_dbl").cuda()
    for iters in (1, 4, 32):
        with torch.no_grad():
            lo8, up8 = m(p1, p2, iters=iters, test_mode=True)
            es, el = [], []
            for i in range(8):
                lo1, up1 = m(p1[i:i + 1], p2[i:i + 1], iters=iters, test_mode=True)
                es.append(epe(up8[i:i + 1], up1))
                el.append(epe(lo8[i:i + 1], lo1))
        print(env, f"iters {iters}: flow_up EPE per pair", " ".join(f"{e:.1e}" for e in es), "| flow_low max", f"{max(el):.1e}", flush=True)
