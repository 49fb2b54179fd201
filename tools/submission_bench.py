"""Submission throughput: the colour-coding kernel, the reference's host colour coding, and the Sintel and KITTI writers of
rnc.harness against a reference-style loop (one pair per forward, host colour coding, files written in line).

    python tools/submission_bench.py [--out DIR]

Prints one JSON line per measurement, each with the card name and power limit read in the same run:
  kernel          rnc.viz.flow_to_image at B = 8, 436x1024: CUDA events around each of 50 launches, median and range;
  host_viz        the reference's flow_to_image on one 436x1024 frame (oracle/_ref/core when built, else oracle/viz_oracle),
                  median of 5 host-clock runs;
  sintel          create_sintel_submission(batch_size=8, warm start) pairs/s with write_png off and on, against the B = 1
                  loop: six synthetic sequences of 8 to 14 frames at 436x1024 (rnc.synth.shift_sequence), 32 iterations;
  kitti           create_kitti_submission(batch_size=8) pairs/s over 40 pairs in 4 sizes near 375x1242, 24 iterations, write_png
                  on, against the B = 1 loop.
With --out, the lines are also appended to DIR/submission_bench.jsonl.  Files go to a temporary directory under DIR (under
the system's temporary directory without --out), removed afterwards.  Each writer pass is one host clock around the whole
call, which returns when every file is written; every shape is warmed up first.
"""
import argparse
import importlib.util
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-ncup_b200")]

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def host_flow_to_image():
    """The reference's flow_to_image when oracle/_ref/core is built, else the oracle's restatement."""
    path = os.path.join(ROOT, "oracle", "_ref", "core", "utils", "flow_viz.py")
    if os.path.exists(path):
        spec = importlib.util.spec_from_file_location("ref_flow_viz", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return "reference", mod.flow_to_image
    from oracle import viz_oracle
    return "oracle", viz_oracle.flow_to_image


def emit(line, out):
    print(json.dumps(line), flush=True)
    if out:
        with open(os.path.join(out, "submission_bench.jsonl"), "a") as f:
            f.write(json.dumps(line) + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("submission_bench needs a CUDA device")
    import cv2
    from rnc.harness import create_kitti_submission, create_sintel_submission
    from rnc.synth import build_model, frames, shift_sequence
    from rnc.viz import flow_to_image
    from utils import frame_utils
    from utils.utils import InputPadder, forward_interpolate

    if args.out:
        os.makedirs(args.out, exist_ok=True)
    cd = card()

    # kernel
    flows = torch.randn(8, 2, 436, 1024, device=DEV) * 8
    for _ in range(5):
        flow_to_image(flows)
    ms = []
    for _ in range(50):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        flow_to_image(flows)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    emit({"card": cd, "what": "kernel", "B": 8, "size": "436x1024", "ms_median": round(statistics.median(ms), 4),
          "ms_min": round(min(ms), 4), "ms_max": round(max(ms), 4)}, args.out)

    # host colour coding
    src, host_viz = host_flow_to_image()
    f = (np.random.default_rng(0).standard_normal((436, 1024, 2)) * 8).astype(np.float32)
    host_viz(f.copy())
    t = []
    for _ in range(5):
        x = f.copy()
        t0 = time.perf_counter()
        host_viz(x)
        t.append(time.perf_counter() - t0)
    host_ms = statistics.median(t) * 1e3
    emit({"card": cd, "what": "host_viz", "source": src, "size": "436x1024", "ms_median": round(host_ms, 2)}, args.out)

    tmp = tempfile.mkdtemp(dir=args.out or None)
    try:
        m = build_model("raft_nc_dbl").to(DEV)

        def clock(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        # Sintel
        lens = [8, 11, 14, 9, 12, 10]
        seqs = [("clean", f"s{s}", shift_sequence(n, 436, 1024, seed=s)) for s, n in enumerate(lens)]
        n_sintel = sum(n - 1 for n in lens)

        def sintel_loop(sq, out, iters=32):
            with torch.no_grad():
                for dstype, scene, fr in sq:
                    flow_prev = None
                    d = os.path.join(out, dstype, scene)
                    os.makedirs(d, exist_ok=True)
                    os.makedirs(os.path.join(out + "_png", dstype, scene), exist_ok=True)
                    for k in range(len(fr) - 1):
                        padder = InputPadder(fr[k].shape)
                        im1, im2 = padder.pad(fr[k][None].to(DEV), fr[k + 1][None].to(DEV))
                        flow_low, flow_pr = m(im1, im2, iters=iters, flow_init=flow_prev, test_mode=True)
                        flow = padder.unpad(flow_pr[0]).permute(1, 2, 0).cpu().numpy()
                        flow_prev = forward_interpolate(flow_low[0])[None]
                        cv2.imwrite(os.path.join(out + "_png", dstype, scene, "frame%04d.png" % (k + 1)), host_viz(flow))
                        frame_utils.writeFlow(os.path.join(d, "frame%04d.flo" % (k + 1)), flow)

        warm = [(d, s, fr[:3]) for d, s, fr in seqs]
        for png in (False, True):
            create_sintel_submission(m, warm, warm_start=True, output_path=os.path.join(tmp, "w"), write_png=png)
        sintel_loop(warm[:1], os.path.join(tmp, "wl"))
        res = {}
        for png in (False, True):
            res[png] = clock(lambda: create_sintel_submission(m, seqs, warm_start=True, output_path=os.path.join(tmp, "s"),
                                                              write_png=png))
        base = clock(lambda: sintel_loop(seqs, os.path.join(tmp, "l")))
        emit({"card": cd, "what": "sintel", "frames": "436x1024", "iters": 32, "warm_start": True, "pairs": n_sintel,
              "batch_size": 8, "pairs_per_s_png_off": round(n_sintel / res[False], 2),
              "pairs_per_s_png_on": round(n_sintel / res[True], 2),
              "b1_loop_host_viz_pairs_per_s": round(n_sintel / base, 2), "host_viz": src}, args.out)

        # KITTI
        sizes = [(375, 1242), (370, 1226), (376, 1241), (374, 1238)]
        pairs = []
        for k in range(40):
            h, w = sizes[k % 4]
            a, b = frames(1, h, w, seed=k)
            pairs.append((f"{k:06d}_10.png", a[0], b[0]))

        def kitti_loop(prs, out):
            os.makedirs(out, exist_ok=True)
            os.makedirs(out + "_png", exist_ok=True)
            with torch.no_grad():
                for fid, a, b in prs:
                    padder = InputPadder(a.shape, mode="kitti")
                    im1, im2 = padder.pad(a[None].to(DEV), b[None].to(DEV))
                    _, flow_pr = m(im1, im2, iters=24, test_mode=True)
                    flow = padder.unpad(flow_pr[0]).permute(1, 2, 0).cpu().numpy()
                    cv2.imwrite(os.path.join(out + "_png", fid + ".png"), host_viz(flow))
                    frame_utils.writeFlowKITTI(os.path.join(out, fid), flow)

        create_kitti_submission(m, pairs, output_path=os.path.join(tmp, "kw"), write_png=True)
        kitti_loop(pairs[:4], os.path.join(tmp, "klw"))
        kt = clock(lambda: create_kitti_submission(m, pairs, output_path=os.path.join(tmp, "k"), write_png=True))
        kb = clock(lambda: kitti_loop(pairs, os.path.join(tmp, "kl")))
        emit({"card": cd, "what": "kitti", "pairs": len(pairs), "sizes": [f"{h}x{w}" for h, w in sizes], "iters": 24,
              "batch_size": 8, "write_png": True, "pairs_per_s": round(len(pairs) / kt, 2),
              "b1_loop_host_viz_pairs_per_s": round(len(pairs) / kb, 2), "host_viz": src}, args.out)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
