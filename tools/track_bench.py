"""Point tracking cost: the chaining kernel alone on dense queries, and track_points end to end split into flow inference and
chaining.

    python tools/track_bench.py [--rounds 3] [--model raft_nc_dbl] [--out DIR]

(a) rnc_track on dense queries, every pixel of frame 0 of one 436x1024 video with T = 50 frames, on smooth random flows and
    5% random masks: CUDA events around 10 launches after a warm-up, the median of --rounds; then the same around
    rnc.track.track, which adds the queries' check and the host's wait for its flags.  Also for eight such videos stacked, as
    track_points calls it.
(b) rnc.harness.track_points on eight synthetic 436x1024 videos of 50 frames (rnc.synth.shift_sequence, frames resident on the
    GPU), 32 iterations, batch_size 8, dense queries on frame 0 of each, against run_sequences_bidirectional alone on the same
    videos, alternating within one process: a host clock around each whole pass that ends in a device synchronise.  The
    difference is the chaining's cost (stacking the pair results, the queries' host check and the launch).
Prints one JSON line with the card name and power limit beside the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-ncup_b200")]

DEV = "cuda:0"
H, W, T, ITERS, VIDEOS = 436, 1024, 50, 32, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def events_ms(fn, rounds, calls=10):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(calls):
            fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / calls)
    return statistics.median(out), out


def random_inputs(V):
    g = torch.Generator(device=DEV).manual_seed(1)
    low = torch.randn(2 * V * (T - 1), 2, H // 16, W // 16, generator=g, device=DEV) * 6
    flows = F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False).view(2, V, T - 1, 2, H, W)
    occ = (torch.rand(2, V, T - 1, H, W, generator=g, device=DEV) < 0.05).to(torch.uint8)
    return flows[0], flows[1], occ[0], occ[1]


@torch.no_grad()                    # the flow passes are inference only
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--model", default="raft_nc_dbl", choices=["raft_nc_dbl", "raft"])
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/track_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("track_bench needs a CUDA device")
    from rnc import native
    from rnc.harness import run_sequences_bidirectional, track_points
    from rnc.synth import build_model, shift_sequence
    from rnc.track import grid_queries, track

    q = grid_queries(H, W, 0).to(DEV)
    line = {"card": card(), "frames": f"{H}x{W}", "T": T, "points_per_video": q.shape[0]}
    for V in (1, VIDEOS):
        fw, bw, o, ob = inputs = random_inputs(V)
        qv = q.expand(V, -1, -1).contiguous()
        tracks, vis = track(*inputs, qv)

        def kernel():                   # rnc_track alone, without track()'s query check on the device and its flag read
            native.rnc.track(fw, *fw.stride(), bw, *bw.stride(), o, *o.stride(), ob, *ob.stride(), qv, V, qv.shape[1], T, H,
                             W, tracks, vis)
        for name, fn in (("kernel", kernel), ("call", lambda: track(*inputs, qv))):
            med, all_ = events_ms(fn, args.rounds)
            line[f"track_{name}_V{V}_ms"] = round(med, 3)
            line[f"track_{name}_V{V}_ms_rounds"] = [round(v, 3) for v in all_]
        del inputs, fw, bw, o, ob, tracks, vis
        torch.cuda.empty_cache()

    seqs = [[f.to(DEV) for f in shift_sequence(T, H, W, seed=s)] for s in range(VIDEOS)]
    qs = [q] * VIDEOS
    m = build_model(args.model).to(DEV)

    def flows_only(sq):
        for _ in run_sequences_bidirectional(m, sq, ITERS, batch_size=VIDEOS, device=DEV):
            pass

    short = [seq[:3] for seq in seqs]
    flows_only(short)
    track_points(m, short, qs, ITERS, batch_size=VIDEOS, device=DEV)
    torch.cuda.synchronize()

    def clock(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    t_flow, t_track = [], []
    for _ in range(args.rounds):
        t_flow.append(clock(lambda: flows_only(seqs))[0])
        t, res = clock(lambda: track_points(m, seqs, qs, ITERS, batch_size=VIDEOS, device=DEV))
        t_track.append(t)
        visible = sum(int(v.sum()) for _, v in res)
        del res
        torch.cuda.empty_cache()
    mf, mt = statistics.median(t_flow), statistics.median(t_track)
    line.update({
        "model": args.model, "iters": ITERS, "videos": VIDEOS, "pairs": VIDEOS * (T - 1), "rounds": args.rounds,
        "run_sequences_bidirectional_s": [round(v, 3) for v in t_flow],
        "track_points_s": [round(v, 3) for v in t_track],
        "chaining_s": round(mt - mf, 3),
        "chaining_share_of_track_points": round((mt - mf) / mt, 4),
        "visible_point_frames": visible,
        "peak_memory_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2),
    })
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "track_bench.json"), "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
