"""Video object segmentation cost: the propagation step and the J and F counts alone, and propagate_masks end to end against
the bidirectional flow pass it runs on.

    python tools/segmentation_bench.py [--rounds 3] [--model raft_nc_dbl] [--out DIR]

(a) rnc_propagate_labels for V = 8 videos at 480x854, one step on smooth random fractional flows, 5% random masks and blocky
    labels: CUDA events around 20 launches after a warm-up, the median of --rounds; also the bytes per pixel the step reads
    and writes by its algorithm (flow, mask, labels, the int map of the column and row passes).
(b) rnc_segmentation_counts for one 70-frame, 3-object 480x854 video (the 68 scored frames of a DAVIS-length video), the same
    way.
(c) rnc.harness.propagate_masks on eight synthetic 480x854 videos of 50 frames (rnc.synth.shift_sequence, frames resident on
    the GPU), 32 iterations, batch_size 8, against run_sequences_bidirectional alone on the same videos, alternating within
    one process: a host clock around each whole pass that ends in a device synchronise.  The difference is the propagation's
    cost; the scoring's is (b) per video.
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
H, W, T, ITERS, VIDEOS = 480, 854, 50, 32, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def events_ms(fn, rounds, calls=20):
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


def blocky(n, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    low = torch.randint(0, K + 1, (n, 1, H // 24, W // 24), generator=g, device=DEV).float()
    return F.interpolate(low, size=(H, W), mode="nearest")[:, 0].to(torch.uint8)


@torch.no_grad()                    # the flow passes are inference only
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--model", default="raft_nc_dbl", choices=["raft_nc_dbl", "raft"])
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/segmentation_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("segmentation_bench needs a CUDA device")
    from rnc import native
    from rnc.harness import propagate_masks, run_sequences_bidirectional
    from rnc.segment import segmentation_counts
    from rnc.synth import build_model, shift_sequence

    line = {"card": card(), "frames": f"{H}x{W}"}
    g = torch.Generator(device=DEV).manual_seed(1)
    low = torch.randn(VIDEOS, 2, H // 16, W // 16, generator=g, device=DEV) * 6
    flow = F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False)
    occ = (torch.rand(VIDEOS, H, W, generator=g, device=DEV) < 0.05).to(torch.uint8)
    lab = blocky(VIDEOS, 20, 2)
    out = torch.empty_like(lab)
    ws = torch.empty(native.rnc.propagate_labels_workspace_bytes(VIDEOS, H, W), dtype=torch.uint8, device=DEV)

    def step():
        native.rnc.propagate_labels(lab, *lab.stride(), flow, *flow.stride(), occ, *occ.stride(), VIDEOS, H, W, out,
                                    *out.stride(), ws, ws.numel())
    med, all_ = events_ms(step, args.rounds)
    unmatched = float((out == 255).float().mean())          # 0 after the fill; kept as a check that it ran
    # vote: flow 8 + mask 1 + 4 label taps + write 1; column pass: read 1, write 4, re-read 4 (and rewrite a part);
    # row pass: read 4, gather 1 and write 1 per unmatched pixel
    bytes_pp = 8 + 1 + 4 + 1 + 1 + 4 + 4 + 4 + 2
    line.update({"propagate_V": VIDEOS, "propagate_step_ms": round(med, 4), "propagate_step_ms_rounds": [round(v, 4) for v in all_],
                 "propagate_bytes_per_pixel_model": bytes_pp,
                 "propagate_GBps_model": round(bytes_pp * VIDEOS * H * W / (med * 1e-3) / 1e9, 1),
                 "unmatched_left": unmatched})
    del flow, occ, lab, out, ws

    N, K = 68, 3
    gt = blocky(N, K, 3)
    pred = torch.roll(gt, shifts=(2, -3), dims=(1, 2)).contiguous()
    counts = torch.empty(N, K, native.SEGMENT_COUNTS, dtype=torch.int64, device=DEV)
    cws = torch.empty(native.rnc.segmentation_counts_workspace_bytes(N, K, H, W), dtype=torch.uint8, device=DEV)

    def score():
        native.rnc.segmentation_counts(pred, *pred.stride(), gt, *gt.stride(), N, K, H, W, counts, cws, cws.numel())
    med, all_ = events_ms(score, args.rounds, calls=5)
    assert torch.equal(counts, segmentation_counts(pred, gt, K))
    line.update({"counts_frames": N, "counts_objects": K, "segmentation_counts_ms": round(med, 3),
                 "segmentation_counts_ms_rounds": [round(v, 3) for v in all_],
                 "segmentation_counts_workspace_gb": round(cws.numel() / 1e9, 2)})
    del gt, pred, counts, cws
    torch.cuda.empty_cache()

    seqs = [[f.to(DEV) for f in shift_sequence(T, H, W, seed=s)] for s in range(VIDEOS)]
    firsts = [blocky(1, 3, 10 + s)[0] for s in range(VIDEOS)]
    m = build_model(args.model).to(DEV)

    def flows_only(sq):
        for _ in run_sequences_bidirectional(m, sq, ITERS, batch_size=VIDEOS, device=DEV):
            pass

    short = [seq[:3] for seq in seqs]
    flows_only(short)
    propagate_masks(m, short, firsts, ITERS, batch_size=VIDEOS, device=DEV)
    torch.cuda.synchronize()

    def clock(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    t_flow, t_prop = [], []
    for _ in range(args.rounds):
        t_flow.append(clock(lambda: flows_only(seqs))[0])
        t, res = clock(lambda: propagate_masks(m, seqs, firsts, ITERS, batch_size=VIDEOS, device=DEV))
        t_prop.append(t)
        del res
    mf, mp = statistics.median(t_flow), statistics.median(t_prop)
    scoring = VIDEOS * line["segmentation_counts_ms"] * 1e-3 * (T - 2) / N
    line.update({
        "model": args.model, "iters": ITERS, "videos": VIDEOS, "T": T, "pairs": VIDEOS * (T - 1), "rounds": args.rounds,
        "run_sequences_bidirectional_s": [round(v, 3) for v in t_flow],
        "propagate_masks_s": [round(v, 3) for v in t_prop],
        "propagation_s": round(mp - mf, 3),
        "scoring_s_from_counts_kernel": round(scoring, 4),
        "propagation_and_scoring_share_of_flow_pass": round((mp - mf + scoring) / mf, 4),
        "peak_memory_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2),
    })
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "segmentation_bench.json"), "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
