"""Video inpainting cost, stage by stage, at the DAVIS frame size: the flow pass, flow completion, the consistency check,
temporal propagation, the spatial fill and the metrics.

    python tools/inpainting_bench.py [--rounds 1] [--sweeps 512] [--model raft_nc_dbl] [--out DIR]

Eight synthetic 480x854 videos of 50 frames (rnc.synth.shift_sequence, frames resident on the GPU), each with a 96x128 hole
that moves 3 px right and 1 px down a frame against content that moves (4, 3) px a frame (3% of each frame), run as
rnc.harness.inpaint_videos runs them: run_sequences_bidirectional (32 iterations, batch_size 8) on the frames with the holes
set to 0, each pair's flows copied into stacked tensors, then rnc.inpaint's steps on the stacks, then PSNR
(interpolation_error) and SSIM of every frame.  CUDA events around each stage after a warm-up on 3-frame videos; the median
over --rounds.  Prints one JSON line with the card name and power limit beside the times.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-ncup_b200")]

DEV = "cuda:0"
H, W, T, ITERS, VIDEOS = 480, 854, 50, 32, 8
STAGES = ("flow_pass", "flow_completion", "consistency", "propagation", "spatial_fill", "metrics")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def hole_masks(n):
    m = torch.zeros(n, H, W, dtype=torch.uint8, device=DEV)
    for t in range(n):
        m[t, 100 + t:196 + t, 200 + 3 * t:328 + 3 * t] = 1
    return m


@torch.no_grad()                    # the flow pass is inference only
def run(m, seqs, masks, sweeps):
    """One inpainting of the videos, stage by stage; returns the stage times in ms and (frames, source, psnr, ssim)."""
    from rnc.harness import run_sequences_bidirectional
    from rnc.inpaint import SOURCE_SPATIAL, harmonic_fill, inpaint_propagate, psnr, ssim
    from rnc.interp import interpolation_error
    from rnc.metrics import fb_consistency
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(STAGES) + 1)]
    V, n = len(seqs), len(seqs[0])
    seen = [[torch.where(h != 0, 0.0, f) for f, h in zip(seq, mk)] for seq, mk in zip(seqs, masks)]
    frames = torch.stack([torch.stack(seq) for seq in seqs])
    hole = torch.stack([torch.stack(mk) for mk in masks])
    torch.cuda.synchronize()
    ev[0].record()
    flows = [torch.zeros(V, n - 1, 2, H, W, device=DEV) for _ in range(2)]
    for s, k, r in run_sequences_bidirectional(m, seen, ITERS, batch_size=VIDEOS, device=DEV):
        flows[0][s, k].copy_(r["flow_up"])
        flows[1][s, k].copy_(r["flow_up_bw"])
    ev[1].record()
    harmonic_fill(flows[0], hole[:, :-1], sweeps, out=flows[0])
    harmonic_fill(flows[1], hole[:, 1:], sweeps, out=flows[1])
    ev[2].record()
    occ, occ_bw, _, _ = fb_consistency(flows[0].view(-1, 2, H, W), flows[1].view(-1, 2, H, W))
    ev[3].record()
    out, source = inpaint_propagate(frames, hole, flows[0], flows[1], occ.view(V, n - 1, H, W), occ_bw.view(V, n - 1, H, W))
    ev[4].record()
    harmonic_fill(out, source == SOURCE_SPATIAL, sweeps, out=out)
    ev[5].record()
    err = interpolation_error(out.view(-1, 3, H, W), frames.view(-1, 3, H, W))
    s, c = ssim(out.view(-1, 3, H, W), frames.view(-1, 3, H, W))
    ev[6].record()
    torch.cuda.synchronize()
    times = {name: ev[i].elapsed_time(ev[i + 1]) for i, name in enumerate(STAGES)}
    p = statistics.mean(psnr(a, b) for a, b in zip(err.sq_sum.tolist(), err.count.tolist()))
    return times, (out, source, p, float((s / c).mean()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--sweeps", type=int, default=512)
    ap.add_argument("--model", default="raft_nc_dbl", choices=["raft_nc_dbl", "raft"])
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/inpainting_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("inpainting_bench needs a CUDA device")
    from rnc.inpaint import SOURCE_SPATIAL
    from rnc.synth import build_model, shift_sequence

    seqs = [[f.to(DEV) for f in shift_sequence(T, H, W, seed=s)] for s in range(VIDEOS)]
    masks = [list(hole_masks(T)) for _ in range(VIDEOS)]
    m = build_model(args.model).to(DEV)
    run(m, [seq[:3] for seq in seqs], [mk[:3] for mk in masks], args.sweeps)          # warm-up: every kernel and shape
    rounds = []
    for _ in range(args.rounds):
        times, (out, source, p, s) = run(m, seqs, masks, args.sweeps)
        rounds.append(times)
    med = {k: round(statistics.median(r[k] for r in rounds), 2) for k in STAGES}
    hole_px = int(torch.stack([torch.stack(mk) for mk in masks]).ne(0).sum())
    line = {"card": card(), "frames": f"{H}x{W}", "model": args.model, "iters": ITERS, "videos": VIDEOS, "T": T,
            "pairs": VIDEOS * (T - 1), "sweeps": args.sweeps, "hole_share": round(hole_px / (VIDEOS * T * H * W), 4),
            "spatial_share_of_hole": round(float((source == SOURCE_SPATIAL).sum()) / hole_px, 4),
            "stage_ms": med, "stage_ms_rounds": rounds, "total_ms": round(sum(med.values()), 1),
            "inpainting_share_of_flow_pass": round(sum(med[k] for k in STAGES[1:5]) / med["flow_pass"], 4),
            "psnr_all_frames_random_weights": round(p, 2), "ssim_all_frames_random_weights": round(s, 4),
            "peak_memory_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2)}
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "inpainting_bench.json"), "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
