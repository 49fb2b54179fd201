"""Temporal-consistency cost, stage by stage, at the DAVIS frame size: the flow pass, the per-step solve and the warping-error
metric, and one step launched eagerly against the same step replayed from a captured CUDA graph.

    python tools/temporal_bench.py [--sweeps 512] [--model raft_nc_dbl] [--out DIR]

Eight synthetic 480x854 videos of 50 frames (rnc.synth.shift_sequence, frames resident on the GPU), processed as
P_t = a_t I_t + b_t + noise (per-frame gain and offset, the flicker of per-frame processing), run as
rnc.harness.validate_temporal_consistency runs them: run_sequences_bidirectional (32 iterations, batch_size 8) on the
original frames, each pair's flow_up_bw and occ_bw stepping its video at once (rnc.temporal.temporal_step, one video per
step, `sweeps` sweeps), then the warping error of P and O at that frame.  CUDA events around every step and metric call;
the flow pass is the rest of the run.  With random weights the occlusion masks cover nearly every pixel, so the warping
errors may be NaN (no frame with a matched pixel); the solve does the same work whatever the weights.  Then one step of 1 and of 8 videos (C = 3), eager and as a graph replay, 5 timed
repetitions each after a warm-up.  Prints one JSON line with the card name and power limit beside the times.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-ncup_b200")]

DEV = "cuda:0"
H, W, T, ITERS, VIDEOS, C = 480, 854, 50, 32, 8, 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def processed(seq, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    I = torch.stack(seq)
    a = 1 + 0.05 * torch.randn(len(seq), 1, 1, 1, generator=g, device=DEV)
    b = 6 * torch.randn(len(seq), 1, 1, 1, generator=g, device=DEV)
    return a * I + b + torch.randn(I.shape, generator=g, device=DEV)


@torch.no_grad()
def run(m, seqs, procs, sweeps):
    """One pass over the videos; returns the stage times in ms and the mean warping errors of P and O."""
    from rnc import native
    from rnc.harness import run_sequences_bidirectional
    from rnc.temporal import temporal_step, warping_error
    outs = [torch.empty_like(p) for p in procs]
    for o, p in zip(outs, procs):
        o[0] = p[0]
    ws = torch.empty(native.rnc.temporal_step_workspace_bytes(1, C, H, W), dtype=torch.uint8, device=DEV)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    marks, parts = [], []
    torch.cuda.synchronize()
    start.record()
    for s, k, r in run_sequences_bidirectional(m, seqs, ITERS, batch_size=VIDEOS, device=DEV):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        o, seq = outs[s], seqs[s]
        temporal_step(o[k][None], procs[s][k + 1][None], seq[k][None], seq[k + 1][None], r["flow_up_bw"][None],
                      r["occ_bw"][None], sweeps=sweeps, out=o[k + 1][None], workspace=ws)
        ev[1].record()
        g, occ = r["flow_up_bw"][None, None], r["occ_bw"][None, None]
        parts.append((warping_error(procs[s][k:k + 2][None], g, occ), warping_error(o[k:k + 2][None], g, occ)))
        ev[2].record()
        marks.append(ev)
    end.record()
    torch.cuda.synchronize()
    total = start.elapsed_time(end)
    solve = sum(e[0].elapsed_time(e[1]) for e in marks)
    metric = sum(e[1].elapsed_time(e[2]) for e in marks)
    scored = [(float(p[0][0] / p[1][0]), float(q[0][0] / q[1][0])) for p, q in parts if int(p[1][0]) > 0]
    wp = statistics.mean(a for a, _ in scored) if scored else math.nan
    wo = statistics.mean(b for _, b in scored) if scored else math.nan
    matched = sum(int(p[1][0]) for p, _ in parts) / (len(parts) * H * W)
    return {"flow_pass": total - solve - metric, "solve": solve, "metric": metric}, len(marks), wp, wo, matched


def step_times(V, sweeps, reps=5):
    """One step of V videos: eager launches against a captured graph's replay, median ms over reps."""
    from rnc import native
    from rnc.temporal import temporal_step
    g = torch.Generator(device=DEV).manual_seed(V)
    O, P = (torch.rand(V, C, H, W, generator=g, device=DEV) * 255 for _ in range(2))
    I0, I1 = (torch.rand(V, 3, H, W, generator=g, device=DEV) * 255 for _ in range(2))
    G = torch.randn(V, 2, H, W, generator=g, device=DEV) * 3
    occ = (torch.rand(V, H, W, generator=g, device=DEV) < 0.05).to(torch.uint8)
    out = torch.empty(V, C, H, W, device=DEV)
    ws = torch.empty(native.rnc.temporal_step_workspace_bytes(V, C, H, W), dtype=torch.uint8, device=DEV)
    step = lambda: temporal_step(O, P, I0, I1, G, occ, sweeps=sweeps, out=out, workspace=ws)  # noqa: E731
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    res = {}
    for name, fn in (("eager", step), ("graph", graph.replay)):
        fn()
        times = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        res[name] = round(statistics.median(times), 3)
    step()
    want = out.clone()
    graph.replay()
    torch.cuda.synchronize()
    res["graph_equals_eager"] = bool(torch.equal(out, want))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=512)
    ap.add_argument("--model", default="raft_nc_dbl", choices=["raft_nc_dbl", "raft"])
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/temporal_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("temporal_bench needs a CUDA device")
    from rnc.synth import build_model, shift_sequence

    seqs = [[f.to(DEV) for f in shift_sequence(T, H, W, seed=s)] for s in range(VIDEOS)]
    procs = [processed(seq, s) for s, seq in enumerate(seqs)]
    m = build_model(args.model).to(DEV)
    run(m, [seq[:3] for seq in seqs], [p[:3] for p in procs], args.sweeps)             # warm-up: every kernel and shape
    torch.cuda.reset_peak_memory_stats()
    times, steps, wp, wo, matched = run(m, seqs, procs, args.sweeps)
    peak = torch.cuda.max_memory_allocated() / 1e9
    line = {"card": card(), "frames": f"{H}x{W}", "model": args.model, "iters": ITERS, "videos": VIDEOS, "T": T, "C": C,
            "pairs": steps, "sweeps": args.sweeps, "stage_ms": {k: round(v, 1) for k, v in times.items()},
            "solve_ms_per_step": round(times["solve"] / steps, 3), "metric_ms_per_step": round(times["metric"] / steps, 3),
            "solve_share_of_flow_pass": round(times["solve"] / times["flow_pass"], 4),
            "matched_share_random_weights": round(matched, 6),
            "warping_error_processed_random_weights": wp, "warping_error_output_random_weights": wo,
            "peak_memory_gb": round(peak, 2),
            "one_step_ms": {f"V={V}": step_times(V, args.sweeps) for V in (1, VIDEOS)}}
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "temporal_bench.json"), "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
