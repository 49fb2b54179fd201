"""Sequence inference throughput: create_sintel_submission's workflow (warm-started pairs of whole sequences).

    python tools/sequence_bench.py [--rounds 2] [--model raft_nc_dbl] [--out DIR]

Twelve synthetic sequences of 20 to 50 frames (Sintel's test-set shape: 436x1024, padded to 440x1024; rnc.synth.shift_sequence),
32 iterations, frames resident on the GPU.  Times, alternating within one process:
  (a) rnc.harness.run_sequence with warm start, sequence after sequence (B = 1; the reference's workflow);
  (b) rnc.harness.run_sequences(batch_size=8) with warm start (each frame encoded once);
  (c) batched B = 8 model(...) calls over the same pairs, cold (the ceiling without reuse; the last call is filled up with
      repeats of its last pair, which are not counted);
  (d) (b) without warm start, and (e) (c) with CUDA graphs off (RNC_GRAPH=0): they separate the cost of the warm start and
      that of eager launches from that of the sequence steps.
Each is a host clock around a whole pass that ends in a device synchronise; every shape is warmed up first.  A separate
pass of (b) and (c) with the engine's CUDA-event brackets on (rnc.engine._Timed) gives the encoder time per step.  Prints
one JSON line with the card name and power limit beside the numbers.
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-ncup_b200")]

DEV = "cuda:0"
H, W, ITERS, B = 436, 1024, 32, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--model", default="raft_nc_dbl", choices=["raft_nc_dbl", "raft"])
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/sequence_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sequence_bench needs a CUDA device")
    from rnc.harness import run_sequence, run_sequences, sequence_schedule
    from rnc.synth import build_model, shift_sequence
    from utils.utils import InputPadder

    rng = random.Random(5)
    lens = [rng.randint(20, 50) for _ in range(12)]
    seqs = [[f.to(DEV) for f in shift_sequence(n, H, W, seed=s)] for s, n in enumerate(lens)]
    pairs = [(s, p) for s, n in enumerate(lens) for p in range(n - 1)]
    m = build_model(args.model).to(DEV)
    eng = m.engine()
    padder = InputPadder((3, H, W))

    def run_a(sq):
        for seq in sq:
            run_sequence(m, seq, ITERS, warm_start=True, device=DEV)

    def run_b(sq, warm=True):
        for _ in run_sequences(m, sq, ITERS, warm_start=warm, batch_size=B, device=DEV):
            pass

    def run_c(sq, prs):
        with torch.no_grad():
            for i in range(0, len(prs), B):
                chunk = prs[i:i + B]
                chunk = chunk + [chunk[-1]] * (B - len(chunk))
                im1 = torch.stack([sq[s][p] for s, p in chunk])
                im2 = torch.stack([sq[s][p + 1] for s, p in chunk])
                p1, p2 = padder.pad(im1, im2)
                m(p1, p2, iters=ITERS, test_mode=True)

    # warm-up: every shape the timed passes use (B = 1 warm and cold, sequence steps at B = 8, a captured B = 8 graph)
    short = [seq[:4] for seq in seqs[:B]]
    run_a([seqs[0][:4]])
    run_b(short)
    run_b(short, warm=False)
    run_c(seqs, pairs[:3 * B])
    torch.cuda.synchronize()

    def clock(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def run_e(sq, prs):
        prev = os.environ.get("RNC_GRAPH")
        os.environ["RNC_GRAPH"] = "0"
        try:
            run_c(sq, prs)
        finally:
            if prev is None:
                del os.environ["RNC_GRAPH"]
            else:
                os.environ["RNC_GRAPH"] = prev

    times = {"a": [], "b": [], "c": [], "d": [], "e": []}
    for _ in range(args.rounds):
        times["a"].append(clock(lambda: run_a(seqs)))
        times["b"].append(clock(lambda: run_b(seqs)))
        times["c"].append(clock(lambda: run_c(seqs, pairs)))
        times["d"].append(clock(lambda: run_b(seqs, warm=False)))
        times["e"].append(clock(lambda: run_e(seqs, pairs)))

    enc = {}
    for k, fn in (("b", lambda: run_b(seqs)), ("c", lambda: run_c(seqs, pairs))):
        eng.profile = {}
        try:
            fn()
            torch.cuda.synchronize()
            ev = eng.profile.get("encoders", [])
            enc[k] = statistics.median(a.elapsed_time(b) for a, b in ev) if ev else None
        finally:
            eng.profile = None

    steps = sequence_schedule(lens, B)
    idle = sum(c.idle for step in steps for c in step)
    n = len(pairs)
    line = {
        "card": card(), "model": args.model, "frames": f"{H}x{W} padded to {(H + 7) // 8 * 8}x{W}", "iters": ITERS,
        "sequences": lens, "pairs": n, "rounds": args.rounds,
        "a_run_sequence_pairs_per_s": [round(n / t, 2) for t in times["a"]],
        "b_run_sequences_b8_pairs_per_s": [round(n / t, 2) for t in times["b"]],
        "c_batched_b8_cold_pairs_per_s": [round(n / t, 2) for t in times["c"]],
        "d_run_sequences_b8_cold_pairs_per_s": [round(n / t, 2) for t in times["d"]],
        "e_batched_b8_cold_eager_pairs_per_s": [round(n / t, 2) for t in times["e"]],
        "encoders_ms_per_step_b": enc["b"], "encoders_ms_per_step_c": enc["c"],
        "steps_b": len(steps), "idle_slot_step_fraction": round(idle / (B * len(steps)), 4),
    }
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sequence_bench.json"), "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
