"""Bidirectional sequence inference throughput: forward flow, backward flow and occlusion masks for every pair of many videos.

    python tools/bidirectional_sequence_bench.py [--rounds 2] [--model raft_nc_dbl] [--out DIR]

The workload of tools/sequence_bench.py: twelve synthetic sequences (rnc.synth.shift_sequence, lengths drawn as there) at
436x1024 (padded to 440x1024), 32 iterations, frames resident on the GPU, batch_size = 8.  Times, cold and warm, alternating
within one process:
  (a) what it takes without the feature: rnc.harness.run_sequences on the sequences, run_sequences on the reversed
      sequences, and rnc.metrics.fb_consistency on each pair's two flows;
  (b) rnc.harness.run_sequences_bidirectional.
One pair is both directions and the masks.  Each time is a host clock around a whole pass that ends in a device
synchronise; every shape is warmed up first.  A separate pass of each with the engine's CUDA-event brackets on
(rnc.engine._Timed) gives the encoders' and the warm start's milliseconds per step.  (b)'s forward flows are compared with
(a)'s in the same run (largest per-pair EPE).  Prints one JSON line with the card name and power limit beside the numbers.
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


@torch.no_grad()                    # run_sequences_bidirectional is inference only
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--model", default="raft_nc_dbl", choices=["raft_nc_dbl", "raft"])
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/bidirectional_sequence_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bidirectional_sequence_bench needs a CUDA device")
    from rnc.harness import run_sequences, run_sequences_bidirectional, sequence_schedule
    from rnc.metrics import fb_consistency
    from rnc.synth import build_model, shift_sequence

    rng = random.Random(5)
    lens = [rng.randint(20, 50) for _ in range(12)]
    seqs = [[f.to(DEV) for f in shift_sequence(n, H, W, seed=s)] for s, n in enumerate(lens)]
    rev = [seq[::-1] for seq in seqs]
    m = build_model(args.model).to(DEV)
    eng = m.engine()

    def run_a(sq, rq, warm, keep=None):
        fw = {}
        for s, p, f in run_sequences(m, sq, ITERS, warm_start=warm, batch_size=B, device=DEV):
            fw[(s, p)] = f
        for s, p, g in run_sequences(m, rq, ITERS, warm_start=warm, batch_size=B, device=DEV):
            k = (s, len(rq[s]) - 2 - p)                   # reversed pair p is (frame k + 1 -> frame k) of the original
            f = fw[k] if keep is not None else fw.pop(k)
            fb_consistency(f[None], g[None])
        if keep is not None:
            keep.update(fw)

    def run_b(sq, warm, keep=None):
        for s, p, r in run_sequences_bidirectional(m, sq, ITERS, warm_start=warm, batch_size=B, device=DEV):
            if keep is not None:
                keep[(s, p)] = r["flow_up"]

    # warm-up: every shape the timed passes use (steps of B and 2B slots, cold and warm)
    short = [seq[:4] for seq in seqs[:B]]
    for warm in (False, True):
        run_a(short, [seq[::-1] for seq in short], warm)
        run_b(short, warm)
    torch.cuda.synchronize()

    def clock(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    times = {k: [] for k in ("a_cold", "b_cold", "a_warm", "b_warm")}
    for _ in range(args.rounds):
        for warm in (False, True):
            tag = "warm" if warm else "cold"
            times["a_" + tag].append(clock(lambda: run_a(seqs, rev, warm)))
            times["b_" + tag].append(clock(lambda: run_b(seqs, warm)))

    prof, epe = {}, {}
    for warm in (False, True):
        tag = "warm" if warm else "cold"
        got = {}
        for k, fn in (("a_" + tag, lambda: run_a(seqs, rev, warm, keep=got.setdefault("a", {}))),
                      ("b_" + tag, lambda: run_b(seqs, warm, keep=got.setdefault("b", {})))):
            eng.profile = {}
            try:
                fn()
                torch.cuda.synchronize()
                prof[k] = {name: round(sum(a.elapsed_time(b) for a, b in ev), 2) for name, ev in eng.profile.items()
                           if name in ("encoders", "warm_start")}
            finally:
                eng.profile = None
        a, b = got["a"], got["b"]
        assert a.keys() == b.keys()
        epe[tag] = max((a[k] - b[k]).pow(2).sum(0).sqrt().mean().item() for k in a)
        epe[tag + "_identical_pairs"] = sum(torch.equal(a[k], b[k]) for k in a)
        del got, a, b

    steps_b = len(sequence_schedule(lens, B))
    steps_a = 2 * steps_b                                  # run_sequences on the sequences and on the reversed ones
    n = sum(lens) - len(lens)
    line = {
        "card": card(), "model": args.model, "frames": f"{H}x{W} padded to {(H + 7) // 8 * 8}x{W}", "iters": ITERS,
        "batch_size": B, "sequences": lens, "pairs": n, "rounds": args.rounds, "steps_b": steps_b, "steps_a": steps_a,
    }
    for k, ts in times.items():
        line[k + "_pairs_per_s"] = [round(n / t, 2) for t in ts]
        line[k + "_ms_per_step"] = round(1e3 * statistics.median(ts) / (steps_a if k[0] == "a" else steps_b), 2)
    for k, p in prof.items():
        st = steps_a if k[0] == "a" else steps_b
        for name, total in p.items():
            line[f"{k}_{name}_ms_per_step"] = round(total / st, 2)
    line["fw_rows_vs_a_worst_epe"] = epe
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bidirectional_sequence_bench.json"), "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
