"""Frame interpolation cost: the interpolation launches alone, and validate_interpolation against the flow pass it runs.

    python tools/interpolation_bench.py [--rounds 3] [--model raft_nc_dbl] [--out DIR]

(a) rnc.interp.interpolate alone (a memset and four launches) on B = 8 pairs of 436x1024 frames with smooth random flows and
    fb_consistency masks, at T = 1 and T = 7 times: CUDA events around 20 calls after a warm-up, the median of --rounds.
(b) rnc.harness.validate_interpolation on the workload of tools/bidirectional_sequence_bench.py (twelve synthetic sequences,
    rnc.synth.shift_sequence, at 436x1024, 32 iterations, batch_size 8, frames resident on the GPU), against
    run_sequences_bidirectional alone on the same even- and odd-indexed subsequences, alternating within one process: a host
    clock around each whole pass that ends in a device synchronise.  (b) - run_sequences_bidirectional is the cost of the
    interpolation and its error, as a share of the pass.
Prints one JSON line with the card name and power limit beside the numbers.
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
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-ncup_b200")]

DEV = "cuda:0"
H, W, ITERS, B = 436, 1024, 32, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def launches_ms(T, rounds):
    from rnc.interp import interpolate
    from rnc.metrics import fb_consistency
    g = torch.Generator().manual_seed(1)
    I0, I1 = (torch.rand(B, 3, H, W, generator=g) * 255).to(DEV), (torch.rand(B, 3, H, W, generator=g) * 255).to(DEV)
    low = torch.randn(B, 2, H // 16, W // 16, generator=g) * 8
    flow = F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False).to(DEV)
    flow_bw = -flow + 0.3 * torch.randn(B, 2, H, W, generator=g).to(DEV)
    occ, occ_bw, _, _ = fb_consistency(flow, flow_bw)
    times = [(k + 1) / (T + 1) for k in range(T)]
    for _ in range(3):
        interpolate(I0, I1, flow, flow_bw, occ, occ_bw, times)
    out = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            interpolate(I0, I1, flow, flow_bw, occ, occ_bw, times)
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / 20)
    return statistics.median(out), out


@torch.no_grad()                    # the flow passes are inference only
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--model", default="raft_nc_dbl", choices=["raft_nc_dbl", "raft"])
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/interpolation_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("interpolation_bench needs a CUDA device")
    from rnc.harness import run_sequences_bidirectional, validate_interpolation
    from rnc.synth import build_model, shift_sequence

    line = {"card": card(), "frames": f"{H}x{W}", "batch": B}
    for T in (1, 7):
        med, all_ = launches_ms(T, args.rounds)
        line[f"interpolate_T{T}_ms"] = round(med, 3)
        line[f"interpolate_T{T}_ms_rounds"] = [round(v, 3) for v in all_]
    torch.cuda.empty_cache()

    rng = random.Random(5)
    lens = [rng.randint(20, 50) for _ in range(12)]
    seqs = [[f.to(DEV) for f in shift_sequence(n, H, W, seed=s)] for s, n in enumerate(lens)]
    subs = [seq[off::2] for seq in seqs for off in (0, 1)]
    m = build_model(args.model).to(DEV)

    def flows_only(sq):
        for _ in run_sequences_bidirectional(m, sq, ITERS, batch_size=B, device=DEV):
            pass

    def validate(sq):
        return validate_interpolation(m, sq, ITERS, batch_size=B, device=DEV)

    short = [seq[:5] for seq in seqs[:B]]
    flows_only([seq[off::2] for seq in short for off in (0, 1)])
    validate(short)
    torch.cuda.synchronize()

    def clock(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    t_flow, t_val, res = [], [], None
    for _ in range(args.rounds):
        t_flow.append(clock(lambda: flows_only(subs))[0])
        t, res = clock(lambda: validate(seqs))
        t_val.append(t)
    n = sum(n - 2 for n in lens)
    mf, mv = statistics.median(t_flow), statistics.median(t_val)
    line.update({
        "model": args.model, "iters": ITERS, "sequences": lens, "triplets": n, "rounds": args.rounds,
        "run_sequences_bidirectional_s": [round(v, 3) for v in t_flow],
        "validate_interpolation_s": [round(v, 3) for v in t_val],
        "interpolation_share_of_pass": round((mv - mf) / mv, 4),
        "interpolation_ms_per_triplet": round(1e3 * (mv - mf) / n, 3),
        "result": res,
    })
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "interpolation_bench.json"), "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
