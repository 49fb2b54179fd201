"""Video-stabilization cost, stage by stage, at the DAVIS frame size: the flow pass, the homography fit, the path, the warp and
the metrics, and the fit alone on exact camera flows, where RANSAC has real inliers.

    python tools/stabilization_bench.py [--model raft_nc_dbl] [--out DIR]

Eight synthetic 480x854 videos of 50 frames (rnc.synth.shift_sequence, frames resident on the GPU), run as
rnc.harness.validate_stabilization runs them: run_sequences (32 iterations, batch_size 8), each pair's flow fitted as it is
yielded (rnc.stabilize.fit_homographies, stride 8, 256 hypotheses, 4 refine rounds), then per video smooth_path (radius 30,
sigma 10, crop) and warp_frames, then the metrics (stabilization_metrics on the host, interpolation_error's partials of the
output and the input on the device).  CUDA events around every fit, path and warp call; the flow pass is the rest of the
flow loop; the metrics are timed by the host clock after a device synchronise.  Then the fit of the 49 exact forward flows
of one rnc.synth.shaky_sequence video, as one call of 49 pairs and as 49 calls of one pair, 5 timed repetitions after a
warm-up.  Prints one JSON line with the card name and power limit beside the times.

    python tools/stabilization_bench.py --fill [--model raft_nc_dbl] [--out DIR]

instead times the full-frame stabilizer, stabilize_videos(crop=False, fill=True) stage by stage on the same videos:
run_sequences_bidirectional (both flows of each pair copied into the stacked tensors as they are yielded), the fit of each
forward flow, the path and the warp per video, then rnc.stabilize's fill steps on the stack as fill_uncovered runs them
(512 sweeps): the residual transfer, the residual completion, the re-add with the consistency check, the propagation and
the spatial fill, each between CUDA events; the filled output is checked against fill_uncovered's.  Prints one JSON line
with the card name and power limit, the peak memory and the shares of filled pixels.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-ncup_b200")]

DEV = "cuda:0"
H, W, T, ITERS, VIDEOS = 480, 854, 50, 32, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def event():
    e = torch.cuda.Event(enable_timing=True)
    e.record()
    return e


@torch.no_grad()
def run(m, seqs):
    """One pass over the videos; returns the stage times in ms, the fits' status counts and the summary."""
    from rnc import native
    from rnc.harness import run_sequences
    from rnc.interp import interpolation_error
    from rnc.stabilize import fit_homographies, smooth_path, stabilization_metrics, summarize_stabilization, warp_frames
    ws = torch.empty(native.rnc.homography_fit_workspace_bytes(1, H, W, 8, 256), dtype=torch.uint8, device=DEV)
    fits = [[None] * (len(s) - 1) for s in seqs]
    fit_marks = []
    torch.cuda.synchronize()
    start = event()
    for s, k, flow in run_sequences(m, seqs, ITERS, batch_size=VIDEOS, device=DEV):
        a = event()
        fits[s][k] = fit_homographies(flow[None], workspace=ws)
        fit_marks.append((a, event()))
    end = event()
    path_marks, warp_marks, res = [], [], []
    for seq, fit in zip(seqs, fits):
        A, inl, mat, st = (torch.cat([f[j] for f in fit]) for j in range(4))
        a = event()
        M, Minv, alpha = smooth_path(A[None], H, W)
        b = event()
        frames, valid = warp_frames(torch.stack(seq), Minv[0])
        c = event()
        path_marks.append((a, b))
        warp_marks.append((b, c))
        res.append((A, M[0], frames, st, alpha))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    records = []
    for seq, (A, M, frames, _, _) in zip(seqs, res):
        inp = torch.stack(seq)
        rows = [interpolation_error(v[1:], v[:-1]) for v in (frames, inp)]
        records.append((stabilization_metrics(A, M), *[list(zip(e.sq_sum.tolist(), e.count.tolist())) for e in rows]))
    summary = summarize_stabilization(records)
    metrics = (time.perf_counter() - t0) * 1e3
    fit = sum(a.elapsed_time(b) for a, b in fit_marks)
    times = {"flow_pass": start.elapsed_time(end) - fit, "fit": fit, "path": sum(a.elapsed_time(b) for a, b in path_marks),
             "warp": sum(a.elapsed_time(b) for a, b in warp_marks), "metrics": metrics}
    status = torch.cat([r[3] for r in res]).cpu()
    return times, len(fit_marks), {"ok": int((status == 0).sum()), "few": int((status != 0).sum())}, summary, \
        [float(r[4]) for r in res]


def exact_fit_times(reps=5):
    """The fit of one shaky video's exact flows: 49 pairs in one call and 49 calls of one pair, median ms."""
    from rnc.stabilize import fit_homographies
    from rnc.synth import shaky_sequence
    _, _, flows = shaky_sequence(T, H, W, seed=0)
    flows = flows.to(DEV)
    out = {}
    for name, fn in (("one_call", lambda: fit_homographies(flows)),
                     ("per_pair", lambda: [fit_homographies(flows[i:i + 1]) for i in range(T - 1)])):
        fn()
        times = []
        for _ in range(reps):
            a = event()
            fn()
            b = event()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        out[name] = round(statistics.median(times), 3)
    inl = fit_homographies(flows)[1].float() / fit_homographies(flows)[2].float()
    out["inlier_share"] = round(float(inl.mean()), 4)
    return out


@torch.no_grad()
def run_fill(m, seqs, check=False):
    """One full-frame pass over the videos (crop=False, fill=True); returns the stage times in ms, the number of pairs and
    the source map."""
    from rnc import native
    from rnc.harness import run_sequences_bidirectional
    from rnc.inpaint import SOURCE_SPATIAL, harmonic_fill, inpaint_propagate
    from rnc.metrics import fb_consistency
    from rnc.stabilize import _readd_, fill_uncovered, fit_homographies, flow_residual, smooth_path, warp_frames
    ws = torch.empty(native.rnc.homography_fit_workspace_bytes(1, H, W, 8, 256), dtype=torch.uint8, device=DEV)
    V, Tn = len(seqs), len(seqs[0])
    fits = [[None] * (Tn - 1) for _ in seqs]
    flows = torch.zeros(2, V, Tn - 1, 2, H, W, device=DEV)
    fit_marks = []
    torch.cuda.synchronize()
    start = event()
    for s, k, r in run_sequences_bidirectional(m, seqs, ITERS, batch_size=VIDEOS, device=DEV):
        a = event()
        fits[s][k] = fit_homographies(r["flow_up"][None], workspace=ws)
        fit_marks.append((a, event()))
        flows[0, s, k].copy_(r["flow_up"])
        flows[1, s, k].copy_(r["flow_up_bw"])
    end = event()
    marks = {"path": [], "warp": []}
    A = torch.stack([torch.cat([f[0] for f in fit]) for fit in fits])
    M, Minv = torch.empty(V, Tn, 3, 3, dtype=torch.float64, device=DEV), torch.empty(V, Tn, 3, 3, dtype=torch.float64, device=DEV)
    frames = torch.empty(V, Tn, 3, H, W, device=DEV)
    valid = torch.empty(V, Tn, H, W, dtype=torch.uint8, device=DEV)
    for v, seq in enumerate(seqs):
        a = event()
        Mv, Mi, _ = smooth_path(A[v:v + 1], H, W, crop=False)
        b = event()
        frames[v], valid[v] = warp_frames(torch.stack(seq), Mi[0])
        c = event()
        M[v], Minv[v] = Mv[0], Mi[0]
        marks["path"].append((a, b))
        marks["warp"].append((b, c))
    e = [event()]
    res, res_bw = flow_residual(flows[0], flows[1], A, M, Minv)
    e.append(event())
    hole = (valid == 0).to(torch.uint8)
    harmonic_fill(res, hole[:, :-1], 512, out=res)
    harmonic_fill(res_bw, hole[:, 1:], 512, out=res_bw)
    e.append(event())
    _readd_(res, res_bw, A, M, Minv)
    n = V * (Tn - 1)
    occ, occ_bw, _, _ = fb_consistency(res.view(n, 2, H, W), res_bw.view(n, 2, H, W), 0.01, 0.5)
    e.append(event())
    out, source = inpaint_propagate(frames, hole, res, res_bw, occ.view(V, Tn - 1, H, W), occ_bw.view(V, Tn - 1, H, W))
    e.append(event())
    harmonic_fill(out, source == SOURCE_SPATIAL, 512, out=out)
    e.append(event())
    torch.cuda.synchronize()
    fit = sum(a.elapsed_time(b) for a, b in fit_marks)
    times = {"flow_pass": start.elapsed_time(end) - fit, "fit": fit}
    times.update({k: sum(a.elapsed_time(b) for a, b in v) for k, v in marks.items()})
    for i, k in enumerate(("transfer", "residual_completion", "readd_and_consistency", "propagation", "spatial_fill")):
        times[k] = e[i].elapsed_time(e[i + 1])
    if check:
        del res, res_bw, occ, occ_bw
        want, src = fill_uncovered(frames, valid, flows[0], flows[1], A, M, Minv)
        assert torch.equal(want, out) and torch.equal(src, source), "the staged fill differs from fill_uncovered"
    return times, len(fit_marks), source


def main_fill(args, m, seqs):
    from rnc.inpaint import SOURCE_KNOWN, SOURCE_SPATIAL
    run_fill(m, [seq[:3] for seq in seqs])                                  # warm-up: every kernel and shape
    torch.cuda.reset_peak_memory_stats()
    times, pairs, source = run_fill(m, seqs)
    peak = torch.cuda.max_memory_allocated() / 1e9
    run_fill(m, seqs, check=True)
    fill = sum(times[k] for k in ("transfer", "residual_completion", "readd_and_consistency", "propagation", "spatial_fill"))
    src = source.flatten(2)
    line = {"card": card(), "frames": f"{H}x{W}", "model": args.model, "iters": ITERS, "videos": VIDEOS, "T": T,
            "pairs": pairs, "crop": False, "fill": True, "sweeps": 512, "stage_ms": {k: round(v, 1) for k, v in times.items()},
            "fill_share_of_flow_pass": round(fill / times["flow_pass"], 4),
            "uncovered_share": round(float((src != SOURCE_KNOWN).float().mean()), 4),
            "spatial_share_random_weights": round(float((src == SOURCE_SPATIAL).float().mean()), 4),
            "source_counts_random_weights": torch.bincount(source.flatten().long(), minlength=5).tolist(),
            "peak_memory_gb": round(peak, 2)}
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "stabilization_fill_bench.json"), "w") as f:
            f.write(json.dumps(line) + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="raft_nc_dbl", choices=["raft_nc_dbl", "raft"])
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/stabilization_bench.json")
    ap.add_argument("--fill", action="store_true", help="time the full-frame stabilizer (crop=False, fill=True) instead")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("stabilization_bench needs a CUDA device")
    from rnc.synth import build_model, shift_sequence

    seqs = [[f.to(DEV) for f in shift_sequence(T, H, W, seed=s)] for s in range(VIDEOS)]
    m = build_model(args.model).to(DEV)
    if args.fill:
        return main_fill(args, m, seqs)
    run(m, [seq[:3] for seq in seqs])                                       # warm-up: every kernel and shape
    torch.cuda.reset_peak_memory_stats()
    times, pairs, status, summary, alphas = run(m, seqs)
    peak = torch.cuda.max_memory_allocated() / 1e9
    line = {"card": card(), "frames": f"{H}x{W}", "model": args.model, "iters": ITERS, "videos": VIDEOS, "T": T,
            "pairs": pairs, "stage_ms": {k: round(v, 1) for k, v in times.items()},
            "fit_ms_per_pair": round(times["fit"] / pairs, 3),
            "fit_path_warp_share_of_flow_pass": round((times["fit"] + times["path"] + times["warp"]) / times["flow_pass"], 4),
            "status_random_weights": status, "alpha_random_weights": [round(a, 4) for a in alphas],
            "summary_random_weights": summary, "peak_memory_gb": round(peak, 2),
            "exact_flow_fit_ms_49_pairs": exact_fit_times()}
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "stabilization_bench.json"), "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
