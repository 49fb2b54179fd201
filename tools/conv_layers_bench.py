"""Per-layer cost of the tensor-core convolution (rnc_conv2d_umma_fwd) in one update-block iteration at the benchmark shape.

    python tools/conv_layers_bench.py [--batch 8] [--launches 50] [--no-breakdown]

Records every uconv call of the second update-block iteration of a B x 440x1024 forward (real buffers, flags and
epilogues), then replays each call back to back and times it with CUDA events after a warm-up:
  ms          the layer as the benchmark runs it
  ms_nob      the same launches with RNC_CONV_PROBE_NOB=1 (weights loaded once per ring fill: the weight stream's cost)
and the useful / tensor-issued FLOP computed from the shapes (three fp16 MMAs per product, padded to whole tiles, K blocks
and column tiles).  `peak_frac` is the issued rate over the dense fp16 peak (989 TFLOP/s at 1830 MHz, data sheet) scaled
to the SM clock sampled during the run.  Then tools/step_breakdown.py splits one step.  The last stdout line is JSON.
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "raft-ncup_b200")):
    sys.path.insert(0, p)

PEAK_FP16_DENSE, PEAK_MHZ = 989e12, 1830.0


def measure(batch, launches):
    """Child process: record one iteration's conv calls and time each (RNC_CONV_PROBE_NOB is read once per process)."""
    os.environ["RNC_GRAPH"] = "0"
    import torch
    from bench import ClockSampler
    from rnc import native
    from rnc.engine_umma import UmmaWeights
    from rnc.synth import build_model, frames

    dev = "cuda:0"
    m = build_model("raft_nc_dbl").to(dev)
    im1, im2 = frames(batch, 440, 1024)
    eng = m.engine()
    calls, state = [], {"n": 0, "rec": False}
    uconv, update_iter = eng.uconv, eng._update_iter

    def rec_uconv(*a, **k):
        if state["rec"]:
            calls.append((a, k))
        return uconv(*a, **k)

    def rec_iter(ws, pk, want_mask, want_delta):
        state["n"] += 1
        state["rec"] = state["n"] == 2
        state["names"] = {id(v): n for n, v in vars(pk).items() if isinstance(v, UmmaWeights)}
        try:
            return update_iter(ws, pk, want_mask, want_delta)
        finally:
            state["rec"] = False

    eng.uconv, eng._update_iter = rec_uconv, rec_iter
    with torch.no_grad():
        m(im1.to(dev), im2.to(dev), iters=3, test_mode=True)
    torch.cuda.synchronize()
    eng.uconv, eng._update_iter = uconv, update_iter

    L = native.lib()
    rows = []
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    for a, k in calls:
        B, H, W, wt = a[0], a[1], a[2], a[6]
        flags = k.get("flags", 0)
        c_in = a[4] + k.get("c1", 0)
        ntiles = L.rnc_conv_umma_tiles(wt.kh, wt.kw, k.get("stride", 1), B, H, W, flags)
        row = {"layer": state["names"].get(id(wt), "?"), "epilogue": a[7], "flags": flags, "k": f"{wt.kh}x{wt.kw}",
               "cin": c_in, "cout": wt.cout, "coutpad": wt.coutpad,
               "gflop_useful": 2.0 * B * H * W * wt.cout * wt.kh * wt.kw * c_in / 1e9,
               "gflop_issued": 3 * 2.0 * ntiles * 128 * wt.coutpad * wt.ktot / 1e9}
        for _ in range(5):
            uconv(*a, **k)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            uconv(*a, **k)
        e1.record()
        torch.cuda.synchronize()
        row["ms"] = e0.elapsed_time(e1) / launches
        rows.append(row)
    clocks = sampler.stop()
    return {"rows": rows, "clocks": clocks}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return {"name": None, "power_limit_w": None, "sm_max_mhz": None}


def child(batch, launches, nob):
    env = dict(os.environ, RNC_CONV_PROBE_NOB="1" if nob else "0")
    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--batch", str(batch), "--launches", str(launches)],
                         env=env, capture_output=True, text=True)
    if out.returncode != 0:
        sys.stderr.write(out.stdout + out.stderr)
        raise SystemExit(f"measurement child failed (RNC_CONV_PROBE_NOB={int(nob)})")
    return json.loads(out.stdout.strip().splitlines()[-1])


def breakdown(batch):
    """tools/step_breakdown.py's split of one step: {bracket: ms} plus the step time."""
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "step_breakdown.py")], env=dict(os.environ, B=str(batch)),
                         capture_output=True, text=True)
    if out.returncode != 0:
        sys.stderr.write(out.stdout + out.stderr)
        raise SystemExit("step_breakdown.py failed")
    res = {}
    for line in out.stdout.splitlines():
        mt = re.match(r"step ([\d.]+) ms", line)
        if mt:
            res["step_ms"] = float(mt.group(1))
        mt = re.match(r"\s+(\S+)\s+(?:x\s*\d+\s+)?([\d.]+) ms", line)
        if mt:
            res[mt.group(1)] = float(mt.group(2))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--no-breakdown", action="store_true")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        print(json.dumps(measure(args.batch, args.launches)))
        return
    base, nob = child(args.batch, args.launches, False), child(args.batch, args.launches, True)
    mhz = base["clocks"].get("sm_mhz") or PEAK_MHZ
    peak = PEAK_FP16_DENSE * mhz / PEAK_MHZ
    rows = base["rows"]
    for r, rn in zip(rows, nob["rows"]):
        r["ms_nob"] = rn["ms"]
        r["peak_frac"] = r["gflop_issued"] * 1e9 / (r["ms"] * 1e-3) / peak
    tot = {k: sum(r[k] for r in rows) for k in ("ms", "ms_nob", "gflop_useful", "gflop_issued")}
    hdr = f"{'layer':10s} {'k':>4s} {'cin':>4s} {'cout':>4s} {'epi':>3s} {'ms':>7s} {'ms_nob':>7s} {'GF use':>7s} {'GF iss':>7s} {'peak':>5s}"
    print(hdr, file=sys.stderr)
    for r in rows:
        print(f"{r['layer']:10s} {r['k']:>4s} {r['cin']:4d} {r['cout']:4d} {r['epilogue']:3d} {r['ms']:7.3f} {r['ms_nob']:7.3f} "
              f"{r['gflop_useful']:7.1f} {r['gflop_issued']:7.1f} {r['peak_frac']:5.2f}", file=sys.stderr)
    print(f"{'total':10s} {'':>4s} {'':>4s} {'':>4s} {'':>3s} {tot['ms']:7.3f} {tot['ms_nob']:7.3f} "
          f"{tot['gflop_useful']:7.1f} {tot['gflop_issued']:7.1f}", file=sys.stderr)
    res = {"card": card(), "clocks": base["clocks"], "batch": args.batch, "shape": [55, 128], "layers": rows, "total": tot,
           "peak_tflops_at_clock": peak / 1e12}
    if not args.no_breakdown:
        res["step_breakdown"] = breakdown(args.batch)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
