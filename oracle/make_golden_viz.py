"""Flow-visualisation golden fixtures from the UNMODIFIED reference `flow_to_image` (core/utils/flow_viz.py:240-275), run on
the CPU (authoring container only; needs the reference):

    python oracle/make_golden_viz.py     ->  tests/golden/viz.npz + viz_meta.json

Per case of CASES, `case_input(name, npz)` gives the float32 [H, W, 2] flow: regenerated from its seed, or read back from the
npz for the small hand-built arrays (stored as `<name>_in`).  Recorded: the reference's uint8 image (`<name>_ref`), the
pixels whose normalised radius exceeds 1 (`<name>_branch`, from viz_oracle, which agrees with the reference on everything
but the arc tangent's last bit), and in the metadata numpy's version and SIMD dispatch, on which numpy's float32 arctan2 and
so the reference's output depend.  TEST INFRASTRUCTURE ONLY.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("RNC_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden")

# name -> (H, W, seed, scale): a seeded random flow, N(0, 1) * scale
RANDOM = {
    "rand_1x1": (1, 1, 1, 5.0),
    "rand_7x13": (7, 13, 2, 5.0),
    "rand_37x53": (37, 53, 3, 5.0),
    "rand_436x1024": (436, 1024, 4, 8.0),
    "large": (64, 96, 5, 3e5),
}
BRANCH_SEEDS = range(100, 400)   # 16x24 flows searched, in order, for ones whose max-radius pixel takes the > 1 branch
N_BRANCH = 3
HAND = ("zero", "unknown", "nan", "axes")


def _random(H, W, seed, scale):
    return (np.random.default_rng(seed).standard_normal((H, W, 2)) * scale).astype(np.float32)


def _hand(name):
    if name == "zero":
        return np.zeros((5, 6, 2), np.float32)
    if name == "unknown":
        f = _random(9, 11, 6, 4.0)
        f[0, 0] = (1e8, 0)
        f[1, 2] = (np.inf, 3)
        f[2, 3] = (-2, -np.inf)
        f[3, 4] = (1e7, 0)              # exactly the threshold: known, and the largest radius
        f[4, 5] = (0, np.float32(10000001.0))   # just above it: unknown
        f[5, 6] = (np.nan, np.inf)      # unknown wins over NaN
        return f
    if name == "nan":
        f = _random(13, 17, 7, 0.2)
        f[6, 8] = (np.nan, 0.5)         # one NaN: maxrad becomes -1 and the flow is negated
        f[0, 0] = (0.0, 1.0)            # rad 1 exactly: the negated flow's own maxrad is 1
        return f
    if name == "axes":
        z, nz = 0.0, -0.0
        px = [(1, z), (1, nz), (-1, z), (-1, nz), (z, 1), (nz, 1), (z, -1), (nz, -1), (z, z), (nz, nz), (nz, z), (z, nz),
              (0.5, z), (0.5, nz), (-0.25, z), (z, -0.75)]
        return np.array(px, np.float32).reshape(4, 4, 2)
    raise KeyError(name)


def branch_cases():
    """The first N_BRANCH seeded 16x24 flows (N(0,1) * 3) in which some pixel's normalised radius rounds above 1."""
    from oracle import viz_oracle
    out = []
    for s in BRANCH_SEEDS:
        f = _random(16, 24, s, 3.0)
        if viz_oracle.branch_mask(f).any():
            out.append(f"branch_{s}")
            if len(out) == N_BRANCH:
                break
    return out


def case_input(name, npz=None):
    if name in RANDOM:
        return _random(*RANDOM[name])
    if name.startswith("branch_"):
        return _random(16, 24, int(name[7:]), 3.0)
    if npz is not None:
        return npz[f"{name}_in"]
    return _hand(name)


def main():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(REF, "core"))
    from utils import flow_viz as ref_viz   # the reference's module
    from numpy._core import _multiarray_umath as mu
    from oracle import viz_oracle

    names = list(RANDOM) + list(HAND) + branch_cases()
    arrays, diff = {}, {}
    for name in names:
        f = case_input(name)
        if name in HAND:
            arrays[f"{name}_in"] = f
        ref = ref_viz.flow_to_image(f.copy())        # the reference zeroes unknown entries of its argument in place
        arrays[f"{name}_ref"] = ref
        arrays[f"{name}_branch"] = viz_oracle.branch_mask(f)
        diff[name] = int((ref != viz_oracle.flow_to_image(f)).sum())
    np.savez_compressed(os.path.join(OUT, "viz.npz"), **arrays)
    meta = {
        "numpy": np.__version__,
        "cpu_baseline": list(mu.__cpu_baseline__),
        "cpu_dispatch": [d for d in mu.__cpu_dispatch__ if mu.__cpu_features__.get(d)],
        "cases": names,
        "branch_pixels": {n: int(arrays[f"{n}_branch"].sum()) for n in names},
        "oracle_channels_differing": diff,
    }
    with open(os.path.join(OUT, "viz_meta.json"), "w") as fh:
        json.dump(meta, fh, indent=1)
    print(json.dumps(meta))


if __name__ == "__main__":
    main()
