"""GPU augmentation (rnc/augment.py, csrc/augment.cu), CPU side: the host draws against the reference's recorded parameters
and RNG states (tests/golden/aug_meta.json, oracle/make_golden_aug.py), argument checks of the entry points, and a
spill-free sm_90a build of augment.cu."""
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle.make_golden_aug import STAGES, rng_digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "raft-ncup_b200", "csrc")
with open(os.path.join(ROOT, "tests", "golden", "aug_meta.json")) as _f:
    META = json.load(_f)


def augmentor(stage):
    from rnc import augment
    sparse, params, _ = STAGES[stage]
    return (augment.SparseFlowAugmentor if sparse else augment.FlowAugmentor)(**params)


@pytest.mark.parametrize("i", range(len(META["samples"])))
def test_draws_match_reference(i):
    s = META["samples"][i]
    np.random.seed(s["seed"])
    torch.manual_seed(s["seed"])
    d = augmentor(s["stage"]).draw(s["H"], s["W"])
    assert json.loads(json.dumps(d)) == s["draw"]
    assert rng_digest() == s["rng"], "the draws consumed np.random / torch differently from the reference"
    assert s["shape"][1:] == list(STAGES[s["stage"]][1]["crop_size"])


def test_golden_covers_every_branch():
    seen = set()
    for s in META["samples"]:
        seen |= set(s["coverage"])
    assert {"asym", "sym", "erase0", "erase1", "erase2", "erase_clipped", "resized", "not_resized", "stretch", "hflip",
            "vflip", "sparse_downscale"} <= seen


def _desc(H=40, W=60, **kw):
    from rnc import native
    d = native.AugDesc()
    d.H, d.W, d.rh, d.rw = H, W, H, W
    d.img1, d.img2, d.flow, d.valid = 0, 3 * H * W, 6 * H * W, 14 * H * W
    for p in range(2):
        for j in range(4):
            d.perm[p][j] = j
        for j in range(3):
            d.factor[p][j] = 1.0
    d.fx = d.fy = d.ifx = d.ify = 1.0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_entry_points_reject_bad_arguments():
    from rnc import native
    L = native.lib()
    H, W, ch, cw = 40, 60, 32, 48
    src_bytes = 18 * H * W
    ws = L.rnc_augment_workspace_bytes(1, ch, cw, 1)
    assert ws >= ch * cw * 4 and L.rnc_augment_workspace_bytes(0, ch, cw, 1) == 0
    assert L.rnc_augment_workspace_bytes(2, ch, cw, 0) < L.rnc_augment_workspace_bytes(2, ch, cw, 1)
    P = 1 << 20   # never dereferenced: every check fails on the host before a launch

    def call(d, B=1, src=P, sb=src_bytes, crop=(ch, cw), sparse=1, out=P, wsp=P, wsb=ws):
        arr = (native.AugDesc * 1)(d)
        return L.rnc_augment(C.addressof(arr), P, B, src, sb, crop[0], crop[1], sparse, out, out, out, out, wsp, wsb, None)

    assert call(_desc(), B=0) == -1
    assert call(_desc(), crop=(0, cw)) == -1
    assert call(_desc(), sparse=2) == -1
    assert call(_desc(), src=0) == -2
    assert call(_desc(), out=0) == -2
    assert call(_desc(), wsp=P + 8) == -2
    assert call(_desc(), wsb=ws - 1) == -5
    assert call(_desc(H=0)) == -1
    assert call(_desc(), crop=(H + 1, cw)) == -1                  # crop larger than the image
    assert call(_desc(y0=H - ch + 1)) == -1                       # crop origin out of range
    assert call(_desc(rh=H + 4)) == -1                            # size change without a resize
    assert call(_desc(resized=1, rh=50, rw=70, fx=0.0)) == -1
    assert call(_desc(vflip=1)) == -1                             # sparse: no v-flip
    assert call(_desc(asym=1)) == -1                              # sparse: symmetric jitter only
    bad_perm = _desc()
    bad_perm.perm[0][3] = 0
    assert call(bad_perm) == -1
    assert call(_desc(n_erase=3)) == -1
    assert call(_desc(), sb=src_bytes - 1) == -1                  # valid plane past the end of src
    assert call(_desc(flow=6 * H * W + 2)) == -2                  # misaligned fp32 plane
    assert call(_desc(hue=(C.c_int * 2)(256, 0))) == -1


def test_augment_cu_does_not_spill(tmp_path):
    from rnc.build import ARCH, nvcc_path
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-c", os.path.join(CSRC, "augment.cu"), "-o", str(tmp_path / "a.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    kernels = re.findall(r"Function properties for \S*(aug_\w+_kernel)", log)
    assert sorted(kernels) == ["aug_contrast_stats_kernel", "aug_eraser_stats_kernel", "aug_gather_kernel",
                               "aug_sparse_scatter_kernel"], kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 4 and all(a == "0" and b == "0" for a, b in spills), spills
    frames = re.findall(r"(\d+) bytes stack frame", log)
    assert all(f == "0" for f in frames), frames
