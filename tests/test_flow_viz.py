"""Flow visualisation and submission writers on the host: the numpy oracle of flow_to_image against the reference's own
output (tests/golden/viz.npz), rnc_flow_to_image's declaration and argument checks, the KITTI size grouping and the
writers' output layout with a stub model."""
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import viz_oracle
from oracle.make_golden_viz import case_input

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "raft-ncup_b200", "csrc")
GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def viz_gold():
    with open(os.path.join(GOLD, "viz_meta.json")) as f:
        meta = json.load(f)
    return meta, np.load(os.path.join(GOLD, "viz.npz"))


def exact_pixels(name, flow, npz):
    """Pixels the oracle must reproduce exactly: unknown, NaN, an all-zero image, and the > 1 branch pixels."""
    u, v = flow[..., 0], flow[..., 1]
    m = (np.abs(u) > 1e7) | (np.abs(v) > 1e7) | np.isnan(u) | np.isnan(v) | npz[f"{name}_branch"]
    return np.ones_like(m) if name == "zero" else m


def test_oracle_matches_the_reference_goldens(viz_gold):
    meta, npz = viz_gold
    assert len(meta["cases"]) >= 12 and sum(meta["branch_pixels"].values()) >= 3
    total = differ = 0
    for name in meta["cases"]:
        flow = case_input(name, npz)
        ref, got = npz[f"{name}_ref"], viz_oracle.flow_to_image(flow)
        assert got.shape == ref.shape == flow.shape[:2] + (3,) and got.dtype == np.uint8
        d = np.abs(got.astype(int) - ref.astype(int))
        assert d.max() <= 1, name
        ex = exact_pixels(name, flow, npz)
        assert np.array_equal(got[ex], ref[ex]), name
        assert np.array_equal(viz_oracle.branch_mask(flow), npz[f"{name}_branch"]), name
        total += d.size
        differ += int((d > 0).sum())
    assert differ <= 1e-4 * total, (differ, total)


def nan_quirk_pair():
    """(g, h, p): g has one NaN pixel p and radii below 0.9 elsewhere, so its maxrad is -1 and it is normalised by -1 + eps;
    h = -g with a radius-1 pixel at p, so it is normalised by 1 + eps.  The two normalised flows differ by 2 ulp, which no
    colour level resolves: the image of g is the image of h with p black."""
    g = np.random.default_rng(0).standard_normal((6, 7, 2)).astype(np.float32) * 0.2
    g = np.clip(g, -0.6, 0.6)
    h = -g
    g[3, 3] = (np.nan, 0.5)
    h[3, 3] = (0, 1)
    return g, h, (3, 3)


def test_oracle_quirks():
    """Unknown and NaN pixels are black; one NaN negates the rest (maxrad -1); -0 and +0 pick opposite wheel ends."""
    f = np.zeros((1, 2, 2), np.float32)
    f[0, 0] = (1, 0)
    f[0, 1] = (1, -0.0)
    img = viz_oracle.flow_to_image(f)
    assert not np.array_equal(img[0, 0], img[0, 1])
    g, h, p = nan_quirk_pair()
    want = viz_oracle.flow_to_image(h)
    want[p] = 0
    assert np.array_equal(viz_oracle.flow_to_image(g), want)
    g[2, 2] = (np.inf, 0)
    assert (viz_oracle.flow_to_image(g)[2, 2] == 0).all()


def test_entry_point_declared_and_bound():
    from rnc import native
    with open(os.path.join(ROOT, "include", "rnc.h")) as f:
        declared = set(re.findall(r"\b(rnc_\w+)\s*\(", f.read()))
    for n in ("rnc_flow_to_image", "rnc_flow_to_image_workspace_bytes"):
        assert n in declared and n in native.SIGNATURES, n
    assert native.ABI_VERSION == 18


def test_entry_point_rejects_bad_arguments():
    from rnc import native
    L = native.lib()
    ws = L.rnc_flow_to_image_workspace_bytes(3)
    assert ws >= 12 and L.rnc_flow_to_image_workspace_bytes(0) == 0 and L.rnc_flow_to_image_workspace_bytes(-1) == 0
    P = 1 << 20   # never dereferenced: every check fails on the host before a launch
    n0 = L.rnc_launch_count()

    def call(B=3, H=4, W=5, flow=P, out=P, wsp=P, wsb=ws):
        return L.rnc_flow_to_image(flow, 40, 20, 5, 1, B, H, W, out, wsp, wsb, None)

    assert call(B=0) == -1 and call(B=-2) == -1 and call(H=0) == -1 and call(W=-1) == -1
    assert call(flow=0) == -2 and call(out=0) == -2 and call(wsp=0) == -2
    assert call(flow=P + 2) == -2 and call(wsp=P + 1) == -2
    assert call(wsb=ws - 1) == -5
    assert L.rnc_launch_count() == n0


def test_cpu_tensors_raise():
    from rnc.native import RncUnavailable
    from rnc.viz import flow_to_image
    with pytest.raises(RncUnavailable):
        flow_to_image(torch.zeros(2, 4, 5))
    with pytest.raises(ValueError):
        flow_to_image(torch.zeros(1, 3, 4, 5))


def test_flow_viz_cu_does_not_spill(tmp_path):
    from rnc.build import ARCH, nvcc_path
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-c", os.path.join(CSRC, "flow_viz.cu"), "-o", str(tmp_path / "v.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    kernels = re.findall(r"Function properties for \S*(viz_\w+_kernel)", log)
    assert sorted(kernels) == ["viz_color_kernel", "viz_maxrad_kernel"], kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 2 and all(a == "0" and b == "0" for a, b in spills), spills
    assert all(f == "0" for f in re.findall(r"(\d+) bytes stack frame", log))


# ----------------------------------------------------------------------------- submission writers


@pytest.mark.parametrize("B", [1, 2, 3, 5])
def test_size_batches(B):
    from rnc.harness import size_batches
    g = np.random.default_rng(B)
    sizes = [[(375, 1242), (370, 1224), (376, 1241)][k] for k in g.integers(0, 3, 23)]
    batches = list(size_batches(range(len(sizes)), B, key=lambda i: sizes[i]))
    flat = [i for b in batches for i in b]
    assert sorted(flat) == list(range(len(sizes)))                      # each pair exactly once
    for b in batches:
        assert 1 <= len(b) <= B and len({sizes[i] for i in b}) == 1
    for s in set(sizes):                                                # first-appearance order within a size
        order = [i for i in flat if sizes[i] == s]
        assert order == sorted(order)
    with pytest.raises(ValueError):
        list(size_batches([1], 0, key=id))


class Stub(torch.nn.Module):
    """Flow = the first two channels of image1 - image2, at padded resolution."""

    def __init__(self):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))

    def forward(self, im1, im2, iters=12, test_mode=True, flow_init=None):
        flow = im1[:, :2] - im2[:, :2]
        return flow[:, :, ::8, ::8], flow


def test_kitti_writer_layout(tmp_path):
    pytest.importorskip("cv2")
    from rnc.harness import create_kitti_submission
    from utils.frame_utils import readFlowKITTI
    g = torch.Generator().manual_seed(0)
    sizes = [(20, 30), (21, 29), (20, 30), (17, 40), (21, 29), (20, 30), (17, 40)]
    pairs = [(f"{k:06d}_10.png", torch.randint(0, 200, (3, h, w), generator=g).float(),
              torch.randint(0, 200, (3, h, w), generator=g).float()) for k, (h, w) in enumerate(sizes)]
    out = str(tmp_path / "kitti")
    create_kitti_submission(Stub(), pairs, iters=1, output_path=out, batch_size=2)
    assert sorted(os.listdir(out)) == sorted(p[0] for p in pairs) and not os.path.exists(out + "_png")
    for fid, a, b in pairs:
        flow, valid = readFlowKITTI(os.path.join(out, fid))
        want = (a[:2] - b[:2]).permute(1, 2, 0).numpy()
        assert flow.shape == want.shape and np.array_equal(flow, want) and (valid == 1).all()


def fake_run_sequences(model, sequences, iters=32, warm_start=False, batch_size=8, device="cuda"):
    """run_sequences' yield order (sequence_schedule) on the host: the flow of pair k is frames[k + 1] - frames[k]."""
    from rnc.harness import sequence_schedule
    for step in sequence_schedule([len(s) for s in sequences], batch_size):
        for c in step:
            if not c.idle:
                yield c.seq, c.pair, sequences[c.seq][c.pair + 1][:2] - sequences[c.seq][c.pair][:2]


def test_sintel_writer_layout(tmp_path, monkeypatch):
    from rnc import harness
    from utils.frame_utils import readFlow
    monkeypatch.setattr(harness, "run_sequences", fake_run_sequences)
    g = torch.Generator().manual_seed(1)
    seqs = [(d, s, [torch.rand(3, 12, 16, generator=g) * 10 for _ in range(n)])
            for d in ("clean", "final") for s, n in (("alley_1", 3), ("ambush_3", 5), ("bamboo_2", 2))]
    out = str(tmp_path / "sintel")
    harness.create_sintel_submission(Stub(), seqs, iters=1, output_path=out, batch_size=2)
    assert sorted(os.listdir(out)) == ["clean", "final"] and not os.path.exists(out + "_png")
    for d, s, frames in seqs:
        names = sorted(os.listdir(os.path.join(out, d, s)))
        assert names == ["frame%04d.flo" % (k + 1) for k in range(len(frames) - 1)]
        for k in range(len(frames) - 1):
            want = (frames[k + 1][:2] - frames[k][:2]).permute(1, 2, 0).numpy()
            assert np.array_equal(readFlow(os.path.join(out, d, s, names[k])), want)


def test_writer_errors_raise_from_the_call(tmp_path, monkeypatch):
    from rnc import harness
    from utils import frame_utils
    monkeypatch.setattr(harness, "run_sequences", fake_run_sequences)
    seqs = [("clean", "a", [torch.zeros(3, 8, 8)] * 4)]

    def broken(path, flow):
        raise OSError(f"disk full writing {path}")
    monkeypatch.setattr(frame_utils, "writeFlow", broken)
    with pytest.raises(OSError, match="disk full"):
        harness.create_sintel_submission(Stub(), seqs, output_path=str(tmp_path / "s"), batch_size=1)
    monkeypatch.undo()
    monkeypatch.setattr(harness, "run_sequences", fake_run_sequences)
    blocker = tmp_path / "file"
    blocker.write_text("")
    with pytest.raises(OSError):
        harness.create_sintel_submission(Stub(), seqs, output_path=str(blocker), batch_size=1)
