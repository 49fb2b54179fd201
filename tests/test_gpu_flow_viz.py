"""Flow visualisation and submission writers on the GPU: rnc.viz.flow_to_image equals the numpy oracle bit for bit on every
golden case (and so keeps the oracle's bounds against the reference), in batches and on strided views, from run to run; the
drop-in utils.flow_viz; and the Sintel and KITTI writers byte for byte against the reference's one-pair-per-forward loop."""
import filecmp
import os

import numpy as np
import pytest
import torch

from conftest import build_model
from oracle import viz_oracle
from oracle.make_golden_viz import case_input
from test_flow_viz import exact_pixels, nan_quirk_pair, viz_gold  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def gpu(flow_hw2):
    from rnc.viz import flow_to_image
    out = flow_to_image(torch.from_numpy(np.ascontiguousarray(flow_hw2)).to(DEV).permute(2, 0, 1))
    return out.cpu().numpy()


def test_kernel_equals_oracle_on_every_golden_case(viz_gold):
    meta, npz = viz_gold
    total = differ = 0
    for name in meta["cases"]:
        flow = case_input(name, npz)
        got = gpu(flow)
        want = viz_oracle.flow_to_image(flow)
        assert got.dtype == np.uint8 and got.shape == want.shape
        bad = np.argwhere(got != want)
        assert not len(bad), f"{name}: {len(bad)} channels differ from the oracle, first {bad[:5].tolist()}"
        ref = npz[f"{name}_ref"]
        d = np.abs(got.astype(int) - ref.astype(int))
        ex = exact_pixels(name, flow, npz)
        assert d.max() <= 1 and np.array_equal(got[ex], ref[ex]), name
        total += d.size
        differ += int((d > 0).sum())
    assert differ <= 1e-4 * total


def test_batch_equals_single_launches_and_repeats():
    from rnc.viz import flow_to_image
    g = np.random.default_rng(11)
    flows = g.standard_normal((3, 37, 53, 2)).astype(np.float32) * np.float32([[[[3.0]]], [[[40.0]]], [[[0.5]]]])
    flows[1, 5, 7] = (np.nan, 1)
    flows[2, 9, 9] = (np.inf, 0)
    t = torch.from_numpy(flows).to(DEV).permute(0, 3, 1, 2)
    batch = flow_to_image(t)
    assert batch.shape == (3, 37, 53, 3) and batch.dtype == torch.uint8
    for b in range(3):
        assert torch.equal(batch[b], flow_to_image(t[b])), b
        assert np.array_equal(batch[b].cpu().numpy(), viz_oracle.flow_to_image(flows[b])), b
    big = torch.from_numpy(g.standard_normal((8, 2, 436, 1024)).astype(np.float32) * 8).to(DEV)
    assert torch.equal(flow_to_image(big), flow_to_image(big))


def test_unpadded_strided_view_equals_its_copy():
    from rnc.viz import flow_to_image
    from utils.utils import InputPadder
    padder = InputPadder((3, 436, 1022))
    flow_up = torch.randn(2, 2, 440, 1024, device=DEV) * 6
    view = padder.unpad(flow_up)
    assert not view.is_contiguous() and view.shape == (2, 2, 436, 1022)
    assert torch.equal(flow_to_image(view), flow_to_image(view.contiguous()))
    hw2 = view.permute(0, 2, 3, 1)                                  # channel-last storage, [B,2,H,W] view of it
    cl = hw2.contiguous().permute(0, 3, 1, 2)
    assert torch.equal(flow_to_image(cl), flow_to_image(view))
    assert torch.equal(flow_to_image(view.double()), flow_to_image(view))   # converted to float32 first


def test_one_nan_negates_the_flow():
    g, h, p = nan_quirk_pair()
    want = gpu(h)
    want[p] = 0
    assert np.array_equal(gpu(g), want)


def test_drop_in_equals_rnc_viz_and_leaves_its_argument(viz_gold):
    from utils import flow_viz
    _, npz = viz_gold
    for name in ("unknown", "rand_37x53", "axes"):
        flow = case_input(name, npz).copy()
        keep = flow.copy()
        img = flow_viz.flow_to_image(flow)
        assert img.dtype == np.uint8 and img.shape == flow.shape[:2] + (3,)
        assert np.array_equal(img, gpu(flow)) and np.array_equal(flow, keep, equal_nan=True), name


# ----------------------------------------------------------------------------- submission writers

ITERS = 6


@pytest.fixture
def det(monkeypatch):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def sintel_sequences():
    from rnc.synth import shift_sequence
    H, W = 92, 180                                  # padded to 96x184: the unpad view has offsets on both axes
    return [(d, f"scene_{s}", shift_sequence(n, H, W, seed=10 * s + (d == "final")))
            for d in ("clean", "final") for s, n in enumerate((2, 5, 3))]


def sintel_loop(m, seqs, out, warm):
    """evaluate.py:23-55, one pair per forward, with the drop-in's writeFlow, flow_viz and cv2.imwrite."""
    import cv2
    from utils import flow_viz, frame_utils
    from utils.utils import InputPadder, forward_interpolate
    with torch.no_grad():
        for dstype, scene, frames in seqs:
            flow_prev = None
            for k in range(len(frames) - 1):
                padder = InputPadder(frames[k].shape)
                im1, im2 = padder.pad(frames[k][None].to(DEV), frames[k + 1][None].to(DEV))
                flow_low, flow_pr = m(im1, im2, iters=ITERS, flow_init=flow_prev, test_mode=True)
                flow = padder.unpad(flow_pr[0]).permute(1, 2, 0).cpu().numpy()
                if warm:
                    flow_prev = forward_interpolate(flow_low[0])[None]
                for root in (out, out + "_png"):
                    os.makedirs(os.path.join(root, dstype, scene), exist_ok=True)
                cv2.imwrite(os.path.join(out + "_png", dstype, scene, "frame%04d.png" % (k + 1)), flow_viz.flow_to_image(flow))
                frame_utils.writeFlow(os.path.join(out, dstype, scene, "frame%04d.flo" % (k + 1)), flow)


def same_trees(a, b):
    names = sorted(os.path.relpath(os.path.join(d, f), a) for d, _, fs in os.walk(a) for f in fs)
    assert names == sorted(os.path.relpath(os.path.join(d, f), b) for d, _, fs in os.walk(b) for f in fs)
    _, mismatch, errors = filecmp.cmpfiles(a, b, names, shallow=False)
    assert not mismatch and not errors, (mismatch, errors)
    return names


@pytest.mark.parametrize("warm", [False, True])
def test_sintel_writer_bytes_equal_the_reference_loop(warm, det, tmp_path):
    pytest.importorskip("cv2")
    from rnc.harness import create_sintel_submission
    m = build_model("raft_nc_dbl").to(DEV)
    seqs = sintel_sequences()
    got, want = str(tmp_path / "got"), str(tmp_path / "want")
    create_sintel_submission(m, seqs, iters=ITERS, warm_start=warm, output_path=got, write_png=True, batch_size=2)
    sintel_loop(m, seqs, want, warm)
    names = same_trees(got, want) + same_trees(got + "_png", want + "_png")
    assert len(names) == 2 * 2 * (1 + 4 + 2)
    assert "clean/scene_1/frame0004.flo" in names and "final/scene_2/frame0002.png" in names


@pytest.mark.parametrize("warm", [False, True])
def test_sintel_writer_default_mode_flows(warm, tmp_path):
    from rnc.harness import create_sintel_submission
    from utils.frame_utils import readFlow
    m = build_model("raft_nc_dbl").to(DEV)
    seqs = sintel_sequences()
    got, want = str(tmp_path / "got"), str(tmp_path / "want")
    create_sintel_submission(m, seqs, iters=ITERS, warm_start=warm, output_path=got, batch_size=2)
    sintel_loop(m, seqs, want, warm)
    worst = 0.0
    for dstype, scene, frames in seqs:
        for k in range(len(frames) - 1):
            rel = os.path.join(dstype, scene, "frame%04d.flo" % (k + 1))
            a, b = readFlow(os.path.join(got, rel)), readFlow(os.path.join(want, rel))
            worst = max(worst, float(np.sqrt(((a - b) ** 2).sum(-1)).mean()))
    assert not os.path.exists(got + "_png")
    assert worst <= (1e-3 if warm else 1e-4), worst


def test_kitti_writer_bytes_equal_the_reference_loop(det, tmp_path):
    import cv2
    from rnc.harness import create_kitti_submission
    from rnc.synth import frames
    from utils import flow_viz, frame_utils
    from utils.utils import InputPadder
    m = build_model("raft_nc_dbl").to(DEV)
    sizes = [(90, 200), (75, 250), (90, 200), (84, 176), (75, 250), (90, 200), (84, 176)]
    pairs = []
    for k, (h, w) in enumerate(sizes):
        a, b = frames(1, h, w, seed=40 + k)
        pairs.append((f"{k:06d}_10.png", a[0], b[0]))
    got, want = str(tmp_path / "got"), str(tmp_path / "want")
    create_kitti_submission(m, pairs, iters=ITERS, output_path=got, write_png=True, batch_size=3)
    os.makedirs(want)
    os.makedirs(want + "_png")
    with torch.no_grad():                                            # evaluate.py:58-87
        for fid, a, b in pairs:
            padder = InputPadder(a.shape, mode="kitti")
            im1, im2 = padder.pad(a[None].to(DEV), b[None].to(DEV))
            _, flow_pr = m(im1, im2, iters=ITERS, test_mode=True)
            flow = padder.unpad(flow_pr[0]).permute(1, 2, 0).cpu().numpy()
            cv2.imwrite(os.path.join(want + "_png", fid + ".png"), flow_viz.flow_to_image(flow))
            frame_utils.writeFlowKITTI(os.path.join(want, fid), flow)
    assert same_trees(got, want) == sorted(p[0] for p in pairs)
    assert same_trees(got + "_png", want + "_png") == sorted(p[0] + ".png" for p in pairs)


def test_writer_error_raises_from_the_call(tmp_path):
    from rnc.harness import create_kitti_submission
    from rnc.synth import frames
    m = build_model("raft_nc_dbl").to(DEV)
    a, b = frames(1, 64, 96, seed=3)
    blocker = tmp_path / "not_a_dir"
    blocker.write_text("")
    with pytest.raises(OSError):
        create_kitti_submission(m, [("000000_10.png", a[0], b[0])], iters=2, output_path=str(blocker / "kitti"),
                                write_png=True)
