"""Validation metrics on the host: summarize on hand-built partials, the host partials against the reference's formulas at the
edges (zero-magnitude ground truth, an image without a valid pixel, values on the thresholds), validate under gloo at world
sizes 2 and 3 against world 1, the sequence and pair assignment of the submission writers, and rnc_flow_metrics' argument
checks."""
import math
import os
import re
import socket
import subprocess

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "raft-ncup_b200", "csrc")


def reference_metrics(flows, gts, valids):
    """evaluate.py:126-137 (no valid) and :160-179 (valid) over lists of [2,H,W] flows and ground truths, as the host loop
    validate() ran before: float32 EPEs pooled in numpy."""
    epe_all, f1_all, epe_img = [], [], []
    for flow, gt, valid in zip(flows, gts, valids):
        epe = torch.sum((flow - gt) ** 2, dim=0).sqrt()
        if valid is None:
            epe_all.append(epe.view(-1).numpy())
        else:
            mag = torch.sum(gt ** 2, dim=0).sqrt().view(-1)
            val = valid.view(-1) >= 0.5
            e = epe.view(-1)
            out = ((e > 3.0) & ((e / mag) > 0.05)).float()
            epe_img.append(e[val].mean().item())
            epe_all.append(e[val].numpy())
            f1_all.append(out[val].numpy())
    e = np.concatenate(epe_all)
    with np.errstate(invalid="ignore"):
        res = {"epe": float(np.mean(e)), "1px": float(np.mean(e < 1)), "3px": float(np.mean(e < 3)),
               "5px": float(np.mean(e < 5))}
        if f1_all:
            res["epe"] = float(np.mean(epe_img))
            res["f1"] = float(100 * np.mean(np.concatenate(f1_all)))
    return res


def assert_matches_reference(got, want):
    assert got.keys() == want.keys()
    for k in ("1px", "3px", "5px"):
        assert got[k] == want[k], (k, got[k], want[k])
    if "f1" in want:                                     # the reference rounds the outlier fraction to float32
        assert got["f1"] == pytest.approx(want["f1"], rel=1e-6, abs=0), (got["f1"], want["f1"])
    if math.isnan(want["epe"]):
        assert math.isnan(got["epe"])
    else:
        assert got["epe"] == pytest.approx(want["epe"], rel=1e-6, abs=0), (got["epe"], want["epe"])


def test_summarize_hand_built_partials():
    from rnc.metrics import Partials, summarize
    counts = torch.tensor([[10, 4, 7, 9, 2], [6, 6, 6, 6, 0], [0, 0, 0, 0, 0]], dtype=torch.int64)
    sums = torch.tensor([25.0, 3.0, 0.0], dtype=torch.float64)
    s = summarize(Partials(counts, sums), "sintel")
    assert list(s) == ["epe", "1px", "3px", "5px"]
    assert s == {"epe": 28.0 / 16, "1px": 10 / 16, "3px": 13 / 16, "5px": 15 / 16}
    assert summarize(Partials(counts, sums), "chairs") == s
    k = summarize(Partials(counts[:2], sums[:2]), "kitti")
    assert k == {"epe": (2.5 + 0.5) / 2, "1px": 10 / 16, "3px": 13 / 16, "5px": 15 / 16, "f1": 100 * 2 / 16}
    kn = summarize(Partials(counts, sums), "kitti")              # an image with no valid pixel: NaN, as in the reference
    assert math.isnan(kn["epe"]) and kn["f1"] == k["f1"]
    empty = summarize(Partials(counts[2:], sums[2:]), "sintel")
    assert all(math.isnan(v) for v in empty.values())
    with pytest.raises(ValueError):
        summarize(Partials(counts, sums), "things")


def edge_case():
    """Two 4x6 images: the first has exact threshold values and zero-magnitude ground truth, the second no valid pixel."""
    gt = torch.zeros(2, 2, 4, 6)
    flow = torch.zeros(2, 2, 4, 6)
    cases = [((3, 0), (0, 0)),       # epe == 3: < 5 but not < 3 and not an outlier (epe > 3)
             ((1, 0), (0, 0)),       # epe == 1: not < 1
             ((5, 0), (0, 0)),       # epe == 5: not < 5; an outlier (5 / 0 = inf)
             ((84, 0), (80, 0)),     # epe 4, epe / mag == 0.05f: not an outlier
             ((83.99, 0), (79.99, 0)),   # epe / mag just above 0.05f: an outlier
             ((4, 0), (0, 0)),       # zero-magnitude gt: epe / 0 = inf, an outlier
             ((0, 0), (0, 0)),       # 0 / 0 = NaN: not an outlier
             ((0, 3.0000002), (0, 0)),   # just above 3, mag 0: an outlier
             ((-2.5, 1.5), (0.5, -2.5))]   # epe 5 with a 3-4-5 triangle
    for i, (f, g) in enumerate(cases):
        y, x = divmod(i, 6)
        flow[0, :, y, x] = torch.tensor(f)
        gt[0, :, y, x] = torch.tensor(g)
    flow[1] = torch.randn(2, 4, 6, generator=torch.Generator().manual_seed(0)) * 4
    valid = torch.ones(2, 4, 6)
    valid[0, 3, 5] = 0.4999                    # below 0.5: invalid
    valid[0, 3, 4] = 0.5                       # exactly 0.5: valid
    valid[1] = 0
    return flow, gt, valid


def test_host_partials_at_the_edges():
    from rnc.metrics import host_partials, summarize
    flow, gt, valid = edge_case()
    p = host_partials(flow, gt, valid)
    assert p.counts.dtype == torch.int64 and p.epe_sum.dtype == torch.float64
    assert p.counts[1].tolist() == [0, 0, 0, 0, 0] and p.epe_sum[1].item() == 0.0
    assert p.counts[0, 0].item() == 23
    want = reference_metrics(list(flow), list(gt), list(valid))
    got = summarize(p, "kitti")
    assert math.isnan(want["epe"]) and math.isnan(got["epe"])
    assert_matches_reference(got, want)
    first = summarize(host_partials(flow[:1], gt[:1], valid[:1]), "kitti")
    assert_matches_reference(first, reference_metrics([flow[0]], [gt[0]], [valid[0]]))
    assert_matches_reference(summarize(host_partials(flow, gt), "sintel"), reference_metrics(list(flow), list(gt), [None] * 2))
    # the threshold pixels, one by one: epe 3, 1, 5, the two 0.05 ratios, 4 / 0, 0 / 0, 3+ / 0, the 3-4-5 triangle
    per = [host_partials(flow[:1, :, i // 6:i // 6 + 1, i % 6:i % 6 + 1], gt[:1, :, i // 6:i // 6 + 1, i % 6:i % 6 + 1]).counts[0]
           for i in range(9)]
    assert [c[1:].tolist() for c in per] == [[0, 0, 1, 0], [0, 1, 1, 0], [0, 0, 0, 1], [0, 0, 1, 0], [0, 0, 1, 1],
                                             [0, 0, 1, 1], [1, 1, 1, 0], [0, 0, 1, 1], [0, 0, 0, 1]]


def test_host_partials_round_as_ieee_float32():
    """Every pixel's EPE is numpy's float32 chain bit for bit, whatever torch's CPU sqrt rounds to on this machine."""
    from rnc.metrics import host_partials
    g = np.random.default_rng(8)
    f, t = (g.standard_normal((20000, 2, 1, 1)) * 6).astype(np.float32), (g.standard_normal((20000, 2, 1, 1)) * 6).astype(np.float32)
    d = f - t
    want = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]).ravel()
    assert want.dtype == np.float32
    p = host_partials(torch.from_numpy(f), torch.from_numpy(t))
    assert np.array_equal(p.epe_sum.numpy(), want.astype(np.float64))


def test_host_partials_with_nan_and_inf():
    from rnc.metrics import host_partials, summarize
    g = torch.Generator().manual_seed(3)
    flow, gt = torch.randn(3, 2, 9, 11, generator=g) * 4, torch.randn(3, 2, 9, 11, generator=g) * 4
    valid = (torch.rand(3, 9, 11, generator=g) > 0.3).float()
    flow[0, 0, 2, 3] = float("inf")
    valid[0, 2, 3] = 1
    flow[2, 1, 4, 4] = float("nan")
    valid[2, 4, 4] = 1
    p = host_partials(flow, gt, valid)
    assert math.isinf(p.epe_sum[0].item()) and math.isnan(p.epe_sum[2].item()) and math.isfinite(p.epe_sum[1].item())
    want = reference_metrics(list(flow), list(gt), list(valid))
    got = summarize(p, "kitti")
    for k in ("1px", "3px", "5px", "f1"):
        assert got[k] == pytest.approx(want[k], rel=1e-6, abs=0), k
    assert math.isnan(got["epe"]) and math.isnan(want["epe"])


def test_flow_metrics_checks_shapes():
    from rnc.metrics import flow_metrics
    with pytest.raises(ValueError):
        flow_metrics(torch.zeros(1, 3, 4, 5), torch.zeros(1, 3, 4, 5))
    with pytest.raises(ValueError):
        flow_metrics(torch.zeros(1, 2, 4, 5), torch.zeros(1, 2, 4, 6))
    with pytest.raises(ValueError):
        flow_metrics(torch.zeros(1, 2, 4, 5), torch.zeros(1, 2, 4, 5), torch.zeros(1, 5, 4))


class Stub(torch.nn.Module):
    """Flow = the first two channels of image1 - image2, at padded resolution; its parameter puts it on the CPU."""

    def __init__(self):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))

    def forward(self, im1, im2, iters=12, test_mode=True, flow_init=None):
        flow = im1[:, :2] - im2[:, :2]
        return flow[:, :, ::8, ::8], flow


def stub_samples(sparse):
    """11 samples, a different frame size in the middle (a KITTI-style mix of sizes)."""
    g = torch.Generator().manual_seed(7 + sparse)
    out = []
    for k in range(11):
        h, w = (20, 30) if k not in (4, 5) else (17, 41)
        a, b = torch.rand(3, h, w, generator=g) * 6, torch.rand(3, h, w, generator=g) * 6
        gt = (a[:2] - b[:2]) + torch.randn(2, h, w, generator=g) * (1 + k)
        if sparse:
            out.append((a, b, gt, (torch.rand(h, w, generator=g) > 0.2 + 0.05 * k).float()))
        else:
            out.append((a, b, gt))
    return out


@pytest.mark.parametrize("sparse", [False, True])
def test_validate_equals_the_reference_loop(sparse):
    from rnc.harness import validate
    samples = stub_samples(sparse)
    flows = [a[:2] - b[:2] for a, b, *_ in samples]
    want = reference_metrics(flows, [s[2] for s in samples], [s[3] if sparse else None for s in samples])
    for bs in (1, 3, 8):
        res = validate(Stub(), samples, iters=1, mode="kitti" if sparse else "sintel", batch_size=bs, device="cpu")
        assert_matches_reference(res, want)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _validate_worker(rank, world, port, sparse, as_iterator, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from rnc.harness import validate
        samples = stub_samples(sparse)
        res = validate(Stub(), iter(samples) if as_iterator else samples, iters=1, batch_size=3, device="cpu")
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def run_ranks(target, world, *args, timeout=180):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, *args, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = sorted((q.get(timeout=timeout) for _ in range(world)), key=lambda t: t[0])
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    return [r[1] for r in res]


@pytest.mark.parametrize("world,sparse,as_iterator", [(2, True, False), (3, False, True), (3, True, True)])
def test_validate_gloo_equals_world_1(world, sparse, as_iterator):
    from rnc.harness import validate
    want = validate(Stub(), stub_samples(sparse), iters=1, batch_size=3, device="cpu")
    for got in run_ranks(_validate_worker, world, sparse, as_iterator):
        assert got == want                                  # bit for bit, on every rank


def test_strided_items_and_gather():
    from rnc.dist import gather_strided, strided_items
    for n in (0, 1, 5, 12):
        for world in (1, 2, 3, 5):
            shares = [list(strided_items(list(range(n)), world, r)) for r in range(world)]
            walked = [list(strided_items(iter(range(n)), world, r)) for r in range(world)]
            assert shares == walked
            assert sorted(i for s in shares for i in s) == list(range(n))
            assert all(i % world == r for r, s in enumerate(shares) for i in s)
    assert gather_strided([1, 2], 1) == [1, 2]
    with pytest.raises(ValueError):
        strided_items([], 2, 2)


def test_greedy_assignment():
    from rnc.dist import greedy_assignment
    g = np.random.default_rng(5)
    for world in (1, 2, 3, 8):
        sizes = [int(x) for x in g.integers(0, 50, 23)]
        owner = greedy_assignment(sizes, world)
        assert owner == greedy_assignment(list(sizes), world)          # deterministic
        assert len(owner) == len(sizes) and set(owner) <= set(range(world))
        load = [sum(s for s, o in zip(sizes, owner) if o == r) for r in range(world)]
        assert max(load) - min(load) <= max(sizes)                       # longest-first greedy bound
    assert greedy_assignment([1, 5, 5, 2], 2) == [1, 0, 1, 0]
    assert greedy_assignment([], 3) == []


def _fake_run_sequences(model, sequences, iters=32, warm_start=False, batch_size=8, device="cuda"):
    from rnc.harness import sequence_schedule
    for step in sequence_schedule([len(s) for s in sequences], batch_size):
        for c in step:
            if not c.idle:
                yield c.seq, c.pair, sequences[c.seq][c.pair + 1][:2] - sequences[c.seq][c.pair][:2]


def writer_inputs():
    g = torch.Generator().manual_seed(2)
    seqs = [(d, s, [torch.rand(3, 12, 16, generator=g) * 10 for _ in range(n)])
            for d in ("clean", "final") for s, n in (("alley_1", 3), ("ambush_3", 6), ("bamboo_2", 2), ("cave_4", 4))]
    pairs = [(f"{k:06d}_10.png", torch.rand(3, 20, 30, generator=g) * 200, torch.rand(3, 20, 30, generator=g) * 200)
             for k in range(7)]
    return seqs, pairs


def _writer_worker(rank, world, port, out, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from rnc import harness
        harness.run_sequences = _fake_run_sequences
        seqs, pairs = writer_inputs()
        harness.create_sintel_submission(Stub(), seqs, iters=1, output_path=os.path.join(out, "sintel"), batch_size=2)
        harness.create_kitti_submission(Stub(), pairs, iters=1, output_path=os.path.join(out, "kitti"), batch_size=2)
        # the writers end with a barrier: every rank's files exist when any rank returns
        q.put((rank, sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs)))
    finally:
        dist.destroy_process_group()


def test_submission_writers_gloo_write_the_world_1_files(tmp_path, monkeypatch):
    pytest.importorskip("cv2")
    from rnc import harness
    monkeypatch.setattr(harness, "run_sequences", _fake_run_sequences)
    seqs, pairs = writer_inputs()
    one = str(tmp_path / "one")
    harness.create_sintel_submission(Stub(), seqs, iters=1, output_path=os.path.join(one, "sintel"), batch_size=2)
    harness.create_kitti_submission(Stub(), pairs, iters=1, output_path=os.path.join(one, "kitti"), batch_size=2)
    names = sorted(os.path.relpath(os.path.join(d, f), one) for d, _, fs in os.walk(one) for f in fs)
    assert len(names) == 2 * (2 + 5 + 1 + 3) + 7
    two = str(tmp_path / "two")
    for listed in run_ranks(_writer_worker, 2, two):
        assert listed == names
    for n in names:
        with open(os.path.join(one, n), "rb") as a, open(os.path.join(two, n), "rb") as b:
            assert a.read() == b.read(), n


# ----------------------------------------------------------------------------- C ABI


def test_entry_point_declared_and_bound():
    from rnc import native
    with open(os.path.join(ROOT, "include", "rnc.h")) as f:
        declared = set(re.findall(r"\b(rnc_\w+)\s*\(", f.read()))
    for n in ("rnc_flow_metrics", "rnc_flow_metrics_workspace_bytes"):
        assert n in declared and n in native.SIGNATURES, n


def test_entry_point_rejects_bad_arguments():
    from rnc import native
    L = native.lib()
    ws = L.rnc_flow_metrics_workspace_bytes(3, 436, 1024)
    assert ws == 3 * 218 * 32 and L.rnc_flow_metrics_workspace_bytes(3, 1, 1) == 3 * 32
    assert L.rnc_flow_metrics_workspace_bytes(0, 4, 5) == 0 and L.rnc_flow_metrics_workspace_bytes(2, -1, 5) == 0
    assert L.rnc_flow_metrics_workspace_bytes(65536, 4, 5) == 0 and L.rnc_flow_metrics_workspace_bytes(1, 1 << 15, 1 << 15) == 0
    P = 1 << 20   # never dereferenced: every check fails on the host before a launch
    n0 = L.rnc_launch_count()

    def call(B=3, H=436, W=1024, flow=P, gt=P, valid=P, counts=P, sums=P, wsp=P, wsb=ws):
        return L.rnc_flow_metrics(flow, 40, 20, 5, 1, gt, 40, 20, 5, 1, valid, 20, 5, 1, B, H, W, counts, sums, wsp, wsb, None)

    assert call(B=0) == -1 and call(B=-2) == -1 and call(H=0) == -1 and call(W=-1) == -1 and call(B=65536) == -1
    assert call(H=1 << 15, W=1 << 15) == -1
    assert call(flow=0) == -2 and call(gt=0) == -2 and call(counts=0) == -2 and call(sums=0) == -2 and call(wsp=0) == -2
    assert call(flow=P + 2) == -2 and call(gt=P + 1) == -2 and call(valid=P + 2) == -2
    assert call(counts=P + 4) == -2 and call(sums=P + 4) == -2 and call(wsp=P + 8) == -2
    assert call(wsb=ws - 1) == -5 and call(valid=0, wsb=0) == -5
    assert L.rnc_launch_count() == n0


def test_cpu_tensors_take_the_host_path():
    from rnc.metrics import flow_metrics, host_partials
    flow, gt, valid = edge_case()
    a, b = flow_metrics(flow, gt, valid), host_partials(flow, gt, valid)
    assert torch.equal(a.counts, b.counts) and torch.equal(a.epe_sum, b.epe_sum)


def test_flow_metrics_cu_does_not_spill(tmp_path):
    from rnc.build import ARCH, nvcc_path
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-I",
           os.path.join(ROOT, "include"), "-I", CSRC, "-c", os.path.join(CSRC, "flow_metrics.cu"), "-o", str(tmp_path / "m.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    kernels = re.findall(r"Function properties for \S*?\d((?:cta|image)_[a-z_]+_kernel)", log)
    assert sorted(kernels) == ["cta_partials_kernel", "image_reduce_kernel"], kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 2 and all(a == "0" and b == "0" for a, b in spills), spills
