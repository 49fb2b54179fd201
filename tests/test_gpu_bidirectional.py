"""Bidirectional inference on the GPU (rnc.harness.bidirectional_flow, model.forward_bidirectional): both directions equal
the two one-directional forwards (bit for bit with the exact lookup in deterministic mode, eager and graph-replayed, cold
and warm-started; within 1e-4 EPE by default, on both encoder routes), fnet and cnet encode each frame once,
rnc_fb_consistency equals host_fb_consistency bit for bit, and validate(consistency=True)."""
import math

import pytest
import torch

from conftest import build_model
from rnc.harness import bidirectional_flow, validate
from rnc.metrics import fb_consistency, host_fb_consistency
from rnc.synth import frames
from test_consistency import check_against_fp64, translation

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H, W, ITERS = 128, 256, 6


@pytest.fixture
def det(monkeypatch):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def inputs(B, seed=11):
    im1, im2 = frames(B, H, W, seed=seed)
    g = torch.Generator().manual_seed(seed)
    fw = torch.randn(B, 2, H // 8, W // 8, generator=g) * 2
    bw = torch.randn(B, 2, H // 8, W // 8, generator=g) * 2
    return im1.to(DEV), im2.to(DEV), fw.to(DEV), bw.to(DEV)


def separate(m, im1, im2, fi, conf=False):
    """The two one-directional forwards: ((low, up[, conf]) of im1 -> im2, the same of im2 -> im1)."""
    with torch.no_grad():
        a = m(im1, im2, iters=ITERS, flow_init=fi[0], test_mode=True, return_confidence=conf)
        b = m(im2, im1, iters=ITERS, flow_init=fi[1], test_mode=True, return_confidence=conf)
    return a, b


def both(m, im1, im2, fi, conf=False):
    with torch.no_grad():
        return bidirectional_flow(m, im1, im2, iters=ITERS, flow_init=fi if any(f is not None for f in fi) else None,
                                  return_confidence=conf)


def epe(a, b):
    return (a - b).pow(2).sum(1).sqrt().mean().item()


@pytest.mark.parametrize("warm", [None, "both", "fw"])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_bit_identical_to_two_forwards_with_the_exact_lookup(name, B, warm, det):
    m = build_model(name).to(DEV)
    im1, im2, fw, bw = inputs(B)
    fi = {None: (None, None), "both": (fw, bw), "fw": (fw, None)}[warm]
    (lo, up), (lo_b, up_b) = separate(m, im1, im2, fi)
    for call in range(3):       # eager, then captured and replayed, then replayed
        r = both(m, im1, im2, fi)
        for k, want in (("flow_low", lo), ("flow_up", up), ("flow_low_bw", lo_b), ("flow_up_bw", up_b)):
            assert torch.equal(r[k], want), f"call {call}: {k} differs, EPE {epe(r[k], want):.3e}"
    eng = m.engine()
    keys = list(eng._graphs)
    assert any(k[-1] == "bidirectional" and "graph" in eng._graphs[k] for k in keys), keys
    assert all(len(k) == 7 for k in keys if k[-1] != "bidirectional")       # the one-directional keys are unchanged


@pytest.mark.parametrize("route", ["umma", "cudnn"])
@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_default_mode_matches_two_forwards(name, route, monkeypatch):
    monkeypatch.setenv("RNC_ENCODER", route)
    m = build_model(name).to(DEV)
    im1, im2, fw, bw = inputs(3, seed=5)
    for fi in ((None, None), (fw, bw)):
        (lo, up), (lo_b, up_b) = separate(m, im1, im2, fi)
        for _ in range(2):
            r = both(m, im1, im2, fi)
            e = max(epe(r["flow_up"], up), epe(r["flow_up_bw"], up_b), epe(r["flow_low"], lo), epe(r["flow_low_bw"], lo_b))
            print(f"{name} {route} warm={fi[0] is not None}: worst EPE vs two forwards {e:.2e}")
            assert e <= 1e-4


def test_fnet_and_cnet_encode_each_frame_once(monkeypatch):
    from rnc.encoder_umma import EncoderRunner
    m = build_model("raft_nc_dbl").to(DEV)
    if m.engine().mode != "umma":
        pytest.skip("tensor-core encoders only")
    monkeypatch.setenv("RNC_GRAPH", "0")            # count eager passes
    images = {"instance": 0, "batch": 0}
    trunk = EncoderRunner._trunk

    def counted(self, pk, bufs, image, N, Hin, Win):
        assert image.shape[0] == N
        images[pk.kind] += N
        return trunk(self, pk, bufs, image, N, Hin, Win)

    monkeypatch.setattr(EncoderRunner, "_trunk", counted)
    B = 3
    im1, im2, _, _ = inputs(B)
    both(m, im1, im2, (None, None))
    assert images == {"instance": 2 * B, "batch": 2 * B}, images


def test_inference_only():
    m = build_model("raft").to(DEV)
    im1, im2, _, _ = inputs(1)
    with pytest.raises(ValueError, match="forward_bidirectional"):
        bidirectional_flow(m, im1, im2, iters=1)
    with torch.no_grad(), pytest.raises(ValueError, match="return_confidence"):
        bidirectional_flow(m, im1, im2, iters=1, return_confidence=True)


@pytest.mark.parametrize("B", [1, 3])
def test_confidence_equals_the_one_directional_confidence(B, det):
    m = build_model("raft_nc_dbl").to(DEV)
    im1, im2, fw, bw = inputs(B, seed=3)
    for fi in ((None, None), (fw, bw)):
        (_, up, c), (_, up_b, c_b) = separate(m, im1, im2, fi, conf=True)
        for _ in range(3):
            r = both(m, im1, im2, fi, conf=True)
            assert torch.equal(r["flow_up"], up) and torch.equal(r["flow_up_bw"], up_b)
            assert torch.equal(r["confidence"], c) and torch.equal(r["confidence_bw"], c_b)


def test_confidence_in_the_default_mode():
    m = build_model("raft_nc_dbl").to(DEV)
    im1, im2, fw, bw = inputs(3, seed=3)
    (_, up, c), (_, up_b, c_b) = separate(m, im1, im2, (None, None), conf=True)
    r = both(m, im1, im2, (None, None), conf=True)
    d = max((r["confidence"] - c).abs().max().item(), (r["confidence_bw"] - c_b).abs().max().item())
    print(f"default mode: largest confidence difference {d:.2e}")
    assert epe(r["flow_up"], up) <= 1e-4 and epe(r["flow_up_bw"], up_b) <= 1e-4 and d <= 1e-3


# ----------------------------------------------------------------------------- rnc_fb_consistency


def random_pair(B, h, w, seed, scale=4.0):
    g = torch.Generator().manual_seed(seed)
    fw = torch.randn(B, 2, h, w, generator=g) * scale
    bw = -fw + torch.randn(B, 2, h, w, generator=g) * scale / 4
    fw.view(-1)[torch.randint(0, fw.numel(), (5,), generator=g)] = float("nan")
    bw.view(-1)[torch.randint(0, bw.numel(), (5,), generator=g)] = float("nan")
    return fw, bw


def assert_same(got, want):
    for k, (x, y) in enumerate(zip(got, want)):
        x = x.cpu()
        assert x.dtype == y.dtype and x.shape == y.shape, k
        assert torch.equal(x.view(torch.uint8) if x.dtype == torch.float32 else x,
                           y.view(torch.uint8) if y.dtype == torch.float32 else y), \
            f"output {k}: {int((x != y).sum())} pixels differ"


@pytest.mark.parametrize("B,h,w", [(3, 23, 37), (2, 436, 1024), (1, 1, 1), (2, 5, 1)])
def test_kernel_equals_the_host_bit_for_bit(B, h, w):
    fw, bw = random_pair(B, h, w, seed=h * w)
    got = fb_consistency(fw.to(DEV), bw.to(DEV))
    assert_same(got, host_fb_consistency(fw, bw))
    assert_same(fb_consistency(fw.to(DEV), bw.to(DEV), 0.05, 0.1), host_fb_consistency(fw, bw, 0.05, 0.1))


def test_strided_unpadded_views():
    fw, bw = random_pair(3, 48, 72, seed=9)
    big_f = fw.to(DEV).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)        # channel-last strides
    big_b = bw.to(DEV)
    vf, vb = big_f[:, :, 4:44, 5:70], big_b.flip(0)[:, :, 3:43, 1:66]
    assert_same(fb_consistency(vf, vb), host_fb_consistency(vf.cpu(), vb.cpu()))


def test_translation_at_sintel_size_against_fp64():
    fw, bw = translation(2, 436, 1024, (37.75, -11.5))
    got = fb_consistency(fw.to(DEV), bw.to(DEV))
    assert_same(got, host_fb_consistency(fw, bw))
    check_against_fp64(fw, bw, "translation 436x1024 (kernel)", got=got)
    fw2, bw2 = random_pair(2, 436, 1024, seed=4, scale=20.0)
    fw2, bw2 = torch.nan_to_num(fw2), torch.nan_to_num(bw2)
    check_against_fp64(fw2, bw2, "random 436x1024 (kernel)", got=fb_consistency(fw2.to(DEV), bw2.to(DEV)))


def test_repeats_and_does_not_depend_on_the_batch():
    fw, bw = random_pair(8, 100, 131, seed=2)
    fw, bw = fw.to(DEV), bw.to(DEV)
    a = fb_consistency(fw, bw)
    b = fb_consistency(fw, bw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    for k in (0, 3, 7):
        one = fb_consistency(fw[k:k + 1], bw[k:k + 1])
        assert all(torch.equal(x[0], y[k]) for x, y in zip(one, a)), k


def test_cuda_arguments_are_checked():
    f = torch.zeros(2, 2, 4, 5, device=DEV)
    with pytest.raises(ValueError):
        fb_consistency(f, f.cpu())
    with pytest.raises(ValueError):
        fb_consistency(f, torch.zeros(2, 2, 4, 6, device=DEV))


# ----------------------------------------------------------------------------- validate(consistency=True)


def synthetic_samples(n=5, h=100, w=180):
    im1, im2 = frames(n, h, w, seed=21)
    g = torch.Generator().manual_seed(22)
    gt = torch.randn(n, 2, h, w, generator=g) * 2
    return [(im1[i], im2[i], gt[i]) for i in range(n)]


def test_validate_consistency_keeps_the_other_keys_bit_for_bit(det):
    m = build_model("raft_nc_dbl").to(DEV)
    samples = synthetic_samples()
    plain = validate(m, samples, iters=2, batch_size=2)
    res = validate(m, samples, iters=2, batch_size=2, consistency=True)
    assert set(res) == set(plain) | {"fb_sparsification", "ideal", "fb_ause"}
    assert {k: res[k] for k in plain} == plain
    assert math.isfinite(res["fb_ause"]) and res["fb_ause"] >= 0
    conf = validate(m, samples, iters=2, batch_size=2, confidence=True)
    res2 = validate(m, samples, iters=2, batch_size=2, confidence=True, consistency=True)
    assert {k: res2[k] for k in conf} == conf                # with confidence too: its keys, bit for bit
    assert res2["fb_sparsification"] == res["fb_sparsification"] and res2["fb_ause"] == res["fb_ause"]
    # nothing is removed at k = 0 whatever the score: the same pixels, summed in the two scores' orders
    assert res2["fb_sparsification"][0] == pytest.approx(res2["sparsification"][0], rel=1e-12)
    print(f"AUSE: NCUP confidence {res2['ause']:.4f}, forward-backward consistency {res2['fb_ause']:.4f}")


def test_validate_consistency_in_the_default_mode():
    m = build_model("raft").to(DEV)
    samples = synthetic_samples(3)
    plain = validate(m, samples, iters=2, batch_size=3)
    res = validate(m, samples, iters=2, batch_size=3, consistency=True)
    print("default mode, bit-equal keys:", {k: res[k] == plain[k] for k in plain})
    for k in plain:
        assert res[k] == pytest.approx(plain[k], rel=1e-4, abs=1e-6), k
    assert math.isfinite(res["fb_ause"]) and res["fb_ause"] >= 0
