"""NCUP output confidence on the GPU: the fused kernels (rnc_ncup_fwd / rnc_ncup_train_fwd / rnc_ncup_bwd given conf_out /
g_conf_out) against fp64, the per-level chain of every other NConvUNet configuration, the model's test mode on both engines (eager,
graph replay, nn.DataParallel), the frozen-trunk and exact training routes against the reference's gradients
(tests/golden/conf.npz, oracle/make_golden_conf.py) and sequence inference."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, build_model, ref_args
from oracle import ncup_oracle as nco
from oracle import raft_oracle as orc
from oracle.make_golden_conf import conf_loss, tf_inputs
from oracle.make_golden_r2 import GRAD_ITERS, grad_fixture, train_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = ((2, 1, 5, 5), (2, 2, 5, 5), (2, 4, 3, 3), (1, 2, 1, 1))


def load_cfg1():
    return np.load(os.path.join(ROOT, "tests", "golden", "cfg1.npz"))


def load_conf():
    z = np.load(os.path.join(ROOT, "tests", "golden", "conf.npz"))
    with open(os.path.join(ROOT, "tests", "golden", "conf_meta.json")) as f:
        return {k: torch.from_numpy(z[k]) for k in z.files}, json.load(f)


def rel(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


def chain_inputs(B, H4, W4, seed):
    """Flow-like data, confidences in (0.01, 0.99) with ~30 % exact zeros, and weight_p of the four live layers."""
    g = torch.Generator().manual_seed(seed)
    x = 5 * torch.randn(B, 2, H4, W4, generator=g)
    c = torch.rand(B, 2, H4, W4, generator=g) * 0.98 + 0.01
    c[torch.rand(B, 2, H4, W4, generator=g) < 0.3] = 0.0
    wp = [0.3 * torch.randn(*s, generator=g) for s in SHAPES]
    return x, c, wp


def live_sd(wp, dtype, device):
    names = ("nconv_in", "nconv_x2.0", "decoder.0", "nconv_out")
    return {f"upsampler.interpolation_net.{n}.weight_p": w.to(device, dtype) for n, w in zip(names, wp)}


def chain64(x, c, wp, out_scale):
    """orc.nconv_unet_live in fp64 on zero-stuffed inputs: (out_scale * out, conf) [B,2,4H4,4W4]."""
    xh, ch = orc.zero_stuff(x), orc.zero_stuff(c)
    b, C, oh, ow = xh.shape
    y, k = orc.nconv_unet_live(live_sd(wp, x.dtype, x.device), xh.view(b * C, 1, oh, ow), ch.view(b * C, 1, oh, ow))
    return out_scale * y.view(b, C, oh, ow), k.view(b, C, oh, ow)


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------------- fused kernels


@pytest.mark.parametrize("B,H4,W4", [(8, 110, 256), (1, 22, 26)])
def test_ncup_fwd_conf_out_matches_fp64(B, H4, W4):
    """At the benchmark shape and at 22x26 (88x104 outputs: partial 30x30 tiles) with exact zero confidences.  The
    confidence is a chain of normalised non-negative averages: measured on an H100, 3.4e-8 (bench shape) and 1.5e-8 from
    fp64, against the 1e-5 bound."""
    from rnc import native
    L = native.lib()
    x, c, wp = chain_inputs(B, H4, W4, seed=B * 1000 + H4)
    xd, cd = x.to(DEV), c.to(DEV)
    ws = [F.softplus(w, beta=10) for w in wp]
    host = torch.cat([w.reshape(-1) for w in ws]).float()
    hw = (ctypes.c_float * 224)(*host.tolist())
    wdev = host.to(DEV)
    shape = (B, 2, 4 * H4, 4 * W4)
    out_ref, out, conf = (torch.empty(shape, device=DEV) for _ in range(3))
    out_t, conf_t = torch.empty(shape, device=DEV), torch.empty(shape, device=DEV)
    native.check(L.rnc_ncup_fwd(xd.data_ptr(), cd.data_ptr(), hw, B, H4, W4, 8.0, ctypes.c_void_p(out_ref.data_ptr()), None,
                                stream()))
    native.rnc.ncup_fwd(xd, cd, hw, B, H4, W4, 8.0, out, conf)
    native.rnc.ncup_train_fwd(xd, cd, wdev, B, H4, W4, 8.0, out_t, conf_t)
    torch.cuda.synchronize()
    o64, c64 = chain64(xd.double(), cd.double(), [w.to(DEV) for w in wp], 8.0)
    err = (conf.double() - c64).abs().max().item()
    print(f"conf {B}x{H4}x{W4}: worst |conf - fp64| {err:.2e}, conf in [{conf.min().item():.3f}, {conf.max().item():.3f}]")
    assert err <= 1e-5
    assert float(conf.min()) >= 0.0 and float(conf.max()) <= 1.0
    assert rel(out, o64) < 1e-5
    assert torch.equal(out, out_ref)
    assert torch.equal(out_t, out) and torch.equal(conf_t, conf)


@pytest.mark.parametrize("name", list(nco.CONFIGS))
def test_per_level_chain_confidence_matches_fp64(name):
    """The cout of rnc/nconv_unet.py's PackedUNet.run (the inference chain of every configuration but the shipped one)."""
    from rnc.modules import NConvUNet
    from rnc.nconv_unet import PackedUNet
    cfg = nco.CONFIGS[name]
    torch.manual_seed(5)
    net = NConvUNet(**nco.unet_kwargs(cfg)).to(DEV)
    x, c, _ = chain_inputs(2, 22, 26, seed=7)
    xh, ch = orc.zero_stuff(x).to(DEV), orc.zero_stuff(c).to(DEV)
    b, C, oh, ow = xh.shape
    xh, ch = xh.view(b * C, 1, oh, ow).contiguous(), ch.view(b * C, 1, oh, ow).contiguous()
    with torch.no_grad():
        _, conf = PackedUNet(net).run(xh, ch, 8.0)
    sd = {k: v.detach().double() for k, v in net.state_dict().items()}
    _, c64 = nco.unet(sd, cfg, xh.double(), ch.double())
    err = (conf.double() - c64).abs().max().item()
    print(f"{name}: worst |conf - fp64| {err:.2e}")
    assert err <= 1e-5 and float(conf.min()) >= 0.0 and float(conf.max()) <= 1.0


# ------------------------------------------------------------------------------------------------------- model, test mode


def variant_model(name):
    if name == "shipped":
        return build_model("raft_nc_dbl")
    import raft_nc_dbl
    a = ref_args("sintel")
    for k, v in nco.args_overrides(nco.CONFIGS[name]).items():
        setattr(a, k, v)
    torch.manual_seed(1234)
    return raft_nc_dbl.RAFT(a).eval()


@pytest.mark.parametrize("mode", ["umma", "ffma"])
def test_model_test_mode_confidence(mode, monkeypatch):
    monkeypatch.setenv("RNC_CONV", mode)
    g, _ = load_conf()
    # teacher-forced upsampler: the shipped (fused) network and the per-level `wide` one through the NConvUpsampler seam
    cfg1 = load_cfg1()
    flow_lr, guid = tf_inputs(cfg1)
    x4, guid = F.interpolate(flow_lr, scale_factor=2, mode="nearest").to(DEV), guid.to(DEV)
    for name in ("shipped", "wide"):
        m = variant_model(name).to(DEV)
        with torch.no_grad():
            out, conf = m.upsampler(x4, guid, return_confidence=True)
            out0 = m.upsampler(x4, guid)
        e = (conf.cpu() - g[f"tf_{name}_conf"]).abs().max().item()
        print(f"{mode} {name}: teacher-forced |conf - reference| {e:.2e}")
        assert e < 5e-5 and torch.equal(out, out0)
        assert float(conf.min()) >= 0.0 and float(conf.max()) <= 1.0

    m = build_model("raft_nc_dbl").to(DEV)
    im1, im2 = (t.to(DEV) for t in orc_frames())
    with torch.no_grad():
        lo0, up0 = m(im1, im2, iters=4, test_mode=True)
        runs = [m(im1, im2, iters=4, test_mode=True, return_confidence=True) for _ in range(3)]
    lo, up, conf = runs[0]
    assert torch.equal(lo, lo0) and torch.equal(up, up0)
    # the third call replays a captured CUDA graph on the umma engine (the second captures it): bit-identical to eager
    assert all(torch.equal(a, b) for r in runs[1:] for a, b in zip(r, runs[0]))
    assert conf.shape == up.shape and float(conf.min()) >= 0.0 and float(conf.max()) <= 1.0
    # End to end the confidence sees the trunk's error only through the weights net's input (the x2 flow and the hidden
    # state), then through a sigmoid (slope <= 1/4) and a normalised average of it.  smoke() and test_gpu_parity bound the
    # flow at 1e-3 EPE from the reference, against flows of about 1 px here; the confidence moves by far less than that
    # relative change times its own size (<= 0.04 here): bound 1e-4 absolute.
    e = (conf.cpu() - g["e2e_conf"]).abs().max().item()
    epe = (up.cpu() - torch.from_numpy(cfg1["raft_nc_dbl_flow_up"])).pow(2).sum(1).sqrt().mean().item()
    print(f"{mode} end to end: |conf - reference| {e:.2e} (flow_up EPE {epe:.2e})")
    assert e < 1e-4 and epe < 1e-3


def orc_frames():
    from rnc.synth import frames
    return frames(1, 128, 256)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="nn.DataParallel needs two GPUs")
def test_data_parallel_gathers_the_confidence():
    m = build_model("raft_nc_dbl").to(DEV)
    dp = torch.nn.DataParallel(m, device_ids=[0, 1])
    from rnc.synth import frames
    im1, im2 = (t.to(DEV) for t in frames(4, 128, 256))
    with torch.no_grad():
        lo, up, conf = dp(im1, im2, iters=2, test_mode=True, return_confidence=True)
        lo1, up1, conf1 = m(im1, im2, iters=2, test_mode=True, return_confidence=True)
        preds, confs = dp(im1, im2, iters=2, return_confidence=True)
    assert conf.shape == up.shape == (4, 2, 128, 256) and len(preds) == len(confs) == 2
    assert (conf - conf1).abs().max().item() < 1e-5 and (up - up1).norm(dim=1).mean().item() < 1e-3
    assert (confs[-1] - conf1).abs().max().item() < 1e-5


# ------------------------------------------------------------------------------------------------------- frozen-trunk route


def chain_grads(fn, x, c, wp, gy, gc, conf_out=True):
    """Gradients of sum(gy * out) + sum(gc * conf) through fn(x, c, *softplus(wp), 8, conf_out): [x, c, weight_p...]."""
    xd, cd = x.to(DEV).requires_grad_(True), c.to(DEV).requires_grad_(True)
    wpd = [w.to(DEV).requires_grad_(True) for w in wp]
    res = fn(xd, cd, *[F.softplus(w, beta=10) for w in wpd], 8.0, conf_out)
    if conf_out:
        out, conf = res
        loss = (out * gy).sum() + ((conf * gc).sum() if gc is not None else 0.0)
    else:
        loss = (res * gy).sum()
    loss.backward()
    return [xd.grad, cd.grad] + [w.grad for w in wpd]


def per_layer(x, c, w1, w2, w3, w4, out_scale, conf_out):
    from rnc.train import NConv2dFn, zero_stuff
    xh, ch = zero_stuff(x), zero_stuff(c)
    b, C, oh, ow = xh.shape
    y, k = NConv2dFn.apply(xh.view(b * C, 1, oh, ow), ch.view(b * C, 1, oh, ow), w1, 1e-20)
    y, k = NConv2dFn.apply(y, k, w2, 1e-20)
    y, k = NConv2dFn.apply(torch.cat((y, y), 1), torch.cat((k, k), 1), w3, 1e-20)
    y, k = NConv2dFn.apply(y, k, w4, 1e-20)
    return out_scale * y.view(b, C, oh, ow), k.view(b, C, oh, ow)


def test_ncup_chain_fn_confidence_backward():
    """NcupChainFn with want_conf against the per-layer NConv2dFn chain and fp64 autograd (the bounds of
    test_gpu_ncup_finetune: 1e-4, 1e-3 for the scale-invariant nconv_out), the flow-only gradient bit-identical to
    want_conf=False's, and determinism."""
    from rnc.train import NcupChainFn
    x, c, wp = chain_inputs(2, 24, 40, seed=31)
    gen = torch.Generator().manual_seed(32)
    with torch.no_grad():
        _, c64 = chain64(x.double(), c.double(), wp, 8.0)
    gy = (torch.randn(c64.shape, generator=gen, dtype=torch.float64) * (c64 > 0)).float().to(DEV)
    gc = torch.randn(c64.shape, generator=gen).to(DEV)
    fused = chain_grads(NcupChainFn.apply, x, c, wp, gy, gc)
    layer = chain_grads(per_layer, x, c, wp, gy, gc)
    xr, cr = x.double().requires_grad_(True), c.double().requires_grad_(True)
    wr = [w.double().requires_grad_(True) for w in wp]
    o64, k64 = chain64(xr, cr, wr, 8.0)
    ((o64 * gy.double().cpu()).sum() + (k64 * gc.double().cpu()).sum()).backward()
    ref = [xr.grad, cr.grad] + [w.grad for w in wr]
    tags = ["x", "conf", "W1", "W2", "W3", "W4"]
    for other, what in ((layer, "per-layer"), (ref, "fp64")):
        errs = {}
        for t, a, b in zip(tags, fused, other):
            ok = torch.isfinite(b.cpu()) & (b.cpu().abs() < 1e6)
            errs[t] = rel(a.cpu()[ok], b.cpu()[ok])
        print(f"fused vs {what}: " + " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
        assert errs.pop("W4") < 1e-3 and all(v < 1e-4 for v in errs.values()), errs
    # the confidence term absent: want_conf=False's gradients, bit for bit
    plain = chain_grads(NcupChainFn.apply, x, c, wp, gy, None, conf_out=False)
    no_conf = chain_grads(NcupChainFn.apply, x, c, wp, gy, None)
    assert all(torch.equal(a, b) for a, b in zip(plain, no_conf))
    # deterministic
    again = chain_grads(NcupChainFn.apply, x, c, wp, gy, gc)
    assert all(torch.equal(a, b) for a, b in zip(fused, again))


def _check_grads(grads, meta, tag, loss, bound_fnet=2e-3, bound=2e-3):
    """Per-parameter gradients against the reference's (make_golden_r2.grad_fixture: norm and seeded projections)."""
    assert abs(float(loss.detach()) - meta[f"{tag}_loss"]) < 1e-4
    gmax = meta[f"{tag}_grad_norm_max"]
    ref = meta[f"{tag}_grads"]
    assert set(grads) == set(ref)
    fix = grad_fixture({k: g.cpu() for k, g in grads.items()})
    worst = 0.0
    for k, g in grads.items():
        b = bound_fnet if k.startswith("fnet.") else bound
        tol = b * ref[k][0] + 1e-5 * gmax
        n = g.numel() ** 0.5
        worst = max(worst, abs(fix[k][0] - ref[k][0]) / tol)
        assert abs(fix[k][0] - ref[k][0]) < tol, k
        assert all(abs(a - r) < tol * n for a, r in zip(fix[k][1:], ref[k][1:])), k
    print(f"{tag}: loss {float(loss.detach()):.6f} (reference {meta[f'{tag}_loss']:.6f}), worst norm error {worst:.2f} of the bound")


@pytest.mark.parametrize("mode", ["ffma", "umma"])
def test_frozen_trunk_want_conf_gradients_match_the_reference(mode, monkeypatch):
    """The frozen-trunk route (trunk on the inference engine, upsampler through NcupChainFn with want_conf) against the reference.
    On the exact-fp32 engine (ffma) the bound is test_gpu_ncup_finetune's 2e-3; measured on an H100: every upsampler
    gradient within 1e-6 of raft_forward_train's.  On the tensor-core engine (umma, the default) the weights net's hidden-layer
    gradients move by up to 8e-3 of their norm (2.7e-3 against the reference): the confidence term's seeded projections
    make those gradients sums with heavy cancellation, so the trunk's fp16-split rounding of the guidance shows; the per-layer
    NConv2dFn chain on the same trunk lands on the same values (7.8e-3 from raft_forward_train), so it is not the fused chain.
    Bound 2e-2 there, test_gpu_ncup_finetune's bound for the similarly conditioned batch-statistics case."""
    import raft_nc_dbl
    import rnc.train
    from rnc.train import sequence_loss
    monkeypatch.setenv("RNC_CONV", mode)
    _, meta = load_conf()
    a = ref_args("sintel")
    a.freeze_raft = True
    torch.manual_seed(1234)
    m = raft_nc_dbl.RAFT(a).to(DEV).train()
    m.freeze_bn()
    used = []
    real = rnc.train.NcupChainFn.apply
    monkeypatch.setattr(rnc.train.NcupChainFn, "apply", lambda *a: used.append(a[7]) or real(*a))
    monkeypatch.setattr(rnc.train, "raft_forward_train", None)     # the frozen-trunk route, not the exact one
    im1, im2, gt, valid = (t.to(DEV) for t in train_inputs())
    preds, confs = m(im1, im2, iters=GRAD_ITERS, return_confidence=True)
    assert len(preds) == len(confs) == GRAD_ITERS and used == [True] * GRAD_ITERS
    loss = sequence_loss(preds, gt, valid, gamma=0.85)[0] + conf_loss(confs)
    loss.backward()
    b = 2e-3 if mode == "ffma" else 2e-2
    _check_grads({k: p.grad for k, p in m.named_parameters() if p.grad is not None}, meta, "frozen", loss, b, b)


def test_exact_training_route_confidence_gradients_match_the_reference():
    """raft_forward_train with the confidences: test_gpu_train's bounds (2e-2 for fnet, 2e-3 for the rest)."""
    from rnc.train import sequence_loss
    _, meta = load_conf()
    m = build_model("raft_nc_dbl").to(DEV).train()
    m.freeze_bn()
    im1, im2, gt, valid = (t.to(DEV) for t in train_inputs())
    preds, confs = m(im1, im2, iters=GRAD_ITERS, return_confidence=True)
    assert len(preds) == len(confs) == GRAD_ITERS and confs[0].shape == preds[0].shape
    loss = sequence_loss(preds, gt, valid, gamma=0.85)[0] + conf_loss(confs)
    loss.backward()
    _check_grads({k: p.grad for k, p in m.named_parameters()}, meta, "full", loss, bound_fnet=2e-2)


# ------------------------------------------------------------------------------------------------------- sequences


def test_run_sequences_confidence_matches_per_pair_calls(monkeypatch):
    from rnc.harness import run_sequences
    from rnc.synth import frames
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    try:
        m = build_model("raft_nc_dbl").to(DEV)
        seqs = [[frames(1, 128, 256, seed=100 * s + t)[0][0] for t in range(n)] for s, n in enumerate([2, 3, 4])]
        got = {}
        for s, p, flow, conf in run_sequences(m, seqs, iters=4, batch_size=2, device=DEV, return_confidence=True):
            assert conf.shape == flow.shape == (2, 128, 256)
            got[(s, p)] = (flow, conf)
        flows = {(s, p): f for s, p, f in run_sequences(m, seqs, iters=4, batch_size=2, device=DEV)}
        assert got.keys() == flows.keys() == {(s, p) for s, seq in enumerate(seqs) for p in range(len(seq) - 1)}
        with torch.no_grad():
            for (s, p), (flow, conf) in got.items():
                _, up, c = m(seqs[s][p][None].to(DEV), seqs[s][p + 1][None].to(DEV), iters=4, test_mode=True,
                             return_confidence=True)
                assert torch.equal(flow, flows[(s, p)]) and torch.equal(flow, up[0]) and torch.equal(conf, c[0]), (s, p)
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
