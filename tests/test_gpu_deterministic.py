"""Deterministic mode (torch.use_deterministic_algorithms(True)) on the GPU: whole training steps repeat bit for bit on every
training route, the gradients still meet the pinned reference bounds, the atomic-free kernels match fp64 and repeat bit for
bit, and inference repeats bit for bit, eager and graph-replayed, within 1e-5 EPE of the default mode."""
import copy
import json
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, build_model
from oracle import raft_oracle as orc
from oracle.make_golden_r2 import GRAD_ITERS, grad_fixture, train_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def rel(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


def _ncup_variant(name, freeze=False):
    import raft_nc_dbl
    from conftest import ref_args
    from oracle import ncup_oracle as nco
    build_model("raft_nc_dbl")
    a = ref_args()
    for k, v in nco.args_overrides(nco.CONFIGS[name]).items():
        setattr(a, k, v)
    a.freeze_raft = freeze
    torch.manual_seed(1234)
    return raft_nc_dbl.RAFT(a)


def _frozen_trunk_bn_batch():
    """--freeze_raft with the trunk's BatchNorm frozen and the weights net's BatchNorm on batch statistics."""
    import raft_nc_dbl
    from conftest import ref_args
    build_model("raft_nc_dbl")
    torch.manual_seed(1234)
    a = ref_args("sintel")
    a.freeze_raft = True
    m = raft_nc_dbl.RAFT(a).train()
    for t in (m.fnet, m.cnet, m.update_block):
        for mod in t.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.eval()
    return m


def _frozen_bn(m):
    m.train()
    m.freeze_bn()
    return m


ROUTES = {
    "full": lambda: _frozen_bn(build_model("raft_nc_dbl")),
    "chairs": lambda: build_model("raft_nc_dbl", "chairs").train(),              # cnet BatchNorm on batch statistics
    "frozen_trunk": _frozen_trunk_bn_batch,
    "raft": lambda: _frozen_bn(build_model("raft")),
    "paper": lambda: _frozen_bn(_ncup_variant("paper")),
    "tf32": lambda: _frozen_bn(build_model("raft_nc_dbl")),
}


@pytest.mark.parametrize("route", list(ROUTES))
def test_train_step_is_bit_identical(det, route, monkeypatch):
    """Two seeded train_steps from identical state: the same loss, every .grad and every updated parameter, bit for bit."""
    import rnc.model
    from rnc.train import fetch_optimizer, train_step
    if route == "tf32":
        monkeypatch.setenv("RNC_TRAIN_CONV", "tf32")
    base = ROUTES[route]().to(DEV)
    im1, im2, gt, valid = (t.to(DEV) for t in train_inputs())
    assert rnc.model.frozen_trunk(base, im1, im2) == (route == "frozen_trunk")
    runs = []
    for _ in range(2):
        m = copy.deepcopy(base)
        opt, sched = fetch_optimizer(m, lr=1e-4, num_steps=10)
        torch.manual_seed(0)
        loss, _ = train_step(m, opt, sched, im1, im2, gt, valid, iters=2)
        grads = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
        params = {k: p.detach().clone() for k, p in m.named_parameters()}
        runs.append((loss, grads, params))
    (l0, g0, p0), (l1, g1, p1) = runs
    assert torch.isfinite(l0) and torch.equal(l0, l1)
    assert g0 and g0.keys() == g1.keys()
    assert all(torch.isfinite(g).all() for g in g0.values())
    bad = [k for k in g0 if not torch.equal(g0[k], g1[k])]
    assert not bad, f"gradients differ between identical steps: {bad[:5]}"
    bad = [k for k in p0 if not torch.equal(p0[k], p1[k])]
    assert not bad, f"parameters differ after identical steps: {bad[:5]}"


def _check_pinned(ref, gmax, grads, bound_of):
    assert set(grads) == set(ref), set(grads) ^ set(ref)
    fix = grad_fixture({k: g.cpu() for k, g in grads.items()})
    for k, g in grads.items():
        tol = bound_of(k) * ref[k][0] + 1e-5 * gmax
        n = g.numel() ** 0.5
        assert abs(fix[k][0] - ref[k][0]) < tol, (k, fix[k][0], ref[k][0])
        assert all(abs(x - y) < tol * n for x, y in zip(fix[k][1:], ref[k][1:])), k


@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft", "paper"])
def test_gradients_meet_pinned_reference_bounds(det, name):
    """Train mode, frozen BatchNorm, 128x160, B = 2, 3 iterations: loss and every gradient against the reference's pinned ones
    (r2.npz / ncup_cfg.npz), with the default mode's bounds: 2e-2 for fnet, 2e-3 elsewhere."""
    from rnc.train import sequence_loss
    if name == "paper":
        with open(os.path.join(ROOT, "tests", "golden", "ncup_cfg_meta.json")) as f:
            meta = json.load(f)
        m = _ncup_variant("paper")
        loss_ref, ref, gmax = meta["paper_train_loss"], meta["paper_train_grads"], meta["paper_train_grad_norm_max"]
    else:
        with open(os.path.join(ROOT, "tests", "golden", "r2_meta.json")) as f:
            meta = json.load(f)
        m = build_model(name)
        loss_ref, ref, gmax = meta[f"train_loss_{name}"], meta[f"train_grads_{name}"], meta[f"train_grad_norm_max_{name}"]
    m = _frozen_bn(m.to(DEV))
    im1, im2, gt, valid = (t.to(DEV) for t in train_inputs())
    loss, _ = sequence_loss(m(im1, im2, iters=GRAD_ITERS), gt, valid, gamma=0.85)
    assert abs(float(loss.detach()) - loss_ref) < 1e-4
    loss.backward()
    grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    _check_pinned(ref, gmax, grads, lambda k: 2e-2 if k.startswith("fnet.") else 2e-3)


WGRAD_SHAPES = [(128, 256, 3, 3, 1), (384, 128, 1, 5, 1), (384, 128, 5, 1, 1), (324, 256, 1, 1, 1), (2, 128, 7, 7, 1),
                (256, 2, 3, 3, 1), (64, 96, 3, 3, 2), (64, 96, 1, 1, 2), (3, 64, 7, 7, 2), (130, 64, 3, 3, 1), (256, 126, 3, 3, 1),
                (64, 96, 3, 3, -2), (64, 96, 1, 1, -2), (64, 64, 3, 3, -1), (96, 128, 3, 3, -2)]


@pytest.mark.parametrize("cin,cout,kh,kw,stride", WGRAD_SHAPES)
def test_weight_gradient_matches_fp64_and_repeats(det, cin, cout, kh, kw, stride):
    """rnc_conv2d_cl_wgrad_det through ConvCL (the weight gradient of both modes): within 5e-6 of fp64 and bit-identical over
    three calls."""
    from rnc.train import ConvCL, to_cl
    g = torch.Generator().manual_seed(cin * 7 + cout + kh)
    B, H, W = 2, 14, 19
    if stride < 0:
        B, H, W, stride = 3, 32, 48, -stride
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    b = torch.randn(cout, generator=g)
    wr, br = w.double().requires_grad_(True), b.double().requires_grad_(True)
    ref = F.conv2d(x.double(), wr, br, stride=stride, padding=(kh // 2, kw // 2))
    gy = torch.randn(ref.shape, generator=g)
    ref.backward(gy.double())
    xd, gyd = to_cl(x.to(DEV)), to_cl(gy.to(DEV))
    outs = []
    for _ in range(3):
        wd, bd = w.to(DEV).requires_grad_(True), b.to(DEV).requires_grad_(True)
        ConvCL.apply(xd, wd, bd, stride).backward(gyd)
        outs.append((wd.grad, bd.grad))
    e_w, e_b = rel(outs[0][0], wr.grad), rel(outs[0][1], br.grad)
    print(f"wgrad_det {cin}->{cout} {kh}x{kw} s{stride}: dw {e_w:.1e} db {e_b:.1e}")
    assert e_w < 5e-6 and e_b < 5e-6
    for gw, gb in outs[1:]:
        assert torch.equal(gw, outs[0][0]) and torch.equal(gb, outs[0][1])


def _lookup_case(kind):
    g = torch.Generator().manual_seed(21)
    B, H, W = 2, 18, 25
    if kind == "random":
        co = orc.coords_grid(B, H, W) + torch.randn(B, 2, H, W, generator=g) * 5
    elif kind == "one_location":                               # every window in one origin cell
        co = torch.empty(B, 2, H, W)
        co[:, 0], co[:, 1] = 11.3, 6.6
    elif kind == "outside":                                    # half the windows miss the grid on every level
        co = orc.coords_grid(B, H, W) + torch.randn(B, 2, H, W, generator=g) * 3
        co[:, 0, :, ::2] = -40.0
        co[:, 1, ::3] = H + 80.0
    else:                                                      # +-1e9 coordinates next to ordinary ones
        co = orc.coords_grid(B, H, W) + torch.randn(B, 2, H, W, generator=g) * 3
        co[:, 0, ::2] = 1e9
        co[:, 1, :, ::3] = -1e9
    f1 = torch.randn(B, 256, H, W, generator=g) * 1.5
    f2 = torch.randn(B, 256, H, W, generator=g) * 1.5
    return f1, f2, co, g


@pytest.mark.parametrize("kind", ["random", "one_location", "outside", "huge"])
def test_lookup_backward_matches_fp64_and_repeats(det, kind):
    """rnc_corr_lookup_bwd_det through CorrLookup: d fmap1 / d fmap2 against fp64 autograd through the reference's 4-D
    pyramid, and bit-identical over repeated calls."""
    from rnc.train import CorrLookup, CorrPyramid, to_cl, to_nchw
    f1, f2, co, g = _lookup_case(kind)
    a, b = f1.double().requires_grad_(True), f2.double().requires_grad_(True)
    ref = orc.corr_lookup(orc.corr_pyramid(a, b), co.double())
    gout = torch.randn(ref.shape, generator=g)
    ref.backward(gout.double())
    outs = []
    for _ in range(3):
        f1d = to_cl(f1.to(DEV)).requires_grad_(True)
        f2d = to_cl(f2.to(DEV)).requires_grad_(True)
        out = CorrLookup.apply(f1d, CorrPyramid.apply(f2d, 4), co.to(DEV), 4)
        out.backward(to_cl(gout.to(DEV)))
        outs.append((to_nchw(f1d.grad), to_nchw(f2d.grad)))
    for got, want in zip(outs[0], (a.grad, b.grad)):
        if want.abs().max() == 0:
            assert got.abs().max() == 0
        else:
            assert rel(got, want) < 1e-5
    for o in outs[1:]:
        assert torch.equal(o[0], outs[0][0]) and torch.equal(o[1], outs[0][1])


@pytest.mark.parametrize("B,H,W,iters", [(1, 128, 256, 4), (8, 440, 1024, 32)])
def test_inference_repeats_and_matches_default_mode(B, H, W, iters):
    """Eager, captured and replayed forwards in deterministic mode are bit-identical, and within 1e-5 EPE of the default
    mode's flows, measured in 1/8-resolution pixels (flow_up carries 8x the flow: 8e-5).  The difference is the InstanceNorm
    statistics' summation order (per-CTA partials instead of the epilogue's atomics), carried through the iterations: 3.8e-6
    / 2.4e-5 at B = 8, 440x1024, 32 iterations (H100)."""
    from rnc.synth import frames
    m = build_model("raft_nc_dbl").to(DEV)
    im1, im2 = (t.to(DEV) for t in frames(B, H, W))
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        with torch.no_grad():
            torch.use_deterministic_algorithms(False)
            lo_def, up_def = m(im1, im2, iters=iters, test_mode=True)
            torch.use_deterministic_algorithms(True, warn_only=False)
            outs = []
            for _ in range(3):                                 # eager, capture, replay
                lo, up = m(im1, im2, iters=iters, test_mode=True)
                outs.append((lo.clone(), up.clone()))
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
    for lo, up in outs[1:]:
        assert torch.equal(lo, outs[0][0]) and torch.equal(up, outs[0][1])
    for got, want, scale in zip(outs[0], (lo_def, up_def), (1, 8)):
        assert torch.isfinite(got).all()
        epe = (got - want).pow(2).sum(1).sqrt().mean().item()
        print(f"B{B} {H}x{W}: deterministic vs default EPE {epe:.2e}")
        assert epe < 1e-5 * scale
