"""Fine-tuning the NCUP upsampler of a frozen RAFT (the reference's --freeze_raft, train.py:295, raft_nc_dbl.py:70-72).

GPU: the fused NCUP chain (rnc_ncup_train_fwd / rnc_ncup_bwd, NcupChainFn) against fp64 autograd of the oracle's NConv chain and
against the per-layer NConv2dFn chain; its determinism; the frozen-trunk forward (trunk on the inference engine, upsampler on
autograd) against the pinned reference gradients and against the exact training path; a few optimiser steps; the fallbacks.
CPU: the routing predicate rnc.model.frozen_trunk."""
import ctypes
import json
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, build_model, ref_args
from oracle import raft_oracle as orc
from oracle.make_golden_r2 import GRAD_ITERS, grad_fixture, tied_leaves, train_inputs

DEV = "cuda:0"
gpu = pytest.mark.gpu


def rel(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


def frozen_model(dataset="sintel", seed=1234):
    """raft_nc_dbl built with freeze_raft through its constructor (the trunk is frozen before the upsampler is built)."""
    build_model("raft_nc_dbl")                       # imports the module
    import raft_nc_dbl
    torch.manual_seed(seed)
    args = ref_args(dataset)
    args.freeze_raft = True
    return raft_nc_dbl.RAFT(args)


def chain_inputs(B, H4, W4, seed):
    g = torch.Generator().manual_seed(seed)
    x = 5 * torch.randn(B, 2, H4, W4, generator=g)
    c = torch.rand(B, 2, H4, W4, generator=g) * 0.98 + 0.01
    c[torch.rand(B, 2, H4, W4, generator=g) < 0.3] = 0.0                # ~30 % exact zeros
    ws = [F.softplus(torch.randn(*s, generator=g)) for s in ((2, 1, 5, 5), (2, 2, 5, 5), (2, 4, 3, 3), (1, 2, 1, 1))]
    return x, c, ws


def chain_ref(x, c, ws, out_scale):
    """The live NConvUNet path on zero-stuffed inputs (upsampler.py:143-177, nconv_modules.py:106-136): (out, conf_out)."""
    xh, ch = orc.zero_stuff(x), orc.zero_stuff(c)
    b, C, oh, ow = xh.shape
    y, k = orc.nconv2d(xh.view(b * C, 1, oh, ow), ch.view(b * C, 1, oh, ow), ws[0])
    y, k = orc.nconv2d(y, k, ws[1])
    y, k = orc.nconv2d(torch.cat([y, y], 1), torch.cat([k, k], 1), ws[2])
    y, k = orc.nconv2d(y, k, ws[3])
    return out_scale * y.view(b, C, oh, ow), k.view(b, C, oh, ow)


def upstream(conf_out, seed):
    """A random output gradient, zero where the chain's final confidence is exactly 0 (there y = 0 / eps and d out / d num is
    1e20 in every implementation)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(conf_out.shape, generator=g, dtype=torch.float64) * (conf_out > 0)


# ------------------------------------------------------------------------------------------------------- fused chain kernels


@gpu
@pytest.mark.parametrize("B,H4,W4", [(1, 7, 9), (2, 24, 40), (2, 96, 128)])
def test_ncup_chain_fn_matches_fp64_autograd(B, H4, W4):
    from rnc import native
    from rnc.train import NcupChainFn
    x, c, ws = chain_inputs(B, H4, W4, seed=H4 * 100 + W4)
    xr, cr = x.double().requires_grad_(True), c.double().requires_grad_(True)
    wr = [w.double().requires_grad_(True) for w in ws]
    out_ref, conf_ref = chain_ref(xr, cr, wr, 8.0)
    gy = upstream(conf_ref.detach(), seed=5)
    (out_ref * gy).sum().backward()

    xd, cd = x.to(DEV).requires_grad_(True), c.to(DEV).requires_grad_(True)
    wd = [w.to(DEV).requires_grad_(True) for w in ws]
    out = NcupChainFn.apply(xd, cd, *wd, 8.0)
    assert out.shape == (B, 2, 4 * H4, 4 * W4)
    e_out = rel(out, out_ref.detach())
    out.backward(gy.float().to(DEV))
    errs = {}
    for tag, got, ref in (("x", xd.grad, xr.grad), ("conf", cd.grad, cr.grad)):
        ok = torch.isfinite(ref) & (ref.abs() < 1e6)
        errs[tag] = rel(got.cpu()[ok], ref[ok])
    for k in range(4):
        assert torch.isfinite(wr[k].grad).all()
        errs[f"W{k + 1}"] = rel(wd[k].grad, wr[k].grad)
    print(f"fused chain {B}x{H4}x{W4}: out {e_out:.2e} " + " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert e_out < 1e-5
    assert all(v < 1e-4 for v in errs.values()), errs

    # the device-weights forward is bit-identical to the inference kernel on the same weights
    L = native.lib()
    host = torch.cat([w.reshape(-1) for w in ws]).float()
    hw = (ctypes.c_float * 224)(*host.tolist())
    ref_out = torch.empty_like(out)
    native.check(L.rnc_ncup_fwd(xd.data_ptr(), cd.data_ptr(), hw, B, H4, W4, 8.0, ctypes.c_void_p(ref_out.data_ptr()), None,
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "ncup")
    assert torch.equal(out.detach(), ref_out)


@gpu
def test_fused_chain_backward_is_deterministic():
    from rnc.train import NcupChainFn
    x, c, ws = chain_inputs(2, 96, 128, seed=11)
    g = torch.randn(2, 2, 384, 512, generator=torch.Generator().manual_seed(12)).to(DEV)
    grads = []
    for _ in range(2):
        xd, cd = x.to(DEV).requires_grad_(True), c.to(DEV).requires_grad_(True)
        wd = [w.to(DEV).requires_grad_(True) for w in ws]
        NcupChainFn.apply(xd, cd, *wd, 8.0).backward(g)
        grads.append([xd.grad, cd.grad] + [w.grad for w in wd])
    assert all(torch.equal(a, b) for a, b in zip(*grads))


@gpu
def test_fused_chain_matches_per_layer_chain():
    """NcupChainFn against the NConv2dFn chain of ncup_upsampler_train (the full-training path) on the same fp32 inputs."""
    from rnc.train import ncup_chain_autograd, nconv_unet_train, zero_stuff
    net = build_model("raft_nc_dbl").upsampler.interpolation_net.to(DEV)
    x, c, _ = chain_inputs(2, 24, 40, seed=21)
    x, c = x.to(DEV), c.to(DEV)

    def run(fused):
        net.zero_grad(set_to_none=True)
        xd, cd = x.clone().requires_grad_(True), c.clone().requires_grad_(True)
        if fused:
            out = ncup_chain_autograd(net, xd, cd, 8.0)
        else:
            xh, ch = zero_stuff(xd), zero_stuff(cd)
            b, C, oh, ow = xh.shape
            y, k = nconv_unet_train(net, xh.view(b * C, 1, oh, ow), ch.view(b * C, 1, oh, ow))
            out = 8.0 * y.view(b, C, oh, ow)
            run.conf = k.view(b, C, oh, ow).detach()
        return out, xd, cd

    out_l, xl, cl = run(False)
    gy = upstream(run.conf.cpu(), seed=22).float().to(DEV)
    out_l.backward(gy)
    gl = {k: p.grad.clone() for k, p in net.named_parameters()}
    out_f, xf, cf = run(True)
    out_f.backward(gy)
    assert rel(out_f, out_l) < 1e-6
    ok_x = xl.grad.abs() < 1e6
    ok_c = cl.grad.abs() < 1e6
    errs = {"x": rel(xf.grad[ok_x], xl.grad[ok_x]), "conf": rel(cf.grad[ok_c], cl.grad[ok_c])}
    # weight gradients relative to their own norm with a floor of 1e-5 of the largest: the 1x1 nconv_out is scale-invariant
    # (out(s * W4) = out(W4)), so its gradient is a sum with heavy cancellation (tests/test_r2_golden.py uses the same floor)
    gmax = max(float(g.norm()) for g in gl.values())
    errs.update({k: float((p.grad - gl[k]).norm() / (gl[k].norm() + 1e-5 * gmax)) for k, p in net.named_parameters()})
    print("fused vs per-layer:", " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    # nconv_out is scale-invariant (out(s * W4) = out(W4)): per position its gradient is W4[1-c] * (A0*B1 - A1*B0) / D^2 with
    # A, B the layer-3 pairs, a difference of the two channels' layer-3 values, so any fp32 evaluation of the forward carries
    # ~1e-4 of it (the per-layer and the fused chain are both 4e-5 .. 1.5e-4 from fp64 here); bound 1e-3, both against each other
    # and against fp64.  Every other gradient: 1e-4.
    names = ("nconv_in", "nconv_x2.0", "decoder.0", "nconv_out")
    leaves = {n + ".weight_p": dict(net.named_parameters())[n + ".weight_p"].detach().double().cpu().requires_grad_(True) for n in names}
    out64, _ = chain_ref(x.double().cpu(), c.double().cpu(), [F.softplus(leaves[n + ".weight_p"], beta=10) for n in names], 8.0)
    (out64 * gy.double().cpu()).sum().backward()
    k = "nconv_out.weight_p"
    e_f, e_l = rel(dict(net.named_parameters())[k].grad, leaves[k].grad), rel(gl[k], leaves[k].grad)
    print(f"   {k}: fused {e_f:.2e}, per-layer {e_l:.2e} from fp64")
    assert errs.pop(k) < 1e-3 and e_f < 1e-3
    assert all(v < 1e-4 for v in errs.values()), errs


# ------------------------------------------------------------------------------------------------------- frozen-trunk forward


def _meta2():
    with open(os.path.join(ROOT, "tests", "golden", "r2_meta.json")) as f:
        return json.load(f)


def _no_exact_path(*a, **k):
    raise AssertionError("the frozen-trunk forward must not take raft_forward_train")


def _upsampler_grads(m):
    return {k: p.grad.detach().clone() for k, p in m.named_parameters() if k.startswith("upsampler.")}


@gpu
def test_frozen_trunk_matches_pinned_reference_gradients(monkeypatch):
    import rnc.train
    from rnc.train import sequence_loss
    meta = _meta2()
    m = frozen_model()
    im1, im2, gt, valid = train_inputs()
    sd, leaves = tied_leaves(m)
    _, _, ups = orc.raft_forward_graph(sd, im1, im2, iters=GRAD_ITERS, model="raft_nc_dbl")
    orc.sequence_loss(ups, gt, valid, gamma=0.85).backward()

    m = m.to(DEV).train()
    m.freeze_bn()
    monkeypatch.setattr(rnc.train, "raft_forward_train", _no_exact_path)
    preds = m(im1.to(DEV), im2.to(DEV), iters=GRAD_ITERS)
    assert len(preds) == GRAD_ITERS and preds[0].shape == (2, 2, 128, 160)
    loss, _ = sequence_loss(preds, gt.to(DEV), valid.to(DEV), gamma=0.85)
    assert abs(float(loss.detach()) - meta["train_loss_raft_nc_dbl"]) < 1e-4
    loss.backward()
    grads = _upsampler_grads(m)
    assert grads
    gmax = meta["train_grad_norm_max_raft_nc_dbl"]
    fix, ref = grad_fixture({k: g.cpu() for k, g in grads.items()}), meta["train_grads_raft_nc_dbl"]
    worst = 0.0
    for k, g in grads.items():
        r = float((g.cpu() - leaves[k].grad).norm() / (leaves[k].grad.norm() + 1e-5 * gmax))
        worst = max(worst, r)
        assert r < 2e-3, (k, r)
        tol = 2e-3 * ref[k][0] + 1e-5 * gmax
        n = g.numel() ** 0.5
        assert abs(fix[k][0] - ref[k][0]) < tol, k
        assert all(abs(a - b) < tol * n for a, b in zip(fix[k][1:], ref[k][1:])), k
    print(f"frozen trunk: loss {float(loss):.6f} (pinned {meta['train_loss_raft_nc_dbl']:.6f}), worst upsampler gradient {worst:.2e}")
    assert all(p.grad is None for k, p in m.named_parameters() if not k.startswith("upsampler."))


def _compare_paths(m, inputs, tag, bound=1e-3):
    """Frozen-trunk forward vs raft_forward_train on the same model: per-iteration EPE within 1e-3, upsampler gradients (each
    parameter, and all of them as one vector) within `bound`."""
    from rnc.train import raft_forward_train, sequence_loss
    im1, im2, gt, valid = inputs
    m.zero_grad(set_to_none=True)
    pf = m(im1, im2, iters=GRAD_ITERS)
    sequence_loss(pf, gt, valid, gamma=0.85)[0].backward()
    gf = _upsampler_grads(m)
    m.zero_grad(set_to_none=True)
    pe = raft_forward_train(m, im1, im2, GRAD_ITERS)
    sequence_loss(pe, gt, valid, gamma=0.85)[0].backward()
    ge = _upsampler_grads(m)
    gmax = max(float(g.norm()) for g in ge.values())
    epe = [float((a - b).detach().norm(dim=1).mean()) for a, b in zip(pf, pe)]
    # a convolution bias followed by a BatchNorm with batch statistics has a gradient that is zero in exact arithmetic: both
    # paths return rounding noise there, bounded in absolute terms
    wn = m.upsampler.weights_est_net
    zero = {f"upsampler.weights_est_net.conv.{i}.0.bias" for i, blk in enumerate(wn.conv) if len(blk) == 3 and blk[1].training}
    errs = {k: float((gf[k] - ge[k]).norm() / (ge[k].norm() + 1e-5 * gmax)) for k in ge if k not in zero}
    worst = max(errs, key=errs.get)
    print(f"{tag}: frozen vs exact path: EPE per iteration {['%.1e' % e for e in epe]}, worst upsampler gradient "
          f"{errs[worst]:.2e} ({worst})" + "".join(f", {k} |g| {float(ge[k].norm()) / gmax:.1e} of the largest" for k in sorted(zero)))
    total = float(torch.cat([(gf[k] - ge[k]).reshape(-1) for k in ge]).norm() / torch.cat([ge[k].reshape(-1) for k in ge]).norm())
    print(f"   all upsampler gradients as one vector: {total:.2e}")
    assert len(pf) == len(pe) == GRAD_ITERS
    assert max(epe) < 1e-3 and total < bound and errs[worst] < bound
    assert all(float(ge[k].norm()) < 1e-4 * gmax and float((gf[k] - ge[k]).norm()) < 1e-4 * gmax for k in zero)


@gpu
def test_frozen_trunk_matches_exact_path():
    m = frozen_model().to(DEV).train()
    m.freeze_bn()
    _compare_paths(m, [t.to(DEV) for t in train_inputs()], "frozen BN")


@gpu
def test_frozen_trunk_train_step(monkeypatch):
    import rnc.train
    from rnc.train import fetch_optimizer, train_step
    m = frozen_model().to(DEV)
    im1, im2, gt, valid = (t.to(DEV) for t in train_inputs())
    m.eval()
    with torch.no_grad():
        _, up_before = m(im1, im2, iters=2, test_mode=True)
    m.train()
    m.freeze_bn()
    opt, sched = fetch_optimizer(m, lr=1e-3, num_steps=20)
    before = {k: p.detach().clone() for k, p in m.named_parameters()}
    monkeypatch.setattr(rnc.train, "raft_forward_train", _no_exact_path)
    losses = [float(train_step(m, opt, sched, im1, im2, gt, valid, iters=2)[0]) for _ in range(3)]
    print("frozen-trunk losses", losses)
    assert all(torch.isfinite(torch.tensor(losses))) and losses[-1] < losses[0]
    for k, p in m.named_parameters():
        if k.startswith("upsampler."):
            assert not torch.equal(before[k], p.detach()), k
        else:
            assert torch.equal(before[k], p.detach()), k
    m.eval()
    with torch.no_grad():
        _, up_after = m(im1, im2, iters=2, test_mode=True)
    assert torch.isfinite(up_after).all() and not torch.equal(up_before, up_after)


@gpu
def test_frozen_trunk_fallbacks(monkeypatch):
    import rnc.model
    import rnc.train
    from rnc.train import sequence_loss
    im1, im2, gt, valid = (t.to(DEV) for t in train_inputs())
    calls = []
    exact = rnc.train.raft_forward_train

    def counting(*a, **k):
        calls.append(1)
        return exact(*a, **k)

    monkeypatch.setattr(rnc.train, "raft_forward_train", counting)
    # trunk BatchNorm with batch statistics (the reference's chairs stage): the exact path
    m = frozen_model().to(DEV).train()
    assert not rnc.model.frozen_trunk(m, im1, im2)
    preds = m(im1, im2, iters=2)
    sequence_loss(preds, gt, valid, gamma=0.85)[0].backward()
    assert len(calls) == 1 and all(torch.isfinite(p.grad).all() for k, p in m.named_parameters() if k.startswith("upsampler."))
    # images that require grad: the exact path, and the images receive gradients
    m.freeze_bn()
    a, b = im1.clone().requires_grad_(True), im2.clone().requires_grad_(True)
    preds = m(a, b, iters=2)
    sequence_loss(preds, gt, valid, gamma=0.85)[0].backward()
    assert len(calls) == 2
    assert a.grad is not None and torch.isfinite(a.grad).all() and a.grad.abs().sum() > 0 and b.grad is not None
    # weights-net BatchNorm with batch statistics, trunk BatchNorm frozen: the frozen-trunk path, matching the exact path
    m = frozen_model("sintel").to(DEV).train()
    for t in (m.fnet, m.cnet, m.update_block):
        for mod in t.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.eval()
    assert any(isinstance(mod, torch.nn.BatchNorm2d) and mod.training for mod in m.upsampler.modules())
    assert rnc.model.frozen_trunk(m, im1, im2)
    n = len(calls)
    # with batch statistics the weights-net gradients are far less well conditioned: the 1e-5 EPE by which the two trunks'
    # predictions differ moved the first BatchNorm's bias gradient (the largest of the upsampler) by 7e-3 of its norm and the
    # whole upsampler gradient by 5e-3 (H100); with frozen statistics the same inputs agree to 5e-4.  Bound 2e-2 here.
    _compare_paths(m, (im1, im2, gt, valid), "weights-net BN in train mode", bound=2e-2)
    assert len(calls) == n + 1                                  # only the explicit exact-path call


# ------------------------------------------------------------------------------------------------------- routing (CPU)


def test_frozen_trunk_predicate():
    from rnc.model import frozen_trunk
    im = torch.zeros(1, 3, 64, 64)
    m = frozen_model().train()
    m.freeze_bn()
    assert frozen_trunk(m, im, im)
    with torch.no_grad():
        assert not frozen_trunk(m, im, im)
    assert not frozen_trunk(m, im.clone().requires_grad_(True), im)
    assert not frozen_trunk(m, im, im, torch.zeros(1, 2, 8, 8, requires_grad=True))
    assert frozen_trunk(m, im, im, torch.zeros(1, 2, 8, 8))
    # weights-net BatchNorm in train mode is fine; trunk BatchNorm in train mode is not
    for mod in m.upsampler.modules():
        mod.train()
    assert frozen_trunk(m, im, im)
    m.cnet.train()
    assert not frozen_trunk(m, im, im)
    m.freeze_bn()
    m.args.mixed_precision = True
    assert not frozen_trunk(m, im, im)
    m.args.mixed_precision = False
    m.update_block.flow_head.conv1.weight.requires_grad_(True)
    assert not frozen_trunk(m, im, im)
    m.update_block.flow_head.conv1.weight.requires_grad_(False)
    for p in m.upsampler.parameters():
        p.requires_grad_(False)
    assert not frozen_trunk(m, im, im)                         # nothing trains
    # the default model trains everything; the convex model has no upsampler
    full = build_model("raft_nc_dbl").train()
    full.freeze_bn()
    assert not frozen_trunk(full, im, im)
    convex = build_model("raft").train()
    for p in convex.parameters():
        p.requires_grad_(False)
    assert not frozen_trunk(convex, im, im)


def test_ncup_train_entry_points_reject_bad_arguments():
    from rnc import native
    L = native.lib()
    v = ctypes.c_void_p
    p = v(16)
    assert L.rnc_ncup_bwd_workspace_bytes(0, 4, 4) == 0
    ws = L.rnc_ncup_bwd_workspace_bytes(2, 96, 128)
    assert ws == 8 * (12 * 16 * 4 * 196 + 196)                 # per-CTA partial rows + the reduced sums
    assert L.rnc_ncup_bwd(p, p, p, 0, 4, 4, 8.0, p, None, p, p, p, p, 1 << 20, None) == -1
    assert L.rnc_ncup_bwd(None, p, p, 1, 4, 4, 8.0, p, None, p, p, p, p, 1 << 20, None) == -2
    assert L.rnc_ncup_bwd(p, p, p, 1, 4, 4, 8.0, p, None, None, None, None, None, 0, None) == -2
    assert L.rnc_ncup_bwd(p, p, p, 1, 4, 4, 8.0, p, None, p, p, p, None, 1 << 20, None) == -2
    assert L.rnc_ncup_bwd(p, p, p, 1, 4, 4, 8.0, p, None, p, p, p, p, 8, None) == -5
    assert L.rnc_ncup_train_fwd(p, p, p, 1, 0, 4, 8.0, p, None, None) == -1
    assert L.rnc_ncup_train_fwd(p, p, None, 1, 4, 4, 8.0, p, None, None) == -2
