"""NConvUNet configurations beyond the shipped one, on the GPU: the seam against the reference's goldens, the kernels'
gradients against fp64 autograd of the oracle (pooling ties, zero confidences, the decoder's up source, bias), determinism,
whole-model flows and training gradients (full and frozen-trunk) against the reference's, and graph replay."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, ref_args
from oracle import ncup_oracle as nco
from oracle import raft_oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CONFIGS = list(nco.CONFIGS)


@pytest.fixture(scope="module")
def ng():
    z = np.load(os.path.join(ROOT, "tests", "golden", "ncup_cfg.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


@pytest.fixture(scope="module")
def nmeta():
    with open(os.path.join(ROOT, "tests", "golden", "ncup_cfg_meta.json")) as f:
        return json.load(f)


def rel(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


def golden_unet(ng, name):
    from nconv_modules import NConvUNet
    net = NConvUNet(**nco.unet_kwargs(nco.CONFIGS[name]))
    p = f"{name}_sd_"
    net.load_state_dict({k[len(p):]: v for k, v in ng.items() if k.startswith(p)})
    return net.to(DEV)


def variant_model(name, seed=1234, freeze=False):
    import raft_nc_dbl
    a = ref_args()
    for k, v in nco.args_overrides(nco.CONFIGS[name]).items():
        setattr(a, k, v)
    a.freeze_raft = freeze
    torch.manual_seed(seed)
    return raft_nc_dbl.RAFT(a).eval()


@pytest.mark.parametrize("inp", ["even", "odd"])
@pytest.mark.parametrize("name", CONFIGS)
def test_seam_matches_reference(ng, name, inp):
    net = golden_unet(ng, name)
    with torch.no_grad():
        x, c = net((ng[f"in_{inp}_data"].to(DEV), ng[f"in_{inp}_conf"].to(DEV)))
    assert (x.cpu() - ng[f"{name}_{inp}_xout"]).abs().max() < 1e-4
    assert (c.cpu() - ng[f"{name}_{inp}_cout"]).abs().max() < 1e-6


@pytest.mark.parametrize("inp", ["even", "odd"])
@pytest.mark.parametrize("name", CONFIGS)
def test_gradients_match_fp64_oracle_and_reference(ng, nmeta, name, inp):
    cfg = nco.CONFIGS[name]
    net = golden_unet(ng, name)
    d0, c0 = ng[f"in_{inp}_data"], ng[f"in_{inp}_conf"]
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in net.state_dict().items()}
    dr, cr = d0.double().requires_grad_(True), c0.double().requires_grad_(True)
    xr, cor = nco.unet(sd, cfg, dr, cr)
    g = torch.Generator().manual_seed(5)
    p1, p2 = torch.randn(xr.shape, generator=g), torch.randn(cor.shape, generator=g)
    ((p1.double() * xr).sum() + (p2.double() * cor).sum()).backward()

    def run():
        net.zero_grad(set_to_none=True)
        d, c = d0.to(DEV).requires_grad_(True), c0.to(DEV).requires_grad_(True)
        x, co = net((d, c))
        ((p1.to(DEV) * x).sum() + (p2.to(DEV) * co).sum()).backward()
        return d.grad.clone(), c.grad.clone(), {n: (None if p.grad is None else p.grad.clone()) for n, p in net.named_parameters()}

    gd, gc, gp = run()
    for got, ref in ((gd, dr.grad), (gc, cr.grad)):
        ok = ref.abs() < 1e6                  # zero-confidence neighbourhoods: ~1e20 * g in every implementation
        assert rel(got.cpu()[ok], ref[ok]) < 1e-4
    assert sorted(n for n, v in gp.items() if v is None) == sorted(nmeta[f"{name}_{inp}_grad_none"])
    for n in nco.live_parameter_names(cfg):
        ref = sd[n].grad
        assert (gp[n].cpu().double() - ref).abs().max() < 1e-4 * max(1.0, ref.abs().max().item()), n
    gd2, gc2, gp2 = run()                     # fixed-order reductions: repeated backwards are bit-identical
    assert torch.equal(gd, gd2) and torch.equal(gc, gc2)
    assert all((v is None and gp2[n] is None) or torch.equal(v, gp2[n]) for n, v in gp.items())


@pytest.mark.parametrize("up_hw,hw", [((5, 7), (11, 15)), ((12, 16), (12, 16)), ((6, 8), (12, 16))])
def test_nconv_layer_up_source_and_bias_match_fp64(up_hw, hw):
    """One layer on cat(nearest-upsampled coarse input, full-resolution input), with bias, against fp64 autograd."""
    from rnc.train import NConv2dFn
    g = torch.Generator().manual_seed(up_hw[0] * 31 + hw[1])
    ux, uc = torch.randn(2, 4, *up_hw, generator=g) * 2, torch.rand(2, 4, *up_hw, generator=g)
    x, c = torch.randn(2, 4, *hw, generator=g) * 2, torch.rand(2, 4, *hw, generator=g)
    uc[uc < 0.3] = 0.0
    c[c < 0.3] = 0.0
    wp, b = torch.rand(4, 8, 5, 5, generator=g) + 0.05, torch.randn(4, generator=g)
    leaves = [t.double().requires_grad_(True) for t in (ux, uc, x, c, wp, b)]
    rux, ruc, rx, rc, rw, rb = leaves
    cat_x = torch.cat((F.interpolate(rux, size=hw, mode="nearest"), rx), 1)
    cat_c = torch.cat((F.interpolate(ruc, size=hw, mode="nearest"), rc), 1)
    den = F.conv2d(cat_c, rw, padding=2)
    y = F.conv2d(cat_x * cat_c, rw, padding=2) / (den + 1e-20) + rb.view(1, -1, 1, 1)
    co = den / rw.reshape(4, -1).sum(-1).view(1, -1, 1, 1)
    gy, gco = torch.randn(y.shape, generator=g), torch.randn(co.shape, generator=g)
    ((y * gy.double()).sum() + (co * gco.double()).sum()).backward()
    dev = [t.to(DEV).requires_grad_(True) for t in (ux, uc, x, c, wp, b)]
    yd, cd = NConv2dFn.apply(dev[2], dev[3], dev[4], 1e-20, dev[5], dev[0], dev[1])
    assert rel(yd, y.detach()) < 1e-5 and rel(cd, co.detach()) < 1e-5
    torch.autograd.backward([yd, cd], [gy.to(DEV), gco.to(DEV)])
    for got, ref in zip(dev, leaves):
        ok = ref.grad.abs() < 1e6
        assert rel(got.grad.cpu()[ok], ref.grad[ok]) < 1e-4


@pytest.mark.parametrize("max_pool_data", [False, True])
def test_pooling_ties_and_gradients_are_exact(max_pool_data):
    from rnc.train import NConvPoolFn
    g = torch.Generator().manual_seed(3)
    d = torch.round(torch.randn(2, 3, 13, 17, generator=g) * 2) / 2       # many ties in the data
    c = torch.round(torch.rand(2, 3, 13, 17, generator=g) * 3) / 3
    c[c < 0.5] = 0.0                                                      # and in the confidence (zero regions)
    dr, cr = d.clone().requires_grad_(True), c.clone().requires_grad_(True)
    xo, co = nco.pool(dr, cr, "max_pooling" if max_pool_data else "conf_based")
    gx, gc = torch.randn(xo.shape, generator=g), torch.randn(co.shape, generator=g)
    ((xo * gx).sum() + (co * gc).sum()).backward()
    dd, cd = d.to(DEV).requires_grad_(True), c.to(DEV).requires_grad_(True)
    xd, cod = NConvPoolFn.apply(dd, cd, max_pool_data)
    assert torch.equal(xd.cpu(), xo.detach()) and torch.equal(cod.cpu(), co.detach())
    ((xd * gx.to(DEV)).sum() + (cod * gc.to(DEV)).sum()).backward()
    assert torch.equal(dd.grad.cpu(), dr.grad) and torch.equal(cd.grad.cpu(), cr.grad)


MODEL_CONFIGS = ("paper", "wide")        # oracle/make_golden_ncup.py:MODEL_CONFIGS


@pytest.mark.parametrize("name", MODEL_CONFIGS)
def test_model_flows_match_reference_and_graph_replay(ng, name):
    """Whole-model test-mode flows at cfg-1 size against the reference's; eager, captured and replayed forwards agree."""
    from rnc.synth import frames
    m = variant_model(name).to(DEV)
    im1, im2 = (t.to(DEV) for t in frames(1, 128, 256))
    outs = []
    with torch.no_grad():
        for _ in range(3):                        # eager, capture, replay
            lo, up = m(im1, im2, iters=4, test_mode=True)
            outs.append((lo.clone(), up.clone()))
    for lo, up in outs[1:]:
        assert torch.equal(lo, outs[0][0]) and torch.equal(up, outs[0][1])
    for key, got in (("flow_low", outs[0][0]), ("flow_up", outs[0][1])):
        epe = (got.cpu() - ng[f"{name}_cfg1_{key}"]).pow(2).sum(1).sqrt().mean().item()
        assert epe < 1e-3, (key, epe)


def _check_pinned(meta, name, grads, bound_of):
    """Per-parameter gradient norm and seeded projections against the reference's (make_golden_r2.grad_fixture), within
    bound * |g| + 1e-5 of the largest gradient norm, as tests/test_gpu_ncup_finetune.py holds the shipped network."""
    from oracle.make_golden_r2 import grad_fixture
    ref, gmax = meta[f"{name}_train_grads"], meta[f"{name}_train_grad_norm_max"]
    fix = grad_fixture({k: g.cpu() for k, g in grads.items()})
    for k in grads:
        tol = bound_of(k) * ref[k][0] + 1e-5 * gmax
        n = grads[k].numel() ** 0.5
        assert abs(fix[k][0] - ref[k][0]) < tol, (k, fix[k][0], ref[k][0])
        assert all(abs(x - y) < tol * n for x, y in zip(fix[k][1:], ref[k][1:])), k


@pytest.mark.parametrize("name", MODEL_CONFIGS)
def test_full_training_matches_pinned_reference_gradients(nmeta, name):
    """Train mode, frozen BatchNorm, 128x160, B = 2, 3 iterations (make_golden_r2): loss and every parameter's gradient
    against the reference's.  fnet's gradients are ill-conditioned in fp32 (tests/test_gpu_train.py): 2e-2 there, 2e-3
    elsewhere."""
    from oracle.make_golden_r2 import GRAD_ITERS, train_inputs
    from rnc.train import sequence_loss
    m = variant_model(name).to(DEV).train()
    m.freeze_bn()
    im1, im2, gt, valid = (t.to(DEV) for t in train_inputs())
    loss, _ = sequence_loss(m(im1, im2, iters=GRAD_ITERS), gt, valid, gamma=0.85)
    assert abs(float(loss.detach()) - nmeta[f"{name}_train_loss"]) < 1e-4
    loss.backward()
    assert sorted(k for k, p in m.named_parameters() if p.grad is None) == sorted(nmeta[f"{name}_train_grad_none"])
    grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    _check_pinned(nmeta, name, grads, lambda k: 2e-2 if k.startswith("fnet.") else 2e-3)


@pytest.mark.parametrize("name", MODEL_CONFIGS)
def test_frozen_trunk_matches_pinned_reference_gradients(nmeta, name, monkeypatch):
    """--freeze_raft: the trunk runs on the inference engine, the upsampler on the per-level chain; the upsampler's gradients
    are the reference's full-training ones (freezing the trunk does not change them)."""
    import rnc.train
    from oracle.make_golden_r2 import GRAD_ITERS, train_inputs
    from rnc.train import sequence_loss

    def no_exact_path(*a, **k):
        raise AssertionError("the frozen-trunk forward must not take raft_forward_train")

    m = variant_model(name, freeze=True).to(DEV).train()
    m.freeze_bn()
    monkeypatch.setattr(rnc.train, "raft_forward_train", no_exact_path)
    im1, im2, gt, valid = (t.to(DEV) for t in train_inputs())
    loss, _ = sequence_loss(m(im1, im2, iters=GRAD_ITERS), gt, valid, gamma=0.85)
    assert abs(float(loss.detach()) - nmeta[f"{name}_train_loss"]) < 1e-4
    loss.backward()
    assert all(p.grad is None for k, p in m.named_parameters() if not k.startswith("upsampler."))
    grads = {k: p.grad for k, p in m.named_parameters() if k.startswith("upsampler.")}
    assert grads and all(g is not None for g in grads.values())
    _check_pinned(nmeta, name, grads, lambda k: 2e-3)


@pytest.mark.parametrize("name", ["paper", "n2_unshared"])
def test_frozen_trunk_train_step_moves_only_the_upsampler(name):
    from rnc.model import frozen_trunk
    from rnc.nconv_unet import unused_parameters
    from rnc.synth import frames
    from rnc.train import fetch_optimizer, train_step
    m = variant_model(name, freeze=True).to(DEV)
    m.train()
    m.freeze_bn()
    im1, im2 = (t.to(DEV) for t in frames(2, 128, 160))
    g = torch.Generator().manual_seed(8)
    gt = (torch.randn(2, 2, 128, 160, generator=g) * 3).to(DEV)
    valid = torch.ones(2, 128, 160, device=DEV)
    assert frozen_trunk(m, im1, im2)
    before = {k: v.detach().clone() for k, v in m.state_dict().items()}
    opt, sched = fetch_optimizer(m, lr=1e-3, num_steps=10)
    loss, _ = train_step(m, opt, sched, im1, im2, gt, valid, iters=2)
    assert torch.isfinite(loss)
    unused = {id(p) for p in unused_parameters(m.upsampler.interpolation_net)}
    for n, p in m.named_parameters():
        if n.startswith("upsampler.") and id(p) not in unused:
            assert p.grad is not None, n
        else:
            assert p.grad is None, n
    after = m.state_dict()
    moved = {k for k in before if not torch.equal(before[k], after[k])}
    assert moved and all(k.startswith("upsampler.") for k in moved)
    if name == "n2_unshared":
        assert "upsampler.interpolation_net.encoder.2.weight_p" not in moved
