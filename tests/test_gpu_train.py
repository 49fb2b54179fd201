"""Training path (SURVEY.md §8f-3, north-star config #5) on the GPU: every backward kernel against fp64 torch autograd, and
the whole model's loss / per-parameter gradients against the differentiable CPU oracle, which tests/test_r2_golden.py pins to
the reference's own autograd."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, build_model
from oracle import raft_oracle as orc
from oracle.make_golden_r2 import GRAD_ITERS, tied_leaves, train_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def rel(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


@pytest.mark.parametrize("cin,cout,kh,kw,stride", [(128, 256, 3, 3, 1), (384, 128, 1, 5, 1), (384, 128, 5, 1, 1), (324, 256, 1, 1, 1),
                                                    (2, 128, 7, 7, 1), (256, 2, 3, 3, 1), (64, 96, 3, 3, 2), (64, 96, 1, 1, 2),
                                                    (3, 64, 7, 7, 2), (130, 64, 3, 3, 1), (256, 126, 3, 3, 1),
                                                    (64, 96, 3, 3, -2), (64, 96, 1, 1, -2), (64, 64, 3, 3, -1), (96, 128, 3, 3, -2)])
@pytest.mark.parametrize("mode", ["ffma", "tf32"])
def test_conv_cl_forward_and_gradients(cin, cout, kh, kw, stride, mode, monkeypatch):
    from rnc.train import ConvCL, to_cl, to_nchw
    monkeypatch.setenv("RNC_TRAIN_CONV", mode)
    g = torch.Generator().manual_seed(cin * 7 + cout + kh)
    B, H, W = 2, 14, 19
    if stride < 0:                                             # larger problem: many M tiles, several K splits in the wgrad
        B, H, W, stride = 3, 32, 48, -stride
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    b = torch.randn(cout, generator=g)
    gy = None
    xr, wr, br = (t.double().requires_grad_(True) for t in (x, w, b))
    ref = F.conv2d(xr, wr, br, stride=stride, padding=(kh // 2, kw // 2))
    gy = torch.randn(ref.shape, generator=g)
    ref.backward(gy.double())
    xd = to_cl(x.to(DEV)).requires_grad_(True)
    wd, bd = w.to(DEV).requires_grad_(True), b.to(DEV).requires_grad_(True)
    y = ConvCL.apply(xd, wd, bd, stride)
    assert y.shape[:3] == (B, ref.shape[2], ref.shape[3])
    # ffma: exact fp32 CUDA cores throughout; tf32: wgmma TF32x3 (~2^-21 per product) for forward and data gradient where the
    # layer's shape allows (the weight gradient stays exact fp32)
    e_y = rel(to_nchw(y, cout), ref.detach())
    assert (y[..., cout:] == 0).all()
    y.backward(to_cl(gy.to(DEV)))
    e_x, e_w, e_b = rel(to_nchw(xd.grad, cin), xr.grad), rel(wd.grad, wr.grad), rel(bd.grad, br.grad)
    print(f"ConvCL[{mode}] {cin}->{cout} {kh}x{kw} s{stride}: rel err y {e_y:.1e} dx {e_x:.1e} dw {e_w:.1e} db {e_b:.1e}")
    tol = 2e-6 if mode == "ffma" else 2e-5
    assert e_y < tol and e_x < tol and e_w < 5e-6 and e_b < 5e-6


def test_corr_lookup_backward_matches_autograd_through_the_4d_pyramid():
    """The reference back-propagates through corr_pyramid + grid_sample (corr.py:7-55); the kernels never build the volume."""
    from rnc.train import CorrLookup, CorrPyramid, to_cl, to_nchw
    g = torch.Generator().manual_seed(12)
    B, H, W = 2, 18, 25                                        # odd sizes: pooling drops rows / columns
    f1 = (torch.randn(B, 256, H, W, generator=g) * 1.5).requires_grad_(True)
    f2 = (torch.randn(B, 256, H, W, generator=g) * 1.5).requires_grad_(True)
    co = orc.coords_grid(B, H, W) + torch.randn(B, 2, H, W, generator=g) * 5
    ref = orc.corr_lookup(orc.corr_pyramid(f1, f2), co)
    gout = torch.randn(ref.shape, generator=g)
    ref.backward(gout)
    f1d = to_cl(f1.detach().to(DEV)).requires_grad_(True)
    f2d = to_cl(f2.detach().to(DEV)).requires_grad_(True)
    out = CorrLookup.apply(f1d, CorrPyramid.apply(f2d, 4), co.to(DEV), 4)
    assert rel(to_nchw(out), ref.detach()) < 1e-5
    out.backward(to_cl(gout.to(DEV)))
    assert rel(to_nchw(f1d.grad), f1.grad) < 1e-5 and rel(to_nchw(f2d.grad), f2.grad) < 1e-5
    # seam: CorrBlock on NCHW feature maps that require grad
    from corr import CorrBlock
    a, b2 = f1.detach().to(DEV).requires_grad_(True), f2.detach().to(DEV).requires_grad_(True)
    CorrBlock(a, b2)(co.to(DEV)).backward(gout.to(DEV))
    assert rel(a.grad, f1.grad) < 1e-5 and rel(b2.grad, f2.grad) < 1e-5


@pytest.mark.parametrize("cin,cout,k", [(1, 2, 5), (2, 2, 5), (4, 2, 3), (2, 1, 1)])
def test_nconv2d_backward_matches_autograd(cin, cout, k):
    from rnc.train import NConv2dFn
    g = torch.Generator().manual_seed(cin * 10 + k)
    data = torch.randn(3, cin, 21, 17, generator=g) * 3
    conf = torch.rand(3, cin, 21, 17, generator=g)
    conf[conf < 0.4] = 0.0                                      # sparse confidences (zero-stuffed lattice in NCUP)
    wp = torch.rand(cout, cin, k, k, generator=g) + 0.05
    dr, cr, wr = (t.double().requires_grad_(True) for t in (data, conf, wp))
    y, c = orc.nconv2d(dr, cr, wr)
    gy, gc = torch.randn(y.shape, generator=g), torch.randn(c.shape, generator=g)
    (y * gy.double()).sum().add((c * gc.double()).sum()).backward()
    dd, cd, wd = (t.to(DEV).requires_grad_(True) for t in (data, conf, wp))
    yd, cdo = NConv2dFn.apply(dd, cd, wd, 1e-20)
    assert rel(yd, y.detach()) < 1e-5 and rel(cdo, c.detach()) < 1e-5
    torch.autograd.backward([yd, cdo], [gy.to(DEV), gc.to(DEV)])
    # positions whose whole neighbourhood has zero confidence have y = 0/(0+eps): their gradient is ~1e20 * gy in both
    # implementations; compare where the reference gradient is finite and of sane size
    ok = dr.grad.abs() < 1e6
    assert rel(dd.grad.cpu()[ok], dr.grad[ok]) < 1e-4
    okc = cr.grad.abs() < 1e6
    assert rel(cd.grad.cpu()[okc], cr.grad[okc]) < 1e-4
    if torch.isfinite(wr.grad).all() and wr.grad.abs().max() < 1e6:
        assert rel(wd.grad, wr.grad) < 1e-4


@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_training_loss_and_gradients_match_the_oracle(name):
    """Config-5-style step at 128x160, B = 2, 3 iterations, train mode with frozen BatchNorm (train.py:185-186): loss and every
    parameter's gradient against the differentiable oracle (= the reference's autograd, tests/test_r2_golden.py), evaluated
      (a) on the CPU in fp32 — the pinned reference numbers, and
      (b) by PyTorch on the same GPU in fp32 (cuDNN / cuBLAS, TF32 off) — what the reference itself computes on a GPU.
    The gradients of the fnet convolutions below layer3 are ill-conditioned in fp32 (a long chain of InstanceNorm backward
    passes, sums with heavy cancellation): cuDNN's own fp32 evaluation of the encoder sits several 1e-3 from fp64
    there, and any two fp32 GPU evaluations differ from each other by as much (test_encoder_gradients_match_torch_fp64).
    Hence two bounds: 2e-2 for fnet, 2e-3 for every other parameter."""
    from rnc.train import sequence_loss
    with open(os.path.join(ROOT, "tests", "golden", "r2_meta.json")) as f:
        meta = json.load(f)
    m = build_model(name)
    im1, im2, gt, valid = train_inputs()
    sd, leaves = tied_leaves(m)
    _, _, ups = orc.raft_forward_graph(sd, im1, im2, iters=GRAD_ITERS, model=name)
    oloss = orc.sequence_loss(ups, gt, valid, gamma=0.85)
    oloss.backward()
    assert abs(float(oloss.detach()) - meta[f"train_loss_{name}"]) < 1e-4
    # (b) the same graph evaluated by torch on the GPU
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd_g, leaves_g = tied_leaves(m)
    moved = {}
    for k, v in sd_g.items():
        if id(v) not in moved:
            moved[id(v)] = v.detach().to(DEV).requires_grad_(v.requires_grad)
        sd_g[k] = moved[id(v)]
    leaves_g = {k: moved[id(v)] for k, v in leaves_g.items()}
    _, _, ups_g = orc.raft_forward_graph(sd_g, im1.to(DEV), im2.to(DEV), iters=GRAD_ITERS, model=name)
    orc.sequence_loss(ups_g, gt.to(DEV), valid.to(DEV), gamma=0.85).backward()

    m = m.to(DEV).train()
    m.freeze_bn()
    preds = m(im1.to(DEV), im2.to(DEV), iters=GRAD_ITERS)
    assert len(preds) == GRAD_ITERS and preds[0].shape == (2, 2, 128, 160)
    loss, metrics = sequence_loss(preds, gt.to(DEV), valid.to(DEV), gamma=0.85)
    assert abs(float(loss.detach()) - float(oloss.detach())) < 1e-4 and 0 <= metrics["1px"] <= 1
    loss.backward()
    gmax = max(float(p.grad.norm()) for p in leaves.values())
    worst = {}
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        grp = "fnet" if k.startswith("fnet.") else "rest"
        for tag, ref in (("cpu", leaves[k].grad), ("gpu", leaves_g[k].grad.cpu())):
            r = float((p.grad.cpu() - ref).norm() / (ref.norm() + 1e-5 * gmax))
            if r > worst.get((grp, tag), (0.0, ""))[0]:
                worst[(grp, tag)] = (r, k)
    print(f"{name}: loss {float(loss.detach()):.6f} (oracle {float(oloss.detach()):.6f}); worst per-parameter relative gradient error "
          + "; ".join(f"{g}/{t} {v[0]:.2e} ({v[1]})" for (g, t), v in sorted(worst.items())))
    for (grp, tag), (r, k) in worst.items():
        assert r < (2e-2 if grp == "fnet" else 2e-3), (grp, tag, k, r)


@pytest.mark.parametrize("mode", ["ffma", "tf32"])
def test_train_step_updates_parameters_and_lowers_the_loss(mode, monkeypatch):
    from rnc.train import fetch_optimizer, train_step
    monkeypatch.setenv("RNC_TRAIN_CONV", mode)
    m = build_model("raft_nc_dbl").to(DEV).train()
    m.freeze_bn()
    im1, im2, gt, valid = (t.to(DEV) for t in train_inputs())
    opt, sched = fetch_optimizer(m, lr=1e-4, num_steps=20)
    before = {k: p.detach().clone() for k, p in m.named_parameters()}
    losses = [float(train_step(m, opt, sched, im1, im2, gt, valid, iters=2)[0]) for _ in range(3)]
    print("losses", losses)
    assert all(torch.isfinite(torch.tensor(losses))) and losses[-1] < losses[0]
    assert all(not torch.equal(before[k], p.detach()) for k, p in m.named_parameters())
    # inference after the step uses re-packed weights (version counters moved) and stays finite
    m.eval()
    with torch.no_grad():
        _, up = m(im1, im2, iters=2, test_mode=True)
    assert torch.isfinite(up).all()


class _FixedReLU:
    """Stand-in for F.relu: the first evaluation records where each ReLU's input is positive, later evaluations (NCHW or
    channel-last) apply the recorded regions in call order.  A few pre-activations of the test encoder lie within fp32
    rounding of zero, and which side of zero an fp32 evaluation puts them on moves the gradients of the parameters upstream
    by up to 4e-3; with the regions fixed, every evaluation computes the same piecewise-linear function and the comparison
    measures arithmetic only."""

    def __init__(self):
        self.masks, self.replay, self.i = [], False, 0

    def start_replay(self):
        self.replay, self.i = True, 0

    def __call__(self, x, inplace=False):
        if not self.replay:
            m = x.detach() > 0
            self.masks.append(m.cpu())
        else:
            m = self.masks[self.i].to(x.device)
            self.i += 1
            if m.shape != x.shape:
                m = m.permute(0, 2, 3, 1)                    # channel-last evaluation
            assert m.shape == x.shape
        return x.mul_(m) if inplace else x * m


@pytest.mark.parametrize("norm", ["instance", "batch"])
def test_encoder_gradients_match_torch_fp64(norm, monkeypatch):
    """BasicEncoder (extractor.py:118-192) forward + backward through the ConvCL / norm graph against the nn.Module's own
    layer graph evaluated in fp64 on the CPU: input gradient flows through both stride-2 residual blocks.  All three
    evaluations use the ReLU regions of the fp64 one (_FixedReLU)."""
    import copy
    from rnc.modules import BasicEncoder
    from rnc.train import encoder_cl, to_cl, to_nchw
    relu = _FixedReLU()
    monkeypatch.setattr(F, "relu", relu)
    torch.manual_seed(5)
    enc = BasicEncoder(output_dim=256, norm_fn=norm).train()
    if norm == "batch":
        enc.eval()                                           # frozen statistics, as after freeze_bn()
    ref = copy.deepcopy(enc).double()
    g = torch.Generator().manual_seed(6)
    x = torch.randn(3, 3, 64, 96, generator=g)
    out_ref = ref(x.double())
    gy = torch.randn(out_ref.shape, generator=g)
    out_ref.backward(gy.double())
    enc = enc.to(DEV)
    # how far does an fp32 GPU evaluation of the SAME layer graph (cuDNN, TF32 off) sit from fp64?  (conditioning yardstick)
    lib = copy.deepcopy(enc)
    torch.backends.cudnn.allow_tf32 = False
    relu.start_replay()
    lib(x.to(DEV)).backward(gy.to(DEV))
    for (k, p), (_, q) in zip(lib.named_parameters(), ref.named_parameters()):
        if q.grad is not None and q.grad.norm() > 1e-9 and rel(p.grad, q.grad) > 1e-4:
            print(f"   [cuDNN fp32 vs fp64] {k}: rel {rel(p.grad, q.grad):.2e}")
    relu.start_replay()
    out = encoder_cl(enc, to_cl(x.to(DEV)))
    assert relu.i == len(relu.masks)
    assert rel(to_nchw(out), out_ref.detach()) < 1e-5
    out.backward(to_cl(gy.to(DEV)))
    worst = 0.0
    for (k, p), (_, q) in zip(enc.named_parameters(), ref.named_parameters()):
        if q.grad is None or q.grad.norm() < 1e-9:
            continue
        r = rel(p.grad, dict(lib.named_parameters())[k].grad)
        worst = max(worst, r)
        assert rel(p.grad, q.grad) < 1e-2, k                 # vs fp64: bounded by fp32 conditioning (cuDNN shows the same)
    print(f"encoder[{norm}]: worst relative gradient difference to cuDNN fp32 on this GPU {worst:.2e}")
    assert worst < (2e-2 if norm == "instance" else 1e-4)    # InstanceNorm chain: fp32-conditioned (cuDNN vs fp64 is as far)
