"""Unsupervised fine-tuning on the GPU (rnc/unsupervised.py, csrc/photometric.cu, model.forward(..., bidirectional=True),
rnc.train.unsupervised_step): the census and smoothness kernels against the fp64 restatements at the shapes training uses,
their determinism and batch independence, the bidirectional forward on every route against the forward of the concatenated
pairs, one encoder pass per frame, the loss's parameter gradients against the host restatements in fp32, and a few steps."""
import pytest
import torch

from conftest import build_model
from rnc.native import rnc
from rnc.synth import frames
from rnc.unsupervised import (_census_fwd, census_loss, host_census_loss, host_smoothness_loss, host_unsupervised_loss,
                              smoothness_loss, unsupervised_loss)
from test_gpu_ncup_finetune import frozen_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = [(1, 8, 8), (3, 48, 64), (4, 384, 512), (2, 440, 1024)]
H, W, ITERS = 128, 160, 3


@pytest.fixture
def det(monkeypatch):
    monkeypatch.setenv("RNC_LOOKUP", "ffma")
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def loss_inputs(N, h, w, seed=0):
    """Channel-last images in 0..255, a flow sliced from a 2N-row channel-last tensor (about 5 % of its samples sent out of the
    frame), and random masks with an all-zero row when N > 1."""
    g = torch.Generator().manual_seed(seed)
    i1 = (torch.rand(N, h, w, 3, generator=g) * 255).to(DEV).permute(0, 3, 1, 2)
    i2 = (torch.rand(N, h, w, 3, generator=g) * 255).to(DEV).permute(0, 3, 1, 2)
    big = torch.randn(2 * N, h, w, 2, generator=g) * 4
    far = torch.rand(2 * N, h, w, generator=g) < 0.05
    big[..., 0][far] += 2.0 * w
    flow = big.to(DEV).permute(0, 3, 1, 2)[N:]
    mask = torch.rand(N, h, w, generator=g) < 0.8
    if N > 1:
        mask[N - 1] = False
    return i1, i2, flow, mask.to(DEV)


def snapped(flow):
    """flow in fp64 with x + F and y + F rounded to float32 as the kernels round them, so that the fp64 restatement takes its
    bilinear taps at the same floor (elsewhere the derivative of the sample jumps)."""
    h, w = flow.shape[-2:]
    xs = torch.arange(w, device=flow.device, dtype=torch.float32).view(1, w)
    ys = torch.arange(h, device=flow.device, dtype=torch.float32).view(h, 1)
    return torch.stack([(xs + flow[:, 0]).double() - xs.double(), (ys + flow[:, 1]).double() - ys.double()], 1)


def grad_of(fn, flow, *args):
    f = flow.detach().clone().requires_grad_()
    loss = fn(*args, f)
    loss.backward()
    return loss.detach(), f.grad


@pytest.mark.parametrize("N,h,w", SHAPES)
def test_census_loss_matches_fp64(N, h, w):
    i1, i2, flow, mask = loss_inputs(N, h, w, seed=N + h)
    loss, grad = grad_of(lambda f: census_loss(i1, i2, f, mask), flow)
    ref, ref_grad = grad_of(lambda f: host_census_loss(i1.double(), i2.double(), f, mask), snapped(flow))
    rel = abs(float(loss) - float(ref)) / abs(float(ref))
    gerr = float((grad.double() - ref_grad).abs().max() / ref_grad.abs().max())
    print(f"census {N}x{h}x{w}: loss {float(loss):.8f} rel err {rel:.2e}; grad max err / max|grad| {gerr:.2e}")
    assert rel < 1e-5 and gerr < 1e-4


@pytest.mark.parametrize("N,h,w", SHAPES)
def test_smoothness_loss_matches_fp64(N, h, w):
    i1, _, flow, _ = loss_inputs(N, h, w, seed=N + w)
    loss, grad = grad_of(lambda f: smoothness_loss(i1, f), flow)
    ref, ref_grad = grad_of(lambda f: host_smoothness_loss(i1.double(), f), flow.double())
    rel = abs(float(loss) - float(ref)) / abs(float(ref))
    gerr = float((grad.double() - ref_grad).abs().max() / ref_grad.abs().max())
    print(f"smoothness {N}x{h}x{w}: loss {float(loss):.8f} rel err {rel:.2e}; grad max err / max|grad| {gerr:.2e}")
    assert rel < 1e-5 and gerr < 1e-4


def test_an_all_zero_mask_gives_zero_loss_and_gradient():
    i1, i2, flow, mask = loss_inputs(2, 48, 64)
    loss, grad = grad_of(lambda f: census_loss(i1, i2, f, torch.zeros_like(mask)), flow)
    assert float(loss) == 0.0 and not grad.any()


def raw(i1, i2, flow, mask):
    """Per-row results of both kernels: S, M, the census gradient at scale 1, the smoothness row sums and its gradient at
    scales (1, 1)."""
    N, _, h, w = flow.shape
    S, M, _, state = _census_fwd(i1, i2, flow, mask)
    one = torch.ones(2, dtype=torch.float32, device=DEV)
    gc = torch.empty(N, 2, h, w, device=DEV)
    rnc.census_loss_bwd(state, N, h, w, one, gc)
    sx, sy = (torch.empty(N, dtype=torch.float64, device=DEV) for _ in range(2))
    total = torch.empty(2, dtype=torch.float64, device=DEV)
    ws = torch.empty(rnc.smoothness_workspace_bytes(N, h, w), dtype=torch.uint8, device=DEV)
    f, im = flow.float(), i1.float()
    rnc.smoothness_fwd(im, *im.stride(), f, *f.stride(), N, h, w, 150.0, sx, sy, total, ws, ws.numel())
    gs = torch.empty(N, 2, h, w, device=DEV)
    rnc.smoothness_bwd(im, *im.stride(), f, *f.stride(), N, h, w, 150.0, one, gs)
    return S, M, gc, sx, sy, gs


def test_bit_identical_run_to_run_and_independent_of_the_batch():
    i1, i2, flow, mask = loss_inputs(3, 384, 512, seed=5)
    mask[2] = mask[0]
    a, b = raw(i1, i2, flow, mask), raw(i1, i2, flow, mask)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    one = raw(i1[1:2], i2[1:2], flow[1:2], mask[1:2])
    assert all(torch.equal(x[1:2], y) for x, y in zip(a, one))
    l1, g1 = grad_of(lambda f: census_loss(i1, i2, f, mask) + 2 * smoothness_loss(i1, f), flow)
    l2, g2 = grad_of(lambda f: census_loss(i1, i2, f, mask) + 2 * smoothness_loss(i1, f), flow)
    assert torch.equal(l1, l2) and torch.equal(g1, g2)


# ------------------------------------------------------------------------------------------------ bidirectional forward


def pairs(B, seed=3):
    im1, im2 = frames(B, H, W, seed=seed)
    return im1.to(DEV), im2.to(DEV)


def epe(a, b):
    return (a - b).pow(2).sum(1).sqrt().mean().item()


def fixed_loss(preds, seed=0):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(preds[0].shape, generator=g).to(DEV)
    return sum((p * w).sum() * (i + 1) for i, p in enumerate(preds))


@pytest.mark.parametrize("mode", ["det", "default"])
def test_inference_routes_equal_the_concatenated_forward(mode, request):
    if mode == "det":
        request.getfixturevalue("det")
    m = build_model("raft_nc_dbl").to(DEV)
    im1, im2 = pairs(2)
    cat1, cat2 = torch.cat([im1, im2]), torch.cat([im2, im1])
    with torch.no_grad():
        for _ in range(2):                                   # eager, then graph replay
            lo, up = m(im1, im2, iters=ITERS, test_mode=True, bidirectional=True)
            rlo, rup = m(cat1, cat2, iters=ITERS, test_mode=True)
            if mode == "det":
                assert torch.equal(lo, rlo) and torch.equal(up, rup)
            else:
                assert epe(up, rup) < 1e-4
        preds = m(im1, im2, iters=ITERS, bidirectional=True)
        ref = m(cat1, cat2, iters=ITERS)
    assert len(preds) == ITERS and preds[0].shape == (4, 2, H, W)
    for p, r in zip(preds, ref):
        assert torch.equal(p, r) if mode == "det" else epe(p, r) < 1e-4


@pytest.mark.parametrize("mode", ["det", "default"])
def test_frozen_trunk_route_equals_the_concatenated_forward(mode, request):
    if mode == "det":
        request.getfixturevalue("det")
    m = frozen_model().to(DEV).train()
    m.freeze_bn()
    im1, im2 = pairs(2)
    out = []
    for args, kw in (((im1, im2), dict(bidirectional=True)), ((torch.cat([im1, im2]), torch.cat([im2, im1])), {})):
        m.zero_grad()
        preds = m(*args, iters=ITERS, **kw)
        fixed_loss(preds).backward()
        out.append(([p.detach() for p in preds], {k: p.grad.clone() for k, p in m.named_parameters() if p.requires_grad}))
    (pa, ga), (pb, gb) = out
    assert ga and all(k.startswith("upsampler.") for k in ga)
    if mode == "det":
        assert all(torch.equal(a, b) for a, b in zip(pa, pb))
        assert all(torch.equal(ga[k], gb[k]) for k in ga)
    else:
        assert all(epe(a, b) < 1e-4 for a, b in zip(pa, pb))
        for k in ga:
            assert float((ga[k] - gb[k]).norm() / (gb[k].norm() + 1e-30)) < 2e-3, k


def param_grad_errors(ga, gb):
    gmax = max(float(g.norm()) for g in gb.values())
    worst = {}
    for k, ref in gb.items():
        grp = "fnet" if k.startswith("fnet.") else "rest"
        r = float((ga[k] - ref).norm() / (ref.norm() + 1e-5 * gmax))
        worst[grp] = max(worst.get(grp, 0.0), r)
    return worst


def check_param_grads(ga, gb):
    assert set(ga) == set(gb)
    worst = param_grad_errors(ga, gb)
    print("worst per-parameter relative gradient error", worst)
    for grp, r in worst.items():
        assert r < (2e-2 if grp == "fnet" else 2e-3), (grp, r)


def full_model():
    m = build_model("raft_nc_dbl").to(DEV).train()
    m.freeze_bn()
    return m


def test_full_route_equals_the_concatenated_forward():
    m = full_model()
    im1, im2 = pairs(1)
    out = []
    for args, kw in (((im1, im2), dict(bidirectional=True)), ((torch.cat([im1, im2]), torch.cat([im2, im1])), {})):
        m.zero_grad()
        preds = m(*args, iters=ITERS, **kw)
        fixed_loss(preds).backward()
        out.append(([p.detach() for p in preds], {k: p.grad.clone() for k, p in m.named_parameters()}))
    (pa, ga), (pb, gb) = out
    assert all(epe(a, b) < 1e-4 for a, b in zip(pa, pb))
    check_param_grads(ga, gb)


def test_each_frame_is_encoded_once_on_every_route(monkeypatch):
    from rnc import train
    from rnc.encoder_umma import EncoderRunner
    monkeypatch.setenv("RNC_GRAPH", "0")
    B = 2
    im1, im2 = pairs(B)
    m = build_model("raft_nc_dbl").to(DEV)
    if m.engine().mode != "umma":
        pytest.skip("tensor-core encoders only")
    images = {"instance": 0, "batch": 0}
    trunk = EncoderRunner._trunk

    def counted(self, pk, bufs, image, N, Hin, Win):
        images[pk.kind] += N
        return trunk(self, pk, bufs, image, N, Hin, Win)

    monkeypatch.setattr(EncoderRunner, "_trunk", counted)
    with torch.no_grad():
        m(im1, im2, iters=1, test_mode=True, bidirectional=True)
        assert images == {"instance": 2 * B, "batch": 2 * B}, images
        m(im1, im2, iters=1, bidirectional=True)
        assert images == {"instance": 4 * B, "batch": 4 * B}, images
    f = frozen_model().to(DEV).train()
    f.freeze_bn()
    f(im1, im2, iters=1, bidirectional=True)
    assert images == {"instance": 6 * B, "batch": 6 * B}, images

    calls = []
    encoder = train.encoder_cl

    def counted_cl(enc, x):
        calls.append(x.shape[0])
        return encoder(enc, x)

    monkeypatch.setattr(train, "encoder_cl", counted_cl)
    full_model()(im1, im2, iters=1, bidirectional=True)
    assert calls == [2 * B, 2 * B], calls


def test_loss_gradients_match_the_host_restatement_in_fp32(det):
    m = full_model()
    im1, im2 = pairs(1, seed=9)
    out = []
    for loss_fn in (unsupervised_loss, host_unsupervised_loss):
        m.zero_grad()
        preds = m(im1, im2, iters=ITERS, bidirectional=True)
        # an untrained model's two directions disagree everywhere: a loose alpha2 keeps the census term in the loss
        loss, metrics = loss_fn(preds, im1, im2, alpha2=1e4)
        loss.backward()
        out.append((float(loss.detach()), metrics, {k: p.grad.clone() for k, p in m.named_parameters()}))
    (la, ma, ga), (lb, mb, gb) = out
    print("loss", la, lb, ma)
    assert abs(la - lb) / abs(lb) < 1e-4
    assert ma["occluded_fw"] == mb["occluded_fw"] < 0.5 and ma["occluded_bw"] == mb["occluded_bw"] < 0.5
    check_param_grads(ga, gb)


def run_steps(route, steps=2, seed=0):
    from rnc.train import fetch_optimizer, unsupervised_step
    m = full_model() if route == "full" else frozen_model().to(DEV).train()
    m.freeze_bn()
    opt, sched = fetch_optimizer(m, lr=1e-4, num_steps=10)
    im1, im2 = pairs(1, seed=seed + 1)
    losses = []
    for _ in range(steps):
        loss, metrics = unsupervised_step(m, opt, sched, im1, im2, iters=2)
        losses.append(float(loss))
        for k, p in m.named_parameters():
            if p.requires_grad:
                assert p.grad is not None and torch.isfinite(p.grad).all(), k
                assert route == "full" or k.startswith("upsampler."), k
            else:
                assert p.grad is None, k
    return losses, {k: p.detach().clone() for k, p in m.named_parameters()}


@pytest.mark.parametrize("route", ["full", "frozen"])
def test_unsupervised_step_is_finite_and_deterministic(route, det):
    la, pa = run_steps(route)
    lb, pb = run_steps(route)
    print(route, "losses", la)
    assert all(torch.isfinite(torch.tensor(la)))
    assert la == lb and all(torch.equal(pa[k], pb[k]) for k in pa)
