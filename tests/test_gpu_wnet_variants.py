"""Weights-net (Simple) configurations beyond the shipped one, on the GPU: the dilated convolution kernels (fp16 hi/lo split,
TF32 and exact fp32) and their gradients against fp64, the Simple seam and its gradients against the reference's goldens,
whole-model flows on both engines (eager and graph-replayed), training gradients (full and frozen-trunk) against the
reference's pinned ones, and bit-identical deterministic steps."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, ref_args

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

with open(os.path.join(ROOT, "tests", "golden", "wnet_cfg_meta.json")) as _f:
    CONFIGS = json.load(_f)["configs"]
MODEL_CONFIGS = ("dilated", "wide_k")        # oracle/make_golden_wnet.py:MODEL_CONFIGS

# (B, H, W, cin, cout, k, dil): odd sizes, an image smaller than the dilated footprint, widths that are not multiples of 32,
# and a phase wide enough for the row-halo tiling
LAYERS = [(2, 23, 37, 40, 48, 3, 2), (1, 5, 7, 20, 24, 7, 4), (2, 19, 29, 132, 96, 5, 3), (1, 30, 300, 64, 32, 3, 2)]


@pytest.fixture(scope="module")
def wg():
    z = np.load(os.path.join(ROOT, "tests", "golden", "wnet_cfg.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


@pytest.fixture(scope="module")
def wmeta():
    with open(os.path.join(ROOT, "tests", "golden", "wnet_cfg_meta.json")) as f:
        return json.load(f)


def rel(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


def layer_data(B, H, W, cin, cout, k, dil):
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + k + dil)
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=(k // 2) * dil, dilation=dil)
    return x, w, b, ref


@pytest.mark.parametrize("shape", LAYERS)
def test_dilated_conv_operand_forms_match_fp64(shape):
    """The dilated convolution's forward on each operand form against fp64: exact fp32 (CUDA cores), the training path's TF32
    hi/lo planes, and the inference weights net's fp16 hi/lo split, launched directly."""
    from rnc import native
    from rnc.engine import engine_for
    from rnc.engine_umma import UmmaWeights
    from rnc.native import rnc
    from rnc.train import _conv_launch, _conv_launch_tf32, _packed, to_cl
    B, H, W, cin, cout, k, dil = shape
    x, w, b, ref = layer_data(*shape)
    ref_cl = ref.permute(0, 2, 3, 1)
    eng = engine_for(DEV)
    Cx = (cin + 7) // 8 * 8
    xc = to_cl(x.to(DEV), pad_to=Cx)
    scale = ref.abs().max().item()
    exact = _conv_launch(eng, xc, _packed(w.to(DEV), "fwd", Cx), cout, k, k, b.to(DEV), dil=dil)
    assert (exact[..., :cout].cpu().double() - ref_cl).abs().max() < 5e-6 * scale
    # the epilogue stores whole 32-channel chunks: an output pitch of ceil32(cout)
    ldo = (cout + 31) // 32 * 32
    tf32 = _conv_launch_tf32(eng, xc, UmmaWeights(w.to(DEV), None, [Cx], tf32=True), ldo, 1, b.to(DEV), dil)
    # fp16 hi/lo split operands, the format of the inference weights net (UmmaWnet)
    M = B * H * W
    hi, lo = (torch.empty(M, Cx, dtype=torch.float16, device=DEV) for _ in range(2))
    rnc.f32_to_split(xc, Cx, Cx, M, hi, lo, Cx, 0)
    f16 = torch.empty(B, H, W, ldo, dtype=torch.float32, device=DEV)
    eng.uconv(B, H, W, (hi.data_ptr(), lo.data_ptr()), Cx, Cx, UmmaWeights(w.to(DEV), b.to(DEV), [Cx]), native.EPI_LINEAR,
              out_f32=f16.data_ptr(), ldo_f32=ldo, dil=dil)
    for fmt, out in (("tf32", tf32), ("f16", f16)):
        assert (out[..., :cout].cpu().double() - ref_cl).abs().max() < 2e-5 * scale, fmt


@pytest.mark.parametrize("shape", LAYERS)
def test_dilated_conv_gradients_match_fp64_and_repeat(shape):
    from rnc.train import ConvCL, to_cl
    B, H, W, cin, cout, k, dil = shape
    x, w, b, _ = layer_data(*shape)
    xr, wr, br = (t.double().requires_grad_(True) for t in (x, w, b))
    y = F.conv2d(xr, wr, br, padding=(k // 2) * dil, dilation=dil)
    gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(4))
    y.backward(gy.double())

    def run():
        xd = to_cl(x.to(DEV)).requires_grad_(True)
        wd, bd = w.to(DEV).requires_grad_(True), b.to(DEV).requires_grad_(True)
        yd = ConvCL.apply(xd, wd, bd, 1, dil)
        yd.backward(to_cl(gy.to(DEV), pad_to=yd.shape[-1]))
        return xd.grad[..., :cin].permute(0, 3, 1, 2).cpu(), wd.grad.cpu(), bd.grad.cpu()

    gx, gw, gb = run()
    assert rel(gx, xr.grad) < 5e-6 and rel(gw, wr.grad) < 5e-6 and rel(gb, br.grad) < 5e-6
    gx2, gw2, gb2 = run()                     # fixed-order weight-gradient sum: bit-identical from call to call
    assert torch.equal(gx, gx2) and torch.equal(gw, gw2) and torch.equal(gb, gb2)


def golden_simple(wmeta, name):
    """The drop-in Simple with the golden's seeded weights and running statistics (their SHAs are the reference's)."""
    from interp_weights_est import Simple
    from oracle.make_golden import tensor_sha
    from oracle.make_golden_wnet import set_running_stats
    num_ch, filter_sz, dilation, dataset = CONFIGS[name]
    torch.manual_seed(4321)
    net = Simple(num_ch=[130] + num_ch, out_ch=2, use_bn=dataset == "sintel", filter_sz=filter_sz, dilation=dilation,
                 final_act=torch.sigmoid)
    set_running_stats(net, 7)
    assert {k: tensor_sha(v) for k, v in net.state_dict().items()} == wmeta[f"{name}_simple_sha"]
    return net.to(DEV)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_simple_seam_matches_reference(wg, wmeta, name):
    from oracle.make_golden_wnet import simple_input
    net = golden_simple(wmeta, name).eval()
    with torch.no_grad():
        out = net(simple_input().to(DEV))
    assert (out.cpu() - wg[f"{name}_eval_out"]).abs().max() < 1e-5


@pytest.mark.parametrize("mode", ["eval", "train"])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_simple_gradients_match_reference(wg, wmeta, name, mode):
    """Outputs, and the input and parameter gradients' norms and seeded projections, against the reference's."""
    from oracle.make_golden_r2 import grad_fixture
    from oracle.make_golden_wnet import simple_input
    net = golden_simple(wmeta, name).train(mode == "train")
    x = simple_input().to(DEV).requires_grad_(True)
    out = net(x)
    assert (out.detach().cpu() - wg[f"{name}_{mode}_out"]).abs().max() < 1e-5
    p = torch.randn(out.shape, generator=torch.Generator().manual_seed(5)).to(DEV)
    (p * out).sum().backward()
    grads = {"input": x.grad, **{pn: prm.grad for pn, prm in net.named_parameters()}}
    fix, ref = grad_fixture({k: g.cpu() for k, g in grads.items()}), wmeta[f"{name}_simple_{mode}_grads"]
    gmax = max(v[0] for v in ref.values())
    for k, g in grads.items():
        # a bias ahead of train-mode BatchNorm has a zero gradient in exact arithmetic: its rounding noise is bounded by gmax
        tol = 1e-4 * ref[k][0] + 1e-6 * gmax
        assert abs(fix[k][0] - ref[k][0]) < tol, (k, fix[k][0], ref[k][0])
        assert all(abs(a - b) < tol * g.numel() ** 0.5 for a, b in zip(fix[k][1:], ref[k][1:])), k


def variant_model(name, seed=1234, freeze=False):
    import raft_nc_dbl
    num_ch, filter_sz, dilation, dataset = CONFIGS[name]
    a = ref_args(dataset)
    a.weights_est_net_num_ch, a.weights_est_net_filter_sz, a.weights_est_net_dilation = num_ch, filter_sz, dilation
    a.freeze_raft = freeze
    torch.manual_seed(seed)
    return raft_nc_dbl.RAFT(a).eval()


@pytest.mark.parametrize("engine", ["umma", "ffma"])
@pytest.mark.parametrize("name", MODEL_CONFIGS)
def test_model_flows_match_reference_and_graph_replay(wg, name, engine, monkeypatch):
    from rnc.synth import frames
    monkeypatch.setenv("RNC_CONV", engine)
    m = variant_model(name).to(DEV)
    im1, im2 = (t.to(DEV) for t in frames(1, 128, 256))
    outs = []
    with torch.no_grad():
        for _ in range(3):                        # eager, capture, replay (the exact engine runs eagerly every time)
            lo, up = m(im1, im2, iters=4, test_mode=True)
            outs.append((lo.clone(), up.clone()))
    for lo, up in outs[1:]:
        assert torch.equal(lo, outs[0][0]) and torch.equal(up, outs[0][1])
    for key, got in (("flow_low", outs[0][0]), ("flow_up", outs[0][1])):
        epe = (got.cpu() - wg[f"{name}_cfg1_{key}"]).pow(2).sum(1).sqrt().mean().item()
        assert epe < 1e-3, (key, epe)


def _check_pinned(meta, name, grads, bound_of):
    from oracle.make_golden_r2 import grad_fixture
    ref, gmax = meta[f"{name}_train_grads"], meta[f"{name}_train_grad_norm_max"]
    fix = grad_fixture({k: g.cpu() for k, g in grads.items()})
    for k in grads:
        tol = bound_of(k) * ref[k][0] + 1e-5 * gmax
        n = grads[k].numel() ** 0.5
        assert abs(fix[k][0] - ref[k][0]) < tol, (k, fix[k][0], ref[k][0])
        assert all(abs(x - y) < tol * n for x, y in zip(fix[k][1:], ref[k][1:])), k


def _train_grads(name, freeze=False):
    from oracle.make_golden_r2 import GRAD_ITERS, train_inputs
    from rnc.train import sequence_loss
    m = variant_model(name, freeze=freeze).to(DEV).train()
    m.freeze_bn()
    im1, im2, gt, valid = (t.to(DEV) for t in train_inputs())
    loss, _ = sequence_loss(m(im1, im2, iters=GRAD_ITERS), gt, valid, gamma=0.85)
    loss.backward()
    return float(loss.detach()), m


@pytest.mark.parametrize("name", MODEL_CONFIGS)
def test_full_training_matches_pinned_reference_gradients(wmeta, name):
    loss, m = _train_grads(name)
    assert abs(loss - wmeta[f"{name}_train_loss"]) < 1e-4
    assert sorted(k for k, p in m.named_parameters() if p.grad is None) == sorted(wmeta[f"{name}_train_grad_none"])
    grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    _check_pinned(wmeta, name, grads, lambda k: 2e-2 if k.startswith("fnet.") else 2e-3)


@pytest.mark.parametrize("name", MODEL_CONFIGS)
def test_frozen_trunk_matches_pinned_reference_gradients(wmeta, name):
    loss, m = _train_grads(name, freeze=True)
    assert abs(loss - wmeta[f"{name}_train_loss"]) < 1e-4
    grads = {k: p.grad for k, p in m.named_parameters() if k.startswith("upsampler.")}
    assert grads and all(g is not None for g in grads.values())
    assert all(p.grad is None for k, p in m.named_parameters() if not k.startswith("upsampler."))
    _check_pinned(wmeta, name, grads, lambda k: 2e-3)


def test_tf32_training_gradients_match_pinned_reference(wmeta, monkeypatch):
    monkeypatch.setenv("RNC_TRAIN_CONV", "tf32")
    loss, m = _train_grads("dilated", freeze=True)
    grads = {k: p.grad for k, p in m.named_parameters() if k.startswith("upsampler.")}
    _check_pinned(wmeta, "dilated", grads, lambda k: 2e-3)


@pytest.mark.parametrize("freeze", [False, True])
def test_deterministic_steps_are_bit_identical(freeze):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            loss, m = _train_grads("wide_k", freeze=freeze)
            runs.append((loss, {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}))
    finally:
        torch.use_deterministic_algorithms(prev)
    assert runs[0][0] == runs[1][0]
    assert runs[0][1].keys() == runs[1][1].keys() and all(torch.equal(v, runs[1][1][k]) for k, v in runs[0][1].items())
