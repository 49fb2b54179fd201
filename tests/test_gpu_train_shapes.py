"""The training step's kernels checked pointwise against fp64 at the reference's training crops (tests/test_train_shapes.py:
T_SHAPES, the references, compare_mag and its tolerances).

Every case runs real training steps (train mode, freeze_bn(), 2 iterations: no shape or signature depends on the count) with
the `apply` of each training autograd Function wrapped: the wrapper records the call's fp32 inputs and routes every
differentiable input and output through an identity Function that records the gradient passing through it, so each call's
upstream gradient and the input gradients its own kernels produced are known.  After the backward every recorded call (with 2
iterations: every call of the first and of the last iteration, the encoders and the pyramid) is evaluated again by its fp64
reference on its own inputs and upstream gradient, and its output and every input gradient are compared pointwise,
|err| <= tol * mag, with mag the same reference on absolute values.  A failure names the route, shape, Function, call index
and layer, tensor, image, pixel and 128-pixel tile.
"""
import time

import pytest
import torch
import torch.nn.functional as F

from oracle import ncup_oracle as nco
from test_gpu_ncup_finetune import chain_ref, frozen_model
from test_gpu_product_shapes import LibProxy
from test_train_shapes import (NCONV_GRID_ELEMS, NCONV_MAX_BLOCKS, NCONV_WEIGHT_PIX, NCUP_NB, T_SHAPES, compare_mag,
                               compare_tiles, conv_ref, lookup_ref, nconv_ref, nconv_weight_grid, pyramid_ref, ulp_tol)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FUNCTIONS = ("ConvCL", "CorrPyramid", "CorrLookup", "NConv2dFn", "NConvPoolFn", "NcupChainFn")
# a kernel built with flush-to-zero drops terms below the smallest normal fp32 number: an absolute allowance per product
FTZ = 2.0 ** -126


class _Tap(torch.autograd.Function):
    """Identity that records the gradient passing through it in slot[key]."""

    @staticmethod
    def forward(ctx, x, slot, key):
        ctx.slot, ctx.key = slot, key
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        ctx.slot[ctx.key] = g.detach()
        return g, None, None


class Call:
    def __init__(self, fn, idx, args, name):
        self.fn, self.idx, self.name = fn, idx, name
        self.args = tuple(a.detach() if torch.is_tensor(a) else a for a in args)
        self.outs, self.g_in, self.g_out = [], {}, {}


class Capture:
    """Wraps the training autograd Functions of rnc.train for one step."""

    def __init__(self, mp, model=None):
        from rnc import train
        self.calls = []
        self.pnames = {id(p): n for n, p in model.named_parameters()} if model is not None else {}
        for fn in FUNCTIONS:
            cls = getattr(train, fn)
            mp.setattr(cls, "apply", self._wrap(fn, cls.apply))

    def _wrap(self, fn, orig):
        def apply(*args):
            name = self.pnames.get(id(args[1]), "") if fn == "ConvCL" else ""
            call = Call(fn, len(self.calls), args, name)
            self.calls.append(call)
            tapped = [_Tap.apply(a, call.g_in, i) if torch.is_tensor(a) and a.requires_grad else a for i, a in enumerate(args)]
            out = orig(*tapped)
            outs = out if isinstance(out, tuple) else (out,)
            call.outs = [o.detach() for o in outs]
            res = tuple(_Tap.apply(o, call.g_out, k) if o.requires_grad else o for k, o in enumerate(outs))
            return res if isinstance(out, tuple) else res[0]
        return apply


def nchw(t, c=None):
    return (t if c is None else t[..., :c]).permute(0, 3, 1, 2)


# ----------------------------------------------------------------------------------------------------------- per-call checks
class Checker:
    def __init__(self, tag, tf32=False):
        self.tag, self.tf32, self.worst = tag, tf32, {}

    def mag(self, call, what, got, rr, extra_tf32=False):
        ref, mag, n = rr[:3]
        floor = FTZ * n + (rr[3] if len(rr) > 3 else 0.0)          # (lookup_ref: the sample-position allowance)
        tol = ulp_tol(n, tf32=self.tf32 and extra_tf32)
        label = f"[{self.tag}] {call.fn}#{call.idx}{' ' + call.name if call.name else ''} {what}"
        w = compare_mag(label, got, ref, mag, tol, floor=floor)
        key = (call.fn, what.split(" (")[0])
        self.worst[key] = max(self.worst.get(key, 0.0), w)

    def check(self, call):
        getattr(self, call.fn)(call)

    def ConvCL(self, call):
        x, w, b, stride = call.args[:4]
        dil = call.args[4] if len(call.args) > 4 else 1
        cout, cin, kh, kw = w.shape
        y = call.outs[0]
        gy = call.g_out.get(0)
        grads = tuple(k for i, k in ((0, "dx"), (1, "dw"), (2, "db")) if i in call.g_in)
        r = conv_ref(nchw(x, cin), w, b, None if gy is None else nchw(gy, cout), stride, dil, grads)
        self.mag(call, "y", nchw(y, cout), r["y"], extra_tf32=True)
        assert not y[..., cout:].any(), f"[{self.tag}] ConvCL#{call.idx}: pad channels of y are not zero"
        if "dx" in r:
            gx = call.g_in[0]
            self.mag(call, "dx", nchw(gx, cin), r["dx"], extra_tf32=True)
            assert not gx[..., cin:].any(), f"[{self.tag}] ConvCL#{call.idx}: pad channels of dx are not zero"
        if "dw" in r:
            self.mag(call, "dw", call.g_in[1], r["dw"])
        if "db" in r:
            self.mag(call, "db", call.g_in[2], r["db"])

    def _pyr_levels(self, flat, B, D, H, W, levels):
        from rnc import native
        L = native.lib()
        L = L._lib if isinstance(L, LibProxy) else L
        out = []
        for l in range(levels):
            o0, o1 = L.rnc_pyramid_offset(B, D, H, W, l), L.rnc_pyramid_offset(B, D, H, W, l + 1)
            out.append(flat[o0:o1].view(B, H >> l, W >> l, D).permute(0, 3, 1, 2))
        return out

    def CorrPyramid(self, call):
        f2, levels = call.args
        B, H, W, D = f2.shape
        got = self._pyr_levels(call.outs[0], B, D, H, W, levels)
        assert torch.equal(got[0], nchw(f2)), f"[{self.tag}] CorrPyramid#{call.idx}: level 0 is not fmap2"
        for l in range(1, levels):
            prev = got[l - 1].double()
            rr = (F.avg_pool2d(prev, 2, stride=2), F.avg_pool2d(prev.abs(), 2, stride=2), 4)
            self.mag(call, f"level {l} ({H >> l}x{W >> l})", got[l], rr)
        if 0 in call.g_out:
            gl = self._pyr_levels(call.g_out[0], B, D, H, W, levels)
            self.mag(call, "adjoint", nchw(call.g_in[0]), pyramid_ref(gl))

    def CorrLookup(self, call):
        f1, pyr, coords, levels = call.args
        B, H, W, D = f1.shape
        f2l = self._pyr_levels(pyr, B, D, H, W, levels)
        g = call.g_out.get(0)
        r = lookup_ref(nchw(f1), f2l, coords, None if g is None else nchw(g), grads=g is not None)
        self.mag(call, "y", nchw(call.outs[0]), r["y"])
        if g is None:
            return
        self.mag(call, "g_f1", nchw(call.g_in[0]), r["g_f1"])
        gl = self._pyr_levels(call.g_in[1], B, D, H, W, levels)
        for l in range(levels):
            self.mag(call, f"g_f2[{l}] ({H >> l}x{W >> l})", gl[l], r[f"g_f2[{l}]"])

    def NConv2dFn(self, call):
        a = list(call.args) + [None] * (7 - len(call.args))
        data, conf, w, eps, bias, ux, uc = a
        gy, gc = call.g_out.get(0), call.g_out.get(1)
        names = {0: "g_data", 1: "g_conf", 2: "g_w", 4: "g_b", 5: "g_ux", 6: "g_uc"}
        want = tuple(names[i] for i in call.g_in if i in names)
        r = nconv_ref(data, conf, w, bias, eps, ux, uc, gy, gc, want)
        self.mag(call, "y", call.outs[0], r["y"])
        self.mag(call, "conf", call.outs[1], r["conf"])
        if gy is None and gc is None:
            return
        for i, k in names.items():
            if i in call.g_in:
                self.mag(call, k, call.g_in[i], r[k])

    def NConvPoolFn(self, call):
        data, conf, max_pool = call.args
        dr, cr = data.cpu().double().requires_grad_(True), conf.cpu().double().requires_grad_(True)
        with torch.enable_grad():
            xo, co = nco.pool(dr, cr, "max_pooling" if max_pool else "conf_based")
        tag = f"[{self.tag}] NConvPoolFn#{call.idx} {tuple(data.shape)}"
        assert torch.equal(call.outs[0].cpu().double(), xo.detach()), f"{tag}: data"
        assert torch.equal(call.outs[1].cpu().double(), co.detach()), f"{tag}: conf"
        gx, gc = call.g_out.get(0), call.g_out.get(1)
        if gx is None and gc is None:
            return
        gx = torch.zeros_like(xo) if gx is None else gx.cpu().double()
        gc = torch.zeros_like(co) if gc is None else gc.cpu().double()
        rd, rc = torch.autograd.grad([xo, co], [dr, cr], [gx, gc])
        for i, ref in ((0, rd), (1, rc)):
            if i in call.g_in:
                assert torch.equal(call.g_in[i].cpu().double(), ref), f"{tag}: gradient {('g_data', 'g_conf')[i]}"
        self.worst[("NConvPoolFn", "exact")] = 0.0

    def NcupChainFn(self, call):
        x, c, w1, w2, w3, w4, out_scale = call.args
        leaves = [t.detach().double().requires_grad_(i in call.g_in) for i, t in enumerate((x, c, w1, w2, w3, w4))]
        with torch.enable_grad():
            out, _ = chain_ref(leaves[0], leaves[1], leaves[2:], out_scale)
        label = f"[{self.tag}] NcupChainFn#{call.idx}"
        self.worst[("NcupChainFn", "out")] = max(self.worst.get(("NcupChainFn", "out"), 0.0),
                                                 compare_tiles(label + " out", call.outs[0], out.detach(), NCUP_NB, 1e-4))
        g = call.g_out.get(0)
        if g is None:
            return
        req = [t for t in leaves if t.requires_grad]
        gs = dict(zip([i for i, t in enumerate(leaves) if t.requires_grad], torch.autograd.grad(out, req, g.double())))
        for i, k in ((0, "g_x"), (1, "g_conf")):
            if i in gs:
                w = compare_tiles(f"{label} {k}", call.g_in[i], gs[i], NCUP_NB // 4, 1e-4)
                self.worst[("NcupChainFn", k)] = max(self.worst.get(("NcupChainFn", k), 0.0), w)
        gmax = max((float(gs[i].norm()) for i in range(2, 6) if i in gs), default=0.0)
        for i in range(2, 6):
            if i in gs:
                # nconv_out (W4) is scale-invariant, its gradient a difference with heavy cancellation: 1e-3, as
                # test_gpu_ncup_finetune.py::test_fused_chain_matches_per_layer_chain; the others 1e-4
                tol = 1e-3 if i == 5 else 1e-4
                ref = gs[i]
                err = float((call.g_in[i].double() - ref).abs().max())
                bound = tol * (float(ref.abs().max()) + 1e-5 * gmax)
                key = ("NcupChainFn", f"W{i - 1}")
                self.worst[key] = max(self.worst.get(key, 0.0), err / bound)
                print(f"  {label} W{i - 1} {tuple(ref.shape)}: max err {err:.2e} (bound {bound:.2e})")
                assert err <= bound, f"{label} W{i - 1}: max err {err:.3e} > {bound:.3e}"


# ----------------------------------------------------------------------------------------------------------- models, inputs
def _raft_nc_dbl(**overrides):
    import raft_nc_dbl
    from conftest import ref_args
    a = ref_args()
    for k, v in overrides.items():
        setattr(a, k, v)
    torch.manual_seed(1234)
    return raft_nc_dbl.RAFT(a)


def _variant(name):
    return _raft_nc_dbl(freeze_raft=True, **nco.args_overrides(nco.CONFIGS[name]))


def _dilated():
    from oracle.make_golden_wnet import CONFIGS
    num_ch, filter_sz, dilation, _ = CONFIGS["dilated"]
    return _raft_nc_dbl(freeze_raft=True, weights_est_net_num_ch=list(num_ch), weights_est_net_filter_sz=list(filter_sz),
                        weights_est_net_dilation=list(dilation))


def _model(route):
    from conftest import build_model
    if route in ("full", "tf32", "det"):
        m = build_model("raft_nc_dbl")
    elif route == "raft":
        m = build_model("raft")
    elif route == "frozen":
        m = frozen_model()
    elif route.startswith("unet-"):
        m = _variant(route[5:])
    elif route == "wnet-dilated":
        m = _dilated()
    else:
        raise KeyError(route)
    m = m.to(DEV).train()
    m.freeze_bn()
    return m


def train_batch(sid, seed=3):
    """Smooth shifted frames, a smooth ground-truth flow, and a valid mask (20 % valid at the KITTI crop, as its sparse ground
    truth is)."""
    from rnc.synth import smooth_shift_frames
    B, H, W = T_SHAPES[sid]
    im1, im2 = smooth_shift_frames(B, H, W, seed=seed)
    yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    gt = torch.stack([torch.stack([6 * torch.sin(yy / 61 + b) + 0.01 * xx - 2, 4 * torch.cos(xx / 83 + b) - 0.005 * yy + 1])
                      for b in range(B)])
    g = torch.Generator().manual_seed(seed)
    valid = (torch.rand(B, H, W, generator=g) < 0.2).float() if sid == "T3" else torch.ones(B, H, W)
    return [t.to(DEV) for t in (im1, im2, gt, valid)]


def run_step(mp, route, sid, capture=True):
    """One forward + sequence_loss + backward of `route` at `sid` (2 iterations) -> (model, Capture or None)."""
    from rnc.train import sequence_loss
    if route == "tf32":
        mp.setenv("RNC_TRAIN_CONV", "tf32")
    m = _model(route)
    im1, im2, gt, valid = train_batch(sid)
    cap = Capture(mp, m) if capture else None
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(route == "det")
    try:
        preds = m(im1, im2, iters=2)
        loss, _ = sequence_loss(preds, gt, valid, gamma=0.85)
        loss.backward()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    return m, cap


def check_calls(cap, tag, tf32=False):
    chk = Checker(tag, tf32)
    for call in cap.calls:
        chk.check(call)
    return chk


def report(tag, chk, ncalls, t0):
    torch.cuda.synchronize()
    props = torch.cuda.get_device_properties(0)
    print(f"[{tag}] {ncalls} calls checked in {time.time() - t0:.1f} s on {props.name}; peak memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB; worst err/bound: "
          + ", ".join(f"{f}.{k} {v:.2e}" for (f, k), v in sorted(chk.worst.items())))


# ----------------------------------------------------------------------------------------------------------- the cases
CASES = [("full", "T1"), ("full", "T2"), ("full", "T3"), ("tf32", "T1"), ("det", "T2"), ("frozen", "T1"), ("frozen", "T2"),
         ("raft", "T3"), ("unet-paper", "T2"), ("unet-n2_maxpool_bias", "T2"), ("unet-wide", "T2"), ("wnet-dilated", "T1")]
# Functions each route must call (a route that stops reaching one fails here instead of silently checking less)
ROUTE_FUNCTIONS = {
    "full": {"ConvCL", "CorrPyramid", "CorrLookup", "NConv2dFn"},
    "tf32": {"ConvCL", "CorrPyramid", "CorrLookup", "NConv2dFn"},
    "det": {"ConvCL", "CorrPyramid", "CorrLookup", "NConv2dFn"},
    "raft": {"ConvCL", "CorrPyramid", "CorrLookup"},
    "frozen": {"ConvCL", "NcupChainFn"},
    "unet-paper": {"ConvCL", "NConv2dFn", "NConvPoolFn"},
    "unet-n2_maxpool_bias": {"ConvCL", "NConv2dFn", "NConvPoolFn"},
    "unet-wide": {"ConvCL", "NConv2dFn", "NConvPoolFn"},
    "wnet-dilated": {"ConvCL", "NcupChainFn"},
}
_T1_NCONV_INPUTS = []          # (data, conf) of the first NConv2dFn call of each iteration of the full T1 step


@pytest.mark.parametrize("route,sid", CASES, ids=[f"{s}-{r}" for r, s in CASES])
def test_train_step_calls_match_fp64(route, sid, monkeypatch):
    """Every call of the training Functions in one training step of `route` at `sid` against its fp64 reference, pointwise."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    tag = f"{sid} {route}"
    m, cap = run_step(monkeypatch, route, sid)
    fns = {c.fn for c in cap.calls}
    assert fns == ROUTE_FUNCTIONS[route], f"[{tag}] Functions called: {sorted(fns)}"
    if route == "wnet-dilated":
        assert any(c.fn == "ConvCL" and (c.args[4] if len(c.args) > 4 else 1) > 1 for c in cap.calls), "no dilated layer"
    if route in ("raft",):
        assert any(c.name.startswith("update_block.mask.") for c in cap.calls), "the mask head did not run on ConvCL"
    if route == "full" and sid == "T1":
        _T1_NCONV_INPUTS[:] = [c.args[:2] for c in cap.calls if c.fn == "NConv2dFn" and c.args[0].shape[1] == 1]
    chk = check_calls(cap, tag, tf32=route == "tf32")
    report(tag, chk, len(cap.calls), t0)
    del m, cap


def test_nconv_chain_past_the_weight_kernels_block_cap(monkeypatch):
    """T1x2: the shipped network's per-layer NConv2dFn chain on the zero-stuffed planes of all 6 samples of a T1 batch
    (N = 12 planes of 400x720, 3.46 M pixels: the weight-gradient kernel's grid is capped and loops), every layer against fp64.
    The inputs are those the T1 training step fed the chain (its two iterations' nconv_in inputs, side by side)."""
    from conftest import build_model
    from rnc.train import nconv_unet_train
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    if len(_T1_NCONV_INPUTS) != 2:
        with monkeypatch.context() as mp:
            _, cap = run_step(mp, "full", "T1")
        _T1_NCONV_INPUTS[:] = [c.args[:2] for c in cap.calls if c.fn == "NConv2dFn" and c.args[0].shape[1] == 1]
        del cap
    assert len(_T1_NCONV_INPUTS) == 2
    data = torch.cat([d for d, _ in _T1_NCONV_INPUTS]).requires_grad_(True)
    conf = torch.cat([c for _, c in _T1_NCONV_INPUTS]).requires_grad_(True)
    N, _, H, W = data.shape
    B6, Hi, Wi = T_SHAPES["T1x2"]
    assert (N, H, W) == (2 * B6, Hi, Wi)
    pix = N * H * W
    assert pix > NCONV_WEIGHT_PIX and nconv_weight_grid(pix) == NCONV_MAX_BLOCKS and pix > 12 * NCONV_GRID_ELEMS
    net = build_model("raft_nc_dbl").upsampler.interpolation_net.to(DEV)
    with monkeypatch.context() as mp:
        cap = Capture(mp, None)
        out, cout = nconv_unet_train(net, data, conf)
        g = torch.randn(out.shape, generator=torch.Generator(device=DEV).manual_seed(9), device=DEV) * (cout.detach() > 0)
        out.backward(g)
    assert [c.fn for c in cap.calls] == ["NConv2dFn"] * 4
    chk = check_calls(cap, "T1x2 nconv chain")
    report("T1x2 nconv chain", chk, len(cap.calls), t0)


# ----------------------------------------------------------------------------------------------------------- coverage guard
# Every librnc entry point a training step of the routes above calls at T3 -> the case that checks it.
STEP = "test_train_step_calls_match_fp64"
PRODUCT = "test_gpu_product_shapes.py::test_update_iteration_layer_by_layer (inference entry point of the frozen trunk's " \
          "forward, checked at S1-S4)"
TRAIN_COVERAGE = {
    "rnc_conv2d_cl_fwd": f"{STEP}: ConvCL y and dx (exact fp32 route)",
    "rnc_conv2d_cl_wgrad_workspace_bytes": "size query",
    "rnc_conv2d_cl_wgrad_det": f"{STEP}: ConvCL dw, db",
    "rnc_conv2d_cl_dil_fwd": f"{STEP}[T1-wnet-dilated]: ConvCL y and dx of the dilated layers",
    "rnc_conv2d_cl_wgrad_dil_workspace_bytes": "size query",
    "rnc_conv2d_cl_wgrad_dil_det": f"{STEP}[T1-wnet-dilated]: ConvCL dw, db of the dilated layers",
    "rnc_f32_to_tf32_split": f"{STEP}[T1-tf32]: ConvCL y and dx (tensor-core operands)",
    "rnc_conv2d_umma_fwd": f"{STEP}[T1-tf32]: ConvCL y and dx; and {PRODUCT}",
    "rnc_pyramid_offset": "size query",
    "rnc_fmap_pyramid": f"{STEP}: CorrPyramid 'level l'; and {PRODUCT}",
    "rnc_pyramid_pool_bwd": f"{STEP}: CorrPyramid 'adjoint'",
    "rnc_corr_lookup_fwd": f"{STEP}: CorrLookup y",
    "rnc_corr_lookup_bwd": f"{STEP}: CorrLookup g_f1, g_f2[l]",
    "rnc_corr_lookup_bwd_workspace_bytes": "size query",
    "rnc_corr_lookup_bwd_det": f"{STEP}[T2-det]: CorrLookup g_f1, g_f2[l]",
    "rnc_nconv2d_fwd": f"{STEP}: NConv2dFn y, conf; test_nconv_chain_past_the_weight_kernels_block_cap",
    "rnc_nconv2d_bwd_workspace_bytes": "size query",
    "rnc_nconv2d_bwd": f"{STEP}: NConv2dFn g_data, g_conf, g_w, g_b, g_ux, g_uc; test_nconv_chain_past_the_weight_kernels_block_cap",
    "rnc_nconv_pool2_fwd": f"{STEP}[T2-unet-*]: NConvPoolFn data, conf (exact)",
    "rnc_nconv_pool2_bwd": f"{STEP}[T2-unet-*]: NConvPoolFn gradients (exact)",
    "rnc_ncup_train_fwd": f"{STEP}[*-frozen, T1-wnet-dilated]: NcupChainFn out",
    "rnc_ncup_bwd_workspace_bytes": "size query",
    "rnc_ncup_bwd": f"{STEP}[*-frozen, T1-wnet-dilated]: NcupChainFn g_conf, W1-W4",
    # the frozen trunk's forward runs on the inference engine
    "rnc_stem_window_prep": PRODUCT,
    "rnc_instnorm_finalize": PRODUCT,
    "rnc_instnorm_apply": PRODUCT,
    "rnc_conv_umma_tiles": "size query",
    "rnc_corr_lookup_umma_workspace_bytes": "size query",
    "rnc_f32_to_f16": PRODUCT,
    "rnc_coords_init": PRODUCT,
    "rnc_corr_lookup_umma_fwd": PRODUCT,
    "rnc_flow_im2col7_split_fwd": PRODUCT,
    "rnc_flow_tap_gather_fwd": PRODUCT,
    "rnc_cl_to_nchw": PRODUCT,
    "rnc_flow_x2_fwd": PRODUCT,
    "rnc_ncup_guidance_fwd": PRODUCT,
}


class _Names:
    def __init__(self):
        self.called = set()

    def native(self, name, fn, args):
        self.called.add(name)
        return fn(*args)


def test_train_coverage_guard(monkeypatch):
    """The librnc entry points called by one training step of every route above at T3 are exactly TRAIN_COVERAGE's: a kernel
    added to the training step fails here until it has a pointwise check."""
    from rnc import native
    rec = _Names()
    for route in dict.fromkeys(r for r, _ in CASES):
        with monkeypatch.context() as mp:
            mp.setattr(native, "_lib", LibProxy(native.lib(), rec))
            run_step(mp, route, "T3", capture=False)
    called = rec.called
    missing = set(TRAIN_COVERAGE) - called
    assert called - set(TRAIN_COVERAGE) == set(), f"entry points without a pointwise check: {sorted(called - set(TRAIN_COVERAGE))}"
    assert missing == set(), f"table lists entry points the steps no longer call: {sorted(missing)}"
