"""InstanceNorm statistics against fp64 where they are fragile: |mean| >> std (flat frames), constant channels, and a model
whose BatchNorm statistics and weight scales look trained (tests/test_norm_conditioning.py: stimuli, transform, bounds).

  (a) the three statistics routes (fused convolution epilogue + rnc_instnorm_finalize, rnc_instnorm_stats,
      rnc_instnorm_stats_det) and rnc_instnorm_apply at |mean|/std from 0 to 1e4, at the encoders' shapes;
  (b) fnet on near-uniform frames, every norm checked on its own fp32 input (teacher forcing: a whole-encoder fp64 reference
      would fail even for exact kernels, because the stem's own fp32 rounding is amplified ~2000x on a grey frame);
  (c) the layer-by-layer check of test_gpu_product_shapes.py on a trained-like model, with per-channel bounds;
  (d) end to end on a grey pair and a grey + noise pair against the oracle.
"""
import math

import pytest
import torch

from conftest import build_model
from test_conv_error_model import C_A, U, a_tol, conv_split_ref, fp64_floor, split_bound
from test_gpu_product_shapes import CONFIGS, Recorder, expected_stages, stimulus
from test_train_shapes import compare_mag
from test_norm_conditioning import (EPS, apply_bound, apply_ref, compare_per_channel, conditioned, near_uniform_frames,
                                    norm_ref, stats_bounds, trained_like, worst_at)
from test_product_shapes import SHAPES, Mismatch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (N, H, W, C) of fnet's norms on the benchmark frames (16 = both frames of B = 8 at 440x1024), and a ragged size
A_SHAPES = {
    "norm1-layer1": (16, 220, 512, 64),
    "layer2": (16, 110, 256, 96),
    "layer3": (16, 55, 128, 128),
    "ragged": (3, 37, 45, 128),             # P = 1665: not a multiple of 32 or of 512
}


def check_stats(what, mr, x, labels, log=print):
    """mean_rstd [N*C*2] of a kernel against the two-pass fp64 statistics of its own fp32 input x [N, P, C].  labels [N, C]:
    the |mean|/std of each channel (nan: constant), named on failure.  Returns (mean, var, rstd) of the reference."""
    N, _, C = x.shape
    mean, var, rstd = norm_ref(x)
    bad, em, er = stats_bounds(mr.view(N, C, 2), mean, var, rstd)
    n, c, r = worst_at(er, labels)
    log(f"  {what}: worst rstd rel err {float(er.max()):.2e} (image {n}, channel {c}, |mean|/std {r:g}), "
        f"worst mean rel err {float(em.max()):.2e}")
    if bad.any():
        per_ratio = {}
        for nn_, cc in bad.nonzero().tolist():
            key = "constant" if math.isnan(float(labels[nn_, cc])) else f"{float(labels[nn_, cc]):g}"
            per_ratio[key] = max(per_ratio.get(key, 0.0), float(er[nn_, cc]))
        n, c, r = worst_at(torch.where(bad, er, torch.zeros_like(er)), labels)
        got = mr.view(N, C, 2)[n, c].tolist()
        raise Mismatch(f"{what}: {int(bad.sum())} (image, channel) statistics out of bound; worst image {n}, channel {c}, "
                       f"|mean|/std {r:g}: mean {got[0]!r} vs {float(mean[n, c])!r}, rstd {got[1]!r} vs "
                       f"{float(rstd[n, c])!r}; worst rstd rel err per |mean|/std: {per_ratio}")
    return mean, var, rstd


def check_apply(what, got, x, mean, var, rstd, mode, res=None, split=False, labels=None):
    """An rnc_instnorm_apply output [N, P, C] (fp32, or hi + lo halves with split=True) against the fp64 normalisation of x by
    the reference statistics; a constant channel's output exactly 0 (mode 0 / 1) or relu(res) (mode 2)."""
    ref = apply_ref(x, mean, rstd, mode, res)
    bound = apply_bound(x, mean, rstd, ref)
    if split:
        bound = bound + 2.0 ** -21 * ref.abs() + 2.0 ** -24             # the 22-bit hi/lo split of the fp32 result
    err = (got.double() - ref).abs()
    rel = err / bound
    N, P, C = x.shape
    flat = int(rel.reshape(-1).argmax())
    n, rem = divmod(flat, P * C)
    p, c = divmod(rem, C)
    r = "?" if labels is None else f"{float(labels[n, c]):g}"
    if bool((rel > 1).any()):
        raise Mismatch(f"{what} mode {mode}: {int((rel > 1).sum())} outputs out of bound; worst image {n}, position {p}, "
                       f"channel {c} (|mean|/std {r}): {float(got[n, p, c])!r} vs {float(ref[n, p, c])!r}, "
                       f"bound {float(bound[n, p, c]):.2e}")
    const = var == 0
    if const.any() and not (split and mode == 2):                      # (relu(res) itself is not a 22-bit value)
        want = torch.zeros_like(got) if mode < 2 else res.clamp_min(0).to(got.dtype)
        sel = const[:, None, :].expand_as(got)
        assert torch.equal(got[sel], want[sel]), f"{what} mode {mode}: a constant channel's output is not exactly " \
                                                 f"{'0' if mode < 2 else 'relu(res)'}"
    return float(rel.max())


def _det_stats(x, N, P, C, mr):
    from rnc.native import rnc
    nbytes = rnc.instnorm_stats_det_workspace_bytes(N, P, C)
    ws = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=DEV)
    rnc.instnorm_stats_det(x, N, P, C, EPS, ws, nbytes, mr)


# ----------------------------------------------------------------------------------------------------------- (a)
@pytest.mark.parametrize("sid", list(A_SHAPES))
def test_stats_routes_at_controlled_conditioning(sid, monkeypatch):
    """x = m + sigma z per (image, channel) at |m|/sigma in {0, 1, 10, 100, 1000, 3000, 1e4}, both signs, and constant
    channels, through the three statistics routes: (1) a LINEAR 1x1 identity rnc_conv2d_umma_fwd with fused statistics, then
    rnc_instnorm_finalize (which must leave the sums zeroed); (2) rnc_instnorm_stats; (3) rnc_instnorm_stats_det (twice:
    bit-identical).  mean and rstd against the two-pass fp64 statistics of the kernel's own fp32 input, with bounds that do
    not depend on the conditioning; rnc_instnorm_apply (modes 0, 1, 2) against fp64 normalisation of the same input."""
    from rnc import native
    from rnc.encoder_umma import UmmaWeights
    from rnc.engine import engine_for
    from rnc.native import rnc
    monkeypatch.setenv("RNC_CONV", "umma")            # the fused statistics are a tensor-core convolution epilogue
    N, H, W, C = A_SHAPES[sid]
    P = H * W
    xin, ratio, _, _ = conditioned(N, P, C, seed=C + N, device=DEV)
    eng = engine_for(torch.device(DEV))
    assert eng.mode == "umma"
    # route 1: the convolution's output is the tensor under test (the hi/lo split input reproduces xin to 22 bits)
    hi = xin.half()
    lo = (xin - hi.float()).half()
    ident = UmmaWeights(torch.eye(C, device=DEV).view(C, C, 1, 1), None, [C])
    x = torch.empty(N, P, C, device=DEV)
    stats = torch.zeros(N * C * 2, dtype=torch.float64, device=DEV)
    mrs = {r: torch.empty(N * C * 2, device=DEV) for r in ("fused", "stats", "det", "det again")}
    eng.uconv(N, H, W, (hi.data_ptr(), lo.data_ptr()), C, C, ident, native.EPI_LINEAR, out_f32=x.data_ptr(), ldo_f32=C,
              stats=stats.data_ptr())
    rnc.instnorm_finalize(stats, N, P, C, EPS, mrs["fused"])
    scratch = torch.empty(N * C * 2, dtype=torch.float64, device=DEV)
    rnc.instnorm_stats(x, N, P, C, EPS, scratch, mrs["stats"])
    _det_stats(x, N, P, C, mrs["det"])
    _det_stats(x, N, P, C, mrs["det again"])
    torch.cuda.synchronize()
    assert (x.double() - xin.double()).abs().max() <= 2.0 ** -21 * float(xin.abs().max())     # the controlled tensor
    assert not stats.any(), "rnc_instnorm_finalize must re-zero the accumulated sums"
    assert torch.equal(mrs["det"], mrs["det again"]), "rnc_instnorm_stats_det: repeats differ"
    res = torch.randn(N, P, C, device=DEV, generator=torch.Generator(device=DEV).manual_seed(N))
    out = torch.empty(N, P, C, device=DEV)
    oh = torch.empty(N, P, C, dtype=torch.float16, device=DEV)
    ol = torch.empty_like(oh)
    failures = []
    for route in ("fused", "stats", "det"):
        what = f"[{sid} {N}x{P}x{C}] route {route}"
        try:
            mean, var, rstd = check_stats(what, mrs[route], x, ratio)
            for mode in (0, 1, 2):
                rnc.instnorm_apply(x, mrs[route], res if mode == 2 else None, N, P, C, mode, out,
                                   oh if mode else None, ol if mode else None)
                torch.cuda.synchronize()
                check_apply(what, out, x, mean, var, rstd, mode, res, labels=ratio)
                if mode:
                    check_apply(what + " split", oh.float() + ol.float(), x, mean, var, rstd, mode, res, True, ratio)
        except Mismatch as e:
            print(f"  FAIL {e}")
            failures.append(str(e))
    assert not failures, "\n".join(failures)


# ----------------------------------------------------------------------------------------------------------- (b)
# (B, H, W): the benchmark's Sintel frames (fnet on 16 images) and KITTI's 376x1248 (fnet on 6)
B_SHAPES = {"S1": (8, 440, 1024), "S2": (3, 376, 1248)}


class NormRecorder:
    """Wraps EncoderRunner._norm: each of fnet's norms is checked, as it runs, against the fp64 statistics and normalisation
    of its own fp32 input (the tensor the kernels left)."""

    def __init__(self, monkeypatch, runner, tag):
        self.tag, self.calls, self.worst, self.ratio = tag, [], {}, 0.0
        orig = runner._norm
        rec = self

        def norm(bufs, x32, N, P, Cc, mode, res=None, out32=None, split=None, fused_stats=False):
            x = x32[:N * P * Cc].view(N, P, Cc).clone()
            r = res[:N * P * Cc].view(N, P, Cc).clone() if res is not None else None
            orig(bufs, x32, N, P, Cc, mode, res=res, out32=out32, split=split, fused_stats=fused_stats)
            torch.cuda.synchronize()
            rec.check(len(rec.calls), bufs.mr[:N * Cc * 2], x, mode, r, out32, split, fused_stats)
            rec.calls.append((P, Cc, mode, fused_stats))

        monkeypatch.setattr(runner, "_norm", norm)

    def check(self, i, mr, x, mode, res, out32, split, fused):
        N, P, C = x.shape
        what = f"{self.tag} norm {i} ({'fused' if fused else 'det'}, {N}x{P}x{C})"
        mean, var, rstd = norm_ref(x)
        labels = torch.where(var > 0, mean.abs() / var.sqrt(), torch.full_like(var, math.nan)).cpu()
        self.ratio = max(self.ratio, float(labels[~labels.isnan()].max()))
        check_stats(what, mr, x, labels, log=lambda s: None)
        w = 0.0
        if out32 is not None:
            w = check_apply(what, out32[:N * P * C].view(N, P, C), x, mean, var, rstd, mode, res, labels=labels)
        if split is not None:
            v = (split.hi.float() + split.lo.float())[:N * P].view(N, P, -1)[..., :C]
            w = max(w, check_apply(what + " split", v, x, mean, var, rstd, mode, res, True, labels))
        self.worst[i] = w


@pytest.mark.parametrize("det", [False, True], ids=["fused", "det"])
@pytest.mark.parametrize("sid", list(B_SHAPES))
def test_fnet_norms_on_near_uniform_frames(sid, det, monkeypatch):
    """fnet on grey, black, white, grey +- 1 and half-flat frames: every InstanceNorm (15 per pass) against fp64 on its own
    input, in the default mode (fused epilogue statistics) and under torch.use_deterministic_algorithms
    (rnc_instnorm_stats_det).  The grey frames put norm1 beyond |mean|/std = 1000."""
    monkeypatch.setenv("RNC_CONV", "umma")
    B, H, W = B_SHAPES[sid]
    frames, kinds = near_uniform_frames(2 * B, H, W, seed=B)
    m = build_model("raft_nc_dbl").to(DEV)
    eng = m.engine()
    ws = eng.workspace(DEV, B, H // 8, W // 8, False, True)
    runner = eng.encoder()
    rec = NormRecorder(monkeypatch, runner, f"[{sid} {'det' if det else 'fused'}]")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        with torch.no_grad():
            runner.run(m, ws, frames[:B].to(DEV), frames[B:].to(DEV))
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    print(f"[{sid} {'det' if det else 'fused'}] frames {kinds}: {len(rec.calls)} norms checked, max |mean|/std "
          f"{rec.ratio:.0f}, worst apply err/bound " + ", ".join(f"{k}:{v:.2f}" for k, v in rec.worst.items()))
    assert len(rec.calls) == 15 and all(f == (not det) for *_, f in rec.calls)
    assert rec.ratio > 1000, "the grey frames must reach |mean|/std > 1000 at norm1"


# ----------------------------------------------------------------------------------------------------------- (c)
# The encoder outputs are compared with a whole-encoder fp64 reference (fnet / cnet end to end, not layer by layer), so
# their error compounds over 13 convolutions.  Their per-channel bound adds ENC_MARGIN times the deviation from fp64 of an
# fp32 evaluation of the same graph, channel by channel: what fp32 arithmetic itself costs there.  The tensor-core engine's
# split operands carry 22 bits where fp32 carries 24 (4x the operand rounding, in two operands).
ENC_MARGIN = 8.0
# GRU gate outputs squash their pre-activation: z = sigmoid(a_z), r*h = sigmoid(a_r) * h (|h| <= 1), and the new
# h = (1 - z) h_old + z tanh(a_q).  An error d in the pre-activation moves them by at most slope * d, and the pre-activation's
# error scales with its own magnitude, not with the squashed output's; so their per-channel bound is taken on the
# pre-activation: tol * slope * max(1, max|a[:, c]|), on top of the output's own.
GATE_PRE = {"z": ("convz", 0.25), "r*h": ("convr", 0.25), "h": ("convq", 1.0), "h (split)": ("convq", 1.0)}


# Tensor-core layers of the update block judged by the error model of tests/test_conv_error_model.py instead of a flat
# per-channel bound: packed stage -> (label of the Recorder's comparison, activation, output stored as split halves)
MODEL_STAGES = {"convc1": ("convc1", True, True), "convc2": ("convc2", True, True), "convf1": ("convf1", True, True),
                "convf2": ("convf2", True, True), "conv": ("conv", True, True), "czr1": ("czr1", False, False),
                "cq1": ("cq1", False, False), "czr2": ("czr2", False, False), "cq2": ("cq2", False, False),
                "fh1": ("fh1", True, True), "fh2": ("fh2 (taps)", False, False)}


class ChannelRecorder(Recorder):
    """The layer-by-layer Recorder with per-output-channel bounds (compare_per_channel).  On the tensor-core engine the
    update block's convolutions (MODEL_STAGES) are instead checked elementwise against the error model, on the split planes
    each layer read and through the engine's real pack: against conv_split_ref with bound A (the kernel computes its own
    arithmetic), and against the fp64 layer of the module's weights with R + A (plus the output split's own rounding)."""

    def __init__(self, mp, model, eng, *a, **kw):
        self.pre, self.enc_floor, self.model = {}, {}, {}
        super().__init__(mp, model, eng, *a, **kw)
        if self.umma:
            from rnc.engine_umma import SplitBuf
            self.planes = [b for b in vars(self.ws).values() if isinstance(b, SplitBuf)]
            inner = eng.uconv

            def uconv(B_, H_, W_, in0, c0, ld0, wt, epi, **k):
                st = self.pk_names.get(id(wt))
                if self.check and st in MODEL_STAGES and not k.get("c1") and not k.get("add"):
                    # convf1 reads the im2col planes, not the flow the Recorder's reference starts from: its fp64 layer
                    # is evaluated here on those planes (the im2col stage is checked on its own)
                    w = None
                    if st == "convf1":
                        wf = self.sd["update_block.encoder.convf1.weight"]
                        w = wf.permute(0, 2, 3, 1).reshape(wf.shape[0], -1, 1, 1)
                    self.model[MODEL_STAGES[st][0]] = (conv_split_ref(self.read_planes(in0, c0, ld0, B_, H_, W_), wt,
                                                                      weight=w), *MODEL_STAGES[st][1:])
                return inner(B_, H_, W_, in0, c0, ld0, wt, epi, **k)
            mp.setattr(eng, "uconv", uconv)

    def read_planes(self, in0, c0, ld0, B, H, W):
        """The (hi, lo) planes [B, c0, H, W] a layer reads from the workspace's split buffer at the addresses in0."""
        for b in self.planes:
            base = b.hi.data_ptr()
            if b.ld == ld0 and base <= in0[0] < base + b.hi.numel() * 2:
                off = (in0[0] - base) // 2
                assert in0[1] - b.lo.data_ptr() == 2 * off and off + c0 <= b.ld
                return tuple(t[:B * H * W, off:off + c0].reshape(B, H, W, c0).permute(0, 3, 1, 2) for t in (b.hi, b.lo))
        raise AssertionError("a tensor-core layer read planes outside the workspace's split buffers")

    def conv(self, name, x, w=None, b=None):
        out = super().conv(name, x, w, b)
        self.pre[name.rsplit(".", 1)[-1][:5]] = out             # the last convz / convr / convq evaluated
        return out

    def encoders_ref_f32(self):
        """fp32 evaluation of encoders_ref's graph (TF32 off)."""
        from oracle import raft_oracle as orc
        sd = {k: v.float() for k, v in self.sd.items() if k.startswith(("fnet.", "cnet."))}
        f1, f2, net, inp = [], [], [], []
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            for i in range(self.B):
                a = 2 * (self.im1[i:i + 1].float() / 255.0) - 1.0
                b = 2 * (self.im2[i:i + 1].float() / 255.0) - 1.0
                f1.append(orc.basic_encoder(sd, "fnet.", a, "instance"))
                f2.append(orc.basic_encoder(sd, "fnet.", b, "instance"))
                c = orc.basic_encoder(sd, "cnet.", a, "batch")
                net.append(torch.tanh(c[:, :128]))
                inp.append(torch.relu(c[:, 128:]))
        return [torch.cat(t, 0) for t in (f1, f2, net, inp)]

    def check_encoders(self, args):
        r64, r32 = self.encoders_ref(), self.encoders_ref_f32()
        for st, a, b in zip(("encoder fmap1", "encoder fmap2", "encoder net", "encoder inp"), r32, r64):
            self.enc_floor[st] = ENC_MARGIN * (a.double() - b).abs().amax((0, 2, 3))
        super().check_encoders(args)

    def cmp(self, st, got, ref, tol, floor=0.0):
        if not self.check:
            return
        if st in self.model:
            return self.cmp_model(st, got, ref)
        floor = floor + self.enc_floor.get(st, 0.0)
        stage, _, out = st.partition(" ")
        if stage[:2] in ("zr", "q1", "q2") and out in GATE_PRE:
            conv, slope = GATE_PRE[out]
            floor = floor + tol * slope * self.pre[conv].abs().amax((0, 2, 3)).clamp_min(1.0)
        w = compare_per_channel(f"{self.tag} {st}", got, ref, tol, floor)
        self.worst[st] = max(self.worst.get(st, 0.0), w)

    def cmp_model(self, st, got, ref):
        """got (the layer's output as stored, after its activation) against the model of the layer's last launch: A
        against conv_split_ref, R + A against ref (fp64 of the module's weights on the same input; for convf1 the model's
        own, on the planes the layer read).  A's epilogue term takes the pre-activation |ref| (an activation that is
        1-Lipschitz moves no error up); a split output adds its own rounding, split_bound of the value."""
        s, act, split = self.model[st]
        C = got.shape[1]
        if s.exact is not None:
            ref = s.exact[:, :C].clamp_min(0) if act else s.exact[:, :C]
        pre = s.ref[:, :C]
        mine = pre.clamp_min(0) if act else pre
        floor = U * pre.abs() + fp64_floor(s)[:, :C] + (split_bound(mine) if split else 0.0)
        tol = a_tol(s.steps)
        w = compare_mag(f"{self.tag} {st} [split]", got, mine, s.mag_a[:, :C], tol, floor)
        w = max(w, compare_mag(f"{self.tag} {st} [exact]", got, ref, s.mag_a[:, :C], tol, floor + s.R[:, :C]))
        self.worst[st] = max(self.worst.get(st, 0.0), w)
        if st == "convc2" and C > 181:
            # the channel of the flat per-channel bound's miss at S3: its error against fp64, and the model's two parts there
            # (all figures at the element of the channel's largest error against fp64)
            c = 181
            err = (got[:, c].double() - ref[:, c].double()).abs()
            i = int(err.reshape(-1).argmax())
            b, yx = divmod(i, err.shape[1] * err.shape[2])
            at = lambda t: float(t[:, c].reshape(-1)[i])      # noqa: E731
            print(f"  {self.tag} convc2 channel {c}: max|ref| {float(ref[:, c].abs().max()):.3e}, flat bound "
                  f"{2e-5 * max(1.0, float(ref[:, c].abs().max())):.3e}; at image {b}, pixel (y={yx // err.shape[2]}, "
                  f"x={yx % err.shape[2]}): |err| vs fp64 {float(err.max()):.3e}, |got - split ref| "
                  f"{abs(float(got[:, c].reshape(-1)[i]) - at(mine)):.3e}, |ref| {abs(at(pre)):.3e}, mag {at(s.mag):.3e}, "
                  f"mag_a {at(s.mag_a):.3e}, R {at(s.R):.3e}, A (C_A {C_A}, {s.steps} K steps) {tol * at(s.mag_a) + U * abs(at(pre)):.3e}")


C_CASES = [pytest.param(cfg, sid, id=f"{sid}-{cfg}") for cfg in ("umma", "ffma") for sid in ("S2", "S3")]


@pytest.mark.parametrize("cfg,sid", C_CASES)
def test_trained_like_layer_by_layer(cfg, sid, monkeypatch):
    """Two iterations of a test-mode raft_nc_dbl forward on a trained-like model (BatchNorm statistics, per-channel weight
    scales, zero channels, spread NConv weights), every stage against its fp64 reference layer built from the module's own
    weights: the host BatchNorm fold and the per-layer power-of-two weight scale see real statistics, and each output
    channel is judged at its own scale, so a small channel cannot hide behind a large one."""
    for k, v in CONFIGS[cfg].items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("RNC_GRAPH", "0")
    B, H8, W8 = SHAPES[sid]
    m = trained_like(build_model("raft_nc_dbl"), seed=17).to(DEV)
    eng = m.engine()
    im1, im2, fi = stimulus(B, H8, W8, seed=3)
    with monkeypatch.context() as mp:
        rec = ChannelRecorder(mp, m, eng, B, H8, W8, tag=f"[{sid} {cfg} trained-like]")
        rec.images(im1, im2, fi)
        with torch.no_grad():
            m(im1, im2, iters=2, flow_init=fi, test_mode=True)
        torch.cuda.synchronize()
    assert rec.stages == expected_stages(cfg, "raft_nc_dbl", 2)
    print(f"[{sid} {cfg} trained-like] worst err/bound: " + ", ".join(f"{k} {v:.2f}" for k, v in rec.worst.items()))


# ----------------------------------------------------------------------------------------------------------- (d)
@pytest.mark.parametrize("kind", ["grey", "grey+-1"])
def test_end_to_end_near_uniform_pair(kind):
    """raft_nc_dbl, 12 iterations, one 440x1024 pair of near-uniform frames (frame 2 of grey +- 1: other noise), against the
    oracle: EPE <= 1e-3."""
    from oracle import raft_oracle as orc
    H, W = 440, 1024
    if kind == "grey":
        im1 = im2 = torch.full((1, 3, H, W), 128.0)
    else:
        g = torch.Generator().manual_seed(11)
        im1, im2 = (128.0 + (torch.rand(1, 3, H, W, generator=g) * 2 - 1) for _ in range(2))
    m = build_model("raft_nc_dbl")
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m = m.to(DEV)
    with torch.no_grad():
        lo, up = m(im1.to(DEV), im2.to(DEV), iters=12, test_mode=True)
    torch.cuda.synchronize()
    olo, oup, _ = orc.raft_forward(sd, im1, im2, iters=12, model="raft_nc_dbl", upsample_every_iter=False)
    epe = lambda a, b: (a.cpu() - b).pow(2).sum(1).sqrt().mean().item()
    e_lo, e_up = epe(lo, olo), epe(up, oup)
    print(f"{kind}: EPE flow_low {e_lo:.3e} flow_up {e_up:.3e} |flow_up| {oup.abs().mean():.3f}")
    assert e_up <= 1e-3 and e_lo <= 1e-3
