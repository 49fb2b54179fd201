"""Every hot-path kernel checked pointwise against an fp64 reference at the shapes the benchmark and the training runs use
(tests/test_product_shapes.py: SHAPES, the comparator and its tolerances).

The update-iteration test runs real test-mode forwards (2 iterations, warm start with a motion boundary) with the engine's
convolution calls and librnc entry points wrapped: each stage is compared, as it finishes, with the fp64 evaluation of the
matching reference layer on the stage's own input as the kernels left it (teacher forcing), with weights taken from the
modules rather than from the packs, so the packing is checked as well.  A failure names the stage, image and 128-pixel tile.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import build_model
from oracle import raft_oracle as orc
from test_product_shapes import CFG5_CONV_SIGNATURES, SHAPES, TOL, cl, compare, unblock

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# the tensor-core engine, with its exact fp32 lookup, and the exact fp32 engine
CONFIGS = {
    "umma": {},
    "umma-lookup-ffma": {"RNC_LOOKUP": "ffma"},
    "ffma": {"RNC_CONV": "ffma"},
}

# librnc entry points that complete a checked stage
NATIVE_STAGES = {
    "rnc_corr_lookup_umma_fwd": "lookup", "rnc_corr_lookup_split_fwd": "lookup", "rnc_corr_lookup_fwd": "lookup",
    "rnc_flow_im2col7_split_fwd": "im2col", "rnc_conv_flow7x7_fwd": "convf1",
    "rnc_flow_tap_gather_fwd": "gather", "rnc_flow_head2_fwd": "flow_head2", "rnc_coords_init": "coords_init",
    "rnc_flow_x2_fwd": "flow_x2", "rnc_ncup_guidance_fwd": "guidance", "rnc_ncup_guidance_split_fwd": "guidance",
    "rnc_conf_head_fwd": "conf",
}
# packed update-block layers (PackedUpdateUmma / PackedUpdateBlock attributes) -> stage
PACKED_STAGES = {"convc1": "convc1", "convc2": "convc2", "convf1_mm": "convf1", "convf2": "convf2", "conv": "conv",
                 "zr1_c": "czr1", "q1_c": "cq1", "zr2_c": "czr2", "q2_c": "cq2", "zr1": "zr1", "q1": "q1", "zr2": "zr2",
                 "q2": "q2", "fh1": "fh1", "fh2": "fh2", "m0": "m0", "m2": "m2"}


def expected_stages(engine, model, iters):
    """The stage order of one test-mode forward: a change to the engine's call sequence fails here, loudly, instead of
    comparing the wrong pairs."""
    umma = engine == "umma"
    seq = ["encoders", "pyramid"] + ([] if umma else ["context"]) + ["coords_init"]
    for it in range(iters):
        last = it == iters - 1
        seq += ["lookup", "convc1", "convc2"] + (["im2col", "convf1"] if umma else ["convf1"]) + ["convf2", "conv"]
        if umma and it == 0:
            seq += ["czr1", "cq1", "czr2", "cq2"]                  # hoisted context addends: once per forward
        seq += ["zr1", "q1", "zr2", "q2", "fh1"] + (["fh2", "gather"] if umma else ["flow_head2"])
        if last and model == "raft":
            seq += ["m0", "m2"]
    seq += ["flow_x2", "guidance", "conf", "ncup"] if model == "raft_nc_dbl" else ["flow_low", "convex"]
    return seq + ["net_out", "flow_low"]


def stimulus(B, H8, W8, seed):
    """Smooth frames (bicubic noise, a translated pair) and a warm start: a smooth flow plus a motion boundary, so the
    tensor-core lookup meets incoherent tiles (exact fallback) as well as coherent ones."""
    from rnc.synth import motion_boundary_flow_init, smooth_shift_frames
    im1, im2 = smooth_shift_frames(B, 8 * H8, 8 * W8, seed=seed)
    yy, xx = torch.meshgrid(torch.arange(H8).float(), torch.arange(W8).float(), indexing="ij")
    smooth = torch.stack([3 * torch.sin(yy / 7 + seed) + 0.02 * xx - 1.3, 2 * torch.cos(xx / 11) - 0.03 * yy + 0.7])
    fi = motion_boundary_flow_init(B, H8, W8) + smooth[None]
    return im1.to(DEV), im2.to(DEV), fi.to(DEV)


class LibProxy:
    """Stands in for the librnc handle: every rnc_* call goes through the recorder."""

    def __init__(self, lib, rec):
        self._lib, self._rec = lib, rec

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("rnc_"):
            return fn
        return lambda *a: self._rec.native(name, fn, a)


class Recorder:
    """Wraps one engine for one forward: records the librnc entry points called and, with check=True, compares every stage
    with its fp64 reference as it completes."""

    def __init__(self, monkeypatch, model, eng, B, H8, W8, check=True, tag=""):
        from rnc import native
        self.m, self.eng, self.check, self.tag = model, eng, check, tag
        self.B, self.H, self.W, self.M = B, H8, W8, B * H8 * W8
        self.umma = eng.mode == "umma"
        self.ncup = model.ncup
        self.called, self.stages, self.worst = set(), [], {}
        self.fallback = None
        self.flow_init = None
        self.sd = {k: v.detach().double() for k, v in model.state_dict().items()}
        pk = eng.packed_update(model.update_block)
        self.pk_names = {id(getattr(pk, a)): s for a, s in PACKED_STAGES.items() if hasattr(pk, a)}
        self.ws = eng.workspace(torch.device(DEV), B, H8, W8, pk.has_mask, self.ncup)
        self.grid = orc.coords_grid(B, H8, W8).to(DEV).double()
        self.pending = {}
        monkeypatch.setattr(native, "_lib", LibProxy(native.lib(), self))
        if self.umma:
            orig_uconv = eng.uconv
            monkeypatch.setattr(eng, "uconv", lambda B_, H_, W_, in0, c0, ld0, wt, epi, **kw:
                                self.layer(self.pk_names.get(id(wt)), lambda: orig_uconv(B_, H_, W_, in0, c0, ld0, wt, epi, **kw)))
            self._wrap(monkeypatch, "finish_fmaps", "encoders", "pyramid")
        else:
            orig_conv = eng.conv
            monkeypatch.setattr(eng, "conv", lambda B_, H_, W_, in0, c0, ld0, packed, *a, **kw:
                                self.layer(self.pk_names.get(id(packed)), lambda: orig_conv(B_, H_, W_, in0, c0, ld0, packed, *a, **kw)))
            self._wrap(monkeypatch, "fmap_prepare", "encoders", "pyramid")
            self._wrap(monkeypatch, "load_state", "context", None)
        self._wrap(monkeypatch, "ncup_chain", None, "ncup")
        self._wrap(monkeypatch, "convex_upsample", None, "convex")
        self._wrap(monkeypatch, "flow_low", None, "flow_low")
        self._wrap(monkeypatch, "net_nchw", None, "net_out")

    def _wrap(self, monkeypatch, meth, pre_stage, post_stage):
        orig = getattr(self.eng, meth)

        def run(*a, **kw):
            if pre_stage:
                self.stage(pre_stage, "pre", a)
            out = orig(*a, **kw)
            if post_stage:
                self.stages.append(post_stage)
                self.stage(post_stage, "post", a, out)
            return out
        monkeypatch.setattr(self.eng, meth, run)

    def native(self, name, fn, args):
        self.called.add(name)
        st = NATIVE_STAGES.get(name)
        if st is None:
            return fn(*args)
        self.stage(st, "before", args)
        r = fn(*args)
        if r == 0:
            self.stage(st, "post", args)
        return r

    def layer(self, st, call):
        if st is None:
            return call()
        self.stage(st, "before", ())
        call()
        self.stage(st, "post", ())

    # ------------------------------------------------------------------ readers
    def val(self, buf):
        return (buf.hi.float() + buf.lo.float()) if hasattr(buf, "hi") else buf

    def nchw(self, t2d, c0, c1, H=None, W=None):
        return cl(t2d[:, c0:c1], self.B, H or self.H, W or self.W).double()

    def hx(self):
        return self.val(self.ws.hx)

    def h32(self):
        return self.ws.h if self.umma else self.ws.hx[:, :128]

    def zgate(self, kh, kw):
        if not self.umma:
            return self.nchw(self.ws.z, 0, 128)
        return self.nchw(unblock(self.ws.z, 128, 128, kh, kw, self.B, self.H, self.W), 0, 128)

    def conv(self, name, x, w=None, b=None):
        mod = self.m.get_submodule(name)
        w = self.sd[name + ".weight"] if w is None else w
        b = self.sd[name + ".bias"] if b is None else b
        return F.conv2d(x, w, b, padding=mod.padding)

    def cmp(self, st, got, ref, tol, floor=0.0):
        if not self.check:
            return
        w = compare(f"{self.tag} {st}", got, ref, tol, floor)
        self.worst[st] = max(self.worst.get(st, 0.0), w)

    def lookup_ref(self, coords):
        M, B, H, W = self.M, self.B, self.H, self.W
        f1 = cl(self.ws.f1_cl, B, H, W).double()
        f2 = cl(self.ws.f2_pyr[:M * 256], B, H, W).double()
        return orc.corr_lookup_direct(f1, f2, coords.double()), f1, f2

    # ------------------------------------------------------------------ stages
    def stage(self, st, when, args, out=None):
        if when in ("before", "pre"):
            self.stages.append(st)
        if not self.check:
            return
        ws, B, H, W = self.ws, self.B, self.H, self.W
        p = "update_block."
        if when == "before":
            if st in ("lookup", "gather", "flow_head2"):
                self.pending[st] = ws.coords1.clone()
            # the flow convf1 sees: at the im2col of the 1x1 form, else at the 7x7 kernel
            if st == "im2col" or (st == "convf1" and self.stages[-2:-1] != ["im2col"]):
                self.pending["flow"] = ws.coords1.double() - self.grid
            if st in ("q1", "q2"):
                self.pending["h_old"] = self.h32().clone()
            return
        if st == "encoders":
            return self.check_encoders(args)
        if st == "context":
            return self.check_context(args)
        if st == "pyramid":
            return self.check_pyramid(args)
        hx = self.hx() if st not in ("coords_init", "flow_low", "convex", "ncup", "net_out") else None
        if st == "coords_init":
            ref = self.grid + (self.flow_init.double() if self.flow_init is not None else 0)
            self.cmp(st, ws.coords1, ref, TOL["move"])
        elif st == "lookup":
            coords = self.pending.pop("lookup")
            if self.umma and self.eng.lookup_mode == "umma":
                # the error model of tests/test_lookup_error_model.py: tensor-core units against the fp64 lookup of the
                # halves, flagged units against the fp64 lookup of the fp32 features, flags against the host records
                from test_gpu_lookup_error_model import check_launch
                lv, _, wr, ex = check_launch(f"{self.tag} lookup", ws, self.eng.corr_nchw(ws), coords.cpu())
                self.worst[st] = max(self.worst.get(st, 0.0), wr, ex, *(r for r, _ in lv))
                self.fallback = int(ws.lookup_flags.sum())
                print(f"  {self.tag} lookup: fallback tiles {self.fallback}/{ws.lookup_flags.numel()}, C_A needed per level "
                      f"{', '.join(f'{c:.3f}' for _, c in lv)}")
                return
            ref, f1, f2 = self.lookup_ref(coords)
            got = self.eng.corr_nchw(ws) if self.umma else cl(ws.corr, B, H, W)
            self.cmp(st + " (exact)", got, ref, TOL["lookup_exact"])
        elif st == "convc1":
            x = self.eng.corr_nchw(ws).double() if self.umma else cl(ws.corr, B, H, W).double()
            self.cmp(st, self.nchw(self.val(ws.c1), 0, 256), F.relu(self.conv(p + "encoder.convc1", x)), TOL["conv"])
        elif st == "convc2":
            x = self.nchw(self.val(ws.c1), 0, 256)
            self.cmp(st, self.nchw(self.val(ws.corflo), 0, 192), F.relu(self.conv(p + "encoder.convc2", x)), TOL["conv"])
        elif st == "im2col":
            flow = self.pending["flow"]
            u = F.unfold(flow, 7, padding=3).view(B, 2, 49, H * W).permute(0, 2, 1, 3).reshape(B, 98, H, W)
            ref = torch.cat([u, torch.zeros(B, 30, H, W, dtype=u.dtype, device=DEV)], 1)
            self.cmp(st, self.nchw(self.val(ws.fcol), 0, 128), ref, TOL["move"])
        elif st == "convf1":
            self.pending["f1_flow"] = self.pending.pop("flow")      # checked at convf2
        elif st == "convf2":
            ref_f1 = F.relu(self.conv(p + "encoder.convf1", self.pending.pop("f1_flow")))
            f1 = self.nchw(self.val(ws.f1), 0, 128)
            self.cmp("convf1", f1, ref_f1, TOL["conv"])
            self.cmp(st, self.nchw(self.val(ws.corflo), 192, 256), F.relu(self.conv(p + "encoder.convf2", f1)), TOL["conv"])
        elif st == "conv":
            x = self.nchw(self.val(ws.corflo), 0, 256)
            ref = F.relu(self.conv(p + "encoder.conv", x))[:, :126]
            self.cmp(st, self.nchw(hx, 256, 382), ref, TOL["conv"])
            self.cmp("flow append", self.nchw(hx, 382, 384), ws.coords1.double() - self.grid, TOL["move"])
        elif st in ("czr1", "cq1", "czr2", "cq2"):
            tag = st[-1]
            gates = ["convz", "convr"] if st.startswith("czr") else ["convq"]
            w = torch.cat([self.sd[f"{p}gru.{g}{tag}.weight"] for g in gates], 0)[:, 128:256]
            b = torch.cat([self.sd[f"{p}gru.{g}{tag}.bias"] for g in gates], 0)
            ref = self.conv(f"{p}gru.{gates[0]}{tag}", self.nchw(hx, 128, 256), w, b)
            buf = getattr(ws, st)
            ld = 256 if st.startswith("czr") else 128                 # the packs' coutpad
            kh, kw = (1, 5) if tag == "1" else (5, 1)
            got = unblock(buf, ld, ld, kh, kw, B, H, W)
            self.cmp(st, self.nchw(got, 0, ld), ref, TOL["conv"])
        elif st in ("zr1", "zr2"):
            tag = st[-1]
            kh, kw = (1, 5) if tag == "1" else (5, 1)
            h = self.nchw(self.h32(), 0, 128)
            xin = self.nchw(hx, 0, 384)                               # [h (as the kernel reads it) | inp | motion | flow]
            z = torch.sigmoid(self.conv(f"{p}gru.convz{tag}", xin))
            r = torch.sigmoid(self.conv(f"{p}gru.convr{tag}", xin))
            self.cmp(st + " z", self.zgate(kh, kw), z, TOL["conv"])
            self.cmp(st + " r*h", self.nchw(self.val(ws.rh), 0, 128), r * h, TOL["conv"])
        elif st in ("q1", "q2"):
            tag = st[-1]
            kh, kw = (1, 5) if tag == "1" else (5, 1)
            h_old = self.nchw(self.pending.pop("h_old"), 0, 128)
            z = self.zgate(kh, kw)
            xin = torch.cat([self.nchw(self.val(ws.rh), 0, 128), self.nchw(hx, 128, 384)], 1)
            q = torch.tanh(self.conv(f"{p}gru.convq{tag}", xin))
            ref = (1 - z) * h_old + z * q
            self.cmp(st + " h", self.nchw(self.h32(), 0, 128), ref, TOL["conv"])
            if self.umma:
                self.cmp(st + " h (split)", self.nchw(hx, 0, 128), ref, TOL["conv"])
        elif st == "fh1":
            x = self.nchw(hx, 0, 128)
            self.cmp(st, self.nchw(self.val(ws.fh), 0, 256), F.relu(self.conv(p + "flow_head.conv1", x)), TOL["conv"])
        elif st == "fh2":
            w2 = self.sd[p + "flow_head.conv2.weight"]
            taps = F.conv2d(self.nchw(self.val(ws.fh), 0, 256), w2.permute(2, 3, 0, 1).reshape(18, w2.shape[1], 1, 1))
            self.cmp("fh2 (taps)", cl(ws.fh2p[:, :18], B, H, W), taps, TOL["conv"])
        elif st in ("gather", "flow_head2"):
            old = self.pending.pop(st).double()
            delta = self.conv(p + "flow_head.conv2", self.nchw(self.val(ws.fh), 0, 256))
            new = ws.coords1.double()
            # coords1 += delta rounds to fp32 coordinates: allow one rounding of |coords1|
            self.cmp("fh2 + coords1 += delta", new - old, delta, TOL["conv"], 2.0 ** -23 * float(new.abs().max()))
        elif st == "m0":
            x = self.nchw(hx, 0, 128)
            self.cmp(st, self.nchw(self.val(ws.mh), 0, 256), F.relu(self.conv(p + "mask.0", x)), TOL["conv"])
        elif st == "m2":
            x = self.nchw(self.val(ws.mh), 0, 256)
            self.cmp(st, self.nchw(ws.mask, 0, 576), 0.25 * self.conv(p + "mask.2", x), TOL["conv"])
        elif st == "flow_x2":
            flow = ws.coords1.double() - self.grid
            self.cmp(st, ws.x4, F.interpolate(flow, scale_factor=2, mode="nearest"), TOL["move"])
        elif st == "guidance":
            gin = self.val(ws.gin)
            H4, W4 = 2 * H, 2 * W
            g4 = F.interpolate(self.nchw(self.h32(), 0, 128), scale_factor=2, mode="nearest")
            ref = torch.cat([ws.x4.double(), g4, torch.zeros(B, 2, H4, W4, dtype=g4.dtype, device=DEV)], 1)
            self.cmp(st, self.nchw(gin, 0, 132, H4, W4), ref, TOL["move"])
            self.pending["gin"] = self.nchw(gin, 0, 130, H4, W4)
        elif st == "conf":
            ref = orc.weights_net(self.sd, self.pending.pop("gin"), use_bn=True)
            self.cmp("weights net conf", ws.conf, ref, TOL["conv"])
        elif st == "ncup":
            _, _, x_lowres, conf, out_scale = args
            xh, ch = orc.zero_stuff(x_lowres.double()), orc.zero_stuff(conf.double())
            b, c, oh, ow = xh.shape
            ref, _ = orc.nconv_unet_live(self.sd, xh.view(b * c, 1, oh, ow), ch.view(b * c, 1, oh, ow))
            self.cmp(st, out, out_scale * ref.view(b, c, oh, ow), TOL["ncup"])
        elif st == "convex":
            _, flow_low, mask_cl, ldm = args
            ref = orc.convex_upsample(flow_low.double(), self.nchw(mask_cl, 0, 576))
            self.cmp(st, out, ref, TOL["convex"])
        elif st == "flow_low":
            self.cmp(st, out, ws.coords1.double() - self.grid, TOL["move"])
        elif st == "net_out":
            self.cmp(st, out, self.nchw(self.h32(), 0, 128), 0.0)

    def images(self, im1, im2, fi):
        self.im1, self.im2, self.flow_init = im1, im2, fi

    def encoders_ref(self):
        """fp64 fnet / cnet of the model's weights (BatchNorm in eval mode), one image at a time."""
        f1, f2, net, inp = [], [], [], []
        for i in range(self.B):
            a = 2 * (self.im1[i:i + 1].double() / 255.0) - 1.0
            b = 2 * (self.im2[i:i + 1].double() / 255.0) - 1.0
            f1.append(orc.basic_encoder(self.sd, "fnet.", a, "instance"))
            f2.append(orc.basic_encoder(self.sd, "fnet.", b, "instance"))
            c = orc.basic_encoder(self.sd, "cnet.", a, "batch")
            net.append(torch.tanh(c[:, :128]))
            inp.append(torch.relu(c[:, 128:]))
        return [torch.cat(t, 0) for t in (f1, f2, net, inp)]

    def check_encoders(self, args):
        ws, B, H, W, M = self.ws, self.B, self.H, self.W, self.M
        r1, r2, rnet, rinp = self.encoders_ref()
        if self.umma:
            f1, f2 = cl(ws.f1_cl, B, H, W), cl(ws.f2_pyr[:M * 256], B, H, W)
        else:
            f1, f2 = args[1], args[2]
        self.cmp("encoder fmap1", f1, r1, TOL["conv"])
        self.cmp("encoder fmap2", f2, r2, TOL["conv"])
        self.pending["context_ref"] = (rnet, rinp)
        if self.umma:
            self.check_context((None, cl(ws.h, B, H, W), self.nchw(self.hx(), 128, 256)))

    def check_context(self, args):
        rnet, rinp = self.pending.pop("context_ref")
        net, inp = args[1], args[2]
        # the bound of test_gpu_encoder.py::test_encoders_match_reference_golden for tanh(net): 1e-4 absolute
        self.cmp("encoder net", net, rnet, 1e-4)
        self.cmp("encoder inp", inp, rinp, TOL["conv"])

    def check_pyramid(self, args):
        ws, B, H, W = self.ws, self.B, self.H, self.W
        if not self.umma:
            assert torch.equal(cl(ws.f1_cl, B, H, W), args[1]), "rnc_fmap_prepare: fmap1 channel-last copy"
        from rnc import native
        L = native.lib()._lib
        prev = cl(ws.f2_pyr[:B * H * W * 256], B, H, W).double()
        for lvl in range(1, ws.levels):
            o0, o1 = L.rnc_pyramid_offset(B, 256, H, W, lvl), L.rnc_pyramid_offset(B, 256, H, W, lvl + 1)
            ref = F.avg_pool2d(prev, 2, stride=2)
            got = cl(ws.f2_pyr[o0:o1], B, H >> lvl, W >> lvl)
            self.cmp(f"pyramid level {lvl}", got, ref, TOL["move"])
            prev = got.double()
        if self.umma and self.eng.lookup_mode == "umma":
            assert torch.equal(ws.f1h, ws.f1_cl.reshape(-1).half()) and torch.equal(ws.f2h, ws.f2_pyr.half())


def run_forward(monkeypatch, cfg, model_name, sid, check=True, seed=1, iters=2):
    for k, v in CONFIGS[cfg].items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("RNC_GRAPH", "0")
    B, H8, W8 = SHAPES[sid]
    m = build_model(model_name).to(DEV)
    eng = m.engine()
    im1, im2, fi = stimulus(B, H8, W8, seed)
    with monkeypatch.context() as mp:
        rec = Recorder(mp, m, eng, B, H8, W8, check=check, tag=f"[{sid} {cfg} {model_name}]")
        rec.images(im1, im2, fi)
        with torch.no_grad():
            lo, up = m(im1, im2, iters=iters, flow_init=fi, test_mode=True)
        torch.cuda.synchronize()
    return rec, m, eng, (lo, up), (im1, im2, fi)


CASES = ([("umma", mdl, s) for mdl in ("raft_nc_dbl", "raft") for s in SHAPES]
         + [("ffma", "raft_nc_dbl", s) for s in SHAPES] + [("ffma", "raft", "S1")]
         + [("umma-lookup-ffma", "raft_nc_dbl", s) for s in ("S1", "S2")])


@pytest.mark.parametrize("cfg,model_name,sid", CASES, ids=[f"{s}-{c}-{m}" for c, m, s in CASES])
def test_update_iteration_layer_by_layer(cfg, model_name, sid, monkeypatch):
    """Two iterations of a test-mode forward, every stage against its fp64 reference layer (teacher forcing): encoders and
    pyramid, lookup, convc1, convc2, convf1 (im2col + 1x1, or the 7x7 of the exact engine), convf2, conv + flow append, the
    hoisted context addends, z / r*h / h of both GRU halves (z read back from the tile-blocked layout), fh1, fh2 in tap form +
    coords1 += delta, the mask head, and the upsampler stages.  The second iteration reuses the hoisted addends."""
    import time
    t0 = time.time()
    rec, m, eng, _, _ = run_forward(monkeypatch, cfg, model_name, sid)
    engine = "umma" if cfg.startswith("umma") else "ffma"
    assert rec.stages == expected_stages(engine, model_name, 2)
    if sid == "S1" and engine == "umma" and eng.lookup_mode == "umma":
        assert rec.fallback and rec.fallback > 0, "the motion boundary must send some lookup tiles to the exact fallback"
    print(f"[{sid} {cfg} {model_name}] {len(rec.stages)} stages checked in {time.time() - t0:.1f} s; worst errors: "
          + ", ".join(f"{k} {v:.1e}" for k, v in rec.worst.items()))


@pytest.mark.parametrize("sid", ["S1", "S2"])
def test_second_forward_and_graph_replay(sid, monkeypatch):
    """A second forward with other images in the same workspace (checked stage by stage), then a CUDA-graph replay with
    images different from those captured, against its own eager run."""
    rec_a, m, eng, (lo_a, up_a), _ = run_forward(monkeypatch, "umma", "raft_nc_dbl", sid, seed=1)
    B, H8, W8 = SHAPES[sid]
    im1, im2, fi = stimulus(B, H8, W8, seed=5)
    with monkeypatch.context() as mp:
        rec = Recorder(mp, m, eng, B, H8, W8, tag=f"[{sid} umma second forward]")
        rec.images(im1, im2, fi)
        with torch.no_grad():
            lo_b, up_b = m(im1, im2, iters=2, flow_init=fi, test_mode=True)
    assert rec.stages == expected_stages("umma", "raft_nc_dbl", 2)
    monkeypatch.setenv("RNC_GRAPH", "1")
    a1, a2, afi = stimulus(B, H8, W8, seed=1)
    with torch.no_grad():
        m(a1, a2, iters=2, flow_init=afi, test_mode=True)          # first sight of the signature: eager
        ga = m(a1, a2, iters=2, flow_init=afi, test_mode=True)     # capture with these images, replay
        gb = m(im1, im2, iters=2, flow_init=fi, test_mode=True)    # replay with other images
    torch.cuda.synchronize()
    assert any("graph" in v for v in eng._graphs.values())
    # the replay runs the eager kernels; the instance-norm statistics use fp64 atomics, so the last bits may differ
    for what, got, ref in (("replay A flow_low", ga[0], lo_a), ("replay A flow_up", ga[1], up_a),
                           ("replay B flow_low", gb[0], lo_b), ("replay B flow_up", gb[1], up_b)):
        compare(f"[{sid}] {what}", got, ref.double(), TOL["conv"])


# ----------------------------------------------------------------------------------------------------------- coverage guard
# Every librnc entry point a test-mode forward of either model calls on either engine -> the test that checks it pointwise.
LAYERS = "test_update_iteration_layer_by_layer"
COVERAGE = {
    "rnc_stem_window_prep": f"{LAYERS}: 'encoder fmap1/fmap2/net/inp' (tensor-core encoders)",
    "rnc_conv2d_umma_fwd": f"{LAYERS}: every tensor-core layer, encoders and weights net through their outputs",
    "rnc_instnorm_finalize": f"{LAYERS}: 'encoder fmap1/fmap2'",
    "rnc_instnorm_apply": f"{LAYERS}: 'encoder fmap1/fmap2/net/inp'",
    "rnc_instnorm_stats_det": f"{LAYERS}: 'encoder fmap1/fmap2' (deterministic mode)",
    "rnc_instnorm_stats_det_workspace_bytes": "size query",
    "rnc_pyramid_offset": "size query",
    "rnc_conv_umma_tiles": "size query; test_product_shapes.py::test_blocked_layout_round_trip",
    "rnc_corr_lookup_umma_workspace_bytes": "size query",
    "rnc_fmap_pyramid": f"{LAYERS}: 'pyramid level l'",
    "rnc_fmap_prepare": f"{LAYERS}: 'pyramid level l' (exact engine)",
    "rnc_f32_to_f16": f"{LAYERS}: pyramid stage, halves copies equal .half()",
    "rnc_nchw_to_cl": f"{LAYERS}: 'encoder net/inp' then every layer reading hx (exact engine)",
    "rnc_coords_init": f"{LAYERS}: 'coords_init' (warm start)",
    "rnc_corr_lookup_umma_fwd": f"{LAYERS}: 'lookup (tensor cores)'",
    "rnc_corr_lookup_split_fwd": f"{LAYERS}[*-umma-lookup-ffma-*]: 'lookup (exact)'",
    "rnc_corr_lookup_fwd": f"{LAYERS}[*-ffma-*]: 'lookup (exact)'",
    "rnc_flow_im2col7_split_fwd": f"{LAYERS}: 'im2col'",
    "rnc_conv_flow7x7_fwd": f"{LAYERS}[*-ffma-*]: 'convf1'",
    "rnc_conv2d_cl_fwd": f"{LAYERS}[*-ffma-*]: every exact-engine layer",
    "rnc_flow_tap_gather_fwd": f"{LAYERS}: 'fh2 + coords1 += delta'",
    "rnc_flow_head2_fwd": f"{LAYERS}[*-ffma-*]: 'fh2 + coords1 += delta'",
    "rnc_cl_to_nchw": f"{LAYERS}: 'net_out'",
    "rnc_coords_to_flow": f"{LAYERS}: 'flow_low'",
    "rnc_flow_x2_fwd": f"{LAYERS}: 'flow_x2'",
    "rnc_ncup_guidance_split_fwd": f"{LAYERS}: 'guidance'",
    "rnc_ncup_guidance_fwd": f"{LAYERS}[*-ffma-*]: 'guidance'",
    "rnc_conf_head_fwd": f"{LAYERS}: 'weights net conf'",
    "rnc_ncup_fwd": f"{LAYERS}: 'ncup'",
    "rnc_convex_upsample_fwd": f"{LAYERS}[*-raft]: 'convex'",
}
QUERIES = {k for k, v in COVERAGE.items() if v.startswith("size query")}
SWITCH_ONLY = {"rnc_corr_lookup_split_fwd", "rnc_instnorm_stats_det"}


def test_coverage_guard(monkeypatch):
    """The librnc entry points of one test-mode forward at S1 of each model on each engine are exactly the table's: a kernel
    added to the forward fails here until it has a pointwise check."""
    called = set()
    for cfg in ("umma", "ffma"):
        for name in ("raft_nc_dbl", "raft"):
            with monkeypatch.context() as mp:
                rec, *_ = run_forward(mp, cfg, name, "S1", check=False)
            called |= rec.called
    assert called - set(COVERAGE) == set(), f"entry points without a pointwise check: {sorted(called - set(COVERAGE))}"
    missing = set(COVERAGE) - QUERIES - SWITCH_ONLY - called
    assert missing == set(), f"table lists entry points the forwards no longer call: {sorted(missing)}"


# ----------------------------------------------------------------------------------------------------------- training layers
def _rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def test_train_conv_signatures_recorded(monkeypatch):
    """One real raft_nc_dbl train_step at config 5 (B = 2, 384x512; 2 iterations: the signatures do not depend on the count)
    calls ConvCL with exactly the written-out signatures."""
    from rnc import train
    from rnc.synth import frames
    seen = set()
    orig = train.ConvCL.apply

    def rec(x, weight, bias, stride, dil=1):
        cout, cin, kh, kw = weight.shape
        seen.add((cin, cout, kh, kw, stride, dil, x.shape[0], x.shape[1], x.shape[2]))
        return orig(x, weight, bias, stride, dil)

    monkeypatch.setattr(train.ConvCL, "apply", rec)
    m = build_model("raft_nc_dbl").to(DEV)
    m.train()
    m.freeze_bn()
    opt, sched = train.fetch_optimizer(m, lr=1e-4, num_steps=10)
    im1, im2 = (t.to(DEV) for t in frames(2, 384, 512))
    gt = (torch.randn(2, 2, 384, 512, generator=torch.Generator().manual_seed(3)) * 5).to(DEV)
    train.train_step(m, opt, sched, im1, im2, gt, torch.ones(2, 384, 512, device=DEV), iters=2)
    assert sorted(seen) == CFG5_CONV_SIGNATURES


@pytest.mark.parametrize("mode", ["ffma", "tf32"])
@pytest.mark.parametrize("sig", CFG5_CONV_SIGNATURES, ids=["-".join(map(str, s)) for s in CFG5_CONV_SIGNATURES])
def test_train_conv_at_config5_shapes(sig, mode, monkeypatch):
    """ConvCL forward, data and weight gradients at a config-5 layer shape against fp64 autograd (the bounds of
    test_gpu_train.py::test_conv_cl_forward_and_gradients, plus a pointwise check of y and dx), the weight gradient's K split
    bit-reproducible over three runs, and its workspace at most 52 MB."""
    from rnc import native
    from rnc.train import ConvCL, to_cl, to_nchw
    monkeypatch.setenv("RNC_TRAIN_CONV", mode)
    cin, cout, kh, kw, stride, dil, B, H, W = sig
    g = torch.Generator(device=DEV).manual_seed(sum(sig))
    x = torch.randn(B, cin, H, W, device=DEV, generator=g)
    w = torch.randn(cout, cin, kh, kw, device=DEV, generator=g) / (cin * kh * kw) ** 0.5
    b = torch.randn(cout, device=DEV, generator=g)
    xr, wr, br = (t.double().requires_grad_(True) for t in (x, w, b))
    ref = F.conv2d(xr, wr, br, stride=stride, padding=(kh // 2, kw // 2))
    gy = torch.randn(ref.shape, device=DEV, generator=g)
    ref.backward(gy.double())
    cx = 136 if cin == 130 else None                  # the weights net's staging pitch (tensor-core eligible), as in training
    xd = to_cl(x, pad_to=cx).requires_grad_(True)
    wd, bd = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    y = ConvCL.apply(xd, wd, bd, stride)
    grads = [torch.autograd.grad(y, (xd, wd, bd), to_cl(gy), retain_graph=True) for _ in range(3)]
    gx, gw, gb = grads[0]
    tag = f"ConvCL[{mode}] {sig}"
    compare(f"{tag} y", to_nchw(y, cout), ref.detach(), TOL["conv"])
    compare(f"{tag} dx", to_nchw(gx, cin), xr.grad, TOL["conv"])
    e = (_rel(to_nchw(y, cout), ref.detach()), _rel(to_nchw(gx, cin), xr.grad), _rel(gw, wr.grad), _rel(gb, br.grad))
    print(f"{tag}: rel err y {e[0]:.1e} dx {e[1]:.1e} dw {e[2]:.1e} db {e[3]:.1e}")
    tol = 2e-6 if mode == "ffma" else 2e-5
    assert e[0] < tol and e[1] < tol and e[2] < 5e-6 and e[3] < 5e-6
    for _, gw2, gb2 in grads[1:]:
        assert torch.equal(gw2, gw) and torch.equal(gb2, gb)
    nbytes = native.lib().rnc_conv2d_cl_wgrad_workspace_bytes(xd.shape[-1], cout, B, H, W, kh, kw, stride)
    assert nbytes <= 52 * 2 ** 20, f"wgrad workspace {nbytes / 2 ** 20:.1f} MB"


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("H,W", [(48, 64), (47, 156)])
def test_corr_lookup_train_at_product_shapes(H, W, det):
    """CorrLookup forward (pointwise) and backward against fp64 autograd through the 4-D corr_pyramid, in the default and the
    deterministic (atomic-free) mode."""
    from rnc.train import CorrLookup, CorrPyramid, to_cl, to_nchw
    B = 2
    g = torch.Generator(device=DEV).manual_seed(H + W)
    f1 = (torch.randn(B, 256, H, W, device=DEV, generator=g) * 1.5).double().requires_grad_(True)
    f2 = (torch.randn(B, 256, H, W, device=DEV, generator=g) * 1.5).double().requires_grad_(True)
    _, _, fi = stimulus(B, H, W, seed=2)
    co = orc.coords_grid(B, H, W).to(DEV) + fi
    ref = orc.corr_lookup(orc.corr_pyramid(f1, f2), co.double())
    gout = torch.randn(ref.shape, device=DEV, generator=g)
    ref.backward(gout)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        f1d = to_cl(f1.detach().float()).requires_grad_(True)
        f2d = to_cl(f2.detach().float()).requires_grad_(True)
        out = CorrLookup.apply(f1d, CorrPyramid.apply(f2d, 4), co, 4)
        out.backward(to_cl(gout))
    finally:
        torch.use_deterministic_algorithms(prev)
    compare(f"CorrLookup {H}x{W} det={det}", to_nchw(out), ref.detach(), TOL["lookup_exact"])
    e1, e2 = _rel(to_nchw(f1d.grad), f1.grad), _rel(to_nchw(f2d.grad), f2.grad)
    print(f"CorrLookup {H}x{W} det={det}: rel grad err f1 {e1:.1e} f2 {e2:.1e}")
    assert e1 < 1e-5 and e2 < 1e-5
