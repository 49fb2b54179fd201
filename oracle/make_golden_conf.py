"""NCUP output-confidence golden fixtures from the UNMODIFIED reference (authoring container only; needs the reference):

    python oracle/make_golden_conf.py     ->  tests/golden/conf.npz + conf_meta.json

The reference computes NConvUNet's output confidence on every upsampler call and discards it (core/upsampler.py:168,
`output, _ = self.interpolation_net(...)`).  A forward hook on `upsampler.interpolation_net` captures that cout, viewed as
[B,2,H,W] like the flow (channels_to_batch):
  * teacher-forced upsampler: RAFT.upsample_flow (raft_nc_dbl.py:107-112) on the top-left TF_CROP (1/8-resolution rows,
    columns) of the cfg-1 iteration-3 flow and hidden state of tests/golden/cfg1.npz (tf_inputs), for the shipped network
    (dataset sintel, BatchNorm weights net) and the `wide` configuration of ncup_oracle.CONFIGS (not fused): the captured
    confidence, [1,2,64,128];
  * end to end: the last upsampler call's confidence of the test-mode forward at cfg-1 size (one 128x256 pair of
    make_golden.frames, 4 iterations, seed 1234), whose flow_low / flow_up are cfg1.npz's raft_nc_dbl_flow_low / _up
    (asserted here);
  * gradients: as make_golden_r2 (train mode, frozen BatchNorm, 128x160, B = 2, 3 iterations) of
    L = sequence_loss(preds, gamma 0.85) + sum_i sum(P_i * conf_i), P_i = conf_projection(i, shape), for the whole model and
    the --freeze_raft model: the loss, make_golden_r2.grad_fixture of the gradients, the largest gradient norm.
The oracle (raft_oracle / ncup_oracle.unet) is asserted against the teacher-forced confidences here.  TEST INFRASTRUCTURE
ONLY.
"""
import json
import os
import sys
import warnings

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from make_golden import OUT, REF, frames, ref_args   # noqa: E402
from make_golden_r2 import GRAD_ITERS, grad_fixture, train_inputs   # noqa: E402
import ncup_oracle as nco                            # noqa: E402

TF_IT = 3                      # teacher-forced iteration of cfg1.npz
TF_CROP = (8, 16)              # teacher-forced crop of its 1/8-resolution inputs: outputs of 64x128
CONF_WEIGHT = 0.01             # scale of the projections P_i of the confidence term


def conf_projection(i, shape):
    """P_i of the gradient fixture's confidence term (seeded per iteration)."""
    g = torch.Generator().manual_seed(700 + i)
    return CONF_WEIGHT * torch.randn(shape, generator=g)


def conf_loss(confs):
    return sum((conf_projection(i, c.shape).to(c) * c).sum() for i, c in enumerate(confs))


def tf_inputs(cfg1):
    """The teacher-forced upsampler inputs (flow_lr [1,2,8,16], guidance [1,128,8,16]) from cfg1.npz's arrays (numpy)."""
    h, w = TF_CROP
    flow = torch.from_numpy(np.ascontiguousarray(cfg1[f"ncup_in_flow_it{TF_IT}"][:, :, :h, :w]))
    guid = torch.from_numpy(np.ascontiguousarray(cfg1[f"net_out_it{TF_IT}"][:, :, :h, :w]))
    return flow, guid


def oracle_conf(sd, cfg_name, flow_lr, guidance, use_bn=True):
    """The oracle's upsampler output and output confidence (no x8) for a state_dict of configuration cfg_name."""
    from oracle import raft_oracle as orc
    x4 = F.interpolate(flow_lr, scale_factor=2, mode="nearest")
    g4 = F.interpolate(guidance, x4.shape[2:], mode="area")
    w4 = orc.weights_net(sd, torch.cat([x4, g4], 1), use_bn)
    xh, wh = orc.zero_stuff(x4), orc.zero_stuff(w4)
    b, c, oh, ow = xh.shape
    if cfg_name == "shipped":
        y, k = orc.nconv_unet_live(sd, xh.view(b * c, 1, oh, ow), wh.view(b * c, 1, oh, ow))
    else:
        y, k = nco.unet(sd, nco.CONFIGS[cfg_name], xh.view(b * c, 1, oh, ow), wh.view(b * c, 1, oh, ow),
                        p="upsampler.interpolation_net.")
    return y.view(b, c, oh, ow), k.view(b, c, oh, ow)


def capture(model):
    """Hook on the reference's interpolation net: every call's cout viewed as [B,2,H,W] lands in the returned list."""
    got = []

    def hook(mod, inp, out):
        c = out[1]
        got.append(c.view(c.shape[0] // 2, 2, c.shape[2], c.shape[3]))

    model.upsampler.interpolation_net.register_forward_hook(hook)
    return got


def main():
    warnings.filterwarnings("ignore")
    sys.path.insert(0, os.path.join(REF, "core"))
    sys.path.insert(0, ROOT)
    import raft_nc_dbl as ref_nc
    from oracle import raft_oracle as orc

    torch.set_num_threads(os.cpu_count())
    gold, meta = {}, {"reference_commit": "51ac387", "torch": torch.__version__, "tf_iteration": TF_IT,
                      "tf_crop": list(TF_CROP), "conf_weight": CONF_WEIGHT, "grad_iters": GRAD_ITERS}
    z = np.load(os.path.join(OUT, "cfg1.npz"))
    flow_lr, guid = tf_inputs(z)

    # ------------------------------------------------------------------ teacher-forced upsampler
    for name in ("shipped", "wide"):
        a = ref_args("sintel")
        if name != "shipped":
            for k, v in nco.args_overrides(nco.CONFIGS[name]).items():
                setattr(a, k, v)
        torch.manual_seed(1234)
        m = ref_nc.RAFT(a).eval()
        got = capture(m)
        with torch.no_grad():
            out = m.upsample_flow(flow_lr, guid)
        assert len(got) == 1
        gold[f"tf_{name}_conf"] = got[0].numpy()
        sd = {k: v.detach().double() for k, v in m.state_dict().items()}
        oy, oc = oracle_conf(sd, name, flow_lr.double(), guid.double())
        d_out, d_conf = (oy - out.double()).abs().max().item(), (oc - got[0].double()).abs().max().item()
        print(f"teacher-forced {name}: conf in [{float(got[0].min()):.4f}, {float(got[0].max()):.4f}], oracle vs reference "
              f"out {d_out:.2e} conf {d_conf:.2e}")
        assert d_out < 1e-3 and d_conf < 1e-6, name
        meta[f"tf_{name}_oracle_vs_reference"] = {"out": d_out, "conf": d_conf}

    # ------------------------------------------------------------------ end to end, cfg-1 size
    torch.manual_seed(1234)
    m = ref_nc.RAFT(ref_args("sintel")).eval()
    got = capture(m)
    im1, im2 = frames(1, 128, 256)
    with torch.no_grad():
        lo, up = m(im1, im2, iters=4, test_mode=True)
    assert len(got) == 4
    assert np.abs(lo.numpy() - z["raft_nc_dbl_flow_low"]).max() < 1e-6
    assert np.abs(up.numpy() - z["raft_nc_dbl_flow_up"]).max() < 1e-5
    gold["e2e_conf"] = got[-1].numpy()

    # ------------------------------------------------------------------ gradients of sequence_loss + the confidence term
    ti1, ti2, gt, valid = train_inputs()
    for tag, freeze in (("full", False), ("frozen", True)):
        a = ref_args("sintel")
        a.freeze_raft = freeze
        torch.manual_seed(1234)
        m = ref_nc.RAFT(a)
        m.train()
        m.freeze_bn()                                         # train.py:185-186
        got = capture(m)
        preds = m(ti1, ti2, iters=GRAD_ITERS)
        assert len(got) == GRAD_ITERS
        flow_loss = orc.sequence_loss(preds, gt, valid, gamma=0.85)
        loss = flow_loss + conf_loss(got)
        loss.backward()
        grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
        meta[f"{tag}_loss"] = float(loss)
        meta[f"{tag}_flow_loss"] = float(flow_loss)
        meta[f"{tag}_grads"] = grad_fixture(grads)
        meta[f"{tag}_grad_norm_max"] = max(float(g.norm()) for g in grads.values())
        meta[f"{tag}_grad_none"] = [k for k, p in m.named_parameters() if p.grad is None]
        print(f"{tag}: loss {float(loss):.6f} (flow {float(flow_loss):.6f}), {len(grads)} gradients")

    np.savez_compressed(os.path.join(OUT, "conf.npz"), **gold)
    with open(os.path.join(OUT, "conf_meta.json"), "w") as f:
        json.dump(meta, f, indent=0, sort_keys=True)
    print("wrote", os.path.join(OUT, "conf.npz"), os.path.getsize(os.path.join(OUT, "conf.npz")), "bytes")


if __name__ == "__main__":
    main()
