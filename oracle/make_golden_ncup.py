"""NConvUNet-configuration golden fixtures from the UNMODIFIED reference (authoring container only; needs the reference):

    python oracle/make_golden_ncup.py     ->  tests/golden/ncup_cfg.npz + ncup_cfg_meta.json

For every configuration of oracle/ncup_oracle.py:CONFIGS:
  * the state_dict keys, shapes and per-tensor SHAs of the reference raft_nc_dbl model built with seed 1234 and the
    configuration's --interp_net_* flags;
  * the reference NConvUNet (seed 4321) on zero-stuffed inputs (one sample with all-zero confidence) and on an odd-size
    input with quantised data (pooling ties in data and confidence); its state_dict;
  * gradients of L = sum(P1 * xout) + sum(P2 * cout) (seeded P) w.r.t. data, conf and every parameter, and the names of the
    parameters whose gradient is None.
For the configurations of MODEL_CONFIGS, the whole reference raft_nc_dbl model (seed 1234):
  * test-mode flow_low / flow_up at cfg-1 size (one 128x256 pair of make_golden.frames, 4 iterations);
  * a training step as in make_golden_r2 (train mode, frozen BatchNorm, 128x160, B = 2, 3 iterations, sequence_loss with
    gamma 0.85): the loss, per-parameter gradient norms and seeded projections (make_golden_r2.grad_fixture), the largest
    gradient norm and the parameters whose gradient is None.
The restated oracle (ncup_oracle.unet) is asserted against the reference outputs here.  TEST INFRASTRUCTURE ONLY.
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from make_golden import OUT, REF, frames, ref_args, tensor_sha   # noqa: E402
from make_golden_r2 import GRAD_ITERS, grad_fixture, train_inputs   # noqa: E402
import ncup_oracle as nco                                # noqa: E402


MODEL_CONFIGS = ("paper", "wide")


def zero_stuff(x, scale=4):
    b, c, h, w = x.shape
    out = torch.zeros(b, c, h * scale, w * scale, dtype=x.dtype)
    out[:, :, scale // 2::scale, scale // 2::scale] = x
    return out


def inputs():
    """(data, conf) pairs: zero-stuffed [3,1,40,48] with sample 2 all-zero confidence; odd-size [2,1,23,37] with
    quantised data and confidence (ties)."""
    g = torch.Generator().manual_seed(91)
    d = zero_stuff(torch.randn(3, 1, 10, 12, generator=g) * 4)
    c = zero_stuff(torch.rand(3, 1, 10, 12, generator=g))
    c[2] = 0.0
    d2 = torch.round(torch.randn(2, 1, 23, 37, generator=g) * 2) / 2
    c2 = torch.round(torch.rand(2, 1, 23, 37, generator=g) * 4) / 4
    c2[c2 < 0.5] = 0.0
    return {"even": (d, c), "odd": (d2, c2)}


def projections(xo, co, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(xo.shape, generator=g, dtype=xo.dtype), torch.randn(co.shape, generator=g, dtype=co.dtype)


def main():
    warnings.filterwarnings("ignore")
    sys.path.insert(0, os.path.join(REF, "core"))
    sys.path.insert(0, ROOT)
    import raft_nc_dbl as ref_nc
    from nconv_modules import NConvUNet

    torch.set_num_threads(os.cpu_count())
    gold, meta = {}, {"reference_commit": "51ac387", "torch": torch.__version__, "configs": nco.CONFIGS}
    ins = inputs()
    for k, (d, c) in ins.items():
        gold[f"in_{k}_data"], gold[f"in_{k}_conf"] = d.numpy(), c.numpy()
    for name, cfg in nco.CONFIGS.items():
        a = ref_args("sintel")
        for k, v in nco.args_overrides(cfg).items():
            setattr(a, k, v)
        torch.manual_seed(1234)
        m = ref_nc.RAFT(a)
        sd = m.state_dict()
        meta[f"{name}_state_sha"] = {k: tensor_sha(v) for k, v in sd.items()}
        meta[f"{name}_state_shape"] = {k: list(v.shape) for k, v in sd.items()}

        torch.manual_seed(4321)
        net = NConvUNet(**nco.unet_kwargs(cfg))
        for k, v in net.state_dict().items():
            gold[f"{name}_sd_{k}"] = v.numpy()
        for kin, (d, c) in ins.items():
            d, c = d.clone().requires_grad_(True), c.clone().requires_grad_(True)
            net.zero_grad(set_to_none=True)
            xo, co = net((d, c))
            p1, p2 = projections(xo, co, 5)
            ((p1 * xo).sum() + (p2 * co).sum()).backward()
            gold[f"{name}_{kin}_xout"], gold[f"{name}_{kin}_cout"] = xo.detach().numpy(), co.detach().numpy()
            gold[f"{name}_{kin}_gdata"], gold[f"{name}_{kin}_gconf"] = d.grad.numpy(), c.grad.numpy()
            none = []
            for pn, p in net.named_parameters():
                if p.grad is None:
                    none.append(pn)
                else:
                    gold[f"{name}_{kin}_g_{pn}"] = p.grad.numpy()
            meta[f"{name}_{kin}_grad_none"] = none
            osd = {k: v.double() for k, v in net.state_dict().items()}
            ox, oc = nco.unet(osd, cfg, d.detach().double(), c.detach().double())
            assert (ox - xo.detach().double()).abs().max() < 1e-4 and (oc - co.detach().double()).abs().max() < 1e-6, name
        print(f"{name}: {len(sd)} state keys, grad None for {meta[f'{name}_even_grad_none']}")

    from oracle import raft_oracle as orc
    im1, im2 = frames(1, 128, 256)
    ti1, ti2, gt, valid = train_inputs()
    for name in MODEL_CONFIGS:
        a = ref_args("sintel")
        for k, v in nco.args_overrides(nco.CONFIGS[name]).items():
            setattr(a, k, v)
        torch.manual_seed(1234)
        m = ref_nc.RAFT(a).eval()
        with torch.no_grad():
            lo, up = m(im1, im2, iters=4, test_mode=True)
        gold[f"{name}_cfg1_flow_low"], gold[f"{name}_cfg1_flow_up"] = lo.numpy(), up.numpy()
        torch.manual_seed(1234)
        m = ref_nc.RAFT(a)
        m.train()
        m.freeze_bn()                                         # train.py:185-186
        loss = orc.sequence_loss(m(ti1, ti2, iters=GRAD_ITERS), gt, valid, gamma=0.85)
        loss.backward()
        grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
        meta[f"{name}_train_loss"] = float(loss)
        meta[f"{name}_train_grads"] = grad_fixture(grads)
        meta[f"{name}_train_grad_norm_max"] = max(float(g.norm()) for g in grads.values())
        meta[f"{name}_train_grad_none"] = [k for k, p in m.named_parameters() if p.grad is None]
        print(f"{name}: cfg-1 |flow_up| mean {float(up.abs().mean()):.4f}, train loss {float(loss):.6f}")

    np.savez_compressed(os.path.join(OUT, "ncup_cfg.npz"), **gold)
    with open(os.path.join(OUT, "ncup_cfg_meta.json"), "w") as f:
        json.dump(meta, f, indent=0, sort_keys=True)
    print("wrote", os.path.join(OUT, "ncup_cfg.npz"), os.path.getsize(os.path.join(OUT, "ncup_cfg.npz")), "bytes")


if __name__ == "__main__":
    main()
