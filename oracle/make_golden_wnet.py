"""Weights-net (Simple) configuration golden fixtures from the UNMODIFIED reference (authoring container only; needs the
reference):

    python oracle/make_golden_wnet.py     ->  tests/golden/wnet_cfg.npz + wnet_cfg_meta.json

For every configuration of CONFIGS (the --weights_est_net_* flags and the dataset, which switches BatchNorm):
  * the state_dict keys, shapes and per-tensor SHAs of the reference raft_nc_dbl model built with seed 1234;
  * the reference Simple (seed 4321, num_ch [130] + hidden, out_ch 2, sigmoid, running statistics set by
    set_running_stats) on the odd-size input simple_input() [2,130,23,37], with BatchNorm in eval mode and in train mode
    (batch statistics): its state_dict SHAs, outputs, and the norms and seeded projections (make_golden_r2.grad_fixture) of
    the gradients of L = sum(P * out) (seeded P) w.r.t. the input and every parameter.  The input and the weights are
    regenerated from their seeds by the tests, which keeps the fixture small.
For the configurations of MODEL_CONFIGS, the whole reference raft_nc_dbl model (seed 1234): test-mode flow_low / flow_up at
cfg-1 size and a training step as in make_golden_r2 (make_golden_ncup.py's recipe).
It also records whether the reference model runs with an even weights-net filter size.  TEST INFRASTRUCTURE ONLY.
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

# name -> (weights_est_net_num_ch, weights_est_net_filter_sz, weights_est_net_dilation, dataset)
CONFIGS = {
    "dilated": ([64, 32], [3, 3, 1], [1, 2, 1], "sintel"),
    "deep": ([64, 64, 32], [3, 3, 3, 1], [1, 2, 4, 1], "sintel"),
    "wide_k": ([96, 48], [5, 7, 3], [2, 1, 3], "kitti"),
    "narrow": ([32, 16], [3, 3, 1], [1, 1, 1], "kitti"),
    "head_only": ([], [5], [2], "sintel"),
}
MODEL_CONFIGS = ("dilated", "wide_k")


def args_for(name):
    num_ch, filter_sz, dilation, dataset = CONFIGS[name]
    a = ref_args(dataset)
    a.weights_est_net_num_ch, a.weights_est_net_filter_sz, a.weights_est_net_dilation = list(num_ch), list(filter_sz), list(dilation)
    return a


def simple_input():
    g = torch.Generator().manual_seed(93)
    return torch.randn(2, 130, 23, 37, generator=g)


def set_running_stats(net, seed):
    g = torch.Generator().manual_seed(seed)
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
            m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)


def main():
    warnings.filterwarnings("ignore")
    sys.path.insert(0, os.path.join(REF, "core"))
    sys.path.insert(0, ROOT)
    import raft_nc_dbl as ref_nc
    from interp_weights_est import Simple

    torch.set_num_threads(os.cpu_count())
    gold, meta = {}, {"reference_commit": "51ac387", "torch": torch.__version__, "configs": CONFIGS}
    x0 = simple_input()
    for name, (num_ch, filter_sz, dilation, dataset) in CONFIGS.items():
        torch.manual_seed(1234)
        sd = ref_nc.RAFT(args_for(name)).state_dict()
        meta[f"{name}_state_sha"] = {k: tensor_sha(v) for k, v in sd.items()}
        meta[f"{name}_state_shape"] = {k: list(v.shape) for k, v in sd.items()}

        torch.manual_seed(4321)
        net = Simple(num_ch=[130] + num_ch, out_ch=2, use_bn=dataset == "sintel", filter_sz=filter_sz, dilation=dilation,
                     final_act=torch.sigmoid)
        set_running_stats(net, 7)
        meta[f"{name}_simple_sha"] = {k: tensor_sha(v) for k, v in net.state_dict().items()}
        for mode in ("eval", "train"):
            net.train(mode == "train")
            x = x0.clone().requires_grad_(True)
            net.zero_grad(set_to_none=True)
            out = net(x)
            p = torch.randn(out.shape, generator=torch.Generator().manual_seed(5))
            (p * out).sum().backward()
            gold[f"{name}_{mode}_out"] = out.detach().numpy()
            meta[f"{name}_simple_{mode}_grads"] = grad_fixture({"input": x.grad, **{pn: prm.grad for pn, prm in net.named_parameters()}})
            if mode == "train":                       # the forward in train mode moved the running statistics: restore them
                set_running_stats(net, 7)
        print(f"{name}: {len(sd)} state keys, Simple out {tuple(out.shape)}")

    from oracle import raft_oracle as orc
    im1, im2 = frames(1, 128, 256)
    ti1, ti2, gt, valid = train_inputs()
    for name in MODEL_CONFIGS:
        a = args_for(name)
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

    # even filter sizes: the reference's padding k//2 grows the output by one pixel per even layer
    a = ref_args("sintel")
    a.weights_est_net_filter_sz = [4, 3, 1]
    torch.manual_seed(1234)
    try:
        with torch.no_grad():
            ref_nc.RAFT(a).eval()(im1, im2, iters=1, test_mode=True)
        meta["even_filter_runs"], meta["even_filter_error"] = True, ""
    except Exception as e:                                    # noqa: BLE001  (any failure of the reference counts)
        meta["even_filter_runs"], meta["even_filter_error"] = False, f"{type(e).__name__}: {e}"
    print("even filter size:", "runs" if meta["even_filter_runs"] else meta["even_filter_error"])

    np.savez_compressed(os.path.join(OUT, "wnet_cfg.npz"), **gold)
    with open(os.path.join(OUT, "wnet_cfg_meta.json"), "w") as f:
        json.dump(meta, f, indent=0, sort_keys=True)
    print("wrote", os.path.join(OUT, "wnet_cfg.npz"), os.path.getsize(os.path.join(OUT, "wnet_cfg.npz")), "bytes")


if __name__ == "__main__":
    main()
