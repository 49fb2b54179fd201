"""NCUP output confidence (CPU): the oracle's confidence and gradients against the reference's (tests/golden/conf.npz, made
by oracle/make_golden_conf.py), the public surface's refusals, and the NCUP entry points (whose conf_out / g_conf_out
request the confidence) in the C header, the binding and the library's argument and grid checks."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT, build_model, ref_args
from oracle import ncup_oracle as nco
from oracle import raft_oracle as orc
from oracle.make_golden_conf import conf_loss, oracle_conf, tf_inputs
from oracle.make_golden_r2 import GRAD_ITERS, grad_fixture, tied_leaves, train_inputs

NCUP = ("rnc_ncup_fwd", "rnc_ncup_train_fwd", "rnc_ncup_bwd")
# folded into NCUP (the confidence is an optional output there) or unused, at ABI 17
REMOVED = ("rnc_ncup_conf_fwd", "rnc_ncup_train_conf_fwd", "rnc_ncup_conf_bwd", "rnc_add_relu_split")


def load_conf():
    z = np.load(os.path.join(ROOT, "tests", "golden", "conf.npz"))
    with open(os.path.join(ROOT, "tests", "golden", "conf_meta.json")) as f:
        return {k: torch.from_numpy(z[k]) for k in z.files}, json.load(f)


def variant_model(name):
    """raft_nc_dbl with seed 1234: the shipped network, or a configuration of ncup_oracle.CONFIGS (identical weights to the
    reference's, tests/test_ncup_variants.py)."""
    if name == "shipped":
        return build_model("raft_nc_dbl")
    import raft_nc_dbl
    a = ref_args("sintel")
    for k, v in nco.args_overrides(nco.CONFIGS[name]).items():
        setattr(a, k, v)
    torch.manual_seed(1234)
    return raft_nc_dbl.RAFT(a).eval()


@pytest.mark.parametrize("name", ["shipped", "wide"])
def test_oracle_confidence_matches_the_reference(name):
    g, _ = load_conf()
    sd = {k: v.detach().double() for k, v in variant_model(name).state_dict().items()}
    flow_lr, guid = tf_inputs(np.load(os.path.join(ROOT, "tests", "golden", "cfg1.npz")))
    _, conf = oracle_conf(sd, name, flow_lr.double(), guid.double())
    assert conf.shape == g[f"tf_{name}_conf"].shape == (1, 2, 64, 128)
    assert (conf - g[f"tf_{name}_conf"].double()).abs().max() < 1e-6
    assert float(conf.min()) >= 0.0 and float(conf.max()) <= 1.0


def test_oracle_gradients_of_the_confidence_loss_match_the_reference(monkeypatch):
    """The oracle's autograd of sequence_loss + sum_i P_i . conf_i (the confidence captured from its NConvUNet, as the
    fixture's hook captures the reference's) against the reference's gradients: the bounds of tests/test_r2_golden.py."""
    _, meta = load_conf()
    m = build_model("raft_nc_dbl")
    im1, im2, gt, valid = train_inputs()
    sd, leaves = tied_leaves(m)
    confs, live = [], orc.nconv_unet_live

    def capturing(*a, **k):
        y, c = live(*a, **k)
        confs.append(c.view(c.shape[0] // 2, 2, c.shape[2], c.shape[3]))
        return y, c

    monkeypatch.setattr(orc, "nconv_unet_live", capturing)
    _, _, ups = orc.raft_forward_graph(sd, im1, im2, iters=GRAD_ITERS, model="raft_nc_dbl")
    assert len(confs) == GRAD_ITERS
    loss = orc.sequence_loss(ups, gt, valid, gamma=0.85) + conf_loss(confs)
    loss.backward()
    assert abs(float(loss.detach()) - meta["full_loss"]) < 1e-4
    gmax = meta["full_grad_norm_max"]
    fix, ref = grad_fixture({k: v.grad for k, v in leaves.items() if v.grad is not None}), meta["full_grads"]
    assert set(fix) == set(ref)
    for k in ref:
        tol = 2e-3 * ref[k][0] + 1e-5 * gmax
        n = leaves[k].numel() ** 0.5
        assert abs(fix[k][0] - ref[k][0]) < tol, k
        assert all(abs(a - b) < tol * n for a, b in zip(fix[k][1:], ref[k][1:])), k


def test_convex_model_refuses_confidence():
    m = build_model("raft")
    im = torch.zeros(1, 3, 64, 64)
    with pytest.raises(ValueError, match="return_confidence"):
        m(im, im, iters=1, test_mode=True, return_confidence=True)


def test_cpu_tensors_are_refused_when_the_confidence_is_requested():
    from rnc.native import RncUnavailable
    from rnc.train import NcupChainFn
    m = build_model("raft_nc_dbl")
    im = torch.zeros(1, 3, 64, 64)
    with torch.no_grad(), pytest.raises(RncUnavailable):
        m(im, im, iters=1, test_mode=True, return_confidence=True)
    with torch.no_grad(), pytest.raises(RncUnavailable):
        m.upsampler(torch.zeros(1, 2, 16, 16), torch.zeros(1, 128, 8, 8), return_confidence=True)
    ws = [torch.ones(*s) for s in ((2, 1, 5, 5), (2, 2, 5, 5), (2, 4, 3, 3), (1, 2, 1, 1))]
    with pytest.raises(RncUnavailable):
        NcupChainFn.apply(torch.zeros(1, 2, 4, 4), torch.zeros(1, 2, 4, 4), *ws, 8.0, True)


def test_ncup_entry_points_are_declared_bound_and_versioned():
    from rnc import native
    with open(os.path.join(ROOT, "include", "rnc.h")) as f:
        header = f.read()
    with open(os.path.join(ROOT, "raft-ncup_b200", "csrc", "layout.cu")) as f:
        layout = f.read()
    declared = set(re.findall(r"\b(rnc_\w+)\s*\(", header))
    assert all(n in declared and n in native.SIGNATURES for n in NCUP)
    assert native.ABI_VERSION == 18 and "(now 18)" in header and "rnc_abi_version(void) { return 18; }" in layout
    L = native.lib()
    assert L.rnc_abi_version() == 18
    for n in REMOVED:
        assert n not in header and n not in native.SIGNATURES and not hasattr(L, n), n


def test_ncup_entry_points_with_confidence_reject_bad_arguments():
    """Status codes of the argument checks, which return before anything is launched."""
    from rnc import native
    L = native.lib()
    p = ctypes.c_void_p(16)
    hw = (ctypes.c_float * 224)(*([1.0] * 224))
    assert L.rnc_ncup_fwd(p, p, hw, 0, 4, 4, 8.0, p, p, None) == -1
    assert L.rnc_ncup_fwd(p, p, hw, 1, 4, 4, 8.0, None, p, None) == -2
    assert L.rnc_ncup_fwd(p, p, None, 1, 4, 4, 8.0, p, p, None) == -2
    assert L.rnc_ncup_train_fwd(p, p, p, 1, 0, 4, 8.0, p, p, None) == -1
    assert L.rnc_ncup_train_fwd(p, p, None, 1, 4, 4, 8.0, p, p, None) == -2
    assert L.rnc_ncup_train_fwd(p, p, p, 1, 4, 4, 8.0, None, p, None) == -2
    # (..., g_out, g_conf_out, g_x_lowres, g_conf, g_weights, workspace, workspace_bytes, stream)
    assert L.rnc_ncup_bwd(p, p, p, 0, 4, 4, 8.0, p, p, p, p, p, p, 1 << 20, None) == -1
    assert L.rnc_ncup_bwd(p, p, p, 1, 4, 4, 8.0, None, None, p, p, p, p, 1 << 20, None) == -2     # no upstream gradient
    assert L.rnc_ncup_bwd(None, p, p, 1, 4, 4, 8.0, None, p, p, p, p, p, 1 << 20, None) == -2
    assert L.rnc_ncup_bwd(p, p, p, 1, 4, 4, 8.0, None, p, None, None, None, None, 0, None) == -2
    assert L.rnc_ncup_bwd(p, p, p, 1, 4, 4, 8.0, p, p, p, p, p, None, 1 << 20, None) == -2
    assert L.rnc_ncup_bwd(p, p, p, 1, 4, 4, 8.0, None, p, p, p, p, p, 8, None) == -5
    assert L.rnc_ncup_bwd(p, p, p, 1, 4, 4, 8.0, p, None, p, p, p, p, 8, None) == -5


@pytest.mark.parametrize("conf_out", [False, True], ids=["flow", "conf"])
def test_ncup_entry_points_reject_grids_past_the_launch_limits(conf_out):
    """2*B and the rows of output tiles are bounded by the 65535 limit of grid.z / grid.y of the grid each call launches:
    30x30 tiles forward (H4 = 500000: 66667 rows), 32x32 backward (H4 = 600000: 75000 rows; 500000 would be 62500, a valid
    grid).  Every case returns RNC_ERR_UNSUPPORTED before anything is launched, with or without the confidence."""
    from rnc import native
    L = native.lib()
    p = ctypes.c_void_p(16)
    c = p if conf_out else None
    hw = (ctypes.c_float * 224)(*([1.0] * 224))
    before = L.rnc_launch_count()
    for B, H4, W4 in ((1, 500000, 4), (40000, 4, 4)):
        assert L.rnc_ncup_fwd(p, p, hw, B, H4, W4, 8.0, p, c, None) == -3, (B, H4, W4)
        assert L.rnc_ncup_train_fwd(p, p, p, B, H4, W4, 8.0, p, c, None) == -3, (B, H4, W4)
    for B, H4, W4 in ((40000, 4, 4), (1, 600000, 4)):
        assert L.rnc_ncup_bwd(p, p, p, B, H4, W4, 8.0, p, c, p, p, p, p, 1 << 40, None) == -3, (B, H4, W4)
    assert L.rnc_launch_count() == before
