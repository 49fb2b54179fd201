"""Parity on the configuration bench.py actually times (BASELINE configs[2]: B = 8, 1024x436 padded to 440, 32 iterations)
and on the two other stimuli of SURVEY.md §8d: every pair of the batch equals the same pair run alone, pairs 0 and 7 are
within the north star's 1e-3 EPE of the CPU oracle, and the smooth-shift / motion-boundary stimuli (the latter drives the
lookup's exact fallback path) hold the same bar end to end."""
import pytest
import torch

from conftest import build_model
from oracle import raft_oracle as orc
from rnc.synth import frames, motion_boundary_flow_init, smooth_shift_frames

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-3                                  # north-star tolerance: EPE of flow_up vs the reference algorithm


def epe(a, b):
    return (a - b).pow(2).sum(1).sqrt().mean().item()


def padded(b, maker=frames, **kw):
    from utils.utils import InputPadder
    im1, im2 = maker(b, 436, 1024, **kw)
    return InputPadder(im1.shape, "sintel").pad(im1, im2)


def fallback_units(model, B, H8, W8):
    eng = model.engine()
    ws = next(w for k, w in eng._ws.items() if k[0] == "umma" and (w.B, w.H8, w.W8) == (B, H8, W8))
    return int((ws.lookup_flags != 0).sum().item()), ws.lookup_flags.numel()


@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_benchmarked_batch_of_8_matches_single_pairs_and_oracle(name):
    m = build_model(name).to(DEV)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    p1, p2 = padded(8)
    with torch.no_grad():
        lo8, up8 = m(p1.to(DEV), p2.to(DEV), iters=32, test_mode=True)
        worst = 0.0
        for i in range(8):
            _, up1 = m(p1[i:i + 1].to(DEV), p2[i:i + 1].to(DEV), iters=32, test_mode=True)
            worst = max(worst, epe(up8[i:i + 1], up1))
    print(f"{name}: B=8 vs B=1 worst EPE {worst:.2e}")
    assert worst < 1e-4
    for i in (0, 7):
        _, oup, _ = orc.raft_forward(sd, p1[i:i + 1], p2[i:i + 1], iters=32, model=name, upsample_every_iter=False)
        e = epe(up8[i:i + 1].cpu(), oup)
        print(f"{name}: pair {i} of the B=8 step vs oracle EPE {e:.2e} (|flow_up| {oup.abs().mean():.1f} px)")
        assert e < TOL


@pytest.mark.parametrize("name", ["raft_nc_dbl", "raft"])
def test_smooth_shift_stimulus_end_to_end(name):
    m = build_model(name).to(DEV)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    p1, p2 = padded(2, smooth_shift_frames)
    with torch.no_grad():
        _, up = m(p1.to(DEV), p2.to(DEV), iters=32, test_mode=True)
    _, oup, _ = orc.raft_forward(sd, p1[:1], p2[:1], iters=32, model=name, upsample_every_iter=False)
    e = epe(up[:1].cpu(), oup)
    print(f"{name} smooth-shift: EPE vs oracle {e:.2e}")
    assert e < TOL


def test_motion_boundary_stimulus_uses_the_fallback_and_stays_exact():
    """Warm start with a 24 px (1/8-res) flow discontinuity: the boundary tiles' windows do not fit the fixed boxes of the
    tensor-core lookup, so they go through the exact kernel; results must not depend on coherence."""
    m = build_model("raft_nc_dbl").to(DEV)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    p1, p2 = padded(2)
    init = motion_boundary_flow_init(2, 55, 128)
    with torch.no_grad():
        lo, up = m(p1.to(DEV), p2.to(DEV), iters=12, flow_init=init.to(DEV), test_mode=True)
    n_fb, n_units = fallback_units(m, 2, 55, 128)
    print(f"motion boundary: {n_fb} of {n_units} (tile, level) units recomputed by the exact kernel in the last iteration")
    assert n_fb > 0
    olo, oup, _ = orc.raft_forward(sd, p1[:1], p2[:1], iters=12, flow_init=init[:1], upsample_every_iter=False)
    e_lo, e_up = epe(lo[:1].cpu(), olo), epe(up[:1].cpu(), oup)
    print(f"motion boundary: EPE flow_low {e_lo:.2e} flow_up {e_up:.2e}")
    assert e_up < TOL and e_lo < TOL / 4


def test_realistic_feature_magnitudes_in_the_lookup():
    """Feature maps 30x larger than the random-init ones (trained checkpoints are not available offline): the tensor-core
    lookup rounds features to fp16 once; its output must stay within its error model (tests/test_lookup_error_model.py) of
    the fp64 lookup, and close to the exact fp32 CorrBlock."""
    from rnc.engine import engine_for
    from test_gpu_lookup_error_model import umma_lookup_model
    eng = engine_for(torch.device(DEV))
    if eng.mode != "umma":
        pytest.skip("tensor-core engine only")
    g = torch.Generator().manual_seed(3)
    f1, f2 = torch.randn(2, 256, 55, 128, generator=g) * 45, torch.randn(2, 256, 55, 128, generator=g) * 45
    co = orc.coords_grid(2, 55, 128) + torch.randn(2, 2, 55, 128, generator=g) * 3
    from corr import CorrBlock
    exact = CorrBlock(f1.to(DEV), f2.to(DEV))(co.to(DEV)).cpu()
    got, flags = umma_lookup_model("|fmap| ~ 45", f1, f2, co)
    scale = exact.abs().max().item()
    err = (got - exact).abs().max().item()
    print(f"lookup with |fmap| ~ 45: max err {err:.3e} on scale {scale:.1f} vs CorrBlock, {int(flags.sum())} units flagged")
    assert err < 1e-3 * scale
