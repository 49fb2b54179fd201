"""Bidirectional sequence inference on the host: rnc.harness.run_sequences_bidirectional's argument checks, which raise
before any launch, and the backward warm-start rule it implements on the device."""
import numpy as np
import pytest
import torch

from rnc.harness import run_sequences_bidirectional


def test_mismatched_frame_sizes_raise():
    seqs = [[torch.zeros(3, 64, 96)] * 3, [torch.zeros(3, 64, 96), torch.zeros(3, 64, 104)]]
    with pytest.raises(ValueError, match=r"\(3, 64, 96\) and \(3, 64, 104\)"):
        next(run_sequences_bidirectional(None, seqs, device="cpu"))


def test_one_frame_sequences_yield_nothing():
    assert list(run_sequences_bidirectional(None, [[torch.zeros(3, 64, 96)]], device="cpu")) == []


class _Stub(torch.nn.Module):
    """A model shell that fails the test if anything past the argument checks touches it."""

    def __init__(self, ncup):
        super().__init__()
        self.ncup = ncup
        self.w = torch.nn.Parameter(torch.zeros(1))

    def _needs_grad(self):
        return torch.is_grad_enabled() and self.w.requires_grad

    def eval(self):
        raise AssertionError("reached the steps")


def test_return_confidence_on_the_convex_model_raises():
    seqs = [[torch.zeros(3, 64, 96)] * 3]
    with torch.no_grad(), pytest.raises(ValueError, match="return_confidence"):
        next(run_sequences_bidirectional(_Stub(ncup=False), seqs, device="cpu", return_confidence=True))


def test_grad_enabled_on_a_model_that_requires_grad_raises():
    seqs = [[torch.zeros(3, 64, 96)] * 3]
    with pytest.raises(ValueError, match="inference only"):
        next(run_sequences_bidirectional(_Stub(ncup=True), seqs, device="cpu"))


def test_batch_size_below_one_raises():
    with pytest.raises(ValueError, match="batch_size"):
        next(run_sequences_bidirectional(None, [[torch.zeros(3, 64, 96)] * 2], batch_size=0, device="cpu"))


def _splat_backward(b):
    """The backward warm-start rule written out directly: every sample of b [2,H,W] moves to x - b(x), samples landing
    strictly inside the frame are kept, and each grid point takes the b(x) of its nearest kept sample (scipy griddata
    'nearest', fill 0), as the reference's forward_interpolate does with x + f(x)."""
    from scipy import interpolate
    f = b.numpy()
    dx, dy = f[0], f[1]
    ht, wd = dx.shape
    x0, y0 = np.meshgrid(np.arange(wd), np.arange(ht))
    x1, y1 = (x0 - dx).reshape(-1), (y0 - dy).reshape(-1)
    dxr, dyr = dx.reshape(-1), dy.reshape(-1)
    ok = (x1 > 0) & (x1 < wd) & (y1 > 0) & (y1 < ht)
    fx = interpolate.griddata((x1[ok], y1[ok]), dxr[ok], (x0, y0), method="nearest", fill_value=0)
    fy = interpolate.griddata((x1[ok], y1[ok]), dyr[ok], (x0, y0), method="nearest", fill_value=0)
    return torch.from_numpy(np.stack([fx, fy], 0)).float()


def _flows():
    g = torch.Generator().manual_seed(3)
    yield torch.randn(2, 9, 13, generator=g) * 3                       # many samples leave the frame
    t = torch.zeros(2, 8, 12)                                         # integer flows: samples land on one point and tie
    t[0, :, ::2], t[0, :, 1::2], t[1, 2:5] = 1.0, -1.0, 2.0
    yield t
    t = torch.full((2, 6, 9), 40.0)                                   # all samples but two leave the frame
    t[:, 2, 3], t[:, 4, 7] = 0.5, -1.5
    yield t
    yield torch.zeros(2, 6, 9)                                        # x = 0 and y = 0 samples are dropped (strict test)


@pytest.mark.parametrize("i", range(4))
def test_backward_rule_is_the_mirrored_forward_interpolate(i):
    from oracle import raft_oracle as orc
    b = list(_flows())[i]
    want = _splat_backward(b)
    got = -orc.forward_interpolate(-b)
    assert torch.equal(got, want)
    if i == 0:
        assert not torch.equal(orc.forward_interpolate(b), want)       # the direction of the splat matters
