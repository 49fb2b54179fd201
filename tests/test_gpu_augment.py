"""GPU augmentation (rnc/augment.py, csrc/augment.cu) against the reference augmentor's golden samples
(tests/golden/aug_meta.json, oracle/make_golden_aug.py): images, valid and flow bit for bit (the flow also to within 1 ulp, checked first),
through the numpy `__call__` and through `batch()`; mixed source sizes in one batch; bit-identical repeats; and a
frozen-trunk training step fed by batch() from a DataLoader."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle.make_golden_aug import STAGES, make_inputs, pick_index

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "tests", "golden", "aug_meta.json")) as _f:
    META = json.load(_f)
PICKS = np.load(os.path.join(ROOT, "tests", "golden", "aug.npz"))["flow_pick"]
DEV = "cuda:0"
gpu = pytest.mark.gpu


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def augmentor(stage):
    from rnc import augment
    sparse, params, _ = STAGES[stage]
    return (augment.SparseFlowAugmentor if sparse else augment.FlowAugmentor)(**params)


def inputs(s):
    sparse = STAGES[s["stage"]][0]
    return make_inputs(s["H"], s["W"], 1000 + s["seed"], s["grey"], sparse)


def ulp_diff(a, b):
    ia = a.astype(np.float32).view(np.int32).astype(np.int64)
    ib = b.astype(np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def check(i, img1, img2, flow, valid):
    """img1, img2 uint8 CHW; flow float32 [2,h,w]; valid float32 [h,w] (numpy)."""
    s = META["samples"][i]
    assert list(img1.shape) == s["shape"]
    assert sha(img1) == s["img1"], "img1 differs from the reference"
    assert sha(img2) == s["img2"], "img2 differs from the reference"
    assert sha(valid) == s["valid"], "valid differs from the reference"
    f = flow.reshape(-1)
    picks = f[pick_index(f.size, s["seed"])]
    assert ulp_diff(picks, PICKS[i]).max() <= 1
    assert abs(np.sqrt((flow.astype(np.float64) ** 2).sum()) - s["flow_norm"]) <= 1e-6 * s["flow_norm"]
    assert sha(flow) == s["flow"], "flow within 1 ulp of the reference but not bit-identical"


@gpu
@pytest.mark.parametrize("i", range(len(META["samples"])))
def test_call_matches_reference(i):
    s = META["samples"][i]
    aug = augmentor(s["stage"])
    img1, img2, flow, valid = inputs(s)
    np.random.seed(s["seed"])
    torch.manual_seed(s["seed"])
    with torch.cuda.device(0):
        out = aug(img1, img2, flow, valid) if valid is not None else aug(img1, img2, flow)
    o1, o2, of = out[:3]
    assert o1.dtype == np.uint8 and of.dtype == np.float32
    ft = of.transpose(2, 0, 1)
    va = out[3].astype(np.float32) if valid is not None else ((np.abs(ft[0]) < 1000) & (np.abs(ft[1]) < 1000)).astype(np.float32)
    check(i, o1.transpose(2, 0, 1), o2.transpose(2, 0, 1), ft, va)


def raw(s):
    img1, img2, flow, valid = inputs(s)
    t1 = torch.from_numpy(img1).permute(2, 0, 1).float()
    t2 = torch.from_numpy(img2).permute(2, 0, 1).float()
    tf = torch.from_numpy(flow).permute(2, 0, 1).float()
    tv = torch.from_numpy(valid).float() if valid is not None else ((tf[0].abs() < 1000) & (tf[1].abs() < 1000)).float()
    return t1, t2, tf, tv


@gpu
@pytest.mark.parametrize("i", range(len(META["samples"])))
def test_batch_matches_reference(i):
    s = META["samples"][i]
    np.random.seed(s["seed"])
    torch.manual_seed(s["seed"])
    i1, i2, fl, va = augmentor(s["stage"]).batch([raw(s)], DEV)
    check(i, i1[0].to(torch.uint8).cpu().numpy(), i2[0].to(torch.uint8).cpu().numpy(), fl[0].cpu().numpy(),
          va[0].cpu().numpy())
    assert torch.equal(i1, i1.round()) and i1.dtype == torch.float32


def mixed_samples(sparse):
    """Golden inputs of several source sizes that all admit one crop."""
    stages = ("sintel_kitti", "sintel_hd1k", "kitti") if sparse else ("chairs", "things", "sintel")
    out = []
    for st in stages:
        s = next(x for x in META["samples"] if x["stage"] == st)
        out.append(raw(s))
    return out


@gpu
@pytest.mark.parametrize("sparse", [False, True])
def test_mixed_batch_equals_per_sample_and_repeats(sparse):
    from rnc import augment
    crop = [280, 480]
    aug = augment.SparseFlowAugmentor(crop, -0.3, 0.5, do_flip=True) if sparse else augment.FlowAugmentor(crop, -0.4, 0.8)
    samples = mixed_samples(sparse) * 3                      # 9 samples, 3 source sizes, different draws
    np.random.seed(77)
    torch.manual_seed(77)
    batch = aug.batch(samples, DEV)
    np.random.seed(77)
    torch.manual_seed(77)
    again = aug.batch(samples, DEV)
    for a, b in zip(batch, again):
        assert torch.equal(a, b), "a repeat is not bit-identical"
    np.random.seed(77)
    torch.manual_seed(77)
    singles = [aug.batch([s], DEV) for s in samples]
    for k in range(4):
        assert torch.equal(batch[k], torch.cat([t[k] for t in singles])), k
    assert batch[0].shape == (9, 3, 280, 480) and batch[2].shape == (9, 2, 280, 480) and batch[3].shape == (9, 280, 480)


class RawDataset(torch.utils.data.Dataset):
    """In-memory raw samples, as a reference FlowDataset built with aug_params=None returns them."""

    def __init__(self, samples):
        self.samples = samples

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        return self.samples[i]


@gpu
def test_frozen_trunk_step_fed_by_batch():
    from conftest import build_model, ref_args
    from rnc import augment
    from rnc.train import fetch_optimizer, train_step
    build_model("raft_nc_dbl")
    import raft_nc_dbl
    torch.manual_seed(1234)
    args = ref_args("sintel")
    args.freeze_raft = True
    m = raft_nc_dbl.RAFT(args).to(DEV)
    m.train()
    m.freeze_bn()
    opt, sched = fetch_optimizer(m, lr=1e-4, num_steps=10)
    loader = torch.utils.data.DataLoader(RawDataset(mixed_samples(False)[:2]), batch_size=2, collate_fn=list)
    aug = augment.FlowAugmentor([256, 384], -0.2, 0.6)
    torch.manual_seed(5)
    np.random.seed(5)
    for raw_batch in loader:
        im1, im2, flow, valid = aug.batch(raw_batch, DEV)
        loss = float(train_step(m, opt, sched, im1, im2, flow, valid, iters=2)[0])
        assert np.isfinite(loss), loss
