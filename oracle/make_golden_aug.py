"""Augmentation golden fixtures from the UNMODIFIED reference augmentor (authoring container only; needs the reference, cv2,
Pillow and torchvision):

    python oracle/make_golden_aug.py     ->  tests/golden/aug.npz + aug_meta.json

For every stage of STAGES (the aug_params of each fetch_dataloader stage, core/datasets.py:201-236, with realistic source and
crop sizes) and each of its seeds: the inputs make_inputs(...) regenerates from the seed, then np.random.seed(seed),
torch.manual_seed(seed) and one reference augmentor call followed by FlowDataset.__getitem__'s tensor conversion
(datasets.py:81-90).  Recorded per sample: SHA-256 of img1, img2 (uint8 CHW) and valid (float32), SHA-256, float64 norm and
N_PICK sampled values of the float32 flow, SHA-256 of both RNG states after the call, and the parameters rnc.augment's draw()
makes from the same seed (the tests check that those repeat).  Seeds are added until every branch occurs (COVERAGE).
TEST INFRASTRUCTURE ONLY.
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("RNC_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden")
N_PICK = 300

# name -> (sparse, aug_params, source (H, W), seeds tried first)
STAGES = {
    "chairs": (False, dict(crop_size=[368, 496], min_scale=-0.1, max_scale=1.0, do_flip=True), (384, 512)),
    "things": (False, dict(crop_size=[400, 720], min_scale=-0.4, max_scale=0.8, do_flip=True), (540, 960)),
    "sintel": (False, dict(crop_size=[368, 768], min_scale=-0.2, max_scale=0.6, do_flip=True), (436, 1024)),
    "sintel_kitti": (True, dict(crop_size=[368, 768], min_scale=-0.3, max_scale=0.5, do_flip=True), (375, 1242)),
    "sintel_hd1k": (True, dict(crop_size=[368, 768], min_scale=-0.5, max_scale=0.2, do_flip=True), (1080, 2560)),
    "kitti": (True, dict(crop_size=[288, 960], min_scale=-0.2, max_scale=0.4, do_flip=False), (375, 1242)),
}
SEEDS_PER_STAGE = 6


def make_inputs(H, W, seed, grey, sparse):
    """Smooth structure plus noise, saturated 0 / 255 blocks, flow values beyond 1000; grey = one channel tiled, as
    datasets.py:68-70 does for grey-scale frames."""
    r = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    imgs = []
    for _ in range(2):
        base = 128 + 110 * np.sin(xx / (20 + 30 * r.rand()) + 6 * r.rand()) * np.cos(yy / (15 + 25 * r.rand()) + 6 * r.rand())
        im = np.clip(base[..., None] + r.randn(H, W, 3) * 25, 0, 255).astype(np.uint8)
        im[: H // 8] = 255
        im[-H // 10:, : W // 6] = 0
        if grey:
            im = np.tile(im[..., :1], (1, 1, 3))
        imgs.append(im)
    flow = (r.randn(H, W, 2) * 6 + 20 * np.sin(xx / 50)[..., None]).astype(np.float32)
    flow[H // 3: H // 3 + 40, W // 2: W // 2 + 60, 0] = 1500.0
    flow[H // 2: H // 2 + 30, W // 4: W // 4 + 50, 1] = -2400.0
    valid = (r.rand(H, W) < 0.4).astype(np.float32) if sparse else None
    return imgs[0], imgs[1], flow, valid


def pick_index(n, seed):
    return np.random.RandomState(seed + 7919).randint(0, n, N_PICK)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def rng_digest():
    st = np.random.get_state()
    h = hashlib.sha256(st[1].tobytes() + str(st[2]).encode())
    h.update(torch.get_rng_state().numpy().tobytes())
    return h.hexdigest()


def record(img1, img2, flow, valid, seed):
    """FlowDataset.__getitem__'s conversion, then the digests the tests compare."""
    i1 = torch.from_numpy(img1).permute(2, 0, 1).float()
    i2 = torch.from_numpy(img2).permute(2, 0, 1).float()
    fl = torch.from_numpy(flow).permute(2, 0, 1).float()
    va = torch.from_numpy(valid).float() if valid is not None else ((fl[0].abs() < 1000) & (fl[1].abs() < 1000)).float()
    f = fl.numpy()
    return {"img1": sha(i1.numpy().astype(np.uint8)), "img2": sha(i2.numpy().astype(np.uint8)), "valid": sha(va.numpy()),
            "flow": sha(f), "flow_norm": float(np.sqrt((f.astype(np.float64) ** 2).sum())),
            "flow_pick": f.reshape(-1)[pick_index(f.size, seed)].tolist(), "shape": list(i1.shape)}


def coverage(d, stage_sparse, H, W):
    c = set()
    c.add("asym" if d["asym"] else "sym")
    c.add(f"erase{len(d['erase'])}")
    if any(x + dx > W or y + dy > H for x, y, dx, dy in d["erase"]):
        c.add("erase_clipped")
    c.add("resized" if d["resized"] else "not_resized")
    if d["fx"] != d["fy"]:
        c.add("stretch")
    if d["hflip"]:
        c.add("hflip")
    if d["vflip"]:
        c.add("vflip")
    if stage_sparse and d["resized"] and d["fx"] < 1:
        c.add("sparse_downscale")
    return c


COVERAGE = {"asym", "sym", "erase0", "erase1", "erase2", "erase_clipped", "resized", "not_resized", "stretch", "hflip",
            "vflip", "sparse_downscale"}


def main():
    sys.path.insert(0, os.path.join(REF, "core"))
    sys.path.insert(1, os.path.join(ROOT, "raft-ncup_b200"))
    import cv2
    import PIL
    import torchvision
    from utils.augmentor import FlowAugmentor, SparseFlowAugmentor     # the reference's
    from rnc import augment as gpu_aug
    cv2.setNumThreads(1)
    samples, seen = [], set()
    for stage, (sparse, params, (H, W)) in STAGES.items():
        ref = (SparseFlowAugmentor if sparse else FlowAugmentor)(**params)
        mine = (gpu_aug.SparseFlowAugmentor if sparse else gpu_aug.FlowAugmentor)(**params)
        possible = COVERAGE - ({"asym", "vflip", "stretch"} if sparse else {"sparse_downscale"})
        if not params["do_flip"]:
            possible -= {"hflip", "vflip"}
        seed, n = 0, 0
        while n < SEEDS_PER_STAGE or (not possible <= seen and seed < 400):
            grey = seed % 3 == 2
            np.random.seed(seed); torch.manual_seed(seed)
            d = mine.draw(H, W)
            cov = coverage(d, sparse, H, W)
            if n >= SEEDS_PER_STAGE and (cov & possible) <= seen:
                seed += 1
                continue
            img1, img2, flow, valid = make_inputs(H, W, 1000 + seed, grey, sparse)
            np.random.seed(seed); torch.manual_seed(seed)
            out = ref(img1, img2, flow, valid) if sparse else ref(img1, img2, flow)
            if not sparse:
                out = tuple(out) + (None,)
            rec = record(*out, seed)
            rec.update(stage=stage, seed=seed, grey=grey, H=H, W=W, rng=rng_digest(), draw=d, coverage=sorted(cov))
            samples.append(rec)
            seen |= cov
            n += 1
            seed += 1
    missing = COVERAGE - seen
    assert not missing, missing
    meta = {"cv2": cv2.__version__, "Pillow": PIL.__version__, "torchvision": torchvision.__version__,
            "numpy": np.__version__, "torch": torch.__version__, "stages": {k: [v[0], v[1], list(v[2])] for k, v in STAGES.items()},
            "n_pick": N_PICK, "samples": samples}
    with open(os.path.join(OUT, "aug_meta.json"), "w") as f:
        json.dump(meta, f, indent=1)
    # the flow picks in full precision (the JSON keeps them too, for reading)
    np.savez_compressed(os.path.join(OUT, "aug.npz"), flow_pick=np.array([s["flow_pick"] for s in samples], np.float32))
    print(f"{len(samples)} samples, coverage {sorted(seen)}")


if __name__ == "__main__":
    main()
