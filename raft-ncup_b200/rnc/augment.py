"""Training-sample augmentation on the GPU: the reference's `FlowAugmentor` and `SparseFlowAugmentor`
(core/utils/augmentor.py) as librnc kernels (csrc/augment.cu).

The random parameters are drawn on the host, consuming `np.random` and torch's global generator in exactly the reference's
order and number (`draw`).  The kernels then apply them with Pillow's and cv2's own rounding, so from the same RNG state a
sample comes out as the reference's augmenting `FlowDataset.__getitem__` returns it: images and `valid` bit for bit, the flow
to float32 rounding.

- `aug(img1, img2, flow[, valid])`: the reference's numpy HWC in / numpy out call, run on the current CUDA device.  The
  returned flow is float32 (the value `FlowDataset` converts it to); everything else has the reference's dtypes.
- `aug.batch(samples, device)`: the training path.  `samples` are raw samples as a reference `FlowDataset` built with
  `aug_params=None` returns them (float `[3,H,W]` images with integer values, `[2,H,W]` flow, `[H,W]` valid), of any
  sizes.  Returns `img1, img2 [B,3,h,w]`, `flow [B,2,h,w]`, `valid [B,h,w]` on `device`: the stack of what the
  augmenting dataset returns for the same RNG state, samples drawn in list order.  Host work is the draws and one packed
  host-to-device copy; the kernels run one launch per pass for the whole batch.
"""
import ctypes as C

import numpy as np
import torch

from . import native

_ALIGN = 16


def _jitter_range(v, center):
    """torchvision ColorJitter._check_input for a scalar."""
    return [max(center - float(v), 0.0), center + float(v)] if center == 1 else [center - float(v), center + float(v)]


class _Augmentor:
    sparse = False

    def __init__(self, crop_size, min_scale, max_scale, do_flip, jitter):
        self.crop_size = crop_size
        self.min_scale = min_scale
        self.max_scale = max_scale
        self.spatial_aug_prob = 0.8
        self.stretch_prob = 0.8
        self.max_stretch = 0.2
        self.do_flip = do_flip
        self.h_flip_prob = 0.5
        self.v_flip_prob = 0.1
        b, c, s, h = jitter
        self.jitter_ranges = (_jitter_range(b, 1), _jitter_range(c, 1), _jitter_range(s, 1), _jitter_range(h, 0))
        self.asymmetric_color_aug_prob = 0.2
        self.eraser_aug_prob = 0.5

    # ---- draws (reference order) -----------------------------------------------------------------------------------
    def _jitter_params(self):
        """ColorJitter.get_params: randperm(4), then one float32 uniform per factor."""
        perm = [int(i) for i in torch.randperm(4)]
        f = [float(torch.empty(1).uniform_(lo, hi)) for lo, hi in self.jitter_ranges]
        hue = int(np.int32(f[3] * 255).astype(np.uint8))
        return perm, f[:3], hue, f[3]

    def _eraser(self, ht, wd):
        rects = []
        if np.random.rand() < self.eraser_aug_prob:
            for _ in range(np.random.randint(1, 3)):
                x0 = np.random.randint(0, wd)
                y0 = np.random.randint(0, ht)
                dx = np.random.randint(50, 100)
                dy = np.random.randint(50, 100)
                rects.append([int(x0), int(y0), int(dx), int(dy)])
        return rects

    def draw(self, ht, wd):
        """Draw one sample's parameters for a `ht` x `wd` source, consuming both RNGs as the reference's `__call__` does."""
        d = {"H": int(ht), "W": int(wd)}
        if not self.sparse and np.random.rand() < self.asymmetric_color_aug_prob:
            d["asym"] = 1
            jit = [self._jitter_params(), self._jitter_params()]
        else:
            d["asym"] = 0
            j = self._jitter_params()
            jit = [j, j]
        d["perm"] = [j[0] for j in jit]
        d["factor"] = [j[1] for j in jit]
        d["hue"] = [j[2] for j in jit]
        d["hue_factor"] = [j[3] for j in jit]
        d["erase"] = self._eraser(ht, wd)
        self._spatial(d, ht, wd)
        return d

    def _resized_size(self, ht, wd, fx, fy):
        return int(np.rint(ht * fy)), int(np.rint(wd * fx))     # cv2.resize's dsize: saturate_cast<int>(size * f)

    # ---- device execution --------------------------------------------------------------------------------------------
    def _run(self, planes, draws, device):
        """planes: per sample (img1 u8 [3,H,W], img2 u8 [3,H,W], flow f32 [2,H,W], valid f32 [H,W] or None), CPU tensors."""
        descs, buf = self._pack(planes, draws)
        return self._launch(descs, buf.to(device, non_blocking=True))

    def _pack(self, planes, draws):
        """One pinned host buffer: the descriptors, then every sample's planes, each 16-byte aligned."""
        B = len(planes)
        descs = (native.AugDesc * B)()
        off = (C.sizeof(descs) + _ALIGN - 1) // _ALIGN * _ALIGN
        layout = []
        for i, ((i1, i2, fl, va), d) in enumerate(zip(planes, draws)):
            o = {}
            for name, t in (("img1", i1), ("img2", i2), ("flow", fl), ("valid", va)):
                if t is None:
                    o[name] = 0
                    continue
                o[name] = off
                off += (t.numel() * t.element_size() + _ALIGN - 1) // _ALIGN * _ALIGN
            layout.append(o)
            self._fill(descs[i], d, o)
        buf = torch.empty(off, dtype=torch.uint8, pin_memory=True)
        buf[:C.sizeof(descs)].numpy()[:] = np.frombuffer(bytes(descs), dtype=np.uint8)
        for (i1, i2, fl, va), o in zip(planes, layout):
            for name, t in (("img1", i1), ("img2", i2), ("flow", fl), ("valid", va)):
                if t is not None:
                    n = t.numel() * t.element_size()
                    buf[o[name]:o[name] + n].view(t.dtype).copy_(t.reshape(-1))
        return descs, buf

    def _launch(self, descs, dev):
        """Run the kernels on the uploaded pack `dev` (device copy of _pack's buffer) on the current stream of its device."""
        B = len(descs)
        ch, cw = int(self.crop_size[0]), int(self.crop_size[1])
        device = dev.device
        img1 = torch.empty(B, 3, ch, cw, device=device)
        img2 = torch.empty_like(img1)
        flow = torch.empty(B, 2, ch, cw, device=device)
        valid = torch.empty(B, ch, cw, device=device)
        ws_bytes = native.rnc.augment_workspace_bytes(B, ch, cw, int(self.sparse))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        with torch.cuda.device(device):
            native.rnc.augment(descs, dev, B, dev, dev.numel(), ch, cw, int(self.sparse), img1, img2, flow, valid, ws, ws_bytes)
        return img1, img2, flow, valid

    def _fill(self, c, d, o):
        c.img1, c.img2, c.flow, c.valid = o["img1"], o["img2"], o["flow"], o["valid"]
        c.H, c.W, c.rh, c.rw = d["H"], d["W"], d["rh"], d["rw"]
        c.resized, c.hflip, c.vflip, c.y0, c.x0, c.asym = d["resized"], d["hflip"], d["vflip"], d["y0"], d["x0"], d["asym"]
        for p in range(2):
            for j in range(4):
                c.perm[p][j] = d["perm"][p][j]
            for j in range(3):
                c.factor[p][j] = d["factor"][p][j]
            c.hue[p] = d["hue"][p]
        c.n_erase = len(d["erase"])
        for e, r in enumerate(d["erase"]):
            for j in range(4):
                c.erase[e][j] = r[j]
        c.fx, c.fy = d["fx"], d["fy"]
        c.ifx, c.ify = 1.0 / d["fx"], 1.0 / d["fy"]

    def _planes_np(self, img1, img2, flow, valid):
        for name, a in (("img1", img1), ("img2", img2)):
            if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.shape[:2] != flow.shape[:2]:
                raise ValueError(f"{name} must be uint8 [H,W,3] of the flow's size, got {a.dtype} {a.shape}")
        if flow.ndim != 3 or flow.shape[2] != 2:
            raise ValueError(f"flow must be [H,W,2], got {flow.shape}")
        i1 = torch.from_numpy(np.ascontiguousarray(img1.transpose(2, 0, 1)))
        i2 = torch.from_numpy(np.ascontiguousarray(img2.transpose(2, 0, 1)))
        fl = torch.from_numpy(np.ascontiguousarray(flow.transpose(2, 0, 1), dtype=np.float32))
        va = None if valid is None else torch.from_numpy(np.ascontiguousarray(valid, dtype=np.float32))
        return i1, i2, fl, va

    def _call(self, img1, img2, flow, valid):
        ht, wd = img1.shape[:2]
        planes = self._planes_np(img1, img2, flow, valid)
        d = self.draw(ht, wd)
        o1, o2, of, ov = self._run([planes], [d], torch.device("cuda", torch.cuda.current_device()))
        o1 = o1[0].permute(1, 2, 0).to(torch.uint8).cpu().numpy()
        o2 = o2[0].permute(1, 2, 0).to(torch.uint8).cpu().numpy()
        of = of[0].permute(1, 2, 0).contiguous().cpu().numpy()
        return o1, o2, of, ov[0].cpu().numpy(), d

    def batch(self, samples, device):
        """Augment raw samples `(img1, img2, flow, valid)` ([3,H,W], [3,H,W], [2,H,W], [H,W]) into stacked crops on `device`."""
        return self._run(*self._draw_batch(samples), torch.device(device))

    def _draw_batch(self, samples):
        if not samples:
            raise ValueError("batch() needs at least one sample")
        planes, draws = [], []
        for s in samples:
            img1, img2, flow, valid = s[:4]
            if img1.dim() != 3 or img1.shape[0] != 3 or img2.shape != img1.shape or tuple(flow.shape) != (2, *img1.shape[1:]):
                raise ValueError(f"expected [3,H,W] images and a [2,H,W] flow, got {tuple(img1.shape)}, {tuple(img2.shape)}, "
                                 f"{tuple(flow.shape)}")
            ht, wd = int(img1.shape[1]), int(img1.shape[2])
            draws.append(self.draw(ht, wd))
            va = None
            if self.sparse:
                va = valid.detach().to("cpu", torch.float32).contiguous()
            planes.append((img1.detach().cpu().to(torch.uint8).contiguous(), img2.detach().cpu().to(torch.uint8).contiguous(),
                           flow.detach().to("cpu", torch.float32).contiguous(), va))
        return planes, draws


class FlowAugmentor(_Augmentor):
    """core/utils/augmentor.py:FlowAugmentor on the GPU (photometric jitter, eraser, scale / stretch, flips, crop)."""

    def __init__(self, crop_size, min_scale=-0.2, max_scale=0.5, do_flip=True):
        super().__init__(crop_size, min_scale, max_scale, do_flip, (0.4, 0.4, 0.4, 0.5 / 3.14))

    def _spatial(self, d, ht, wd):
        min_scale = np.maximum((self.crop_size[0] + 8) / float(ht), (self.crop_size[1] + 8) / float(wd))
        scale = 2 ** np.random.uniform(self.min_scale, self.max_scale)
        scale_x = scale
        scale_y = scale
        if np.random.rand() < self.stretch_prob:
            scale_x *= 2 ** np.random.uniform(-self.max_stretch, self.max_stretch)
            scale_y *= 2 ** np.random.uniform(-self.max_stretch, self.max_stretch)
        scale_x = np.clip(scale_x, min_scale, None)
        scale_y = np.clip(scale_y, min_scale, None)
        d["fx"], d["fy"] = float(scale_x), float(scale_y)
        d["resized"] = int(np.random.rand() < self.spatial_aug_prob)
        d["rh"], d["rw"] = self._resized_size(ht, wd, d["fx"], d["fy"]) if d["resized"] else (ht, wd)
        d["hflip"] = d["vflip"] = 0
        if self.do_flip:
            d["hflip"] = int(np.random.rand() < self.h_flip_prob)
            d["vflip"] = int(np.random.rand() < self.v_flip_prob)
        d["y0"] = int(np.random.randint(0, d["rh"] - self.crop_size[0]))
        d["x0"] = int(np.random.randint(0, d["rw"] - self.crop_size[1]))

    def __call__(self, img1, img2, flow):
        o1, o2, of, _, _ = self._call(img1, img2, flow, None)
        return o1, o2, of


class SparseFlowAugmentor(_Augmentor):
    """core/utils/augmentor.py:SparseFlowAugmentor on the GPU (symmetric jitter, eraser, scale, sparse resize, h-flip,
    margin crop)."""
    sparse = True

    def __init__(self, crop_size, min_scale=-0.2, max_scale=0.5, do_flip=False):
        super().__init__(crop_size, min_scale, max_scale, do_flip, (0.3, 0.3, 0.3, 0.3 / 3.14))

    def _spatial(self, d, ht, wd):
        min_scale = np.maximum((self.crop_size[0] + 1) / float(ht), (self.crop_size[1] + 1) / float(wd))
        scale = 2 ** np.random.uniform(self.min_scale, self.max_scale)
        d["fx"] = float(np.clip(scale, min_scale, None))
        d["fy"] = float(np.clip(scale, min_scale, None))
        d["resized"] = int(np.random.rand() < self.spatial_aug_prob)
        d["rh"], d["rw"] = self._resized_size(ht, wd, d["fx"], d["fy"]) if d["resized"] else (ht, wd)
        d["hflip"] = d["vflip"] = 0
        if self.do_flip and np.random.rand() < 0.5:
            d["hflip"] = 1
        margin_y, margin_x = 20, 50
        y0 = np.random.randint(0, d["rh"] - self.crop_size[0] + margin_y)
        x0 = np.random.randint(-margin_x, d["rw"] - self.crop_size[1] + margin_x)
        d["y0"] = int(np.clip(y0, 0, d["rh"] - self.crop_size[0]))
        d["x0"] = int(np.clip(x0, 0, d["rw"] - self.crop_size[1]))

    def __call__(self, img1, img2, flow, valid):
        if valid is None or np.shape(valid) != flow.shape[:2]:
            raise ValueError("SparseFlowAugmentor needs a [H,W] valid mask")
        o1, o2, of, ov, d = self._call(img1, img2, flow, valid)
        return o1, o2, of, (ov.astype(np.int32) if d["resized"] else ov.astype(np.asarray(valid).dtype))
