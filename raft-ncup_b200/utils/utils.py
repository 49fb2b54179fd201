"""Drop-in for `core/utils/utils.py`: InputPadder, forward_interpolate, coords_grid, upflow8 — the host-side helpers the
evaluation loops call around the model (evaluate.py:38-40, 125-129)."""
import torch
import torch.nn.functional as F


class InputPadder:
    """Replicate-pads frames to a multiple of 8 (utils.py:7-25): 'sintel' splits the padding evenly, otherwise it is
    put at the bottom."""

    def __init__(self, dims, mode="sintel"):
        self.ht, self.wd = dims[-2:]
        ph = (8 - self.ht % 8) % 8
        pw = (8 - self.wd % 8) % 8
        if mode == "sintel":
            self._pad = [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2]
        else:
            self._pad = [pw // 2, pw - pw // 2, 0, ph]

    def pad(self, *inputs):
        return [F.pad(x, self._pad, mode="replicate") for x in inputs]

    def unpad(self, x):
        l, r, t, b = self._pad
        return x[..., t:x.shape[-2] - b, l:x.shape[-1] - r]


def forward_interpolate(flow):
    """utils.py:28-56 — warm-start initialisation for the next frame: flow [2,H,W] (or [B,2,H,W]) on a CUDA device.
    The reference round-trips through scipy on the CPU; this runs librnc's exact nearest-sample kernel on the GPU and
    returns a tensor on the input's device (the reference returns a CPU tensor that its caller moves back with .cuda())."""
    from rnc.engine import _require_cuda
    from rnc.native import rnc
    _require_cuda(flow)
    squeeze = flow.dim() == 3
    f = (flow[None] if squeeze else flow).detach().float().contiguous()
    B, two, H, W = f.shape
    if two != 2:
        raise ValueError("flow must be [2,H,W] or [B,2,H,W]")
    out = torch.empty_like(f)
    rnc.forward_interpolate_fwd(f, B, H, W, out)
    return out[0] if squeeze else out


def bilinear_sampler(img, coords, mode="bilinear", mask=False):
    """utils.py:59-73 — grid_sample(align_corners=True) with pixel coordinates: img [N,C,H,W], coords [N,h,w,2] -> [N,C,h,w]
    (and, with mask=True, the in-bounds mask [N,h,w,1]).  Runs librnc's sampler kernel; zero padding outside the image."""
    from rnc.engine import _require_cuda
    from rnc.native import rnc
    if mode != "bilinear":
        raise NotImplementedError("only bilinear sampling is built (the reference never passes another mode)")
    dev = _require_cuda(img, coords)
    N, Cc, H, W = img.shape
    if coords.dim() != 4 or coords.shape[0] != N or coords.shape[-1] != 2:
        raise ValueError("coords must be [N,h,w,2]")
    h, w = coords.shape[1:3]
    with torch.cuda.device(dev):
        out = torch.empty(N, Cc, h, w, dtype=torch.float32, device=dev)
        m = torch.empty(N, h, w, 1, dtype=torch.float32, device=dev) if mask else None
        rnc.bilinear_sample_fwd(img.detach().float().contiguous(), coords.detach().float().contiguous(), N, Cc, H, W, h, w, out, m)
    return (out, m) if mask else out


def coords_grid(batch, ht, wd):
    ys, xs = torch.meshgrid(torch.arange(ht), torch.arange(wd), indexing="ij")
    return torch.stack([xs, ys], 0).float()[None].repeat(batch, 1, 1, 1)


def upflow8(flow, mode="bilinear"):
    return 8 * F.interpolate(flow, size=(8 * flow.shape[2], 8 * flow.shape[3]), mode=mode, align_corners=True)
