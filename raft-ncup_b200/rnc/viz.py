"""Flow visualisation on the GPU: the reference's `flow_to_image` (core/utils/flow_viz.py:240-275) as a librnc kernel
(csrc/flow_viz.cu) over a batch of flows.

`flow_to_image(flow)` colour-codes a CUDA flow `[B,2,H,W]` (or `[2,H,W]`) of any strides into uint8 `[B,H,W,3]` (or
`[H,W,3]`) in the reference's channel order, each image normalised by its own maximum radius.  The arithmetic follows the
reference's numpy 2.x dtype chain rounding by rounding; only the float64 arc tangent is CUDA's rather than numpy's, so a
channel could differ from the reference's by one level (see include/rnc.h, V1).
"""
import torch

from . import native
from .engine import _require_cuda


def flow_to_image(flow):
    """flow: CUDA tensor [B,2,H,W] or [2,H,W] (float32, or converted to it).  Returns a uint8 [B,H,W,3] (or [H,W,3]) tensor on
    the same device, enqueued on its current stream."""
    single = flow.dim() == 3
    if single:
        flow = flow[None]
    if flow.dim() != 4 or flow.shape[1] != 2:
        raise ValueError(f"flow_to_image: expected a [B,2,H,W] or [2,H,W] flow, got {tuple(flow.shape)}")
    dev = _require_cuda(flow)
    if flow.dtype != torch.float32:
        flow = flow.float()
    B, _, H, W = flow.shape
    out = torch.empty(B, H, W, 3, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        ws = torch.empty(native.rnc.flow_to_image_workspace_bytes(B), dtype=torch.uint8, device=dev)
        native.rnc.flow_to_image(flow, *flow.stride(), B, H, W, out, ws, ws.numel())
    return out[0] if single else out
