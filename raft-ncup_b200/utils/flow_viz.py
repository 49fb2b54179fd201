"""Drop-in for `core/utils/flow_viz.py` as the reference's scripts use it (demo.py:viz, evaluate.py:51,84 with
write_png=True): `flow_to_image` only, computed on the current CUDA device by librnc (rnc.viz)."""
import numpy as np
import torch


def flow_to_image(flow):
    """Middlebury colour coding of a float32 flow [H, W, 2] (flow_viz.py:240-275): returns uint8 [H, W, 3] in the
    reference's channel order, which the reference hands straight to cv2.imwrite.

    Unlike the reference, the argument is left unchanged: the reference zeroes the caller's unknown entries (|u| or |v| above
    1e7) in place before colour-coding."""
    from rnc.native import RncUnavailable
    from rnc.viz import flow_to_image as gpu_flow_to_image
    flow = np.asarray(flow)
    if flow.ndim != 3 or flow.shape[2] != 2:
        raise ValueError(f"flow_to_image: expected an [H, W, 2] flow array, got {flow.shape}")
    if not torch.cuda.is_available():
        raise RncUnavailable("flow_to_image runs on a CUDA device (sm_90a); none is available and there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device())
    f = torch.from_numpy(np.ascontiguousarray(flow, np.float32)).to(dev)
    return gpu_flow_to_image(f.permute(2, 0, 1)).cpu().numpy()
