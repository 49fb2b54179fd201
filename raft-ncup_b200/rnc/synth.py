"""Synthetic workloads of SURVEY.md §8d (there is no dataset or checkpoint offline): the flag Namespace every reference
script ships, seeded random-init models, and the three stimuli the benchmark and the parity tests use.  Host-side only."""
import argparse
import importlib

import torch
import torch.nn.functional as F


def ref_args(dataset="sintel"):
    """The flag values every reference script ships (eval_raft_nc_sintel.sh:12-34; SURVEY.md §5)."""
    return argparse.Namespace(
        small=False, mixed_precision=False, load_pretrained=None, freeze_raft=False, dataset=dataset, align_corners=True,
        final_upsampling="NConvUpsampler", final_upsampling_scale=4, final_upsampling_use_data_for_guidance=True,
        final_upsampling_channels_to_batch=True, final_upsampling_use_residuals=False, final_upsampling_est_on_high_res=False,
        interp_net="NConvUNet", interp_net_channels_multiplier=2, interp_net_num_downsampling=1,
        interp_net_data_pooling="conf_based", interp_net_encoder_filter_sz=5, interp_net_decoder_filter_sz=3,
        interp_net_out_filter_sz=1, interp_net_shared_encoder=True, interp_net_use_double_conv=False, interp_net_use_bias=False,
        weights_est_net="Simple", weights_est_net_num_ch=[64, 32], weights_est_net_filter_sz=[3, 3, 1],
        weights_est_net_dilation=[1, 1, 1])


def build_model(name="raft_nc_dbl", dataset="sintel", seed=1234):
    """Seeded model on CPU in eval mode — bit-identical weights to the reference built with the same seed (train.py:345)."""
    torch.manual_seed(seed)
    mod = importlib.import_module(name)
    return mod.RAFT(ref_args(dataset)).eval()


def frames(b, h, w, seed=7):
    """Stimulus 1: uniform-random frames in [0, 255] (SURVEY.md §8d)."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(b, 3, h, w, generator=g) * 255, torch.rand(b, 3, h, w, generator=g) * 255


def smooth_shift_frames(b, h, w, seed=7, dy=3, dx=4):
    """Stimulus 2 (SURVEY.md §8d): bicubic-upsampled 20x36 noise; frame 2 = frame 1 translated by dy px vertically and dx px
    horizontally (coherent flow).  Both frames are crops of one larger canvas, so the translation is exact."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(b, 3, 20, 36, generator=g)
    big = F.interpolate(low, size=(h + dy, w + dx), mode="bicubic", align_corners=False).clamp(0, 1) * 255
    return big[:, :, dy:, dx:].contiguous(), big[:, :, :h, :w].contiguous()


def shift_sequence(n, h, w, seed=7, dy=3, dx=4):
    """A sequence of n frames [3,h,w] for warm-started inference: crops of one smooth canvas (bicubic-upsampled 20x36 noise, as
    smooth_shift_frames), frame t + 1 being frame t translated by dy px vertically and dx px horizontally."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(1, 3, 20, 36, generator=g)
    big = F.interpolate(low, size=(h + (n - 1) * dy, w + (n - 1) * dx), mode="bicubic", align_corners=False).clamp(0, 1) * 255
    return [big[0, :, (n - 1 - t) * dy:(n - 1 - t) * dy + h, (n - 1 - t) * dx:(n - 1 - t) * dx + w].contiguous() for t in range(n)]


def motion_boundary_flow_init(b, h8, w8, jump=24.0):
    """Stimulus 3: a warm-start flow field (raft_nc_dbl.py:144-145) with a motion boundary — the right half moves `jump` px (at
    1/8 resolution) further than the left half, and the lower third moves vertically too — so the lookup windows of the tiles on
    the boundaries are incoherent and do not fit the tensor-core kernel's fixed boxes (exact fallback path)."""
    f = torch.zeros(b, 2, h8, w8)
    f[:, 0, :, w8 // 2:] = jump
    f[:, 1, 2 * h8 // 3:, :] = -jump * 0.75
    return f
