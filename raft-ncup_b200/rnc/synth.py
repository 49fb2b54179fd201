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


def shaky_sequence(n, h, w, seed=0, pan=(2.0, 0.5), jitter_px=3.0, jitter_rot=0.01, jitter_scale=0.01):
    """A handheld-looking video of n frames [3,h,w] with known camera motion, for video stabilization: frame t shows a smooth
    canvas (a seeded sum of sinusoids per channel, 0..255, evaluated in fp64 at the exact point, so no resampling blurs it)
    through the camera homography C_t, canvas -> frame t pixel coordinates: C_t = Tc R(theta_t) s_t Tc^-1 Tr(-o_t), Tc the
    translation to the frame centre, o_t = pan t plus a seeded translation jitter of std jitter_px, and theta_t and s_t - 1
    seeded jitters of std jitter_rot (radians) and jitter_scale.  Returns (frames: list of float32 [3,h,w], C fp64 [n,3,3],
    flows float32 [n-1,2,h,w]), flow k being the exact forward flow C_{k+1} C_k^-1 p - p of frame k's pixels p."""
    import numpy as np
    rng, freq, amp, phase = _shaky_canvas_draws(seed)
    jit = rng.normal(0, 1, (n, 4))
    cx, cy = (w - 1) / 2, (h - 1) / 2
    Tc = np.array([[1.0, 0, cx], [0, 1.0, cy], [0, 0, 1]])
    Tci = np.array([[1.0, 0, -cx], [0, 1.0, -cy], [0, 0, 1]])
    C = np.empty((n, 3, 3))
    for t in range(n):
        th, s = jitter_rot * jit[t, 0], 1 + jitter_scale * jit[t, 1]
        ox, oy = pan[0] * t + jitter_px * jit[t, 2], pan[1] * t + jitter_px * jit[t, 3]
        R = np.array([[s * np.cos(th), -s * np.sin(th), 0], [s * np.sin(th), s * np.cos(th), 0], [0, 0, 1]])
        C[t] = Tc @ R @ Tci @ np.array([[1.0, 0, -ox], [0, 1.0, -oy], [0, 0, 1]])
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    P = np.stack([xs, ys, np.ones_like(xs)]).reshape(3, -1)
    frames = []
    for t in range(n):
        X, Y, Wh = np.linalg.inv(C[t]) @ P
        X, Y = X / Wh, Y / Wh
        img = _shaky_canvas(freq, amp, phase, X, Y)
        frames.append(torch.from_numpy(img.reshape(3, h, w)).float())
    return frames, torch.from_numpy(C), _shaky_flows(C, h, w, False)


def _shaky_canvas_draws(seed):
    """The generator of shaky_sequence after its canvas draws, and those draws: (rng, freq, amp, phase)."""
    import numpy as np
    rng = np.random.default_rng(seed)
    K = 8
    freq = rng.uniform(2 * np.pi / 60, 2 * np.pi / 12, (3, K)) * np.exp(1j * rng.uniform(0, 2 * np.pi, (3, K)))
    amp = rng.uniform(0.5, 1.0, (3, K))
    amp *= 110 / amp.sum(1, keepdims=True)
    phase = rng.uniform(0, 2 * np.pi, (3, K))
    return rng, freq, amp, phase


def _shaky_canvas(freq, amp, phase, X, Y):
    import numpy as np
    return 127.5 + (amp[..., None] * np.sin(freq.real[..., None] * X + freq.imag[..., None] * Y + phase[..., None])).sum(1)


def _shaky_flows(C, h, w, backward):
    import numpy as np
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    P = np.stack([xs, ys, np.ones_like(xs)]).reshape(3, -1)
    flows = np.empty((C.shape[0] - 1, 2, h, w))
    for k in range(C.shape[0] - 1):
        a, b = (k, k + 1) if backward else (k + 1, k)
        X, Y, Wh = C[a] @ np.linalg.inv(C[b]) @ P
        flows[k, 0] = (X / Wh - P[0]).reshape(h, w)
        flows[k, 1] = (Y / Wh - P[1]).reshape(h, w)
    return torch.from_numpy(flows).float()


def shaky_canvas(x, y, seed=0):
    """shaky_sequence(..., seed)'s canvas (the same draws) at canvas points x, y (fp64 arrays of one shape), evaluated in fp64
    as shaky_sequence renders it.  Returns fp64 [3, *x.shape] (numpy): the true content of any output pixel, e.g. of a
    stabilized frame's uncovered border, whose canvas point is C_t^-1 M_t^-1 u."""
    import numpy as np
    _, freq, amp, phase = _shaky_canvas_draws(seed)
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    return _shaky_canvas(freq, amp, phase, x.reshape(-1), y.reshape(-1)).reshape(3, *x.shape)


def shaky_backward_flows(C, h, w):
    """The exact backward flows of a shaky_sequence video with cameras C (fp64 [n,3,3]) at h x w: float32 [n-1,2,h,w], flow
    k being C_k C_{k+1}^-1 p - p of frame k+1's pixels p."""
    return _shaky_flows(torch.as_tensor(C).double().numpy(), h, w, True)
