"""ctypes binding of librnc.so (include/rnc.h).

``rnc.<entry point without the rnc_ prefix>`` is how the product calls the library, e.g.
``rnc.nchw_to_cl(net, B, 128, H, W, ws.hx, HX_LD, 0)``: a ``void*`` argument takes a tensor (its ``data_ptr()``, so a view
carries its own offset), ``None`` (NULL) or a raw address; descriptors and arrays pass through; the stream argument is left
out and the current CUDA stream (``stream()``) appended; a non-zero ``rnc_status`` raises through ``check()`` naming the
entry point.  Size queries and the info calls return their value.  ``lib()`` is the raw ctypes handle; every call reads it
at call time, so a test that swaps ``_lib`` sees every entry point.

The library is REQUIRED on the product path: ``lib()`` raises ``RncUnavailable`` if it cannot be loaded —
there is no CPU or PyTorch fallback for the hot path.
"""
import ctypes as C
import os
import threading
import types

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RNC_LIB") or os.path.join(_HERE, "librnc.so")      # RNC_LIB: developer override (variant builds)
ABI_VERSION = 18
CONV_NO_HALO, CONV_AUX_BLOCKED, CONV_OUT_BLOCKED, CONV_TF32, CONV_WINDOW = 1, 16, 32, 64, 128   # rnc_conv_umma_desc.flags

(EPI_LINEAR, EPI_RELU, EPI_SIGMOID, EPI_GRU_ZR, EPI_GRU_Q, EPI_RELU_FLOW, EPI_RELU_ADD_RELU, EPI_TANH_RELU,
 EPI_FLOW_DELTA) = range(9)

_vp, _i, _f = C.c_void_p, C.c_int, C.c_float


class RncUnavailable(RuntimeError):
    pass


class RncError(RuntimeError):
    pass


class ConvDesc(C.Structure):
    """Mirror of rnc_conv_desc (include/rnc.h)."""
    _fields_ = [("in0", _vp), ("c0", _i), ("ld0", _i),
                ("in1", _vp), ("c1", _i), ("ld1", _i),
                ("weight", _vp), ("bias", _vp),
                ("out", _vp), ("ldo", _i),
                ("h", _vp), ("ldh", _i),
                ("aux0", _vp), ("ldaux", _i),
                ("B", _i), ("H", _i), ("W", _i),
                ("cout", _i), ("kh", _i), ("kw", _i), ("epilogue", _i)]


class UmmaConvDesc(C.Structure):
    """Mirror of rnc_conv_umma_desc (include/rnc.h)."""
    _fields_ = [("in0_hi", _vp), ("in0_lo", _vp), ("c0", _i), ("ld0", _i),
                ("in1_hi", _vp), ("in1_lo", _vp), ("c1", _i), ("ld1", _i),
                ("w_hi", _vp), ("w_lo", _vp), ("ktot", _i), ("coutpad", _i),
                ("bias", _vp), ("unscale", _f),
                ("out_f32", _vp), ("ldo_f32", _i),
                ("out_hi", _vp), ("out_lo", _vp), ("ldo_split", _i),
                ("h", _vp), ("ldh", _i),
                ("aux0", _vp), ("ldaux", _i),
                ("B", _i), ("H", _i), ("W", _i),
                ("cout", _i), ("kh", _i), ("kw", _i), ("epilogue", _i),
                ("stride", _i), ("hin", _i), ("win", _i),
                ("res", _vp), ("ldres", _i), ("flags", _i), ("stats", _vp), ("add", _vp), ("ldadd", _i), ("win_pitch", _i),
                ("dil", _i)]


class AugDesc(C.Structure):
    """Mirror of rnc_aug_desc (include/rnc.h): one augmented sample's sizes, byte offsets and drawn parameters."""
    _fields_ = [("img1", C.c_longlong), ("img2", C.c_longlong), ("flow", C.c_longlong), ("valid", C.c_longlong),
                ("H", _i), ("W", _i), ("rh", _i), ("rw", _i),
                ("resized", _i), ("hflip", _i), ("vflip", _i), ("y0", _i), ("x0", _i), ("asym", _i),
                ("perm", (_i * 4) * 2), ("factor", (_f * 3) * 2), ("hue", _i * 2),
                ("n_erase", _i), ("erase", (_i * 4) * 2), ("pad", _i),
                ("fx", C.c_double), ("fy", C.c_double), ("ifx", C.c_double), ("ify", C.c_double)]


# name -> (restype, argtypes); every symbol include/rnc.h declares
SIGNATURES = {
    "rnc_abi_version": (_i, []),
    "rnc_build_info": (C.c_char_p, []),
    "rnc_status_string": (C.c_char_p, [_i]),
    "rnc_last_cuda_error": (_i, []),
    "rnc_launch_count": (C.c_longlong, []),
    "rnc_launch_count_reset": (None, []),
    "rnc_pyramid_offset": (C.c_size_t, [_i, _i, _i, _i, _i]),
    "rnc_fmap_prepare": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "rnc_corr_lookup_fwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _vp]),
    "rnc_corr_lookup_split_fwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _vp]),
    "rnc_corr_lookup_umma_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "rnc_corr_lookup_umma_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _vp, C.c_size_t, _vp]),
    "rnc_f32_to_f16": (_i, [_vp, _vp, C.c_size_t, _vp]),
    "rnc_conv2d_cl_fwd": (_i, [C.POINTER(ConvDesc), _vp]),
    "rnc_conv2d_cl_dil_fwd": (_i, [C.POINTER(ConvDesc), _i, _vp]),
    "rnc_conv_umma_tiles": (C.c_longlong, [_i, _i, _i, _i, _i, _i, _i]),
    "rnc_conv2d_umma_fwd": (_i, [C.POINTER(UmmaConvDesc), _vp]),
    "rnc_f32_to_split": (_i, [_vp, _i, _i, C.c_longlong, _vp, _vp, _i, _i, _vp]),
    "rnc_f32_to_tf32_split": (_i, [_vp, _i, _i, C.c_longlong, _vp, _vp, _i, _i, _vp]),
    "rnc_stem_conv7x7s2_fwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "rnc_stem_window_prep": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "rnc_instnorm_stats": (_i, [_vp, _i, _i, _i, _f, _vp, _vp, _vp]),
    "rnc_instnorm_finalize": (_i, [_vp, _i, _i, _i, _f, _vp, _vp]),
    "rnc_instnorm_stats_det_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "rnc_instnorm_stats_det": (_i, [_vp, _i, _i, _i, _f, _vp, C.c_size_t, _vp, _vp]),
    "rnc_instnorm_apply": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "rnc_fmap_pyramid": (_i, [_vp, _i, _i, _i, _i, _i, _vp]),
    "rnc_conv_flow7x7_fwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _i, _vp]),
    "rnc_flow_head2_fwd": (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "rnc_flow_im2col7_split_fwd": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp]),
    "rnc_flow_tap_gather_fwd": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "rnc_forward_interpolate_fwd": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "rnc_forward_interpolate_bidir_fwd": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "rnc_coords_init": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "rnc_coords_to_flow": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "rnc_nchw_to_cl": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _vp]),
    "rnc_cl_to_nchw": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "rnc_convex_upsample_fwd": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "rnc_flow_x2_fwd": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "rnc_ncup_guidance_fwd": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _i, _vp]),
    "rnc_ncup_guidance_split_fwd": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp]),
    "rnc_conf_head_fwd": (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "rnc_ncup_fwd": (_i, [_vp, _vp, C.POINTER(_f), _i, _i, _i, _f, _vp, _vp, _vp]),
    "rnc_ncup_train_fwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _f, _vp, _vp, _vp]),
    "rnc_ncup_bwd_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "rnc_ncup_bwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _vp, C.c_size_t, _vp]),
    "rnc_bilinear_sample_fwd": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "rnc_nconv2d_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _f, _vp, _vp, _i, _i, _i, _f, _vp, _vp, _vp]),
    "rnc_corr_lookup_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "rnc_pyramid_pool_bwd": (_i, [_vp, _i, _i, _i, _i, _i, _vp]),
    "rnc_corr_lookup_bwd_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i]),
    "rnc_corr_lookup_bwd_det": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, C.c_size_t, _vp]),
    "rnc_conv2d_cl_wgrad_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i, _i, _i, _i, _i]),
    "rnc_conv2d_cl_wgrad_det": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _vp, _vp, C.c_size_t, _vp]),
    "rnc_conv2d_cl_wgrad_dil_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i, _i, _i, _i, _i]),
    "rnc_conv2d_cl_wgrad_dil_det": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _vp, _vp, C.c_size_t, _vp]),
    "rnc_nconv2d_bwd_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i, _i, _i, _i]),
    "rnc_nconv2d_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _f, _vp, _vp, _i, _i, _i,
                             _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_size_t, _vp]),
    "rnc_nconv_pool2_fwd": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "rnc_nconv_pool2_bwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "rnc_augment_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i]),
    "rnc_augment": (_i, [_vp, _vp, _i, _vp, C.c_size_t, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, C.c_size_t, _vp]),
    "rnc_flow_to_image_workspace_bytes": (C.c_size_t, [_i]),
    "rnc_flow_to_image": (_i, [_vp, C.c_longlong, C.c_longlong, C.c_longlong, C.c_longlong, _i, _i, _i, _vp, _vp, C.c_size_t,
                               _vp]),
    "rnc_flow_metrics_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "rnc_flow_metrics": (_i, [_vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 3, _i, _i, _i, _vp, _vp,
                              _vp, C.c_size_t, _vp]),
    "rnc_sparsification_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "rnc_sparsification": (_i, [_vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 3,
                                _vp, *[C.c_longlong] * 3, _i, _i, _i, _vp, _vp, _vp, _vp, C.c_size_t, _vp]),
    "rnc_fb_consistency": (_i, [_vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _i, _i, _i, _f, _f, _vp, _vp, _vp, _vp,
                                _vp]),
    "rnc_boundary_dist2": (_i, [_vp, *[C.c_longlong] * 3, _i, _i, _i, _vp, _vp]),
    "rnc_region_metrics_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i]),
    "rnc_region_metrics": (_i, [_i, _vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 3,
                                _vp, *[C.c_longlong] * 3, _vp, _vp, *[C.c_longlong] * 3, _i, _i, _i, _vp, _vp, _vp,
                                C.c_size_t, _vp]),
    "rnc_interpolate_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i]),
    "rnc_interpolate": (_i, [_vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _vp,
                             *[C.c_longlong] * 4, _vp, _vp, C.POINTER(_f), _i, _i, _i, _i, _vp, _vp, C.c_size_t, _vp]),
    "rnc_interp_error_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "rnc_interp_error": (_i, [_vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _i, _i, _i, _vp, _vp, _vp, C.c_size_t, _vp]),
    "rnc_census_loss_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "rnc_census_loss_fwd": (_i, [_vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _vp, _i, _i, _i,
                                 _vp, _vp, _vp, _vp, _vp, C.c_size_t, _vp]),
    "rnc_census_loss_bwd": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
    "rnc_smoothness_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "rnc_smoothness_fwd": (_i, [_vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _i, _i, _i, _f, _vp, _vp, _vp, _vp,
                                C.c_size_t, _vp]),
    "rnc_smoothness_bwd": (_i, [_vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _i, _i, _i, _f, _vp, _vp, _vp]),
    "rnc_track": (_i, [_vp, *[C.c_longlong] * 5, _vp, *[C.c_longlong] * 5, _vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4,
                       _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "rnc_track_metrics_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "rnc_track_metrics": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, C.c_size_t, _vp]),
    "rnc_propagate_labels_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "rnc_propagate_labels": (_i, [_vp, *[C.c_longlong] * 3, _vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 3, _i, _i, _i,
                                  _vp, *[C.c_longlong] * 3, _vp, C.c_size_t, _vp]),
    "rnc_segmentation_counts_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i]),
    "rnc_segmentation_counts": (_i, [_vp, *[C.c_longlong] * 3, _vp, *[C.c_longlong] * 3, _i, _i, _i, _i, _vp, _vp, C.c_size_t,
                                     _vp]),
    "rnc_harmonic_fill_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i, _i]),
    "rnc_harmonic_fill": (_i, [_vp, *[C.c_longlong] * 5, _vp, *[C.c_longlong] * 4, _i, _i, _i, _i, _i, _i, _vp,
                               *[C.c_longlong] * 5, _vp, C.c_size_t, _vp]),
    "rnc_inpaint_propagate": (_i, [_vp, *[C.c_longlong] * 5, _vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 5, _vp,
                                   *[C.c_longlong] * 5, _vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _i, _i, _i, _i, _i,
                                   _vp, _vp, _vp]),
    "rnc_ssim_partials_workspace_bytes": (C.c_size_t, [_i, _i, _i]),
    "rnc_ssim_partials": (_i, [_vp, *[C.c_longlong] * 4, _vp, *[C.c_longlong] * 4, _i, _i, _i, _vp, _vp, _vp, C.c_size_t, _vp]),
    "rnc_temporal_step_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i]),
    "rnc_temporal_step": (_i, [*[_vp, *[C.c_longlong] * 4] * 5, _vp, *[C.c_longlong] * 3, _i, _i, _i, _i, _f, _f, _f, _i, _vp,
                               *[C.c_longlong] * 4, _vp, C.c_size_t, _vp]),
    "rnc_warping_error_partials_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i, _i]),
    "rnc_warping_error_partials": (_i, [_vp, *[C.c_longlong] * 5, _vp, *[C.c_longlong] * 5, _vp, *[C.c_longlong] * 4, _i, _i,
                                        _i, _i, _i, _vp, _vp, _vp, C.c_size_t, _vp]),
    "rnc_homography_fit_workspace_bytes": (C.c_size_t, [_i, _i, _i, _i, _i]),
    "rnc_homography_fit": (_i, [_vp, *[C.c_longlong] * 4, _i, _i, _i, _i, _i, C.c_double, _i, C.c_ulonglong, _vp, _vp, _vp,
                                _vp, _vp, C.c_size_t, _vp]),
    "rnc_stabilize_path": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _i, C.c_double, _vp, _vp, _vp, _vp]),
    "rnc_stabilize_warp": (_i, [_vp, *[C.c_longlong] * 4, _vp, _i, _i, _i, _i, _vp, *[C.c_longlong] * 4, _vp,
                                *[C.c_longlong] * 3, _vp]),
    "rnc_stabilize_flow_residual": (_i, [_vp, *[C.c_longlong] * 5, _vp, *[C.c_longlong] * 5, _vp, _vp, _vp, _i, _i, _i, _i,
                                         _vp, _vp, _vp]),
    "rnc_stabilize_flow_readd": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
}
DIST2_NONE = 2147483647                                    # RNC_DIST2_NONE
REGIONS_SINTEL, REGIONS_KITTI = 0, 1                       # rnc_region_metrics' kind
REGION_CELLS = {REGIONS_SINTEL: 32, REGIONS_KITTI: 4}
INTERP_MAX_TIMES = 64                                      # RNC_INTERP_MAX_TIMES
TRACK_THRESHOLDS, TRACK_COUNTS = 5, 18                     # RNC_TRACK_THRESHOLDS, RNC_TRACK_COUNTS
SEGMENT_COUNTS = 6                                         # RNC_SEGMENT_COUNTS
HARMONIC_MAX_CHANNELS = 4                                  # RNC_HARMONIC_MAX_CHANNELS
# RNC_INPAINT_KNOWN, _FORWARD, _BACKWARD, _BOTH, _SPATIAL: rnc_inpaint_propagate's source map
INPAINT_KNOWN, INPAINT_FORWARD, INPAINT_BACKWARD, INPAINT_BOTH, INPAINT_SPATIAL = range(5)
HOMOGRAPHY_OK, HOMOGRAPHY_FEW = 0, 1                       # RNC_HOMOGRAPHY_OK, RNC_HOMOGRAPHY_FEW: rnc_homography_fit's status

_lib = None
_lock = threading.Lock()


def lib():
    """Load librnc.so once; raise loudly if it is missing or stale."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RncUnavailable(
                f"{LIB_PATH} not found: build it with `python raft-ncup_b200/rnc/build.py` "
                "(the RAFT-NCUP hot path has no CPU/PyTorch fallback)")
        try:
            handle = C.CDLL(LIB_PATH)
        except OSError as e:
            raise RncUnavailable(f"cannot load {LIB_PATH}: {e}") from e
        for name, (res, args) in SIGNATURES.items():
            try:
                fn = getattr(handle, name)
            except AttributeError as e:
                raise RncUnavailable(f"{LIB_PATH} does not export {name} (stale build?)") from e
            fn.restype = res
            fn.argtypes = args
        if handle.rnc_abi_version() != ABI_VERSION:
            raise RncUnavailable(f"librnc ABI {handle.rnc_abi_version()} != expected {ABI_VERSION}; rebuild")
        _lib = handle
    return _lib


def check(status, what="rnc"):
    """Translate a negative rnc_status into a Python exception (the reference's error channel, SURVEY §8b)."""
    if status == 0:
        return
    l = lib()
    msg = l.rnc_status_string(status).decode()
    if status == -4:
        msg += f" (cudaError {l.rnc_last_cuda_error()})"
    if status in (-1, -3):
        raise ValueError(f"{what}: {msg}")
    raise RncError(f"{what}: {msg}")


def stream():
    """The raw cudaStream_t of torch's current stream, on which the bound entry points enqueue their work."""
    return torch.cuda.current_stream().cuda_stream


def _bind(name, restype, argtypes):
    # kernel entry points return an rnc_status and take the stream last; which arguments are void* is fixed here, once
    kernel = restype is _i and len(argtypes) > 0 and argtypes[-1] is _vp
    ptrs = tuple(i for i, t in enumerate(argtypes[:-1] if kernel else argtypes) if t is _vp)

    def call(*args):
        args = list(args)
        for i in ptrs:
            if isinstance(args[i], torch.Tensor):
                args[i] = args[i].data_ptr()
        if not kernel:
            return getattr(lib(), name)(*args)
        status = getattr(lib(), name)(*args, stream())
        if status:
            check(status, name)

    call.__name__ = call.__qualname__ = name
    return call


rnc = types.SimpleNamespace(**{name[4:]: _bind(name, *sig) for name, sig in SIGNATURES.items()})


def launch_count():
    return int(rnc.launch_count())


def launch_count_reset():
    rnc.launch_count_reset()
