"""``diff_gaussian_rasterization._C`` -- host-side binding of ``libgsrast.so``.

Mirrors the three functions the reference's pybind11 module exports
(``submodules/diff-gaussian-rasterization/ext.cpp:15-19``), same positional arguments, same
returned tuples (``rasterize_points.cu:35-119,121-204,206-225``), but implemented as a thin
ctypes shim over the C ABI in ``include/gsrast.h``: torch is used only to allocate device
memory and to name the current stream.  There is no CPU fallback -- if the CUDA library is
missing the import fails loudly.
"""
from __future__ import annotations

import ctypes
import os
import warnings
from ctypes import POINTER, Structure, byref, c_char_p, c_float, c_int, c_size_t, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.normpath(os.path.join(_HERE, "..", "lib", "libgsrast.so"))

NUM_CHANNELS = 3


class GsrForwardArgs(Structure):
    _fields_ = [
        ("P", c_int), ("D", c_int), ("M", c_int), ("W", c_int), ("H", c_int),
        ("background", c_void_p), ("means3D", c_void_p), ("shs", c_void_p), ("colors_precomp", c_void_p),
        ("opacities", c_void_p), ("scales", c_void_p), ("scale_modifier", c_float), ("rotations", c_void_p),
        ("cov3D_precomp", c_void_p), ("viewmatrix", c_void_p), ("projmatrix", c_void_p), ("campos", c_void_p),
        ("tan_fovx", c_float), ("tan_fovy", c_float), ("kernel_size", c_float), ("subpixel_offset", c_void_p),
        ("prefiltered", c_int), ("debug", c_int), ("tile_y0", c_int), ("tile_y1", c_int),
        ("out_color", c_void_p), ("radii", c_void_p), ("peer_images", c_void_p), ("n_peer_images", c_int),
    ]


class GsrBackwardArgs(Structure):
    _fields_ = [
        ("P", c_int), ("D", c_int), ("M", c_int), ("R", c_int), ("W", c_int), ("H", c_int),
        ("background", c_void_p), ("means3D", c_void_p), ("shs", c_void_p), ("colors_precomp", c_void_p),
        ("scales", c_void_p), ("scale_modifier", c_float), ("rotations", c_void_p), ("cov3D_precomp", c_void_p),
        ("viewmatrix", c_void_p), ("projmatrix", c_void_p), ("campos", c_void_p),
        ("tan_fovx", c_float), ("tan_fovy", c_float), ("kernel_size", c_float), ("subpixel_offset", c_void_p),
        ("radii", c_void_p), ("geom_buffer", c_void_p), ("binning_buffer", c_void_p), ("img_buffer", c_void_p),
        ("dL_dpix", c_void_p), ("debug", c_int), ("tile_y0", c_int), ("tile_y1", c_int),
        ("accum_scratch", c_void_p), ("accum_is_zero", c_int),
        ("dL_dmean2D", c_void_p), ("dL_dconic", c_void_p), ("dL_dopacity", c_void_p), ("dL_dcolor", c_void_p),
        ("dL_dmean3D", c_void_p), ("dL_dcov3D", c_void_p), ("dL_dsh", c_void_p), ("dL_dscale", c_void_p),
        ("dL_drot", c_void_p), ("deterministic", c_int), ("det_scratch", c_void_p), ("det_marks", c_void_p),
    ]


class GsrAppearanceArgs(Structure):
    _fields_ = [
        ("P", c_int), ("sh_degree", c_int),
        ("features_dc", c_void_p), ("features_rest", c_void_p), ("embeddings", c_void_p), ("means3D", c_void_p),
        ("campos", c_void_p), ("packed_weights", c_void_p), ("colors_raw", c_void_p), ("colors_toned", c_void_p),
        ("dL_dcolors_raw", c_void_p), ("dL_dcolors_toned", c_void_p), ("dL_dfeatures_dc", c_void_p),
        ("dL_dfeatures_rest", c_void_p), ("dL_dembeddings", c_void_p), ("dL_dmeans3D", c_void_p),
        ("grad_pack", c_void_p), ("status", c_void_p), ("deterministic", c_int), ("det_scratch", c_void_p),
    ]


class GsrAdamSegment(Structure):      # include/gsrast.h
    _fields_ = [("param", c_void_p), ("grad", c_void_p), ("exp_avg", c_void_p), ("exp_avg_sq", c_void_p),
                ("n", ctypes.c_longlong), ("step", ctypes.c_longlong), ("lr", ctypes.c_double), ("weight_decay", ctypes.c_double)]


ADAM_MAX_SEGMENTS = 32


class GsrDensifyArgs(Structure):      # include/gsrast.h
    _fields_ = ([("P", c_int)] +
                [(n, c_void_p) for n in ("xyz_grad", "denom", "accum_abs", "xyz", "scales", "rotations", "opacities")] +
                [(n, c_float) for n in ("max_grad", "clone_max_scale", "min_opacity", "prune_max_scale")] +
                [("size_pruning", c_int), ("split_scale_mul", c_float), ("scratch", c_void_p), ("counts", c_void_p),
                 ("normals", c_void_p)])


class GsrDensifySegment(Structure):   # include/gsrast.h
    _fields_ = [("src", c_void_p), ("dst", c_void_p), ("width", c_int), ("kind", c_int)]


DENSIFY_COUNTS = 8
DENSIFY_MAX_SEGMENTS = 48
DENSIFY_MAX_P = 0x3FFFFFFF
DENSIFY_COPY, DENSIFY_ZERO_NEW, DENSIFY_XYZ, DENSIFY_SCALES = 0, 1, 2, 3


class GsrUncertaintyArgs(Structure):      # include/gsrast.h
    _fields_ = ([(n, c_int) for n in ("C", "th", "tw", "Hp", "Wp", "pad_top", "pad_left", "H", "W", "nh", "nw", "ch", "cw",
                                      "nHp", "nWp", "npad_top", "npad_left")] +
                [(n, c_float) for n in ("clip_min", "reg_weight", "bn_eps", "bn_momentum")] +
                [(n, c_void_p) for n in ("feat", "feat_gt_down", "feat_pred_down", "mask", "conv_w", "conv_b", "bn_w", "bn_b",
                                         "running_mean", "running_var", "num_batches_tracked", "gt", "pred", "ssim", "msssim",
                                         "loss_mult", "loss", "metrics", "scratch", "dL_dloss", "d_conv_w", "d_conv_b",
                                         "d_bn_w", "d_bn_b")])


class GsrUncertaintyModeArgs(Structure):      # include/gsrast.h
    _fields_ = ([(n, c_int) for n in ("mode", "training", "C", "th", "tw", "Hp", "Wp", "pad_top", "pad_left", "uh", "uw",
                                      "H", "W", "nh", "nw", "ch", "cw", "nHp", "nWp", "npad_top", "npad_left")] +
                [(n, c_float) for n in ("clip_min", "reg_weight", "bn_eps", "bn_momentum")] +
                [(n, c_void_p) for n in ("feat", "feat_gt_down", "feat_pred_down", "mask", "conv_w", "conv_b", "bn_w", "bn_b",
                                         "running_mean", "running_var", "num_batches_tracked", "gt", "pred", "ssim", "msssim",
                                         "msssim_down", "loss_mult", "loss", "metrics", "scratch", "dL_dloss", "d_conv_w",
                                         "d_conv_b", "d_bn_w", "d_bn_b")])


UNC_MODES = {"l2reg": 0, "l1reg": 1, "dino": 2, "dino+mssim": 3}       # GSR_UNC_MODE_*


class GsrTrainLossArgs(Structure):      # include/gsrast.h
    _fields_ = ([("H", c_int), ("W", c_int), ("c_l1", c_float), ("c_ssim", c_float)] +
                [(n, c_void_p) for n in ("toned", "raw", "gt", "mask", "weight", "grad_scale", "raw_scaled", "ssim_map",
                                         "ssim_partials", "loss", "metrics", "scratch", "dL_dloss", "dL_dmap", "d_toned",
                                         "d_raw")])


class GsrMetricsArgs(Structure):      # include/gsrast.h
    _fields_ = ([(n, c_int) for n in ("B", "H", "W", "C", "a_u8", "b_u8")] + [("a", c_void_p), ("b", c_void_p)] +
                [("taps", ctypes.c_double * 11), ("c1", ctypes.c_double), ("c2", ctypes.c_double)] +
                [(n, c_void_p) for n in ("lpips_a", "lpips_b", "sums", "scratch")])


class GsrDisplayArgs(Structure):      # include/gsrast.h
    _fields_ = [("out_color", c_void_p), ("out_accum", c_void_p), ("depth", c_int), ("out_depth", c_void_p),
                ("depth_values", c_void_p), ("depth_scratch", c_void_p)]


class GsrStats(Structure):
    _fields_ = [("num_rendered", c_int), ("num_visible", c_int), ("num_tiles", c_int), ("num_coarse", c_int)]


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is deliberately no CPU fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    lib.gsr_abi_version.restype = c_int
    lib.gsr_last_error.restype = c_char_p
    lib.gsr_forward_sizes.argtypes = [c_int, c_int, c_int, c_int, POINTER(c_size_t), POINTER(c_size_t)]
    lib.gsr_forward_geometry.argtypes = [POINTER(GsrForwardArgs), c_void_p, c_void_p, c_void_p, POINTER(c_int), POINTER(c_int)]
    lib.gsr_binning_sizes.argtypes = [c_int, c_int, c_int, c_int, c_int, POINTER(c_size_t), POINTER(c_size_t)]
    lib.gsr_forward_render.argtypes = [POINTER(GsrForwardArgs), c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]
    lib.gsr_forward_recolor.argtypes = [POINTER(GsrForwardArgs), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.gsr_forward_display.argtypes = [POINTER(GsrForwardArgs), POINTER(GsrDisplayArgs), c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_int, c_int, c_void_p]
    lib.gsr_forward_display.restype = c_int
    lib.gsr_backward_scratch_bytes.argtypes = [c_int]
    lib.gsr_backward_scratch_bytes.restype = c_size_t
    lib.gsr_backward_deterministic_sizes.argtypes = [c_int, c_int, POINTER(c_size_t), POINTER(c_size_t)]
    lib.gsr_backward_deterministic_sizes.restype = c_int
    lib.gsr_appearance_deterministic_scratch_bytes.restype = c_size_t
    lib.gsr_backward.argtypes = [POINTER(GsrBackwardArgs), c_void_p]
    lib.gsr_backward_partials.argtypes = [POINTER(GsrBackwardArgs), c_void_p]
    lib.gsr_backward_finalize.argtypes = [POINTER(GsrBackwardArgs), c_void_p]
    lib.gsr_backward_partials_peers.argtypes = [POINTER(GsrBackwardArgs), c_void_p, c_int, c_void_p, c_void_p]
    lib.gsr_backward_partials_marked.argtypes = [POINTER(GsrBackwardArgs), c_void_p, c_void_p]
    lib.gsr_backward_partials_marked.restype = c_int
    lib.gsr_backward_finalize_pull.argtypes = [POINTER(GsrBackwardArgs), c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]
    lib.gsr_backward_finalize_pull.restype = c_int
    lib.gsr_mark_visible.argtypes = [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.gsr_img_views.argtypes = [c_void_p, c_int, c_int, POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p)]
    lib.gsr_binning_views.argtypes = [c_void_p, c_int, POINTER(c_void_p)]
    lib.gsr_geom_views.argtypes = [c_void_p, c_int, c_int, POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p)]
    lib.gsr_get_stats.argtypes = [c_void_p, c_int, c_int, c_void_p, POINTER(GsrStats)]
    lib.gsr_appearance_packed_weight_bytes.restype = c_size_t
    lib.gsr_appearance_grad_pack_bytes.restype = c_size_t
    lib.gsr_appearance_pack_weights.argtypes = [c_void_p] * 9
    lib.gsr_appearance_colors_forward.argtypes = [POINTER(GsrAppearanceArgs), c_void_p]
    lib.gsr_appearance_colors_backward.argtypes = [POINTER(GsrAppearanceArgs), c_void_p]
    lib.gsr_appearance_unpack_grads.argtypes = [c_void_p] * 11
    lib.gsr_appearance_embedding_backward.argtypes = [POINTER(GsrAppearanceArgs), c_void_p]
    lib.gsr_backward_colors.argtypes = [POINTER(GsrBackwardArgs), c_void_p]
    lib.gsr_backward_colors.restype = c_int
    for name in ("gsr_appearance_pack_weights", "gsr_appearance_colors_forward", "gsr_appearance_colors_backward",
                 "gsr_appearance_unpack_grads", "gsr_appearance_embedding_backward"):
        getattr(lib, name).restype = c_int
    lib.gsr_gaussian_activations_forward.argtypes = [c_int] + [c_void_p] * 8
    lib.gsr_gaussian_activations_forward.restype = c_int
    lib.gsr_gaussian_activations_backward.argtypes = [c_int] + [c_void_p] * 11
    lib.gsr_gaussian_activations_backward.restype = c_int
    lib.gsr_sh_colors_forward.argtypes = [c_int, c_int] + [c_void_p] * 6
    lib.gsr_sh_colors_forward.restype = c_int
    lib.gsr_sh_colors_backward.argtypes = [c_int, c_int] + [c_void_p] * 9
    lib.gsr_sh_colors_backward.restype = c_int
    lib.gsr_densification_stats.argtypes = [c_int] + [c_void_p] * 8
    lib.gsr_densification_stats.restype = c_int
    lib.gsr_adam_step.argtypes = [POINTER(GsrAdamSegment), c_int, ctypes.c_double, ctypes.c_double, ctypes.c_double, c_int, c_void_p]
    lib.gsr_adam_step.restype = c_int
    lib.gsr_densify_scratch_bytes.argtypes = [c_int]
    lib.gsr_densify_scratch_bytes.restype = c_size_t
    lib.gsr_densify_plan.argtypes = [POINTER(GsrDensifyArgs), c_void_p]
    lib.gsr_densify_plan.restype = c_int
    lib.gsr_densify_apply.argtypes = [POINTER(GsrDensifyArgs), POINTER(GsrDensifySegment), c_int, c_void_p]
    lib.gsr_densify_apply.restype = c_int
    lib.gsr_reset_opacity.argtypes = [c_int] + [c_void_p] * 5
    lib.gsr_reset_opacity.restype = c_int
    lib.gsr_filter3d_scratch_bytes.argtypes = [c_int]
    lib.gsr_filter3d_scratch_bytes.restype = c_size_t
    lib.gsr_compute_3d_filter.argtypes = [c_int, c_void_p, c_int, c_void_p, c_float, c_void_p, c_void_p, c_void_p]
    lib.gsr_compute_3d_filter.restype = c_int
    lib.gsr_knn_scratch_bytes.argtypes = [c_int]
    lib.gsr_knn_scratch_bytes.restype = c_size_t
    lib.gsr_knn_mean_dist2.argtypes = [c_int, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.gsr_knn_mean_dist2.restype = c_int
    lib.gsr_ssim_forward.argtypes = [c_int, c_int, c_int] + [c_void_p] * 5
    lib.gsr_ssim_forward.restype = c_int
    lib.gsr_ssim_backward.argtypes = [c_int, c_int, c_int] + [c_void_p] * 6
    lib.gsr_ssim_backward.restype = c_int
    lib.gsr_msssim_scratch_bytes.argtypes = [c_int] * 4
    lib.gsr_msssim_scratch_bytes.restype = c_size_t
    lib.gsr_msssim_forward.argtypes = [c_int] * 6 + [c_void_p] * 5
    lib.gsr_msssim_forward.restype = c_int
    lib.gsr_ssim_down_scratch_bytes.argtypes = [c_int] * 3
    lib.gsr_ssim_down_scratch_bytes.restype = c_size_t
    lib.gsr_ssim_down_forward.argtypes = [c_int] * 5 + [c_void_p] * 5
    lib.gsr_ssim_down_forward.restype = c_int
    lib.gsr_attention_scratch_bytes.argtypes = [c_int] * 3
    lib.gsr_attention_scratch_bytes.restype = c_size_t
    lib.gsr_attention_forward.argtypes = [c_int] * 3 + [c_void_p] * 4
    lib.gsr_attention_forward.restype = c_int
    lib.gsr_vit_tokens.argtypes = [c_int] * 6 + [c_void_p] * 8
    lib.gsr_vit_tokens.restype = c_int
    lib.gsr_vit_linear.argtypes = [c_int] * 4 + [c_void_p] * 3 + [c_float] + [c_void_p] * 6
    lib.gsr_vit_linear.restype = c_int
    lib.gsr_vit_output.argtypes = [c_int] * 5 + [c_void_p] * 3 + [c_float] + [c_void_p] * 3
    lib.gsr_vit_output.restype = c_int
    lib.gsr_uncertainty_scratch_bytes.argtypes = [POINTER(GsrUncertaintyArgs)]
    lib.gsr_uncertainty_scratch_bytes.restype = c_size_t
    lib.gsr_uncertainty_forward.argtypes = [POINTER(GsrUncertaintyArgs), c_void_p]
    lib.gsr_uncertainty_forward.restype = c_int
    lib.gsr_uncertainty_backward.argtypes = [POINTER(GsrUncertaintyArgs), c_void_p]
    lib.gsr_uncertainty_backward.restype = c_int
    lib.gsr_uncertainty_mode_scratch_bytes.argtypes = [POINTER(GsrUncertaintyModeArgs)]
    lib.gsr_uncertainty_mode_scratch_bytes.restype = c_size_t
    lib.gsr_uncertainty_mode_forward.argtypes = [POINTER(GsrUncertaintyModeArgs), c_void_p]
    lib.gsr_uncertainty_mode_forward.restype = c_int
    lib.gsr_uncertainty_mode_backward.argtypes = [POINTER(GsrUncertaintyModeArgs), c_void_p]
    lib.gsr_uncertainty_mode_backward.restype = c_int
    lib.gsr_train_loss_scratch_bytes.argtypes = []
    lib.gsr_train_loss_scratch_bytes.restype = c_size_t
    lib.gsr_train_loss_forward.argtypes = [POINTER(GsrTrainLossArgs), c_void_p]
    lib.gsr_train_loss_forward.restype = c_int
    lib.gsr_train_loss_backward.argtypes = [POINTER(GsrTrainLossArgs), c_void_p]
    lib.gsr_train_loss_backward.restype = c_int
    lib.gsr_unpack_u8.argtypes = [c_int, c_int] + [c_void_p] * 5
    lib.gsr_unpack_u8.restype = c_int
    lib.gsr_metrics_scratch_bytes.argtypes = [c_int] * 4
    lib.gsr_metrics_scratch_bytes.restype = c_size_t
    lib.gsr_metrics_forward.argtypes = [POINTER(GsrMetricsArgs), c_void_p]
    lib.gsr_metrics_forward.restype = c_int
    lib.gsr_profile_enable.argtypes = [c_int]
    lib.gsr_profile_enable.restype = None
    lib.gsr_profile_stage_count.restype = c_int
    lib.gsr_profile_stage_name.argtypes = [c_int]
    lib.gsr_profile_stage_name.restype = c_char_p
    lib.gsr_profile_read.argtypes = [POINTER(c_float), c_int]
    lib.gsr_launch_count.restype = ctypes.c_ulonglong
    for name in ("gsr_forward_sizes", "gsr_forward_geometry", "gsr_binning_sizes", "gsr_forward_render",
                 "gsr_forward_recolor", "gsr_backward", "gsr_backward_partials", "gsr_backward_finalize",
                 "gsr_backward_partials_peers",
                 "gsr_mark_visible", "gsr_img_views", "gsr_binning_views",
                 "gsr_geom_views", "gsr_get_stats"):
        getattr(lib, name).restype = c_int
    if lib.gsr_abi_version() != 2:
        raise ImportError(f"{LIB_PATH}: ABI version {lib.gsr_abi_version()} != 2")
    return lib


_lib = _load()

# Tile-row shard used by the calls below (multi-GPU partition, see parallel.py); (0, 0) = whole image.
_shard = (0, 0)


def set_tile_row_shard(y0: int, y1: int) -> None:
    global _shard
    _shard = (int(y0), int(y1))


def get_tile_row_shard():
    return _shard


# ---- geometry reuse across consecutive forward calls (SURVEY.md 8f-1) ------------------------------------------
# One entry (the previous forward).  An entry is reused only if every geometry input is THE SAME tensor object the
# caller passed last time (identity of the ORIGINAL objects, before any dtype / contiguity conversion -- method.py:1516
# passes a transposed, non-contiguous view matrix whose contiguous copy is a new tensor on every call) with the same
# version counter (no in-place modification since), on the same stream, with the same scalar settings.  The entry
# keeps those tensors and their converted copies alive, so their addresses cannot be recycled for other data.
# Modifying a tensor behind autograd's back (``x.data.add_(...)``, a raw kernel writing through data_ptr) does not
# bump the version: call clear_geometry_cache() after such writes or set_geometry_cache(False).  The entry is dropped
# when a backward pass starts (no further forward on this geometry can follow before the parameters change).
_GEOM_CACHE_ON = True
_geom_cache: dict = {}


def _geometry_key(dev, stream, P, W, H, M, scalars, shard, tensors):
    return (str(dev), int(stream), P, W, H, M, tuple(scalars), tuple(shard),
            # "absent" inputs are fresh zero-element tensors on every call (__init__.py:218-228): they compare equal
            tuple((id(t), t.data_ptr(), t._version, tuple(t.shape)) if t.numel() else None for t in tensors))


def set_geometry_cache(on: bool) -> None:
    """Enable / disable the reuse (benchmarks of a full forward switch it off)."""
    global _GEOM_CACHE_ON
    _GEOM_CACHE_ON = bool(on)
    if not on:
        _geom_cache.pop("entry", None)


def clear_geometry_cache() -> None:
    """Drop the cached geometry/binning state of the previous forward (frees its buffers)."""
    _geom_cache.pop("entry", None)


def geometry_cache_hits() -> int:
    return int(_geom_cache.get("hits", 0))


# ---- reproducible runs under torch.use_deterministic_algorithms(True) ------------------------------------------------
# The flag is read on every call: when it is set, the backward composite, the colour-only backward and the colour op add
# their partial sums in a fixed order (GsrBackwardArgs / GsrAppearanceArgs.deterministic), and the paths that have no such
# form refuse to run, as PyTorch's own ops do.
def deterministic() -> bool:
    return torch.are_deterministic_algorithms_enabled()


def refuse_nondeterministic(path: str) -> None:
    """Under ``torch.use_deterministic_algorithms(True)`` raise ``RuntimeError`` naming ``path``, or warn when the flag
    was set with ``warn_only=True``; nothing otherwise."""
    if not torch.are_deterministic_algorithms_enabled():
        return
    msg = (f"{path} does not have a deterministic implementation, but you set "
           "'torch.use_deterministic_algorithms(True)'. Run it on one GPU without a tile-row split across processes, "
           "or call torch.use_deterministic_algorithms(True, warn_only=True) to run it anyway with a warning.")
    if torch.is_deterministic_algorithms_warn_only_enabled():
        warnings.warn(msg)
    else:
        raise RuntimeError(msg)


# Mark bits of the deterministic backward: all-zero between calls (each call clears the bits it set), so one buffer is
# kept per (device, stream) and grown with zeros; a call that failed leaves it dirty and it is re-zeroed.
_det_marks: dict = {}


def deterministic_buffers(P: int, R: int, dev):
    """(scratch, marks) for a deterministic ``GsrBackwardArgs`` call with P Gaussians and R instances.  Call
    ``deterministic_done(marks)`` after the library call returned 0."""
    sb, mb = c_size_t(0), c_size_t(0)
    _check(_lib.gsr_backward_deterministic_sizes(int(P), int(R), byref(sb), byref(mb)), "gsr_backward_deterministic_sizes")
    key = (str(dev), int(_stream(dev)))
    ent = _det_marks.get(key)
    if ent is None or ent[0].numel() < mb.value:
        ent = [torch.zeros((max(mb.value, 256),), dtype=torch.uint8, device=dev), "zero"]
        _det_marks[key] = ent
    elif ent[1] != "zero":
        ent[0].zero_()
    ent[1] = "dirty"
    return torch.empty((sb.value,), dtype=torch.uint8, device=dev), ent[0]


def deterministic_done(marks) -> None:
    for ent in _det_marks.values():
        if ent[0] is marks:
            ent[1] = "zero"


def _check(rc: int, what: str) -> None:
    if rc != 0:
        msg = _lib.gsr_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what} failed ({rc}): {msg}")


def _ptr(t: torch.Tensor | None):
    """Device pointer of a tensor, NULL for the reference's "absent" zero-element tensors
    (``__init__.py:218-228``: empty CPU tensors stand for None)."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def _f32c(t: torch.Tensor, device) -> torch.Tensor:
    if t.numel() == 0:
        return t
    if t.device != device or t.dtype != torch.float32:
        t = t.to(device=device, dtype=torch.float32)
    return t.contiguous()


def _stream(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def forward_args(*, background, means3D, colors, opacities, scales, rotations, viewmatrix, projmatrix, campos, tan_fovx,
                 tan_fovy, kernel_size, subpixel_offset, H, W, radii, out_color=None, scale_modifier=1.0,
                 cov3D_precomp=None, sh=None, degree=0, prefiltered=False, debug=False, shard=(0, 0), peer_images=None):
    """``GsrForwardArgs`` of contiguous fp32 tensors on one device.  None or a zero-element tensor (the reference's
    "absent" input) becomes NULL; P is the number of rows of ``means3D``, M the number of SH coefficients of ``sh``.
    ``shard`` is in the ABI's form (``_abi_shard``), ``peer_images = (device address of the array of per-rank image
    pointers, number of ranks)``."""
    a = GsrForwardArgs()
    a.P, a.D, a.W, a.H = int(means3D.size(0)), int(degree), int(W), int(H)
    a.M = int(sh.size(1)) if sh is not None and sh.numel() != 0 else 0
    a.background, a.means3D, a.shs, a.colors_precomp = _ptr(background), _ptr(means3D), _ptr(sh), _ptr(colors)
    a.opacities, a.scales, a.rotations = _ptr(opacities), _ptr(scales), _ptr(rotations)
    a.scale_modifier, a.cov3D_precomp = float(scale_modifier), _ptr(cov3D_precomp)
    a.viewmatrix, a.projmatrix, a.campos = _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos)
    a.tan_fovx, a.tan_fovy, a.kernel_size = float(tan_fovx), float(tan_fovy), float(kernel_size)
    a.subpixel_offset = _ptr(subpixel_offset)
    a.prefiltered, a.debug = int(bool(prefiltered)), int(bool(debug))
    a.tile_y0, a.tile_y1 = shard
    a.out_color, a.radii = _ptr(out_color), _ptr(radii)
    if peer_images is not None:
        a.peer_images, a.n_peer_images = int(peer_images[0]), int(peer_images[1])
    return a


def _forward_geometry(a, dev, stream):
    """First phase of the forward, shared by the training composite (``gsr_forward_render``) and the display composite
    (``gsr_forward_display``): allocates the geometry and image buffers, runs projection, depth ordering and the
    coarse-item offsets (``gsr_forward_geometry``, whose instance-count read-back is the forward's host
    synchronisation) and allocates the binning buffers for those counts.  Returns ``(geom, img, binning, scratch, R,
    N1)``."""
    byte = dict(dtype=torch.uint8, device=dev)
    gb, ib = c_size_t(0), c_size_t(0)
    _check(_lib.gsr_forward_sizes(a.P, a.M, a.W, a.H, byref(gb), byref(ib)), "gsr_forward_sizes")
    geom, img = torch.empty((gb.value,), **byte), torch.empty((ib.value,), **byte)
    R, N1 = c_int(0), c_int(0)
    _check(_lib.gsr_forward_geometry(byref(a), geom.data_ptr(), img.data_ptr(), stream, byref(R), byref(N1)),
           "gsr_forward_geometry")
    bb, sb = c_size_t(0), c_size_t(0)
    _check(_lib.gsr_binning_sizes(a.P, a.W, a.H, R.value, N1.value, byref(bb), byref(sb)), "gsr_binning_sizes")
    return geom, img, torch.empty((bb.value,), **byte), torch.empty((sb.value,), **byte), R.value, N1.value


def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                        viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset, image_height,
                        image_width, sh, degree, campos, prefiltered, debug):
    """Drop-in for ``RasterizeGaussiansCUDA`` (rasterize_points.cu:35-119).

    Returns ``(num_rendered, out_color[3,H,W], radii[P] int32, geomBuffer, binningBuffer, imgBuffer)``.
    """
    return rasterize_gaussians_shard(_shard, background, means3D, colors, opacity, scales, rotations, scale_modifier,
                                     cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size,
                                     subpixel_offset, image_height, image_width, sh, degree, campos, prefiltered, debug)


# ---- host-buffer pipelines: let the colour inputs arrive while the geometry stage runs ------------------------------------
# The projection / depth-ordering / binning stages read only the geometry inputs (means, scales, rotations, opacities,
# camera); colours, background and sub-pixel offsets are first read by the composite.  A caller that uploads its inputs
# on a copy stream can therefore start the forward as soon as the geometry inputs have landed and hand over the event
# that marks the arrival of the rest: the next forward on this thread waits for it right before its composite stage.
_render_wait = {"event": None}


def defer_composite_inputs(event) -> None:
    """One-shot: the next forward waits for `event` (a torch.cuda.Event recorded on the stream that produces colours /
    background / subpixel_offset) immediately before enqueueing its composite stage instead of before its first kernel."""
    _render_wait["event"] = event


def _wait_for_composite_inputs(dev):
    ev = _render_wait["event"]
    if ev is not None:
        _render_wait["event"] = None
        torch.cuda.current_stream(dev).wait_event(ev)


def _abi_shard(shard, H):
    """(y0, y1) as the C ABI wants it: (0, 0) is its "whole image" sentinel, so an EMPTY band (a rank with no tile
    rows) is expressed as the empty band below the last row."""
    y0, y1 = int(shard[0]), int(shard[1])
    if (y0, y1) == (0, 0):
        return 0, 0
    if y1 <= y0:
        gy = (int(H) + 15) // 16
        return gy, gy
    return y0, y1


def rasterize_gaussians_shard(shard, background, means3D, colors, opacity, scales, rotations, scale_modifier,
                              cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset,
                              image_height, image_width, sh, degree, campos, prefiltered, debug, peer_images=None):
    """``rasterize_gaussians`` restricted to the tile rows ``shard = (y0, y1)`` ((0, 0): whole image).
    ``peer_images = (device address of the array of per-rank [4,H,W] image pointers, number of ranks)``: the band is
    stored into the images of all ranks by the composite itself (``out_color`` is then returned as None)."""
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    if not means3D.is_cuda:
        raise RuntimeError("diff_gaussian_rasterization (sm_90a build) needs CUDA tensors; there is no CPU path")
    dev = means3D.device
    P, H, W = int(means3D.size(0)), int(image_height), int(image_width)
    shard = _abi_shard(shard, H)
    with torch.cuda.device(dev):
        byte = dict(dtype=torch.uint8, device=dev)
        if P == 0:
            e = torch.empty((0,), **byte)
            return (0, torch.zeros((NUM_CHANNELS, H, W), dtype=torch.float32, device=dev),
                    torch.zeros((P,), dtype=torch.int32, device=dev), e, e.clone(), e.clone())
        # every pixel of the rendered rows and every radii entry is written by the kernels: the reference's
        # zero-fills (rasterize_points.cu:67-68) are only needed for the rows a tile-row shard leaves out
        alloc_img = torch.empty if shard == (0, 0) else torch.zeros
        out_color = None if peer_images is not None else alloc_img((NUM_CHANNELS, H, W), dtype=torch.float32, device=dev)
        M = int(sh.size(1)) if sh.numel() != 0 else 0
        stream = _stream(dev)

        # Geometry reuse (SURVEY.md 8f-1): wild-gaussians composites the SAME Gaussians two or three times per step
        # with different colours (raw / appearance-toned / depth; method.py:1573-1631).  When every geometry input is
        # the identical, unmodified tensor object of the previous call, projection, depth ordering and tile binning
        # are not repeated: only the composite runs, on the previous call's geom / binning state.
        geo_orig = (means3D, opacity, scales, rotations, cov3D_precomp, viewmatrix, projmatrix, subpixel_offset)
        scalars = (float(scale_modifier), float(tan_fovx), float(tan_fovy), float(kernel_size), int(bool(prefiltered)),
                   int(bool(debug)))
        geo_key = _geometry_key(dev, stream, P, W, H, M, scalars, shard, geo_orig)
        hit = _geom_cache.get("entry") if (_GEOM_CACHE_ON and M == 0 and peer_images is None) else None
        if hit is not None and not (hit["key"] == geo_key and all(
                (x is y) or (x.numel() == 0 and y.numel() == 0)      # "absent" inputs are fresh empty tensors per call
                for x, y in zip(hit["orig"], geo_orig))):
            hit = None

        if hit is not None:
            (means3D, opacity, scales, rotations, cov3D_precomp, viewmatrix, projmatrix, subpixel_offset) = hit["conv"]
            background, colors, campos = (_f32c(t, dev) for t in (background, colors, campos))
        else:
            (background, means3D, colors, opacity, scales, rotations, cov3D_precomp, viewmatrix, projmatrix,
             subpixel_offset, sh, campos) = (_f32c(t, dev) for t in (
                 background, means3D, colors, opacity, scales, rotations, cov3D_precomp, viewmatrix, projmatrix,
                 subpixel_offset, sh, campos))

        radii = hit["radii"] if hit is not None else torch.empty((P,), dtype=torch.int32, device=dev)
        a = forward_args(background=background, means3D=means3D, colors=colors, opacities=opacity, scales=scales,
                         rotations=rotations, viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos,
                         tan_fovx=tan_fovx, tan_fovy=tan_fovy, kernel_size=kernel_size, subpixel_offset=subpixel_offset,
                         H=H, W=W, radii=radii, out_color=out_color, scale_modifier=scale_modifier,
                         cov3D_precomp=cov3D_precomp, sh=sh, degree=degree, prefiltered=prefiltered, debug=debug,
                         shard=shard, peer_images=peer_images)

        if hit is not None:
            _wait_for_composite_inputs(dev)
            img2 = torch.empty_like(hit["img"])
            _check(_lib.gsr_forward_recolor(byref(a), hit["geom"].data_ptr(), hit["binning"].data_ptr(),
                                            hit["img"].data_ptr(), img2.data_ptr(), stream), "gsr_forward_recolor")
            _geom_cache["hits"] = _geom_cache.get("hits", 0) + 1
            # the caller gets its own radii tensor: the cached one must survive in-place edits by the caller
            return hit["R"], out_color, hit["radii"].clone(), hit["geom"], hit["binning"], img2

        # the instance counts: the reference blocks on them in the middle of its forward (rasterizer_impl.cu:283-284),
        # and so does _forward_geometry; binning and composite follow on buffers sized for them
        geom, img, binning, scratch, R, N1 = _forward_geometry(a, dev, stream)
        _wait_for_composite_inputs(dev)
        _check(_lib.gsr_forward_render(byref(a), geom.data_ptr(), img.data_ptr(), binning.data_ptr(),
                                       scratch.data_ptr(), R, N1, stream), "gsr_forward_render")
        # `scratch` goes back to torch's stream-ordered caching allocator here: any later
        # allocation on this stream is ordered after the kernels that use it.
        del scratch
        if _GEOM_CACHE_ON and M == 0 and peer_images is None:
            _geom_cache["entry"] = dict(
                key=geo_key, orig=geo_orig,
                conv=(means3D, opacity, scales, rotations, cov3D_precomp, viewmatrix, projmatrix, subpixel_offset),
                R=R, radii=radii.clone(), geom=geom, binning=binning, img=img)
    return R, out_color, radii, geom, binning, img


def _backward_impl(mode, accum, background, means3D, radii, colors, scales, rotations, scale_modifier,
                   cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset,
                   dL_dout_color, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, debug,
                   want_cov3D=True, peer=None, shard=None, marked=None, pull=None):
    """mode: "both" (gsr_backward), "partials" (returns the [P,12] accumulator), "finalize" (consumes it).
    want_cov3D=False (autograd path with scales/rotations): dL_dcov3D is an intermediate nobody reads, so it
    is neither allocated nor written (24 B per Gaussian) and None is returned in its place."""
    dev = means3D.device
    P = int(means3D.size(0))
    H, W = int(dL_dout_color.size(1)), int(dL_dout_color.size(2))
    M = int(sh.size(1)) if sh.numel() != 0 else 0
    # a backward pass has started: no further forward on the cached geometry can follow before the parameters
    # change, so the cache entry (one frame's geom / binning / img buffers) is released with the autograd graph
    _geom_cache.pop("entry", None)
    with torch.cuda.device(dev):
        f32 = dict(dtype=torch.float32, device=dev)
        have_scales = scales.numel() != 0
        outs = None
        if mode != "partials":
            # every row of every output is written by the kernel: empty, not zeros
            alloc = torch.empty if P > 0 else torch.zeros
            dL_dmeans3D = alloc((P, 3), **f32)
            dL_dmeans2D = alloc((P, 3), **f32)
            dL_dcolors = alloc((P, NUM_CHANNELS), **f32)
            dL_dopacity = alloc((P, 1), **f32)
            skip_cov3D = have_scales and not want_cov3D
            dL_dcov3D = None if skip_cov3D else alloc((P, 6), **f32)
            dL_dsh = alloc((P, M, 3), **f32)
            dL_dscales = alloc((P, 3), **f32) if have_scales else torch.zeros((P, 3), **f32)
            dL_drotations = alloc((P, 4), **f32) if have_scales else torch.zeros((P, 4), **f32)
            outs = (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations)
        if P == 0:
            return outs if mode != "partials" else torch.zeros((0, 12), **f32)

        keep = [_f32c(t, dev) for t in (background, means3D, colors, scales, rotations, cov3D_precomp, viewmatrix,
                                        projmatrix, subpixel_offset, dL_dout_color, sh, campos)]
        (background, means3D, colors, scales, rotations, cov3D_precomp, viewmatrix, projmatrix, subpixel_offset,
         dL_dout_color, sh, campos) = keep
        radii = radii.contiguous()
        own_accum = accum is None
        if own_accum:
            accum = _zero_accumulator(P, dev)
        assert accum.data_ptr() % 256 == 0 and accum.numel() >= P * 12

        a = GsrBackwardArgs()
        a.P, a.D, a.M, a.R, a.W, a.H = P, int(degree), M, int(R), W, H
        a.background = _ptr(background); a.means3D = _ptr(means3D); a.shs = _ptr(sh)
        a.colors_precomp = _ptr(colors); a.scales = _ptr(scales); a.scale_modifier = float(scale_modifier)
        a.rotations = _ptr(rotations); a.cov3D_precomp = _ptr(cov3D_precomp)
        a.viewmatrix = _ptr(viewmatrix); a.projmatrix = _ptr(projmatrix); a.campos = _ptr(campos)
        a.tan_fovx = float(tan_fovx); a.tan_fovy = float(tan_fovy); a.kernel_size = float(kernel_size)
        a.subpixel_offset = _ptr(subpixel_offset); a.radii = radii.data_ptr()
        a.geom_buffer = _ptr(geomBuffer); a.binning_buffer = _ptr(binningBuffer); a.img_buffer = _ptr(imageBuffer)
        a.dL_dpix = _ptr(dL_dout_color); a.debug = int(bool(debug))
        a.tile_y0, a.tile_y1 = _abi_shard(_shard if shard is None else shard, H)
        a.accum_scratch = accum.data_ptr()
        a.accum_is_zero = 1 if (own_accum or peer is not None) else 0
        if outs is not None:
            a.dL_dmean2D = dL_dmeans2D.data_ptr(); a.dL_dconic = None
            a.dL_dopacity = dL_dopacity.data_ptr(); a.dL_dcolor = dL_dcolors.data_ptr()
            a.dL_dmean3D = dL_dmeans3D.data_ptr()
            a.dL_dcov3D = None if dL_dcov3D is None else dL_dcov3D.data_ptr()
            a.dL_dsh = _ptr(dL_dsh)
            a.dL_dscale = dL_dscales.data_ptr() if have_scales else None
            a.dL_drot = dL_drotations.data_ptr() if have_scales else None
        keep_det = None
        if deterministic() and peer is None and marked is None and pull is None and mode != "finalize" and int(R) > 0:
            keep_det = deterministic_buffers(P, int(R), dev)
            a.deterministic = 1
            a.det_scratch, a.det_marks = keep_det[0].data_ptr(), keep_det[1].data_ptr()
        if marked is not None:        # pull-mode first half: local sums + marks
            a.accum_is_zero = 1
            _check(_lib.gsr_backward_partials_marked(byref(a), marked.data_ptr(), _stream(dev)), "gsr_backward_partials_marked")
            return accum
        if pull is not None:          # pull-mode second half: gather the marked rows of all ranks, chain rule
            accum_ptrs, touched_ptrs, n_peers, self_rank, clear_accum, clear_touched = pull
            arr_a = (c_void_p * int(n_peers))(*[int(x) for x in accum_ptrs])
            arr_t = (c_void_p * int(n_peers))(*[int(x) for x in touched_ptrs])
            _check(_lib.gsr_backward_finalize_pull(byref(a), arr_a, arr_t, int(n_peers), int(self_rank),
                                                   None if clear_accum is None else clear_accum.data_ptr(),
                                                   None if clear_touched is None else clear_touched.data_ptr(), _stream(dev)),
                   "gsr_backward_finalize_pull")
            return outs
        if peer is not None:
            peers_dev, n_peers, mc = peer
            _check(_lib.gsr_backward_partials_peers(byref(a), peers_dev or None, int(n_peers), mc or None, _stream(dev)),
                   "gsr_backward_partials_peers")
            return accum
        fn = {"both": _lib.gsr_backward, "partials": _lib.gsr_backward_partials,
              "finalize": _lib.gsr_backward_finalize}[mode]
        if mode != "finalize":
            _accum_state[id(accum)] = "dirty"          # until a finalize has consumed (and thereby cleared) it
        _check(fn(byref(a), _stream(dev)), "gsr_backward" + ("" if mode == "both" else "_" + mode))
        if keep_det is not None:
            deterministic_done(keep_det[1])
        if mode != "partials":
            _accum_state[id(accum)] = "zero"
    return accum if mode == "partials" else outs


# ---- the [P,12] partial-sum accumulator of the backward ----------------------------------------------------------------
# gsr_backward_finalize zero-fills the buffer after consuming it, so it is all-zero again after each complete backward: it is
# kept per (device, stream, P) and handed to the next pass with accum_is_zero = 1 (no 48 B x P fill, no allocation).  A
# pass that was started but never finalised (an exception in between) leaves it marked dirty and it is re-zeroed.
_accum_cache: dict = {}
_accum_state: dict = {}


def _zero_accumulator(P, dev):
    key = (str(dev), int(_stream(dev)), int(P))
    t = _accum_cache.get(key)
    if t is None:
        if len(_accum_cache) >= 4:
            _accum_cache.clear(); _accum_state.clear()
        # +64 floats so a 256-byte aligned view of P rows always fits
        t = _accum_cache[key] = torch.zeros((P * 12 + 64,), dtype=torch.float32, device=dev)
        _accum_state[id(t)] = "zero"
    elif _accum_state.get(id(t)) != "zero":
        t.zero_()
        _accum_state[id(t)] = "zero"
    return t


def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                 cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size,
                                 subpixel_offset, dL_dout_color, sh, degree, campos, geomBuffer, R, binningBuffer,
                                 imageBuffer, debug):
    """Drop-in for ``RasterizeGaussiansBackwardCUDA`` (rasterize_points.cu:121-204).

    Returns ``(dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations)``.
    """
    return _backward_impl("both", None, background, means3D, radii, colors, scales, rotations, scale_modifier,
                          cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset,
                          dL_dout_color, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, debug)


def rasterize_gaussians_backward_lean(*args):
    """Same as ``rasterize_gaussians_backward`` but without materialising ``dL_dcov3D`` when scales/rotations
    are given (its slot in the returned tuple is None).  Used by the autograd function of this package."""
    return _backward_impl("both", None, *args, want_cov3D=False)


def rasterize_gaussians_backward_partials(*args, shard=None):
    """First half of the backward for the tile-row sharded path: this shard's per-Gaussian partial sums as a
    flat fp32 tensor whose first ``P*12`` entries are the ``[P,12]`` accumulator (same 23 arguments)."""
    return _backward_impl("partials", None, *args, shard=shard)


def rasterize_gaussians_backward_partials_peers(accum, peers_dev_ptr, n_peers, multicast_ptr, *args, shard=None):
    """Reduction-fused first half (``gsr_backward_partials_peers``): this shard's sums are added directly into the
    accumulators of all ranks.  ``accum`` is this rank's symmetric buffer (zeroed on every rank, barrier passed);
    ``peers_dev_ptr`` the address of the DEVICE array holding the ranks' buffer pointers, ``multicast_ptr`` the
    NVSwitch multicast address of the buffer or 0."""
    return _backward_impl("partials", accum, *args, peer=(int(peers_dev_ptr), int(n_peers), int(multicast_ptr)),
                          shard=shard)


def rasterize_gaussians_backward_partials_marked(accum, touched, *args, shard=None):
    """Pull-mode first half (``gsr_backward_partials_marked``): this shard's sums go into THIS rank's symmetric accumulator
    only, ``touched`` (uint8 [P], symmetric) gets a 1 for every Gaussian added to."""
    return _backward_impl("partials", accum, *args, shard=shard, marked=touched)


def rasterize_gaussians_backward_finalize_pull(accum, accum_ptrs, touched_ptrs, n_peers, self_rank, clear_accum,
                                               clear_touched, *args, shard=None):
    """Pull-mode second half (``gsr_backward_finalize_pull``): complete sums = rows of all ranks (peer reads of the marked
    rows, rank order), chain rule -> the 8 gradient tensors; zeroes the previous pass's marked rows / marks."""
    return _backward_impl("finalize", accum, *args, want_cov3D=False, shard=shard,
                          pull=(accum_ptrs, touched_ptrs, n_peers, self_rank, clear_accum, clear_touched))


def rasterize_gaussians_backward_finalize(accum, *args, shard=None):
    """Second half: per-Gaussian chain rule from the (all-reduced) accumulator to the 8 gradient tensors."""
    return _backward_impl("finalize", accum, *args, want_cov3D=False, shard=shard)


def mark_visible(means3D, viewmatrix, projmatrix):
    """Drop-in for ``markVisible`` (rasterize_points.cu:206-225): bool[P], view-space z > 0.2."""
    if not means3D.is_cuda:
        raise RuntimeError("diff_gaussian_rasterization (sm_90a build) needs CUDA tensors; there is no CPU path")
    dev = means3D.device
    P = int(means3D.size(0))
    with torch.cuda.device(dev):
        present = torch.zeros((P,), dtype=torch.bool, device=dev)
        if P != 0:
            m = _f32c(means3D, dev)
            v = _f32c(viewmatrix, dev)
            pm = _f32c(projmatrix, dev)
            _check(_lib.gsr_mark_visible(P, m.data_ptr(), v.data_ptr(), pm.data_ptr(), present.data_ptr(),
                                         _stream(dev)), "gsr_mark_visible")
    return present


# ---- extras (not part of the reference surface; used by parity tests and the benchmark) ----------

def _as_tensor(ptr: int, nbytes: int, owner: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """View of `nbytes` bytes at device address `ptr` inside `owner` (a uint8 buffer)."""
    off = ptr - owner.data_ptr()
    assert 0 <= off and off + nbytes <= owner.numel(), "view outside its buffer"
    return owner[off:off + nbytes].view(dtype)


def debug_views(geomBuffer, binningBuffer, imgBuffer, P, M, W, H, R):
    """Expose the integer artefacts the parity tests compare bit-exactly."""
    out = {}
    T = ((W + 15) // 16) * ((H + 15) // 16)
    ft, nc, rg = c_void_p(), c_void_p(), c_void_p()
    _check(_lib.gsr_img_views(imgBuffer.data_ptr(), W, H, byref(ft), byref(nc), byref(rg)), "gsr_img_views")
    out["final_T"] = _as_tensor(ft.value, 4 * W * H, imgBuffer, torch.float32).view(H, W)
    out["n_contrib"] = _as_tensor(nc.value, 4 * W * H, imgBuffer, torch.int32).view(H, W)
    out["ranges"] = _as_tensor(rg.value, 8 * T, imgBuffer, torch.int32).view(T, 2)
    if R > 0:
        pl = c_void_p()
        _check(_lib.gsr_binning_views(binningBuffer.data_ptr(), R, byref(pl)), "gsr_binning_views")
        out["point_list"] = _as_tensor(pl.value, 4 * R, binningBuffer, torch.int32)
    else:
        out["point_list"] = torch.empty((0,), dtype=torch.int32, device=imgBuffer.device)
    d, rec, tt, rgb = c_void_p(), c_void_p(), c_void_p(), c_void_p()
    _check(_lib.gsr_geom_views(geomBuffer.data_ptr(), P, M, byref(d), byref(rec), byref(tt), byref(rgb)), "gsr_geom_views")
    out["depths"] = _as_tensor(d.value, 4 * P, geomBuffer, torch.float32)
    out["records"] = _as_tensor(rec.value, 32 * P, geomBuffer, torch.float32).view(P, 8)
    out["tiles_touched"] = _as_tensor(tt.value, 4 * P, geomBuffer, torch.int32)
    if M > 0:
        out["rgb"] = _as_tensor(rgb.value, 12 * P, geomBuffer, torch.float32).view(P, 3)
    return out


def stats(geomBuffer, P, M):
    s = GsrStats()
    _check(_lib.gsr_get_stats(geomBuffer.data_ptr(), P, M, _stream(geomBuffer.device), byref(s)), "gsr_get_stats")
    return {"num_rendered": s.num_rendered, "num_visible": s.num_visible, "num_coarse": s.num_coarse}


def profile_enable(on: bool) -> None:
    """Per-stage device timing of the following calls (cudaEvents inside the library)."""
    _lib.gsr_profile_enable(int(bool(on)))


def profile_read() -> dict:
    """Stage name -> milliseconds of the most recent forward/backward (synchronise first)."""
    n = _lib.gsr_profile_stage_count()
    buf = (c_float * n)()
    _lib.gsr_profile_read(buf, n)
    return {_lib.gsr_profile_stage_name(i).decode(): float(buf[i]) for i in range(n) if buf[i] >= 0}


def launch_count() -> int:
    return int(_lib.gsr_launch_count())
