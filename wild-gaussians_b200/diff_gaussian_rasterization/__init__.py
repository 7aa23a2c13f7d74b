"""Drop-in ``diff_gaussian_rasterization`` package backed by the sm_90a rasterizer.

Public surface = the reference's (``submodules/diff-gaussian-rasterization/
diff_gaussian_rasterization/__init__.py``):

* ``GaussianRasterizationSettings`` -- NamedTuple, 15 fields, same order (``:175-190``)
* ``GaussianRasterizer(raster_settings)`` -- ``nn.Module`` with ``forward(means3D, means2D,
  opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None)
  -> (color, radii, accumulation)`` and ``markVisible(positions)`` (``:192-241``)
* ``rasterize_gaussians(...)`` and the autograd function ``_RasterizeGaussians`` (``:21-173``)
* submodule ``_C`` with ``rasterize_gaussians`` / ``rasterize_gaussians_backward`` /
  ``mark_visible`` (``ext.cpp:15-19``)

so ``wildgaussians/method.py`` (``:26``, ``:1529-1631``) runs on it unchanged.  Error behaviour
is kept: ``Exception`` for the shs/colors and scale-rotation/cov3D exclusivity checks,
``RuntimeError`` for a mis-shaped ``means3D``, and with ``debug=True`` a CPU snapshot of the
arguments is written to ``snapshot_fw.dump`` / ``snapshot_bw.dump`` before re-raising.
"""
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _C

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians", "defer_composite_inputs"]

# extension of the reference surface for host-buffer pipelines (see _C.defer_composite_inputs)
defer_composite_inputs = _C.defer_composite_inputs


def cpu_deep_copy_tuple(input_tuple):
    return tuple(item.cpu().clone() if isinstance(item, torch.Tensor) else item for item in input_tuple)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings)


def _call_with_snapshot(fn, args, debug, dump_name, what):
    if not debug:
        return fn(*args)
    cpu_args = cpu_deep_copy_tuple(args)  # copy before anything can corrupt them
    try:
        return fn(*args)
    except Exception:
        torch.save(cpu_args, dump_name)
        print(f"\nAn error occured in {what}. Please forward {dump_name} for debugging.")
        raise


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        s = raster_settings
        args = (s.bg, means3D, colors_precomp, opacities, scales, rotations, s.scale_modifier, cov3Ds_precomp,
                s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.kernel_size, s.subpixel_offset,
                s.image_height, s.image_width, sh, s.sh_degree, s.campos, s.prefiltered, s.debug)
        num_rendered, color, radii, geomBuffer, binningBuffer, imgBuffer = _call_with_snapshot(
            _C.rasterize_gaussians, args, s.debug, "snapshot_fw.dump", "forward")

        ctx.raster_settings = s
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer,
                              binningBuffer, imgBuffer)

        accumulation = None
        if s.return_accumulation:
            H, W = int(s.image_height), int(s.image_width)
            if imgBuffer.numel() == 0:
                accumulation = torch.zeros((H, W), dtype=torch.float32, device=color.device)
            else:
                # final transmittance is the first 128-byte aligned array of imgBuffer
                # (same layout contract as the reference, __init__.py:101-113)
                offset = (128 - imgBuffer.data_ptr()) % 128
                final_T = imgBuffer[offset:offset + 4 * H * W].view(torch.float32)
                accumulation = (1.0 - final_T).view(H, W)
        return color, radii, accumulation

    @staticmethod
    def backward(ctx, grad_out_color, _1, _2):
        s = ctx.raster_settings
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer, binningBuffer,
         imgBuffer) = ctx.saved_tensors
        args = (s.bg, means3D, radii, colors_precomp, scales, rotations, s.scale_modifier, cov3Ds_precomp,
                s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.kernel_size, s.subpixel_offset, grad_out_color,
                sh, s.sh_degree, s.campos, geomBuffer, ctx.num_rendered, binningBuffer, imgBuffer, s.debug)
        (grad_means2D, grad_colors_precomp, grad_opacities, grad_means3D, grad_cov3Ds_precomp, grad_sh, grad_scales,
         grad_rotations) = _call_with_snapshot(_C.rasterize_gaussians_backward_lean, args, s.debug, "snapshot_bw.dump",
                                               "backward")
        return (grad_means3D, grad_means2D, grad_sh, grad_colors_precomp, grad_opacities, grad_scales,
                grad_rotations, grad_cov3Ds_precomp, None)


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    kernel_size: float
    subpixel_offset: torch.Tensor
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool
    return_accumulation: bool


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        """Boolean mask of the points in front of the near plane of this camera."""
        with torch.no_grad():
            s = self.raster_settings
            return _C.mark_visible(positions, s.viewmatrix, s.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        if (shs is None) == (colors_precomp is None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')

        empty = torch.Tensor([])
        shs = empty if shs is None else shs
        colors_precomp = empty if colors_precomp is None else colors_precomp
        scales = empty if scales is None else scales
        rotations = empty if rotations is None else rotations
        cov3D_precomp = empty if cov3D_precomp is None else cov3D_precomp

        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                   cov3D_precomp, self.raster_settings)
