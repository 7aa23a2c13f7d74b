"""Opt-in fast path for the CALLER of the rasterizer, ``GaussianModel._render_internal`` (wildgaussians/method.py:1479-1632),
and for the statistics that consume its outputs (SURVEY.md 8f-2 / 8f-3 / 8f-4).  ``method.py`` itself is not modified:

    import wildgaussians_fused
    wildgaussians_fused.enable(model)        # model: wildgaussians.method.GaussianModel

rebinds ``model._render_internal`` to ``render_internal`` below, which returns the same dictionary but

* evaluates the parameter activations + 3D filter (``get_gaussians``, method.py:1060-1086) with one kernel per direction;
* evaluates the raw and the appearance-toned colours with ONE fused kernel per direction (``fused_colors``:
  wgmma MLP + SH evaluation, ``csrc/appearance.cu``) instead of ~60 PyTorch launches and several P x 128 / P x 48
  fp32 intermediates (method.py:1570-1598);
* for a model without appearance, evaluates the SH colours with one bandwidth-bound kernel per direction
  (``fused_sh_colors``, ``csrc/sh_colors.cu``) and composites once, as the reference does (method.py:1555-1583);
* caches the per-camera constants -- the numpy 4x4 inversions, ``getWorld2View2``, the projection matrix, the camera
  centre, tan(fov) (method.py:1502-1527) -- per (pose, intrinsics, size), and the all-zero ``subpixel_offset`` /
  background tensors per (H, W, device): no per-call H2D copies, ``zeros(H, W, 2)`` fills or device-side 4x4 inverse;
* does not synchronise on ``active_sh_degree.cpu().item()`` (method.py:1540) every call: the value is read back only when
  the buffer's version counter changed;
* both rasterizer passes share one projection / depth order / tile binning (the drop-in package's geometry reuse).

``add_densification_stats`` (model method) / ``densification_stats`` (function) fuse method.py:1997-1998 and :1470-1477
into one kernel.  ``enable(model, ssim=True)`` also routes the loss's SSIM (method.py:644-673) through ``fused_ssim``,
``enable(model, msssim=True)`` the uncertainty loss's ``msssim`` and ``ssim_down`` (method.py:126-187), and
``enable(model, dino=True)`` the uncertainty backbone's ``get_intermediate_layers`` through ``fused_dino`` (early exit
after the last block asked for, fused attention), and ``enable(model, uncertainty=True)`` the uncertainty model's
``_compute_losses`` through ``fused_uncertainty`` (the head and the ``dino``-mode loss as kernels, a feature cache that hits),
and ``enable(model, densify=True)`` ``densify_and_prune`` and ``reset_opacity`` through ``fused_densify`` (one gather kernel
into final-size tensors, a GPU quantile without torch's 2^24-element limit, one synchronisation).  ``enable_method(method)`` does what ``enable`` does for
``method.model`` and routes ``method.optimize_embedding`` (test-time appearance optimisation, method.py:1755-1830)
through ``fused_embedding``; ``enable_method(method, train=True)`` also routes ``method.train_iteration``
(method.py:1880-2024) through ``fused_train``: the loss block and its metrics as kernels, training images staged as
bytes in pinned memory, one metric read-back per step.  ``enable_metrics(evaluation)`` routes the evaluation's
``compute_metrics`` (wildgaussians/evaluation.py:331-352) through ``fused_metrics``: SSIM, MSE and MAE as kernels, LPIPS
fed from device memory, one synchronisation per call.
Two configurations are accelerated, which covers all three presets the reference ships: appearance on with separate
tuned colour, ``appearance_model_sh`` off, SH degree 3, 24 + 32 embedding features (the default, and the phototourism
preset), and appearance off with SH degree 3 (the NeRF On-the-go preset; ``embedding`` is then ignored, as the
reference ignores it).  Anything else falls through to the original method, so ``enable`` is always safe.
"""
from __future__ import annotations

import math
import sys
import types

import numpy as np
import torch

from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer, _C
from fused_colors import fused_activations, fused_colors, fused_sh_colors

_cam_cache: dict = {}
_zero_cache: dict = {}
_deg_cache: dict = {}
_CAM_CACHE_MAX = 4096


def _camera_constants(m, cam, device):
    """The tensors / scalars of method.py:1502-1527 for one camera, computed once with the reference's own helper functions."""
    poses = np.ascontiguousarray(cam.poses)
    intr = np.asarray(cam.intrinsics, dtype=np.float64)
    width, height = (int(x) for x in cam.image_sizes)
    key = (poses.tobytes(), intr.tobytes(), width, height, str(device))
    hit = _cam_cache.get(key)
    if hit is not None:
        return hit
    pose = np.concatenate([np.copy(poses), np.array([[0, 0, 0, 1]], dtype=poses.dtype)], axis=0)
    pose = np.linalg.inv(pose)
    R = np.transpose(pose[:3, :3])
    T = pose[:3, 3]
    fx, fy, cx, cy = cam.intrinsics
    world_view = torch.tensor(m.getWorld2View2(R, T, np.array([0.0, 0.0, 0.0], dtype=np.float32), 1.0)).transpose(0, 1).to(device=device)
    # (float() arguments: the helper assigns its results into a torch tensor element, which rejects numpy.float32 scalars)
    proj = m.getProjectionMatrixFromOpenCV(width, height, float(fx), float(fy), float(cx), float(cy), 0.01, 100.0) \
        .transpose(0, 1).to(device=device)
    full_proj = (world_view.unsqueeze(0).bmm(proj.unsqueeze(0))).squeeze(0)
    cam_center = world_view.inverse()[3, :3]
    out = dict(world_view=world_view.contiguous(), full_proj=full_proj.contiguous(), cam_center=cam_center.contiguous(),
               tanfovx=math.tan(m.focal2fov(float(fx), float(width)) * 0.5),
               tanfovy=math.tan(m.focal2fov(float(fy), float(height)) * 0.5), width=width, height=height)
    if len(_cam_cache) >= _CAM_CACHE_MAX:
        _cam_cache.clear()
    _cam_cache[key] = out
    return out


def _zeros(shape, device):
    key = (tuple(shape), str(device))
    t = _zero_cache.get(key)
    if t is None:
        t = _zero_cache[key] = torch.zeros(shape, dtype=torch.float32, device=device)
    return t


def _active_degree(model) -> int:
    t = model.active_sh_degree
    key = id(t)
    hit = _deg_cache.get(key)
    if hit is None or hit[0] != t._version or hit[2] is not t:
        hit = _deg_cache[key] = (t._version, int(t.item()), t)
    return hit[1]


def _supported(model, config) -> bool:
    """The appearance-on configuration the fused colour op covers (the reference's default)."""
    c = model.config
    return (bool(c.appearance_enabled) and bool(c.appearance_separate_tuned_color) and not bool(c.appearance_model_sh)
            and int(c.sh_degree) == 3 and model.features_rest is not None and model.embeddings is not None
            and model.appearance_mlp is not None and model.embeddings.shape[1] == 24 and int(c.appearance_embedding_dim) == 32
            and model.xyz.is_cuda and not bool(config.debug))


def _supported_sh(model, config) -> bool:
    """The appearance-off configuration (e.g. the NeRF On-the-go preset) that ``fused_sh_colors`` covers: SH degree 3
    storage; storage degree 0 (no ``features_rest``) is a different branch of the reference and falls through."""
    c = model.config
    return (not bool(c.appearance_enabled) and int(c.sh_degree) == 3 and model.features_rest is not None
            and model.xyz.is_cuda and not bool(config.debug))


def render_internal(self, viewpoint_camera, config, *, kernel_size, scaling_modifier=1.0, embedding, return_raw=True,
                    render_depth=False):
    """Drop-in for ``GaussianModel._render_internal``: same arguments, same output dictionary."""
    appearance = embedding is not None and _supported(self, config)
    if not (appearance or _supported_sh(self, config)):
        return type(self)._render_internal(self, viewpoint_camera, config, kernel_size=kernel_size,
                                           scaling_modifier=scaling_modifier, embedding=embedding, return_raw=return_raw,
                                           render_depth=render_depth)
    m = sys.modules[type(self).__module__]
    device = self.xyz.device
    assert len(viewpoint_camera.poses.shape) == 2, "Expected a single camera"
    assert viewpoint_camera.image_sizes is not None, "Expected image sizes to be set"
    cc = _camera_constants(m, viewpoint_camera, device)
    H, W = cc["height"], cc["width"]

    # zero tensor whose .grad receives the screen-space gradients (method.py:1495-1499)
    screenspace_points = torch.zeros_like(self.xyz, dtype=self.xyz.dtype, requires_grad=True, device=device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    deg = _active_degree(self)
    settings = GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=cc["tanfovx"], tanfovy=cc["tanfovy"], kernel_size=kernel_size,
        subpixel_offset=_zeros((H, W, 2), device), bg=_zeros((3,), device), scale_modifier=scaling_modifier,
        viewmatrix=cc["world_view"], projmatrix=cc["full_proj"], sh_degree=deg, campos=cc["cam_center"], prefiltered=False,
        debug=False, return_accumulation=True)
    rasterizer = GaussianRasterizer(raster_settings=settings)

    # activations + 3D filter (get_gaussians, method.py:1060-1086) in one kernel per direction
    means3D = self.xyz
    scales, opacity, rotations = fused_activations(self.scales, self.opacities, self.rotations, self.filter_3D)
    kw = dict(means3D=means3D, means2D=screenspace_points, opacities=opacity, scales=scales, rotations=rotations, shs=None,
              cov3D_precomp=None)
    if appearance:
        colors_raw, colors_toned = fused_colors(self.features_dc, self.features_rest, self.embeddings, embedding,
                                                self.appearance_mlp.mlp, means3D, cc["cam_center"], deg,
                                                want_raw=bool(return_raw))
        raw_image = radii = accumulation = None
        if return_raw:
            raw_image, radii, accumulation = rasterizer(colors_precomp=colors_raw, **kw)
        image, radii2, accumulation2 = rasterizer(colors_precomp=colors_toned, **kw)
        radii = radii2 if radii is None else radii
        accumulation = accumulation2 if accumulation is None else accumulation
    else:
        # no appearance model (method.py:1573-1583): one pass with the SH colours; `embedding` is ignored
        colors = fused_sh_colors(self.features_dc, self.features_rest, means3D, cc["cam_center"], deg)
        image, radii, accumulation = rasterizer(colors_precomp=colors, **kw)
        raw_image = image
    out = {"render": image, "viewspace_points": screenspace_points, "visibility_filter": radii > 0,
           "accumulation": accumulation, "radii": radii}
    if return_raw:
        out["raw_render"] = raw_image
    if render_depth:
        dist = torch.norm(means3D - cc["cam_center"][None], dim=-1).unsqueeze(-1).repeat(1, 3)
        out["depth"] = rasterizer(colors_precomp=dist, **kw)[0][0]
    return out


def densification_stats(model, viewspace_point_tensor, radii) -> None:
    """method.py:1997-1998 + ``add_densification_stats`` (:1470-1477) in one kernel (in place on the model's buffers)."""
    grad = viewspace_point_tensor.grad
    P = int(radii.shape[0])
    dev = radii.device
    use_abs = bool(model.config.use_gof_abs_gradient)
    bufs = [model.max_radii2D, model.xyz_grad, model.denom] + ([model.xyz_gradient_accum_abs, model.xyz_gradient_accum_abs_max] if use_abs else [])
    if not (radii.is_cuda and grad is not None and grad.dtype == torch.float32 and grad.is_contiguous() and radii.dtype == torch.int32
            and radii.is_contiguous() and all(b.dtype == torch.float32 and b.is_contiguous() and b.numel() == P for b in bufs)):
        vis = radii > 0
        model.max_radii2D[vis] = torch.max(model.max_radii2D[vis], radii[vis])
        model.add_densification_stats(viewspace_point_tensor, vis)
        return
    with torch.cuda.device(dev):
        _C._check(_C._lib.gsr_densification_stats(
            P, radii.data_ptr(), grad.data_ptr(), model.max_radii2D.data_ptr(), model.xyz_grad.data_ptr(),
            model.xyz_gradient_accum_abs.data_ptr() if use_abs else None,
            model.xyz_gradient_accum_abs_max.data_ptr() if use_abs else None, model.denom.data_ptr(),
            torch.cuda.current_stream(dev).cuda_stream), "gsr_densification_stats")


def camera_table(cameras) -> tuple:
    """The per-camera constants of ``compute_3D_filter`` (method.py:1147-1181) for all cameras as one [C, 20] float32 array
    (layout: include/gsrast.h, gsr_compute_3d_filter) and the focal length of the highest-resolution camera (:1178-1179).
    Built with the reference's own statements (numpy 4x4 inverse, transposed rotation) in one pass on the host."""
    rows, focal = [], 0.0
    for camera in cameras:
        assert camera.image_sizes is not None, "Camera image size is not set"
        fx, fy, _, _ = camera.intrinsics
        width, height = camera.image_sizes
        pose = np.copy(camera.poses)
        pose = np.concatenate([pose, np.array([[0, 0, 0, 1]], dtype=pose.dtype)], axis=0)
        pose = np.linalg.inv(pose)
        R = np.transpose(pose[:3, :3]).astype(np.float32)
        T = pose[:3, 3].astype(np.float32)
        f32 = np.float32
        rows.append(np.concatenate([R.reshape(-1), T, np.array(
            [f32(fx), f32(fy), f32(width / 2.0), f32(height / 2.0), f32(-0.15 * width), f32(width * 1.15), f32(-0.15 * height),
             f32(1.15 * height)], dtype=np.float32)]))
        if focal < fx:
            focal = fx
    table = np.stack(rows).astype(np.float32) if rows else np.zeros((0, 20), dtype=np.float32)
    return table, float(focal)


def compute_3D_filter(model, cameras) -> None:
    """``GaussianModel.compute_3D_filter`` (method.py:1140-1190) in two kernels over all cameras (csrc/filter3d.cu) instead of
    ~20 PyTorch launches + 2 H2D copies + 2 host synchronisations PER CAMERA; registers the same ``filter_3D`` buffer."""
    xyz = model.xyz
    if not (xyz.is_cuda and xyz.dtype == torch.float32 and xyz.is_contiguous()):
        return type(model).compute_3D_filter(model, cameras)
    table, focal = camera_table(cameras)
    if table.shape[0] == 0 or not focal > 0:
        return type(model).compute_3D_filter(model, cameras)
    dev, P = xyz.device, int(xyz.shape[0])
    with torch.no_grad(), torch.cuda.device(dev):
        cams = torch.from_numpy(table).to(dev)
        scratch = torch.empty((_C._lib.gsr_filter3d_scratch_bytes(P) + 15) // 16 * 4, dtype=torch.float32, device=dev)
        out = torch.empty((P,), dtype=torch.float32, device=dev)
        _C._check(_C._lib.gsr_compute_3d_filter(P, xyz.data_ptr(), int(table.shape[0]), cams.data_ptr(), focal, out.data_ptr(),
                                                scratch.data_ptr(), torch.cuda.current_stream(dev).cuda_stream),
                  "gsr_compute_3d_filter")
        filter_3D = out.to(dtype=model.filter_3D.dtype, device=model.filter_3D.device)
        del model.filter_3D
        model.register_buffer("filter_3D", filter_3D[..., None])


def _ssim_hook(original):
    """A stand-in for method.py's module-level ``ssim`` (:644-673): ``fused_ssim.ssim`` where it supports the input,
    ``original`` otherwise (CPU tensors, other dtypes or window sizes, a gradient wanted for img2, ...)."""
    import fused_ssim

    def ssim(img1, img2, window_size=11, size_average=True):
        if fused_ssim.supported(img1, img2, window_size):
            return fused_ssim.ssim(img1, img2, window_size, size_average)
        return original(img1, img2, window_size, size_average)

    ssim.__wrapped__ = original
    return ssim


def _stats_hook(original, fused, supported):
    """A stand-in for method.py's module-level ``msssim`` (:171-187) or ``ssim_down`` (:126-135): the fused forward where
    it supports the input, ``original`` otherwise (CPU tensors, other dtypes or shapes, a gradient wanted, ...)."""

    def hook(*args, **kwargs):
        if supported(*args, **kwargs):
            return fused(*args, **kwargs)
        return original(*args, **kwargs)

    hook.__name__ = getattr(original, "__name__", fused.__name__)
    hook.__wrapped__ = original
    return hook


def dino_get_intermediate_layers(self, x, n=1, reshape=False, return_class_token=False, norm=True):
    """Drop-in for ``DinoVisionTransformer.get_intermediate_layers`` (dinov2.py:789-813): ``fused_dino`` where it supports
    the input, the class's own method otherwise (CPU tensors, other dtypes, a gradient wanted, other head sizes, ...)."""
    import fused_dino
    if fused_dino.supported(self, x, n):
        return fused_dino.get_intermediate_layers(self, x, n, reshape, return_class_token, norm)
    return type(self).get_intermediate_layers(self, x, n, reshape, return_class_token, norm)


def uncertainty_compute_losses(self, gt, prediction, prefix='', _cache_entry=None):
    """Drop-in for ``UncertaintyModel._compute_losses`` (method.py:363-433): ``fused_uncertainty`` where it supports the
    call (``dino`` mode, batch 1, fp32 on the GPU, training mode, no cross-process BatchNorm), the class's own method
    otherwise."""
    import fused_uncertainty
    if fused_uncertainty.supported(self, gt, prediction):
        return fused_uncertainty.compute_losses(self, gt, prediction, prefix, _cache_entry=_cache_entry)
    return type(self)._compute_losses(self, gt, prediction, prefix, _cache_entry=_cache_entry)


def densify_and_prune(self, max_grad, min_opacity, extent, enable_size_pruning, skyradius=None):
    """Drop-in for ``GaussianModel.densify_and_prune`` (method.py:1420-1468): ``fused_densify`` where it supports the
    model, the class's own method otherwise."""
    import fused_densify
    return fused_densify.densify_and_prune(self, max_grad, min_opacity, extent, enable_size_pruning, skyradius=skyradius)


def reset_opacity(self):
    """Drop-in for ``GaussianModel.reset_opacity`` (method.py:1249-1278): ``fused_densify`` where it supports the model,
    the class's own method otherwise."""
    import fused_densify
    return fused_densify.reset_opacity(self)


def enable(model, optimizer: bool = True, ssim: bool = False, msssim: bool = False, dino: bool = False,
           uncertainty: bool = False, densify: bool = False):
    """Route this model's ``_render_internal`` and ``compute_3D_filter`` through the fused paths (instance attributes; the
    class is untouched) and, with ``optimizer``, turn its Adam into the single-kernel ``fused_adam.FusedAdam`` in place.

    With ``ssim``, the module-level ``ssim`` of the model's method module (the photometric loss, method.py:1949, and
    appearance optimisation, :1801) is rebound to ``fused_ssim.ssim`` for supported input.  With ``msssim``, its
    ``msssim`` and ``ssim_down`` (the uncertainty loss, method.py:360, :368-369, :407) are rebound to ``fused_ssim.msssim``
    and ``fused_ssim.ssim_down`` for supported input.  Those names are shared by every model of the module; ``disable``
    restores the originals.  With ``dino``, ``model.uncertainty_model.backbone.get_intermediate_layers`` (every DINOv2
    call of the uncertainty loss, method.py:260) is rebound, as an instance attribute, to ``dino_get_intermediate_layers``.
    With ``uncertainty``, ``model.uncertainty_model._compute_losses`` (reached from ``get_loss``) is rebound, as an
    instance attribute, to ``uncertainty_compute_losses``: the fused head and ``dino``-mode loss with a feature cache
    that hits.  With ``densify``, ``model.densify_and_prune`` and ``model.reset_opacity`` are rebound, as instance
    attributes, to the ``fused_densify`` kernels (same results, one synchronisation per densification, any number of
    Gaussians)."""
    model._render_internal = types.MethodType(render_internal, model)
    model.compute_3D_filter = types.MethodType(compute_3D_filter, model)
    if optimizer and type(getattr(model, "optimizer", None)) is torch.optim.Adam:
        import fused_adam
        fused_adam.adopt(model.optimizer)
    if ssim:
        m = sys.modules[type(model).__module__]
        if not hasattr(m.ssim, "__wrapped__"):
            m.ssim = _ssim_hook(m.ssim)
    if msssim:
        import fused_ssim
        m = sys.modules[type(model).__module__]
        if not hasattr(m.msssim, "__wrapped__"):
            m.msssim = _stats_hook(m.msssim, fused_ssim.msssim, fused_ssim.supported_msssim)
        if not hasattr(m.ssim_down, "__wrapped__"):
            m.ssim_down = _stats_hook(m.ssim_down, fused_ssim.ssim_down, fused_ssim.supported_ssim_down)
    backbone = _dino_backbone(model)
    if dino and backbone is not None and "get_intermediate_layers" not in backbone.__dict__:
        backbone.get_intermediate_layers = types.MethodType(dino_get_intermediate_layers, backbone)
    um = getattr(model, "uncertainty_model", None)
    if uncertainty and um is not None and "_compute_losses" not in um.__dict__:
        um._compute_losses = types.MethodType(uncertainty_compute_losses, um)
    if densify:
        model.densify_and_prune = types.MethodType(densify_and_prune, model)
        model.reset_opacity = types.MethodType(reset_opacity, model)
    return model


def _dino_backbone(model):
    return getattr(getattr(model, "uncertainty_model", None), "backbone", None)


def disable(model):
    model.__dict__.pop("_render_internal", None)
    model.__dict__.pop("compute_3D_filter", None)
    model.__dict__.pop("densify_and_prune", None)
    model.__dict__.pop("reset_opacity", None)
    backbone = _dino_backbone(model)
    if backbone is not None:
        backbone.__dict__.pop("get_intermediate_layers", None)
    um = getattr(model, "uncertainty_model", None)
    if um is not None:
        um.__dict__.pop("_compute_losses", None)
    if type(getattr(model, "optimizer", None)).__name__ == "FusedAdam":
        model.optimizer.__class__ = torch.optim.Adam
    m = sys.modules.get(type(model).__module__)
    if m is not None:
        for name in ("ssim", "msssim", "ssim_down"):
            if hasattr(getattr(m, name, None), "__wrapped__"):
                setattr(m, name, getattr(m, name).__wrapped__)
    return model


def optimize_embedding(method, dataset, *, embedding=None):
    """``WildGaussians.optimize_embedding`` on one geometry pass (``fused_embedding``); unsupported configurations run
    the method's own implementation."""
    import fused_embedding
    return fused_embedding.optimize_embedding(method, dataset, embedding=embedding)


def _metrics_hook(original, evaluation):
    """A stand-in for evaluation.py's ``compute_metrics`` (:331-352): ``fused_metrics.compute_metrics`` where it supports
    the input, ``original`` otherwise (no CUDA device, images under 11 pixels, other dtypes or shapes)."""
    import fused_metrics

    def compute_metrics(pred, gt, *, reduce=True, run_lpips_vgg=False):
        if fused_metrics.supported(pred, gt):
            return fused_metrics.compute_metrics(pred, gt, reduce=reduce, run_lpips_vgg=run_lpips_vgg, evaluation=evaluation)
        return original(pred, gt, reduce=reduce, run_lpips_vgg=run_lpips_vgg)

    compute_metrics.__wrapped__ = original
    return compute_metrics


def _modules_binding(evaluation, fn):
    """The evaluation module and every loaded module whose global ``compute_metrics`` is ``fn``."""
    mods = [evaluation] + [m for m in list(sys.modules.values()) if m is not evaluation]
    return [m for m in mods if getattr(m, "__dict__", {}).get("compute_metrics") is fn]


def enable_metrics(evaluation):
    """Rebind ``compute_metrics`` of the reference's ``evaluation`` module, and of every loaded module that imported the
    same function by name (``train.py``'s ``from .evaluation import compute_metrics``), to a hook that runs
    ``fused_metrics.compute_metrics`` for supported input and the original otherwise.  Objects that captured the function
    earlier keep it: ``NerfWEvaluationProtocol`` stores it in ``__init__``, so an instance built after this call takes the
    fused path and one built before keeps the original.  ``disable_metrics`` undoes the rebinding."""
    original = evaluation.compute_metrics
    if hasattr(original, "__wrapped__"):
        return evaluation
    hook = _metrics_hook(original, evaluation)
    for m in _modules_binding(evaluation, original):
        m.compute_metrics = hook
    return evaluation


def disable_metrics(evaluation):
    """Restore the original ``compute_metrics`` in every module ``enable_metrics`` rebound."""
    hook = evaluation.compute_metrics
    original = getattr(hook, "__wrapped__", None)
    if original is not None:
        for m in _modules_binding(evaluation, hook):
            m.compute_metrics = original
    return evaluation


def enable_method(method, train: bool = False, **kw):
    """``enable(method.model, **kw)`` and ``method.optimize_embedding`` rebound (instance attribute) to
    ``optimize_embedding`` above, so that callers such as the evaluation loop reach the fused path unchanged.  With
    ``train``, ``method.train_iteration`` is rebound (instance attribute) to ``fused_train.train_iteration``: its loss
    always runs as the fused op, while the backbone, ``msssim``, the uncertainty head and densification (``densify``)
    follow their own flags."""
    enable(method.model, **kw)
    method.optimize_embedding = types.MethodType(optimize_embedding, method)
    if train:
        import fused_train
        method.train_iteration = types.MethodType(fused_train.train_iteration, method)
    return method


def disable_method(method):
    method.__dict__.pop("optimize_embedding", None)
    method.__dict__.pop("train_iteration", None)
    disable(method.model)
    return method
