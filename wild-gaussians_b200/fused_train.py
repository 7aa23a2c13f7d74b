"""Fused training iteration of wild-gaussians: ``WildGaussians.train_iteration`` (wildgaussians/method.py:1880-2024) with
the loss block as kernels (``csrc/train_loss.cu``), training images staged as bytes, and one metric read-back per step.

``train_iteration(method, step)`` runs the reference's statements in the reference's order -- the ``step`` bookkeeping,
the learning-rate update, the SH-degree increase, the ``_viewpoint_stack`` / ``randint`` camera draw, the render
(``model._render_internal``, the fused caller when enabled), the uncertainty warm-up / centring / scale-grad logic, the
protected-iteration detach, the densification block on the model's own methods, ``optimizer.step()`` and
``zero_grad(set_to_none=True)`` -- and returns the same metric keys as Python floats.  What differs:

* Ground truth.  At the first call, each training image and mask of ``method.train_images`` / ``train_masks`` is
  checked once: when ``round(x * 255) / 255`` reproduces every fp32 value bit for bit, it is kept as uint8 HWC bytes
  (a quarter of the fp32 list's host memory per byte-staged image; the lists themselves are not touched), otherwise it
  is copied from the reference's fp32 tensor at each use.  Per step, the chosen camera's data is copied into one of two
  pinned slots and sent to the device on a side stream while the render's composites run; the compute stream waits for
  it just before the first use and unpacks bytes with ``x / 255.0f`` (the bits of the reference's ``astype(float32) / 255.0``).
  No copy from pageable memory, so no copy synchronises the stream.  The one-time check makes about seven passes
  over each image with one fp32 and one bool temporary of its size (measured: about 29 ms per 1920x1080 image, so
  about 50 s for a 1,700-image scene).  The slot is filled once the render's kernels are queued, so the host's copy
  (about 1.5 ms at 1920x1080) overlaps the composites instead of preceding the render's first launch; at 1920x1080
  the copy outlasts the composites, so its tail is still exposed.
* Dispatch.  ``supported`` checks every image and mask once per (image list, mask list) and then only the lists'
  identity and length, so a step's host work does not grow with the number of training images.
* Loss.  ``train_loss`` below: scale_grads by the mask and ``loss_mult``, L1, the weighted means and every metric sum in
  three launches forward (one is the fused SSIM) and two backward, no float atomics.
* Uncertainty.  With ``enable(model, uncertainty=True)`` the fused loss's metrics stay on the device
  (``fused_uncertainty.compute_losses_on_device``); otherwise ``get_loss`` runs as the reference calls it.
* Densification statistics: one kernel (``wildgaussians_fused.densification_stats``).
* Metrics: one device vector, copied into pinned memory and read after one event synchronisation at the end of the step.

Host synchronisations per ordinary step: that metric read-back, plus the rasterizer's instance-count read-back inside
the render (which sizes its binning buffers; unchanged here).  Steps that densify, reset the opacity, raise the SH
degree or recompute the 3D filter keep the reference's own synchronisations there.

``supported(method)`` tells which methods this covers; ``wildgaussians_fused.enable_method(method, train=True)`` binds
it and falls back to the class's own ``train_iteration`` for the rest.
"""
from __future__ import annotations

import ctypes
import math
import sys
import weakref

import numpy as np
import torch

from diff_gaussian_rasterization import _C

__all__ = ["train_iteration", "supported", "train_loss", "as_bytes", "METRICS"]

_lib = _C._lib
# the loss op's metric vector (csrc/train_loss.cu), then the step's total loss
METRICS = ("l1_loss", "ssim", "mse", "psnr", "mask_percentage", "ssim_masked", "mse_masked", "l1_loss_masked")
_stagers: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()
_image_checks: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()


# ---- loss op ---------------------------------------------------------------------------------------------------------

def _plane(t, H, W):
    return None if t is None else t.detach().reshape(H, W).to(torch.float32).contiguous()


class _TrainLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, toned, raw, gt, mask, weight, grad_scale, c_l1, c_ssim):
        H, W = int(toned.shape[1]), int(toned.shape[2])
        dev = toned.device
        t, r, g = (x.detach().contiguous() for x in (toned, raw, gt))
        m, w, s = (_plane(x, H, W) for x in (mask, weight, grad_scale))
        want_grad = bool(ctx.needs_input_grad[0] or ctx.needs_input_grad[1])
        f32 = dict(dtype=torch.float32, device=dev)
        raw_scaled = torch.empty_like(r) if (m is not None or s is not None) else None
        ssim_map = torch.empty((H, W), **f32)
        partials = torch.empty((9, H, W), **f32) if want_grad else None
        loss = torch.empty((), **f32)
        metrics = torch.empty((len(METRICS),), **f32)
        scratch = torch.empty(((_lib.gsr_train_loss_scratch_bytes() + 15) // 16 * 4,), **f32)
        a = _C.GsrTrainLossArgs()
        a.H, a.W, a.c_l1, a.c_ssim = H, W, c_l1, c_ssim
        ptr = lambda x: None if x is None else x.data_ptr()
        a.toned, a.raw, a.gt, a.mask, a.weight, a.grad_scale = (ptr(x) for x in (t, r, g, m, w, s))
        a.raw_scaled, a.ssim_map, a.ssim_partials = ptr(raw_scaled), ssim_map.data_ptr(), ptr(partials)
        a.loss, a.metrics, a.scratch = loss.data_ptr(), metrics.data_ptr(), scratch.data_ptr()
        with torch.cuda.device(dev):
            _C._check(_lib.gsr_train_loss_forward(ctypes.byref(a), torch.cuda.current_stream(dev).cuda_stream),
                      "gsr_train_loss_forward")
        ctx.args = a
        ctx.keep = (t, r, g, m, w, s, raw_scaled, ssim_map, partials) if want_grad else None
        ctx.mark_non_differentiable(metrics)
        return loss, metrics

    @staticmethod
    def backward(ctx, g_loss, g_metrics):
        a = ctx.args
        t = ctx.keep[0]
        dev = t.device
        g = g_loss.detach().to(dtype=torch.float32).contiguous()
        d_toned, d_raw = torch.empty_like(t), torch.empty_like(t)
        dmap = torch.empty(t.shape[1:], dtype=torch.float32, device=dev)
        a.dL_dloss, a.dL_dmap, a.d_toned, a.d_raw = g.data_ptr(), dmap.data_ptr(), d_toned.data_ptr(), d_raw.data_ptr()
        with torch.cuda.device(dev):
            _C._check(_lib.gsr_train_loss_backward(ctypes.byref(a), torch.cuda.current_stream(dev).cuda_stream),
                      "gsr_train_loss_backward")
        return d_toned, d_raw, None, None, None, None, None, None


def train_loss(toned, raw, gt, lambda_dssim, mask=None, weight=None, grad_scale=None):
    """The loss block of method.py:1920-1992 without the uncertainty term.  toned, raw, gt: [3,H,W] fp32 CUDA tensors;
    mask (``scale_grads`` of both images and the masked metrics), weight (``loss_mult`` inside the two means) and
    grad_scale (``scale_grads`` by ``loss_mult``, ``uncertainty_scale_grad``): [1,H,W] / [H,W] or None.
    Returns ``(loss, metrics)``: a 0-d tensor whose gradient reaches ``toned`` and ``raw``, and the [8] device tensor of
    the values under ``METRICS`` (the masked ones are zero without a mask)."""
    if not all(isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 for x in (toned, raw, gt)):
        raise RuntimeError("fused_train.train_loss expects fp32 CUDA tensors")
    if toned.dim() != 3 or toned.shape[0] != 3 or toned.shape != raw.shape or toned.shape != gt.shape:
        raise RuntimeError(f"fused_train.train_loss expects three [3,H,W] images, got {tuple(toned.shape)}, "
                           f"{tuple(raw.shape)} and {tuple(gt.shape)}")
    H, W = int(toned.shape[1]), int(toned.shape[2])
    for name, x in (("mask", mask), ("weight", weight), ("grad_scale", grad_scale)):
        if x is not None and not (isinstance(x, torch.Tensor) and x.numel() == H * W and x.device == toned.device):
            raise RuntimeError(f"fused_train.train_loss expects {name} with H*W elements on the images' device")
    lam = float(lambda_dssim)
    return _TrainLoss.apply(toned, raw, gt, mask, weight, grad_scale, 1.0 - lam, lam)


# ---- image staging ---------------------------------------------------------------------------------------------------

def as_bytes(x: np.ndarray):
    """uint8 values u with ``u.astype(float32) / 255`` equal to the fp32 array ``x`` bit for bit, or None.  Temporary
    memory: one fp32 array and one bool array of x's size."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    t = np.multiply(x, np.float32(255))
    with np.errstate(invalid="ignore"):
        np.rint(t, out=t)
        np.clip(t, 0, 255, out=t)
        u8 = t.astype(np.uint8)
    np.divide(u8, np.float32(255), out=t, dtype=np.float32)
    return u8 if np.array_equal(t.view(np.uint32), x.view(np.uint32)) else None


def _align(n: int) -> int:
    return (n + 255) // 256 * 256


class _Entry:
    """One training image (and mask): the bytes to send, or the reference's fp32 tensor when bytes would not be exact."""

    def __init__(self, image, mask):
        self.H, self.W = int(image.shape[1]), int(image.shape[2])
        self.img_u8 = as_bytes(image.permute(1, 2, 0).numpy())           # [H,W,3]; the lists hold HWC memory
        self.img_f32 = image if self.img_u8 is None else None
        self.img_bytes = _align(self.H * self.W * (3 if self.img_u8 is not None else 12))
        self.mask_u8 = self.mask_f32 = None
        self.mask_binary = True
        self.mask_bytes = 0
        if mask is not None:
            mv = mask.reshape(self.H, self.W).numpy()
            self.mask_u8 = as_bytes(mv)
            self.mask_f32 = mask if self.mask_u8 is None else None
            self.mask_bytes = _align(self.H * self.W * (1 if self.mask_u8 is not None else 4))
            self.mask_binary = bool(np.all((mv == 0) | (mv == 1)))


class _Stager:
    """Two pinned host slots and two device slots; a side stream carries the host-to-device copies."""

    def __init__(self, images, masks, device):
        self.images, self.masks = images, masks
        self.entries = [_Entry(img, None if masks is None else masks[i]) for i, img in enumerate(images)]
        cap = max((e.img_bytes + e.mask_bytes for e in self.entries), default=256)
        self.device = device
        self.host = [torch.empty((cap,), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        self.dev = [torch.empty((cap,), dtype=torch.uint8, device=device) for _ in range(2)]
        self.copied = [None, None]       # H2D of the slot done (side stream)
        self.consumed = [None, None]     # the compute stream is done reading the device slot
        self.stream = torch.cuda.Stream(device)
        self.turn = 0
        self.metrics_host = torch.empty((64,), dtype=torch.float32, pin_memory=True)

    def upload(self, cid: int):
        e = self.entries[cid]
        k, self.turn = self.turn, self.turn ^ 1
        ev = self.copied[k]
        if ev is not None and not ev.query():      # the slot's previous transfer (normally long done)
            ev.synchronize()
        host = self.host[k]
        n_img = e.H * e.W * 3
        if e.img_u8 is not None:
            np.copyto(host[:n_img].numpy().reshape(e.H, e.W, 3), e.img_u8)
        else:
            host[:4 * n_img].view(torch.float32).view(3, e.H, e.W).copy_(e.img_f32)
        if e.mask_u8 is not None:
            np.copyto(host[e.img_bytes:e.img_bytes + e.H * e.W].numpy().reshape(e.H, e.W), e.mask_u8)
        elif e.mask_f32 is not None:
            host[e.img_bytes:e.img_bytes + 4 * e.H * e.W].view(torch.float32).view(1, e.H, e.W).copy_(e.mask_f32)
        total = e.img_bytes + e.mask_bytes
        if self.consumed[k] is not None:
            self.stream.wait_event(self.consumed[k])
        with torch.cuda.stream(self.stream):
            self.dev[k][:total].copy_(host[:total], non_blocking=True)
            self.copied[k] = torch.cuda.Event()
            self.copied[k].record(self.stream)
        return k, e

    def receive(self, pending):
        """(gt [3,H,W], mask [1,H,W] or None, mask is 0/1) on the current stream, which waits for the upload."""
        k, e = pending
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(self.copied[k])
        f32 = dict(dtype=torch.float32, device=self.device)
        d = self.dev[k]
        gt = torch.empty((3, e.H, e.W), **f32)
        mask = torch.empty((1, e.H, e.W), **f32) if e.mask_bytes else None
        img_src = d[:e.H * e.W * 3].data_ptr() if e.img_u8 is not None else None
        mask_src = d[e.img_bytes:].data_ptr() if e.mask_u8 is not None else None
        if img_src is not None or mask_src is not None:
            _C._check(_lib.gsr_unpack_u8(e.H, e.W, img_src, mask_src, gt.data_ptr(),
                                         None if mask is None else mask.data_ptr(), cur.cuda_stream), "gsr_unpack_u8")
        if e.img_f32 is not None:
            gt.copy_(d[:12 * e.H * e.W].view(torch.float32).view(3, e.H, e.W))
        if e.mask_f32 is not None:
            mask.copy_(d[e.img_bytes:e.img_bytes + 4 * e.H * e.W].view(torch.float32).view(1, e.H, e.W))
        self.consumed[k] = torch.cuda.Event()
        self.consumed[k].record(cur)
        return gt, mask, e.mask_binary


def _lists_key(method):
    """The identity and length of the method's image and mask lists: what the per-method caches below are valid for."""
    images, masks = method.train_images, method.train_masks
    return (id(images), None if images is None else len(images), id(masks), None if masks is None else len(masks))


def _stager(method, device) -> _Stager:
    s = _stagers.get(method)
    key = _lists_key(method)
    if s is None or s.key != key or s.images is not method.train_images or s.device != device:
        s = _stagers[method] = _Stager(method.train_images, method.train_masks, device)
        s.key = key
    return s


# ---- the step --------------------------------------------------------------------------------------------------------

def _unsupported(method) -> str | None:
    import wildgaussians_fused as wf
    model, cfg = method.model, method.config
    if bool(cfg.debug):
        return "debug mode runs the reference"
    xyz = model.xyz
    if not (xyz.is_cuda and xyz.dtype == torch.float32):
        return "needs fp32 CUDA parameters"
    if not (wf._supported(model, cfg) or wf._supported_sh(model, cfg)):
        return "covers the configurations the fused render covers"
    um = getattr(model, "uncertainty_model", None)
    if um is not None and (um.config.uncertainty_mode != "dino" or um.config.uncertainty_dino_max_size is not None):
        return "covers uncertainty mode 'dino' (uncertainty_dino_max_size None) or no uncertainty"
    return _images_unsupported(method)


def _images_unsupported(method) -> str | None:
    """The check of every training image and mask, made once per (image list, mask list) of the method: a step pays
    only the comparison of the lists' identities and lengths, whatever the size of the dataset."""
    key = _lists_key(method)
    hit = _image_checks.get(method) if _cacheable(method) else None
    if hit is not None and hit[0] == key and hit[1] is method.train_images and hit[2] is method.train_masks:
        return hit[3]
    why = _check_images(method.train_images, method.train_masks)
    if _cacheable(method):
        _image_checks[method] = (key, method.train_images, method.train_masks, why)
    return why


def _cacheable(obj) -> bool:
    """Whether `obj` can key a WeakKeyDictionary (WildGaussians can)."""
    try:
        weakref.ref(obj)
        hash(obj)
        return True
    except TypeError:
        return False


def _check_images(images, masks) -> str | None:
    if not images or not all(isinstance(x, torch.Tensor) and not x.is_cuda and x.dtype == torch.float32 and x.dim() == 3
                             and x.shape[0] == 3 for x in images):
        return "expects training images as [3,H,W] fp32 CPU tensors"
    if masks is not None and not (len(masks) == len(images) and all(
            isinstance(m, torch.Tensor) and not m.is_cuda and m.dtype == torch.float32 and m.numel() == x.shape[1] * x.shape[2]
            for m, x in zip(masks, images))):
        return "expects masks as [1,H,W] fp32 CPU tensors matching the images"
    return None


def supported(method) -> bool:
    """True when ``train_iteration`` covers this method (see the module docstring)."""
    return _unsupported(method) is None


def _uncertainty_loss(um, gt, toned, camera_id):
    """``get_loss`` (method.py:435-442) with the fused loss's metrics left on the device when ``enable(model,
    uncertainty=True)`` routes this model: (loss, metrics dict, device metrics or None, loss_mult [1,H,W])."""
    import fused_uncertainty as fu
    import wildgaussians_fused as wf
    entry = ("train", camera_id)
    hook = um.__dict__.get("_compute_losses")
    if getattr(hook, "__func__", None) is wf.uncertainty_compute_losses and fu.supported(um, gt[None], toned[None]):
        loss, met, loss_mult = fu.compute_losses_on_device(um, gt.unsqueeze(0), toned.unsqueeze(0), _cache_entry=entry)
        return loss, {}, met, loss_mult.squeeze(0)
    loss, metrics, loss_mult = um.get_loss(gt, toned, _cache_entry=entry)
    return loss, metrics, None, loss_mult


def _uncertainty_metrics(values) -> dict:
    import fused_uncertainty as fu
    d = dict(zip(fu.METRICS, values))
    d["uncertainty_loss"] = d.pop("loss")           # get_loss, method.py:440-441
    d.pop("ssim")
    return d


def train_iteration(method, step):
    """Drop-in for ``WildGaussians.train_iteration`` (see the module docstring); unsupported methods run the class's."""
    if not supported(method):
        return type(method).train_iteration(method, step)
    import wildgaussians_fused as wf
    self = method
    m = sys.modules[type(self).__module__]
    assert self.train_cameras is not None, "Method not initialized"
    assert self.model.optimizer is not None, "Method not initialized"
    assert self.train_cameras.image_sizes is not None, "Image sizes are required for training"

    self.step = step
    iteration = step + 1
    del step
    model, cfg = self.model, self.config

    model.train()
    model.update_learning_rate(iteration)
    device = model.xyz.device
    if iteration % 1000 == 0:
        model.oneupSHdegree()

    if not self._viewpoint_stack:
        self._viewpoint_stack = list(range(len(self.train_cameras)))
    camera_id = self._viewpoint_stack.pop(m.randint(0, len(self._viewpoint_stack) - 1))
    viewpoint_cam = self.train_cameras[camera_id]
    assert viewpoint_cam.image_sizes is not None, "Image sizes are required for training"
    image_width, image_height = viewpoint_cam.image_sizes

    stager = _stager(self, device)
    embedding = model.get_embedding(train_image_id=camera_id)
    render_pkg = model._render_internal(viewpoint_cam, config=cfg, embedding=embedding, kernel_size=cfg.kernel_size)
    image_toned, image, viewspace_point_tensor, radii = (render_pkg["render"], render_pkg["raw_render"],
                                                         render_pkg["viewspace_points"], render_pkg["radii"])
    assert image.shape == (3, image_height, image_width), f"image.shape={image.shape}"
    # the render's kernels are queued: the host fills the pinned slot and the copy travels on a side stream while they
    # run; the compute stream waits for it here, before the first use
    gt_image, mask, mask_binary = stager.receive(stager.upload(camera_id))

    uncertainty_loss = 0
    metrics: dict = {}
    unc_metrics = None
    loss_mult = 1.
    grad_scale = None
    if model.uncertainty_model is not None:
        toned_in = image_toned.detach()
        if mask is not None and not mask_binary:
            with torch.no_grad():                 # the value scale_grads(image_toned, mask) has (method.py:1923)
                toned_in = m.scale_grads(toned_in, mask)
        uncertainty_loss, metrics, unc_metrics, loss_mult = _uncertainty_loss(model.uncertainty_model, gt_image, toned_in,
                                                                              camera_id)
        loss_mult = (loss_mult > 1).to(dtype=loss_mult.dtype)
        if iteration < cfg.uncertainty_warmup_start:
            loss_mult = 1
        elif iteration < cfg.uncertainty_warmup_start + cfg.uncertainty_warmup_iters:
            p = (iteration - cfg.uncertainty_warmup_start) / cfg.uncertainty_warmup_iters
            loss_mult = 1 + p * (loss_mult - 1)
        if cfg.uncertainty_center_mult:
            loss_mult = loss_mult.sub(loss_mult.mean() - 1).clamp(0, 2)
        if cfg.uncertainty_scale_grad:
            grad_scale = loss_mult
            loss_mult = 1
    weight = loss_mult if isinstance(loss_mult, torch.Tensor) else None
    grad_scale = grad_scale if isinstance(grad_scale, torch.Tensor) else None
    assert weight is not None or loss_mult == 1

    last_densify_iter = min(iteration, cfg.densify_until_iter - 1)
    last_dentify_iter = (last_densify_iter // cfg.opacity_reset_interval) * cfg.opacity_reset_interval
    if iteration < last_dentify_iter + cfg.uncertainty_protected_iters:
        try:
            uncertainty_loss = uncertainty_loss.detach()  # type: ignore
        except AttributeError:
            pass

    loss, loss_metrics = train_loss(image_toned, image, gt_image, cfg.lambda_dssim, mask=mask, weight=weight,
                                    grad_scale=grad_scale)
    if isinstance(uncertainty_loss, torch.Tensor):
        loss = loss + uncertainty_loss
    loss.backward()

    with torch.no_grad():
        parts = [loss_metrics, loss.detach().reshape(1)] + ([unc_metrics] if unc_metrics is not None else [])
        vec = torch.cat(parts)
        n = int(vec.numel())
        host = stager.metrics_host[:n]
        host.copy_(vec, non_blocking=True)
        read = torch.cuda.Event()
        read.record(torch.cuda.current_stream(device))
        num_gaussians = len(model.xyz)

        # Densification
        if iteration < cfg.densify_until_iter:
            wf.densification_stats(model, viewspace_point_tensor, radii)
            if iteration > cfg.densify_from_iter and iteration % cfg.densification_interval == 0:
                model.densify_and_prune(
                    cfg.densify_grad_threshold,
                    0.005,
                    self.cameras_extent,
                    enable_size_pruning=iteration > cfg.opacity_reset_interval,
                    skyradius=self._sky_distance)
                model.compute_3D_filter(cameras=self.train_cameras)
            if iteration % cfg.opacity_reset_interval == 0:
                model.reset_opacity()

        if iteration % 100 == 0 and iteration > cfg.densify_until_iter:
            if iteration < cfg.iterations - 100:
                model.compute_3D_filter(cameras=self.train_cameras)

        if iteration < cfg.iterations:
            model.optimizer.step()
            model.optimizer.zero_grad(set_to_none=True)

    read.synchronize()
    values = host.tolist()
    v = dict(zip(METRICS, values))
    if unc_metrics is not None:
        metrics = _uncertainty_metrics(values[len(METRICS) + 1:])
    metrics.update({
        "l1_loss": v["l1_loss"],
        "ssim": v["ssim"],
        "mse": v["mse"],
        "loss": values[len(METRICS)],
        "psnr": v["psnr"],
        "num_gaussians": num_gaussians,
    })
    if mask is not None:
        metrics["mask_percentage"] = v["mask_percentage"]
        metrics["ssim_masked"] = v["ssim_masked"]
        metrics["mse_masked"] = masked_mse = v["mse_masked"]
        metrics["psnr_masked"] = 20 * math.log10(1.) - 10 * math.log10(masked_mse)
        metrics["l1_loss_masked"] = v["l1_loss_masked"]

    self.step = self.step + 1
    model.eval()
    return metrics
