"""Fused uncertainty loss for every ``uncertainty_mode``, in training and evaluation mode, with a capped head input: host
side of ``gsr_uncertainty_mode_*`` in ``csrc/uncertainty.cu``.

``compute_losses(model, gt, prediction, prefix, _cache_entry)`` is a drop-in for ``UncertaintyModel._compute_losses``
(wildgaussians/method.py:339-433) with ``uncertainty_mode`` ``l2reg``, ``l1reg``, ``dino`` or ``dino+mssim``, the model
in training or evaluation mode and any ``uncertainty_dino_max_size``: it returns the same ``(loss, metrics, loss_mult)``.
``loss`` is a 0-d tensor whose gradient reaches ``conv_seg.weight``, ``conv_seg.bias``, ``bn.weight`` and ``bn.bias``
(``optimize_embedding`` calls ``get_loss`` under ``torch.enable_grad()`` in evaluation mode, and the reference's loss
has a graph there too); ``metrics`` holds Python floats under the reference's keys, read back at once; ``loss_mult`` is
``[1, 1, H, W]`` and detached: unclamped for ``l2reg`` / ``l1reg``, clamped at 3 for the ``dino`` modes.

What stays PyTorch glue, in the reference's order: the model's own ``_scale_input`` (the head input, resized under a
cap), the normalisation and padding, the dropout2d draw in training mode only (an evaluation-mode call leaves the RNG
stream untouched, as the reference's does), the method module's (possibly hooked) ``ssim_down``, ``msssim`` and
``dino_downsample``, and the backbone's (possibly hooked) ``get_intermediate_layers``.  ``l2reg`` and ``l1reg`` need no
350-px backbone call: their only features are those of the head input, which the cache serves.

Feature cache: as ``fused_uncertainty._features``, under the key the reference stores under, in its own
``_images_cache``.  Keys cannot collide here either.  A head input that a cap resized and a 350-px image that
``dino_downsample`` resized are both resizes of the same ground truth to sizes that are multiples of the patch: the same
token grid is the same size and so the same image.  An unresized head input is the ground truth, whose longer side has
at least 26 patches whenever the 350-px image (at most 25) is a resize, and which is the 350-px image otherwise.  The
case left, a capped head input beside an unresized 350-px image, only arises for the ``dino`` modes, where the
reference raises and ``supported`` refuses.  When ``prediction`` and ``gt`` view the same memory
(``optimize_embedding``'s ``get_loss(gt, gt)``) the 350-px features are computed once: the backbone is frozen and
deterministic.

``supported(model, gt, prediction)`` tells which calls this covers; ``wildgaussians_fused.enable(model,
uncertainty=True, uncertainty_modes=True)`` routes them here when ``fused_uncertainty`` does not take them.
"""
from __future__ import annotations

import ctypes
import sys

import torch
import torch.nn.functional as F

import fused_uncertainty as fu
from diff_gaussian_rasterization import _C

__all__ = ["compute_losses", "compute_losses_on_device", "supported"]

_lib = _C._lib
DINO_MAX_SIZE = fu.DINO_MAX_SIZE
METRICS = fu.METRICS


def _down_size(H: int, W: int, max_size: int):
    """The size ``dino_downsample`` and ``_scale_input`` resize to (method.py:190-201, :339-350), or (H, W)."""
    s = min(max_size / H, max_size / W)
    if s >= 1:
        return H, W
    return ((int(H * s) + 13) // 14) * 14, ((int(W * s) + 13) // 14) * 14


def head_size(model, H: int, W: int):
    """The size of ``model._scale_input(gt, uncertainty_dino_max_size)`` for an H x W image."""
    cap = model.config.uncertainty_dino_max_size
    return (H, W) if cap is None else _down_size(H, W, cap)


def _unsupported_model(model) -> str | None:
    cfg = model.config
    if cfg.uncertainty_mode not in _C.UNC_MODES:
        return "covers uncertainty_mode l2reg, l1reg, dino and dino+mssim only (the reference raises on others)"
    bn = model.bn
    if bool(model.training) != bool(bn.training):
        return "needs the model and its BatchNorm in the same (training or evaluation) mode"
    if not (bn.track_running_stats and bn.affine and bn.running_mean is not None and bn.num_batches_tracked is not None):
        return "needs a BatchNorm with affine parameters and running statistics"
    if model.training and bn.momentum is None:
        return "needs a BatchNorm with a momentum in training mode"
    if model.training and fu._distributed_bn(bn):
        return "does not synchronise BatchNorm statistics across processes"
    return None


def _unsupported(model, gt, prediction) -> str | None:
    why = _unsupported_model(model)
    if why is None:
        why = fu._unsupported_inputs(model, gt, prediction)
    if why is not None:
        return why
    p = int(model.patch_size)
    H, W = (int(s) for s in gt.shape[2:])
    if max(H, W) >= 2 ** 15:
        return "image too large"
    uh, uw = head_size(model, H, W)
    if model.training and -(-uh // p) * -(-uw // p) < 2:
        return "needs more than one token (the reference's BatchNorm raises)"
    if (model.config.uncertainty_mode in ("dino", "dino+mssim") and
            _down_size(uh, uw, DINO_MAX_SIZE) != _down_size(H, W, DINO_MAX_SIZE)):
        return "the cap gives a 350-px grid other than the image's (the reference raises)"
    return None


def supported(model, gt, prediction) -> bool:
    """True when ``compute_losses`` covers this call of ``model._compute_losses(gt, prediction)``."""
    return _unsupported(model, gt, prediction) is None


class _Loss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, conv_w, conv_b, bn_w, bn_b, args, keep):
        dev = conv_w.device
        loss = torch.empty((), dtype=torch.float32, device=dev)
        metrics = torch.empty((len(METRICS),), dtype=torch.float32, device=dev)
        loss_mult = torch.empty((1, 1, args.H, args.W), dtype=torch.float32, device=dev)
        nbytes = _lib.gsr_uncertainty_mode_scratch_bytes(ctypes.byref(args))
        scratch = torch.empty(((nbytes + 3) // 4,), dtype=torch.float32, device=dev)
        args.loss, args.metrics, args.loss_mult, args.scratch = (loss.data_ptr(), metrics.data_ptr(), loss_mult.data_ptr(),
                                                                 scratch.data_ptr())
        _C._check(_lib.gsr_uncertainty_mode_forward(ctypes.byref(args), torch.cuda.current_stream(dev).cuda_stream),
                  "gsr_uncertainty_mode_forward")
        ctx.args, ctx.keep = args, keep + [scratch, conv_w, conv_b, bn_w, bn_b]
        ctx.mark_non_differentiable(metrics, loss_mult)
        return loss, metrics, loss_mult

    @staticmethod
    def backward(ctx, g_loss, g_metrics, g_loss_mult):
        args = ctx.args
        conv_w, conv_b, bn_w, bn_b = ctx.keep[-4:]
        dev = conv_w.device
        g = g_loss.detach().to(dtype=torch.float32).contiguous()
        grads = [torch.empty_like(t) for t in (conv_w, conv_b, bn_w, bn_b)]
        args.dL_dloss = g.data_ptr()
        args.d_conv_w, args.d_conv_b, args.d_bn_w, args.d_bn_b = (t.data_ptr() for t in grads)
        _C._check(_lib.gsr_uncertainty_mode_backward(ctypes.byref(args), torch.cuda.current_stream(dev).cuda_stream),
                  "gsr_uncertainty_mode_backward")
        return (*grads, None, None)


def head_loss(mode, training, feat, feat_gt_down, feat_pred_down, mask, conv, bn, head_hw, gt, prediction, ssim, msssim,
              msssim_down, patch, clip_min, reg_weight):
    """The kernels' part of ``compute_losses``.  feat: [1, C, th, tw] features of the padded head input of size
    ``head_hw``; feat_*_down: [1, C, ch, cw] features of the padded 350-px images (``dino`` modes, else None);
    mask: [C] dropout2d scales (training mode, else None); gt / prediction: [1, 3, H, W]; ssim / msssim: [1, H, W];
    msssim_down: [1, nh, nw] (``dino+mssim``, else None).  Returns (loss, metrics [7] on the device, loss_mult)."""
    H, W = int(gt.shape[2]), int(gt.shape[3])
    a = _C.GsrUncertaintyModeArgs()
    a.mode, a.training = _C.UNC_MODES[mode], int(bool(training))
    a.C, a.th, a.tw = int(feat.shape[1]), int(feat.shape[2]), int(feat.shape[3])
    a.uh, a.uw = head_hw
    a.Hp, a.Wp, a.H, a.W = a.th * patch, a.tw * patch, H, W
    a.pad_top, a.pad_left = fu._pad_pair(a.uh, patch)[0], fu._pad_pair(a.uw, patch)[0]
    a.clip_min, a.reg_weight = float(clip_min), float(reg_weight)
    a.bn_eps, a.bn_momentum = float(bn.eps), float(bn.momentum if bn.momentum is not None else 0.0)
    tensors = [t.detach().contiguous() for t in (feat, gt, prediction, ssim, msssim)]
    a.feat, a.gt, a.pred, a.ssim, a.msssim = (t.data_ptr() for t in tensors)
    if feat_gt_down is not None:
        nh, nw = _down_size(H, W, DINO_MAX_SIZE)
        a.nh, a.nw = nh, nw
        a.ch, a.cw = int(feat_gt_down.shape[2]), int(feat_gt_down.shape[3])
        a.nHp, a.nWp = a.ch * patch, a.cw * patch
        a.npad_top, a.npad_left = fu._pad_pair(nh, patch)[0], fu._pad_pair(nw, patch)[0]
        down = [t.detach().contiguous() for t in (feat_gt_down, feat_pred_down)]
        a.feat_gt_down, a.feat_pred_down = (t.data_ptr() for t in down)
        tensors += down
    for name, t in (("mask", mask), ("msssim_down", msssim_down)):
        if t is not None:
            t = t.detach().contiguous()
            setattr(a, name, t.data_ptr())
            tensors.append(t)
    keep = tensors + [bn.running_mean, bn.running_var, bn.num_batches_tracked]
    a.conv_w, a.conv_b, a.bn_w, a.bn_b = (t.data_ptr() for t in (conv.weight, conv.bias, bn.weight, bn.bias))
    a.running_mean, a.running_var = bn.running_mean.data_ptr(), bn.running_var.data_ptr()
    a.num_batches_tracked = bn.num_batches_tracked.data_ptr() if training else None
    with torch.cuda.device(gt.device):
        return _Loss.apply(conv.weight, conv.bias, bn.weight, bn.bias, a, keep)


def _same_image(a, b) -> bool:
    """Whether two tensors view the same memory the same way (``get_loss(gt, gt)`` passes two such views)."""
    return (a.data_ptr() == b.data_ptr() and a.shape == b.shape and a.stride() == b.stride() and a.dtype == b.dtype and
            a.device == b.device)


def compute_losses(model, gt, prediction, prefix="", _cache_entry=None):
    """Drop-in for ``UncertaintyModel._compute_losses`` on supported input; raises otherwise."""
    loss, metrics_t, loss_mult = compute_losses_on_device(model, gt, prediction, _cache_entry)
    with torch.cuda.device(gt.device):
        values = metrics_t.tolist()
    metrics = {f"{prefix}{k}": v for k, v in zip(METRICS, values)}
    return loss, metrics, loss_mult


def compute_losses_on_device(model, gt, prediction, _cache_entry=None):
    """``compute_losses`` without its read-back: ``(loss, metrics, loss_mult)`` with ``metrics`` the [7] device tensor of
    the values under ``METRICS``; nothing synchronises with the host.  Raises on unsupported input."""
    why = _unsupported(model, gt, prediction)
    if why is not None:
        raise RuntimeError("fused_uncertainty_modes.compute_losses " + why)
    m = sys.modules[type(model).__module__]
    cfg = model.config
    mode, training = cfg.uncertainty_mode, bool(model.training)
    # method.py:364 and :300-309: the (capped) head input's features, then the dropout draw in training mode
    head_in = model._scale_input(gt, cfg.uncertainty_dino_max_size)
    x, _ = fu._normalised_padded(model, head_in)
    feat = fu._features(model, x, _cache_entry)
    C = int(feat.shape[1])
    mask = None
    if training:
        mask = F.dropout2d(torch.ones((1, C, 1, 1), dtype=torch.float32, device=gt.device), p=cfg.uncertainty_dropout,
                           training=True).reshape(C)
    # method.py:368-369: the image statistics, through the module's (possibly hooked) functions
    _ssim = m.ssim_down(gt, prediction, max_size=400).contiguous()
    _msssim = m.msssim(gt, prediction, max_size=400, min_size=80).contiguous()
    fgd = fpd = msssim_down = None
    if mode in ("dino", "dino+mssim"):
        # method.py:386-391 / :400-405 and :267-289: the 350-px images and their features
        gt_down = m.dino_downsample(gt, max_size=DINO_MAX_SIZE)
        pred_down = m.dino_downsample(prediction, max_size=DINO_MAX_SIZE)
        with torch.no_grad():
            # the same size as the head input is the same image (see the module's docstring)
            same = gt_down.shape == head_in.shape
            fgd = feat if same else fu._features(model, fu._normalised_padded(model, gt_down)[0], _cache_entry)
            fpd = fgd if _same_image(prediction, gt) else fu._features(model, fu._normalised_padded(model, pred_down)[0],
                                                                        None)
        if mode == "dino+mssim":
            msssim_down = m.msssim(gt_down, pred_down, min_size=80).contiguous()       # method.py:407
    return head_loss(mode, training, feat, fgd, fpd, mask, model.conv_seg, model.bn,
                     (int(head_in.shape[2]), int(head_in.shape[3])), gt, prediction, _ssim, _msssim, msssim_down,
                     int(model.patch_size), cfg.uncertainty_clip_min, cfg.uncertainty_regularizer_weight)
