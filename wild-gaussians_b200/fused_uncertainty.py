"""Fused head and ``dino``-mode loss of wild-gaussians' uncertainty model: host side of ``csrc/uncertainty.cu``.

``compute_losses(model, gt, prediction, prefix, _cache_entry)`` is a drop-in for ``UncertaintyModel._compute_losses``
(wildgaussians/method.py:363-433) with ``uncertainty_mode == "dino"``: it returns the same ``(loss, metrics, loss_mult)``.
``loss`` is a 0-d tensor whose gradient reaches ``conv_seg.weight``, ``conv_seg.bias``, ``bn.weight`` and ``bn.bias``;
``metrics`` holds Python floats under the reference's keys, read back from the device at once; ``loss_mult`` is
``[1, 1, H, W]``, detached, clamped at 3.

What stays PyTorch glue, in the reference's order: the normalisation and padding of the images, the dropout2d draw (on a
``[1, C, 1, 1]`` tensor of ones: the reference's ``bernoulli_`` draws on the same noise shape, so the RNG stream stays
aligned with it), the method module's ``ssim_down`` and ``msssim`` (so ``enable(model, msssim=True)`` still applies) and
the backbone's ``get_intermediate_layers`` (so ``enable(model, dino=True)`` still applies).  Everything after the
backbone is six kernels forward and three backward.

Feature cache.  The reference's ``_get_dino_cached`` (method.py:257-265) looks entries up under the shape of the
backbone's input but stores them under the shape of its output, so it never hits.  Here the lookup uses the key the
reference stores under, ``(cache_entry, (1, C, Hp / 14, Wp / 14))``, in the reference's own ``model._images_cache``
with the same CPU fp32 values: entries written by either path are hit by the other.  The backbone is frozen,
deterministic and draws no random numbers, so a hit returns what running it again would.  The full-resolution and the
350-px features cannot collide under one entry: when ``dino_downsample`` resizes, the 350-px image has at most 25
patches on its longer side and the full-resolution one at least 26; when it does not, both are the same image.  Cached
features are copied in with ``non_blocking=True`` from pageable memory.  On a model marked by
``wildgaussians_fused.enable(model, resident_features=True)`` (or ``enable_method(..., resident=True)``) a new entry is
instead a device clone owned by the cache while the cache's device entries fit its byte budget, so a hit copies
nothing; the reference's ``_get_dino_cached`` reads such entries unchanged (``.to(x.device)`` of a device tensor is the
tensor).  ``release_features`` moves them back to host tensors.

``supported(model, gt, prediction)`` tells which calls this covers; ``wildgaussians_fused.enable(model,
uncertainty=True)`` routes the rest to the reference's own method.
"""
from __future__ import annotations

import ctypes
import itertools
import sys

import torch
import torch.nn.functional as F

from diff_gaussian_rasterization import _C

__all__ = ["compute_losses", "compute_losses_on_device", "supported", "release_features"]

_lib = _C._lib
DINO_MAX_SIZE = 350                               # method.py:386-387
METRICS = ("loss", "ssim", "msssim", "ssim_discounted", "mse_discounted", "psnr_discounted", "beta")
# Set on an uncertainty model by enable(..., resident_features=True): [budget in bytes of the feature cache's device
# entries], None until the first store, which takes half of the device memory then free.
RESIDENT_MARK = "_fused_resident_features"


def _distributed_bn(bn) -> bool:
    """True when SyncBatchNorm would synchronise its statistics across processes."""
    dist = torch.distributed
    if not (dist.is_available() and dist.is_initialized()):
        return False
    group = bn.process_group if getattr(bn, "process_group", None) is not None else dist.group.WORLD
    return dist.get_world_size(group) > 1


def _unsupported_model(model) -> str | None:
    cfg = model.config
    if cfg.uncertainty_mode != "dino":
        return "covers uncertainty_mode 'dino' only"
    if cfg.uncertainty_dino_max_size is not None:
        return "covers uncertainty_dino_max_size None only"
    if not model.training:
        return "covers training mode only"
    bn = model.bn
    if not (bn.training and bn.track_running_stats and bn.affine and bn.momentum is not None
            and bn.running_mean is not None and bn.num_batches_tracked is not None):
        return "needs a BatchNorm in training mode with affine parameters and running statistics"
    if _distributed_bn(bn):
        return "does not synchronise BatchNorm statistics across processes"
    return None


def _unsupported(model, gt, prediction) -> str | None:
    why = _unsupported_model(model)
    if why is None:
        why = _unsupported_inputs(model, gt, prediction)
    if why is not None:
        return why
    p = int(model.patch_size)
    H, W = gt.shape[2:]
    if -(-H // p) * -(-W // p) < 2:
        return "needs more than one token (the reference's BatchNorm raises)"
    if max(H, W) >= 2 ** 15:
        return "image too large"
    return None


def _unsupported_inputs(model, gt, prediction) -> str | None:
    """What the kernels need of the images and the head's parameters: fp32 [1, 3, H, W] images on one CUDA device, a
    1 x 1 ``conv_seg`` with at most 2048 input channels, contiguous fp32 parameters and statistics beside the images."""
    bn, conv = model.bn, model.conv_seg
    if not (isinstance(gt, torch.Tensor) and isinstance(prediction, torch.Tensor)):
        return "expects tensors"
    if gt.dim() != 4 or gt.shape != prediction.shape or gt.shape[0] != 1 or gt.shape[1] != 3:
        return "expects two [1, 3, H, W] images"
    if gt.dtype != torch.float32 or prediction.dtype != torch.float32:
        return "supports fp32 only"
    if not (gt.is_cuda and prediction.is_cuda) or gt.device != prediction.device:
        return "needs both images on one CUDA device"
    C = int(model.backbone.embed_dim)
    if not (1 <= C <= 2048 and conv.weight.shape == (1, C, 1, 1) and conv.bias is not None):
        return "expects a 1 x 1 conv_seg with C <= 2048 input channels"
    prm = (conv.weight, conv.bias, bn.weight, bn.bias, bn.running_mean, bn.running_var)
    if any(p.dtype != torch.float32 or p.device != gt.device or not p.is_contiguous() for p in prm):
        return "expects contiguous fp32 head parameters on the images' device"
    if bn.num_batches_tracked.dtype != torch.int64:
        return "expects an int64 num_batches_tracked"
    return None


def supported(model, gt, prediction) -> bool:
    """True when ``compute_losses`` covers this call of ``model._compute_losses(gt, prediction)``."""
    return _unsupported(model, gt, prediction) is None


def _pads(model, x):
    """``[left, right, top, bottom]`` as method.py:282 / :304 computes them."""
    return list(itertools.chain.from_iterable(model._get_pad(m) for m in x.shape[:1:-1]))


def _normalised_padded(model, x):
    x = (x - model.img_norm_mean[None, :, None, None]) / model.img_norm_std[None, :, None, None]
    pads = _pads(model, x)
    return F.pad(x, pads), pads


def _features(model, x, cache_entry):
    """The backbone's features of the normalised, padded image ``x``, through ``model._images_cache``."""
    C, p = int(model.backbone.embed_dim), int(model.patch_size)
    key = (cache_entry, torch.Size((x.shape[0], C, x.shape[2] // p, x.shape[3] // p)))
    if cache_entry is not None:
        hit = model._images_cache.get(key)
        if hit is not None:
            return hit.to(x.device, non_blocking=True)
    with torch.no_grad():
        f = model.backbone.get_intermediate_layers(x, n=[model.backbone.num_heads - 1], reshape=True)[-1]
    if cache_entry is not None:
        model._images_cache[(cache_entry, f.shape)] = _cached(model, f)
    return f


def _cached(model, f):
    """What the cache stores for the features ``f``: a device clone within a marked model's budget, else a host copy."""
    mark = model.__dict__.get(RESIDENT_MARK)
    if mark is not None and f.is_cuda:
        if mark[0] is None:
            mark[0] = torch.cuda.mem_get_info(f.device)[0] // 2
        used = sum(v.nbytes for v in model._images_cache.values() if isinstance(v, torch.Tensor) and v.is_cuda)
        if used + f.nbytes <= mark[0]:
            return f.detach().clone(memory_format=torch.contiguous_format)
    return f.detach().cpu()


def release_features(model) -> None:
    """Unmark ``model`` and turn the device entries of its feature cache into the host tensors it would hold unmarked."""
    model.__dict__.pop(RESIDENT_MARK, None)
    cache = getattr(model, "_images_cache", None)
    if cache:
        for k, v in list(cache.items()):
            if isinstance(v, torch.Tensor) and v.is_cuda:
                cache[k] = v.cpu()


class _Loss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, conv_w, conv_b, bn_w, bn_b, args, keep):
        dev = conv_w.device
        loss = torch.empty((), dtype=torch.float32, device=dev)
        metrics = torch.empty((len(METRICS),), dtype=torch.float32, device=dev)
        loss_mult = torch.empty((1, 1, args.H, args.W), dtype=torch.float32, device=dev)
        nbytes = _lib.gsr_uncertainty_scratch_bytes(ctypes.byref(args))
        scratch = torch.empty(((nbytes + 3) // 4,), dtype=torch.float32, device=dev)
        args.loss, args.metrics, args.loss_mult, args.scratch = (loss.data_ptr(), metrics.data_ptr(), loss_mult.data_ptr(),
                                                                 scratch.data_ptr())
        _C._check(_lib.gsr_uncertainty_forward(ctypes.byref(args), torch.cuda.current_stream(dev).cuda_stream),
                  "gsr_uncertainty_forward")
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
        _C._check(_lib.gsr_uncertainty_backward(ctypes.byref(args), torch.cuda.current_stream(dev).cuda_stream),
                  "gsr_uncertainty_backward")
        return (*grads, None, None)


def _pad_pair(size, patch):
    p = -(-size // patch) * patch - size
    return p // 2, p - p // 2


def head_loss(feat, feat_gt_down, feat_pred_down, mask, conv, bn, gt, prediction, ssim, msssim, down_size, patch,
              clip_min, reg_weight):
    """The kernels' part of ``compute_losses``: everything after the backbone and the image statistics.  feat:
    [1, C, th, tw] features of the padded ground truth, feat_*_down: [1, C, ch, cw] of the padded 350-px images of size
    ``down_size``, mask: [C] dropout2d scales, conv / bn: the head's modules (bn's running statistics are updated),
    gt / prediction: [1, 3, H, W], ssim / msssim: [1, H, W].  Returns (loss, metrics [7] on the device, loss_mult)."""
    H, W = int(gt.shape[2]), int(gt.shape[3])
    nh, nw = down_size
    C = int(feat.shape[1])
    a = _C.GsrUncertaintyArgs()
    a.C, a.th, a.tw = C, int(feat.shape[2]), int(feat.shape[3])
    a.Hp, a.Wp, a.H, a.W, a.nh, a.nw = a.th * patch, a.tw * patch, H, W, nh, nw
    a.pad_top, a.pad_left = _pad_pair(H, patch)[0], _pad_pair(W, patch)[0]
    a.ch, a.cw = int(feat_gt_down.shape[2]), int(feat_gt_down.shape[3])
    a.nHp, a.nWp = a.ch * patch, a.cw * patch
    a.npad_top, a.npad_left = _pad_pair(nh, patch)[0], _pad_pair(nw, patch)[0]
    a.clip_min, a.reg_weight = float(clip_min), float(reg_weight)
    a.bn_eps, a.bn_momentum = float(bn.eps), float(bn.momentum)
    tensors = [t.detach().contiguous() for t in (feat, feat_gt_down, feat_pred_down, mask, gt, prediction, ssim, msssim)]
    keep = tensors + [bn.running_mean, bn.running_var, bn.num_batches_tracked]
    a.feat, a.feat_gt_down, a.feat_pred_down, a.mask, a.gt, a.pred, a.ssim, a.msssim = (t.data_ptr() for t in tensors)
    a.conv_w, a.conv_b, a.bn_w, a.bn_b = (t.data_ptr() for t in (conv.weight, conv.bias, bn.weight, bn.bias))
    a.running_mean, a.running_var = bn.running_mean.data_ptr(), bn.running_var.data_ptr()
    a.num_batches_tracked = bn.num_batches_tracked.data_ptr()
    with torch.cuda.device(gt.device):
        return _Loss.apply(conv.weight, conv.bias, bn.weight, bn.bias, a, keep)


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
        raise RuntimeError("fused_uncertainty.compute_losses " + why)
    m = sys.modules[type(model).__module__]
    cfg = model.config
    # method.py:300-309: features of the ground truth, then the dropout draw
    x, _ = _normalised_padded(model, gt)
    feat = _features(model, x, _cache_entry)
    C = int(feat.shape[1])
    mask = F.dropout2d(torch.ones((1, C, 1, 1), dtype=torch.float32, device=gt.device), p=cfg.uncertainty_dropout,
                       training=model.training)
    # method.py:368-369: the image statistics, through the module's (possibly hooked) functions
    _ssim = m.ssim_down(gt, prediction, max_size=400).contiguous()
    _msssim = m.msssim(gt, prediction, max_size=400, min_size=80).contiguous()
    # method.py:386-391 and :267-289: the 350-px images and their features
    gt_down = m.dino_downsample(gt, max_size=DINO_MAX_SIZE)
    pred_down = m.dino_downsample(prediction, max_size=DINO_MAX_SIZE)
    xd, _ = _normalised_padded(model, gt_down)
    yd, _ = _normalised_padded(model, pred_down)
    with torch.no_grad():
        fgd = feat if gt_down is gt else _features(model, xd, _cache_entry)
        fpd = _features(model, yd, None)
    loss, metrics_t, loss_mult = head_loss(feat, fgd, fpd, mask.reshape(C), model.conv_seg, model.bn, gt, prediction, _ssim,
                                           _msssim, (int(gt_down.shape[2]), int(gt_down.shape[3])), int(model.patch_size),
                                           cfg.uncertainty_clip_min, cfg.uncertainty_regularizer_weight)
    return loss, metrics_t, loss_mult
