"""Float64 oracle of the loss block of wild-gaussians' training step (wildgaussians/method.py:1920-1992, without the
uncertainty term), built on ``ssim_oracle``.

The reference's statements in order, autograd-capable: ``scale_grads`` (method.py:120-123) by the mask and, with
``uncertainty_scale_grad``, by ``loss_mult``; ``l1_loss`` with ``reduction='none'``; the SSIM map; the loss of
:1961-1964 with ``loss_mult`` inside both means; the metrics of :1968-1992 (``_reduce_masked`` divides a three-channel
sum by the one-channel mask sum).  ``dtype=torch.float32`` evaluates the same statements in fp32, the reference's own
rounding, which bounds the error inherent to the formulation.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import ssim_oracle

METRICS = ("l1_loss", "ssim", "mse", "psnr", "mask_percentage", "ssim_masked", "mse_masked", "l1_loss_masked")


def scale_grads(values, scale):
    return values * scale + values.detach() * (1 - scale)


def loss_and_grads(toned, raw, gt, lambda_dssim, mask=None, weight=None, grad_scale=None, dtype=torch.float64):
    """(loss, {metric: value}, dL/dtoned, dL/draw) of the loss block evaluated in `dtype`.  mask, weight, grad_scale:
    [1,H,W] or None (weight None: loss_mult = 1 in the loss)."""
    c = lambda t: None if t is None else t.detach().to(dtype).reshape(1, *toned.shape[1:])
    T = toned.detach().to(dtype).requires_grad_(True)
    R = raw.detach().to(dtype).requires_grad_(True)
    G, M, Wt, S = gt.detach().to(dtype), c(mask), c(weight), c(grad_scale)
    with torch.enable_grad():
        image_toned, image = T, R
        if M is not None:
            image, image_toned = scale_grads(image, M), scale_grads(image_toned, M)
        if S is not None:
            image, image_toned = scale_grads(image, S), scale_grads(image_toned, S)
        loss_mult = Wt if Wt is not None else 1.
        Ll1 = F.l1_loss(image_toned, G, reduction="none")
        ssim_value = ssim_oracle.ssim(image, G, size_average=False, dtype=dtype)
        loss = ((1.0 - lambda_dssim) * (Ll1 * loss_mult).mean() + lambda_dssim * ((1.0 - ssim_value) * loss_mult).mean())
        loss.backward()
    with torch.no_grad():
        mse = (image_toned - G).pow(2)
        out = {"l1_loss": Ll1.mean(), "ssim": ssim_value.mean(), "mse": mse.mean(),
               "psnr": 20 * math.log10(1.) - 10 * torch.log10(mse.mean())}
        if M is not None:
            red = lambda t: (t * M).sum() / M.sum()
            out.update(mask_percentage=M.mean(), ssim_masked=red(ssim_value), mse_masked=red(mse), l1_loss_masked=red(Ll1))
    return loss.detach(), {k: float(v) for k, v in out.items()}, T.grad, R.grad
