"""Float64 restatement of the uncertainty loss in every ``uncertainty_mode`` (wildgaussians/method.py:339-433): the
head on the (possibly capped) head input of ``_scale_input``, BatchNorm in training mode (batch statistics, running-
statistics update) or evaluation mode (running statistics, no update), the ``l2reg``, ``l1reg``, ``dino`` and
``dino+mssim`` branches, their gradients with respect to the head's four parameters, and the metrics.

As ``uncertainty_oracle.compute`` (whose padding and ``dino_downsample`` sizes it uses), it takes the dropout2d channel
scales, the backbone's features and the image statistics as inputs, so one draw of each can be compared across
implementations.  Runs on any device; all arithmetic is float64.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle.uncertainty_oracle import METRICS, down_size, pads  # noqa: F401  (METRICS: the order of "metrics")

MODES = ("l2reg", "l1reg", "dino", "dino+mssim")


def head_size(H: int, W: int, max_size=None):
    """The size ``_scale_input`` (method.py:339-350) resizes the head input to, or (H, W)."""
    return (H, W) if max_size is None else down_size(H, W, max_size)


def compute_mode(feat, feat_gt_down, feat_pred_down, mask, conv_w, conv_b, bn_w, bn_b, running_mean, running_var, gt,
                 pred, ssim, msssim, msssim_down=None, *, mode, training=True, head_hw=None, clip_min=0.1, reg_weight=0.5,
                 eps=1e-5, momentum=0.1, dL_dloss=1.0):
    """``uncertainty_oracle.compute`` for every ``uncertainty_mode`` (method.py:371-412), both BatchNorm modes and a
    capped head input.  feat: [1, C, th, tw] features of the padded head input of size ``head_hw`` ((H, W) when None);
    feat_*_down: the 350-px features (``dino`` modes); mask: the dropout2d scales (ignored in evaluation mode, where
    BatchNorm uses the running statistics and leaves them unchanged); msssim_down: [1, nh, nw] (``dino+mssim``).
    Returns ``compute``'s dict; loss_mult is the branch's full-resolution map, unclamped for ``l2reg`` / ``l1reg``."""
    assert mode in MODES, mode
    d = lambda t: t.detach().to(torch.float64)
    H, W = gt.shape[2:]
    uh, uw = head_hw if head_hw is not None else (H, W)
    leaves = {k: d(v).clone().requires_grad_(True) for k, v in
              (("conv_w", conv_w), ("conv_b", conv_b), ("bn_w", bn_w), ("bn_b", bn_b))}
    rm, rv = d(running_mean).clone(), d(running_var).clone()
    C = feat.shape[1]
    with torch.enable_grad():
        x = d(feat) * d(mask).reshape(1, C, 1, 1) if training else d(feat)
        x = F.batch_norm(x, rm, rv, leaves["bn_w"], leaves["bn_b"], training, momentum, eps)
        logits = torch.einsum("nchw,c->nhw", x, leaves["conv_w"].reshape(C)).unsqueeze(1) + leaves["conv_b"].reshape(1, 1, 1, 1)
        logits = F.softplus(logits + math.log(math.exp(1) - 1))
        p = pads(uh, uw)
        u = F.interpolate(logits, size=(uh + p[2] + p[3], uw + p[0] + p[1]), mode="bilinear", align_corners=False)
        u = u.clamp(min=clip_min)[:, :, p[2]:uh + p[2], p[0]:uw + p[0]]
        beta = torch.log(u).mean()
        resize = (lambda t: F.interpolate(t, size=(H, W), mode="bilinear", align_corners=False)) if (uh, uw) != (H, W) \
            else (lambda t: t)
        if mode in ("l2reg", "l1reg"):
            uf = resize(u)
            loss_mult = 1 / (2 * uf.pow(2)) if mode == "l2reg" else 1 / uf
            loss = ((1 - d(msssim).unsqueeze(1)) * loss_mult).mean() + reg_weight * beta
        else:
            lm = 1 / (2 * u.pow(2))
            nh, nw = down_size(H, W)
            assert down_size(uh, uw) == (nh, nw), "the reference's broadcast raises"
            lm_down = F.interpolate(lm, size=(nh, nw), mode="bilinear") if (nh, nw) != (uh, uw) else lm
            cos = F.cosine_similarity(d(feat_gt_down), d(feat_pred_down), dim=1).unsqueeze(1)
            q = pads(nh, nw)
            cos = F.interpolate(cos, size=(nh + q[2] + q[3], nw + q[0] + q[1]), mode="bilinear", align_corners=False)
            cos = cos[:, :, q[2]:nh + q[2], q[0]:nw + q[0]]
            part = (1 - cos.sub(0.5).div(0.5)).clip(0.0, 1)
            if mode == "dino+mssim":
                part = torch.min(part, 1 - d(msssim_down).unsqueeze(1))
            loss = (part * lm_down).mean() + reg_weight * beta
            loss_mult = resize(lm).clamp_max(3)
        loss.backward(torch.as_tensor(dL_dloss, dtype=torch.float64, device=loss.device))
    loss_mult = loss_mult.detach()
    s, ms = d(ssim).unsqueeze(1), d(msssim).unsqueeze(1)
    ssim_disc = (s * loss_mult).sum() / loss_mult.sum()
    mse_disc = ((d(gt) - d(pred)).pow(2) * loss_mult).sum() / loss_mult.sum()
    loss, beta = loss.detach(), beta.detach()
    metrics = [float(loss), float(s.mean()), float(ms.mean()), float(ssim_disc), float(mse_disc),
               float(10 * torch.log10(1 / mse_disc)), float(beta)]
    return dict(loss=float(loss), metrics=metrics, loss_mult=loss_mult,
                grads={k: v.grad.detach() for k, v in leaves.items()}, running_mean=rm, running_var=rv)
