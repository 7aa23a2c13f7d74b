"""Float64 restatement of the uncertainty head and the ``dino``-mode loss (wildgaussians/method.py:300-323, :363-433),
their gradients with respect to the head's four parameters, and the BatchNorm running-statistics update.

Unlike the reference, it takes the dropout2d channel scales (``mask``: 0 or 1 / (1 - p) per channel), the backbone's
features and the two image statistics (``ssim_down``, ``msssim``) as inputs, so one draw of each can be compared across
implementations.  Runs on any device; all arithmetic is float64.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

PATCH = 14
METRICS = ("loss", "ssim", "msssim", "ssim_discounted", "mse_discounted", "psnr_discounted", "beta")


def pads(H: int, W: int, patch: int = PATCH):
    """``[left, right, top, bottom]`` zero padding to multiples of the patch size (method.py:231-236, :304)."""
    out = []
    for s in (W, H):
        p = math.ceil(s / patch) * patch - s
        out += [p // 2, p - p // 2]
    return out


def down_size(H: int, W: int, max_size: int = 350):
    """The size ``dino_downsample`` (method.py:190-201) resizes to, or (H, W) when it does not."""
    if max_size < H or max_size < W:
        s = min(max_size / H, max_size / W)
        return ((int(H * s) + 13) // 14) * 14, ((int(W * s) + 13) // 14) * 14
    return H, W


def compute(feat, feat_gt_down, feat_pred_down, mask, conv_w, conv_b, bn_w, bn_b, running_mean, running_var, gt, pred,
            ssim, msssim, *, clip_min=0.1, reg_weight=0.5, eps=1e-5, momentum=0.1, dL_dloss=1.0):
    """feat: [1, C, th, tw] features of the padded ground truth; feat_*_down: [1, C, ch, cw] of the 350-px images;
    gt, pred: [1, 3, H, W]; ssim, msssim: [1, H, W].  Returns a dict: loss, metrics (list of 7 in METRICS order),
    loss_mult [1, 1, H, W], grads {conv_w, conv_b, bn_w, bn_b}, running_mean, running_var."""
    d = lambda t: t.detach().to(torch.float64)
    H, W = gt.shape[2:]
    leaves = {k: d(v).clone().requires_grad_(True) for k, v in
              (("conv_w", conv_w), ("conv_b", conv_b), ("bn_w", bn_w), ("bn_b", bn_b))}
    rm, rv = d(running_mean).clone(), d(running_var).clone()
    C = feat.shape[1]
    with torch.enable_grad():
        x = d(feat) * d(mask).reshape(1, C, 1, 1)
        x = F.batch_norm(x, rm, rv, leaves["bn_w"], leaves["bn_b"], True, momentum, eps)
        logits = torch.einsum("nchw,c->nhw", x, leaves["conv_w"].reshape(C)).unsqueeze(1) + leaves["conv_b"].reshape(1, 1, 1, 1)
        logits = F.softplus(logits + math.log(math.exp(1) - 1))
        p = pads(H, W)
        Hp, Wp = H + p[2] + p[3], W + p[0] + p[1]
        u = F.interpolate(logits, size=(Hp, Wp), mode="bilinear", align_corners=False).clamp(min=clip_min)
        u = u[:, :, p[2]:H + p[2], p[0]:W + p[0]]
        loss_mult = 1 / (2 * u.pow(2))
        nh, nw = down_size(H, W)
        lm_down = F.interpolate(loss_mult, size=(nh, nw), mode="bilinear") if (nh, nw) != (H, W) else loss_mult
        cos = F.cosine_similarity(d(feat_gt_down), d(feat_pred_down), dim=1).unsqueeze(1)
        q = pads(nh, nw)
        cos = F.interpolate(cos, size=(nh + q[2] + q[3], nw + q[0] + q[1]), mode="bilinear", align_corners=False)
        cos = cos[:, :, q[2]:nh + q[2], q[0]:nw + q[0]]
        dino_part = (1 - cos.sub(0.5).div(0.5)).clip(0.0, 1)
        beta = torch.log(u).mean()
        loss = (dino_part * lm_down).mean() + reg_weight * beta
        loss.backward(torch.as_tensor(dL_dloss, dtype=torch.float64, device=loss.device))
    loss_mult = loss_mult.detach().clamp_max(3)
    s, ms = d(ssim).unsqueeze(1), d(msssim).unsqueeze(1)
    ssim_disc = (s * loss_mult).sum() / loss_mult.sum()
    mse_disc = ((d(gt) - d(pred)).pow(2) * loss_mult).sum() / loss_mult.sum()
    loss, beta = loss.detach(), beta.detach()
    metrics = [float(loss), float(s.mean()), float(ms.mean()), float(ssim_disc), float(mse_disc),
               float(10 * torch.log10(1 / mse_disc)), float(beta)]
    return dict(loss=float(loss), metrics=metrics, loss_mult=loss_mult,
                grads={k: v.grad.detach() for k, v in leaves.items()}, running_mean=rm, running_var=rv)
