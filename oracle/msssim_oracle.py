"""Float64 oracle of the image-quality statistics in wild-gaussians' uncertainty loss (wildgaussians/method.py:126-187).

A torch restatement of ``_ssim_parts`` (:138-168), ``msssim`` (:171-187) and ``ssim_down`` (:126-135), evaluated in
``dtype`` (float64 by default) on the inputs' device:

* the window is ``ssim_oracle.window_2d`` (the fp32-built window of the photometric SSIM, cast to ``dtype``), and
  ``ssim_down``'s SSIM map is ``ssim_oracle.ssim``;
* per level: five depthwise 11x11 convolutions with zero padding 5, sigma = sqrt(clamp_min(E[x^2] - mu^2, 0)),
  C1 = 0.01^2, C2 = 0.03^2, C3 = C2 / 2, and the luminance, contrast and structure maps of :165-167;
* the area resize of :173-176 / :128-131 (``scale_factor``, so the output size is int(H * s)), the 2x2 average-pooled
  pyramid of :180-183 whose contrast and structure maps are bilinearly upsampled (align_corners=False) to the level-0
  size one by one, their product, the bilinear upsampling back to the input size and the channel mean.

``dtype=torch.float32`` evaluates the same statements in fp32 (the reference's own rounding, the yardstick for the
fused kernels' error).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.ssim_oracle import C1, C2, ssim, window_2d

C3 = C2 / 2


def ssim_parts(x: torch.Tensor, y: torch.Tensor, window_size: int = 11):
    """(luminance, contrast, structure) maps of method.py:138-168, each [B,C,H,W] in x's dtype."""
    C = x.shape[-3]
    w = window_2d(window_size).to(device=x.device, dtype=x.dtype).expand(C, 1, window_size, window_size).contiguous()

    def blur(t):
        return F.conv2d(t, w, padding=window_size // 2, groups=C)

    mu_x, mu_y = blur(x), blur(y)
    mu_xx, mu_yy, mu_xy = mu_x.pow(2), mu_y.pow(2), mu_x * mu_y
    var_x = blur(x * x) - mu_xx
    var_y = blur(y * y) - mu_yy
    cov_xy = blur(x * y) - mu_xy
    sd_x, sd_y = torch.sqrt(var_x.clamp_min(0)), torch.sqrt(var_y.clamp_min(0))
    lum = (2 * mu_xy + C1) / (mu_xx + mu_yy + C1)
    con = (2 * sd_x * sd_y + C2) / (var_x + var_y + C2)
    struct = (cov_xy + C3) / (sd_x * sd_y + C3)
    return lum, con, struct


def resized_size(H: int, W: int, max_size, clamp: bool):
    """Output size of the area resize: int(H * s) with s = max(max_size / H, max_size / W), capped at 1 by msssim."""
    if max_size is None:
        return H, W
    s = max(max_size / H, max_size / W)
    if clamp:
        s = min(1, s)
    return int(H * s), int(W * s)


def msssim(x: torch.Tensor, y: torch.Tensor, max_size=None, min_size: int = 200,
           dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """method.py:171-187 in `dtype`; x, y: [B,3,H,W]; returns [B,H,W] ([B,h,w] at level-0 size when max_size is None)."""
    x, y = x.to(dtype), y.to(dtype)
    H, W = x.shape[-2:]
    if max_size is not None:
        h, w = resized_size(H, W, max_size, clamp=True)
        x, y = F.adaptive_avg_pool2d(x, (h, w)), F.adaptive_avg_pool2d(y, (h, w))
    lum, con, struct = ssim_parts(x, y)
    out = lum * con * struct
    size0 = x.shape[-2:]
    while x.shape[-2] > min_size and x.shape[-1] > min_size:
        x, y = F.avg_pool2d(x, 2), F.avg_pool2d(y, 2)
        _, con, struct = ssim_parts(x, y)
        out = out * F.interpolate(con, size=size0, mode="bilinear", align_corners=False)
        out = out * F.interpolate(struct, size=size0, mode="bilinear", align_corners=False)
    if max_size is not None:
        out = F.interpolate(out, size=(H, W), mode="bilinear", align_corners=False)
    return out.mean(1)


def ssim_down(x: torch.Tensor, y: torch.Tensor, max_size=None, dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """method.py:126-135 in `dtype`; x, y: [B,3,H,W]; returns [B,H,W]."""
    x, y = x.to(dtype), y.to(dtype)
    H, W = x.shape[-2:]
    if max_size is not None:
        h, w = resized_size(H, W, max_size, clamp=False)
        x, y = F.adaptive_avg_pool2d(x, (h, w)), F.adaptive_avg_pool2d(y, (h, w))
    out = ssim(x, y, size_average=False, dtype=dtype).unsqueeze(1)
    if max_size is not None:
        out = F.interpolate(out, size=(H, W), mode="bilinear", align_corners=False)
    return out.squeeze(1)
