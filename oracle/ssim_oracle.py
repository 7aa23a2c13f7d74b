"""Float64 oracle of the SSIM in wild-gaussians' photometric loss (wildgaussians/method.py:644-673).

A torch restatement, autograd-capable, so that it is the reference for the map, its mean and dL/dimg1 at any size:

* the window is built in fp32 as method.py:648-652 builds it -- fp32(exp(.)) per tap (:648), normalised by its fp32 sum
  (:649), fp32 outer product (:650) -- and then cast to the compute dtype (:652, ``type_as``);
* five depthwise 11x11 convolutions with zero padding 5 (:654-663), C1 = 0.01^2, C2 = 0.03^2 (:665-666), the SSIM map
  expression of :668, and the reductions of :670-673 (mean over everything, or over the channel dimension).

``dtype=torch.float32`` evaluates the same statements in fp32 (the reference's own rounding, used to bound the error
that is inherent to the formulation on near-flat images).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

C1 = 0.01 ** 2
C2 = 0.03 ** 2


def window_1d(window_size: int = 11, sigma: float = 1.5) -> torch.Tensor:
    """The normalised fp32 1-D Gaussian of method.py:648-649."""
    taps = [math.exp(-(i - window_size // 2) ** 2 / float(2 * sigma ** 2)) for i in range(window_size)]
    g = torch.tensor(taps, dtype=torch.float32)
    return g / g.sum()


def window_2d(window_size: int = 11, sigma: float = 1.5) -> torch.Tensor:
    """The fp32 [window_size, window_size] window of method.py:650."""
    g = window_1d(window_size, sigma)[:, None]
    return g.mm(g.t())


def ssim(img1: torch.Tensor, img2: torch.Tensor, window_size: int = 11, size_average: bool = True,
         dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """method.py:644-673 evaluated in `dtype` (float64 by default) on img1's device; img1 / img2: [C,H,W] or [B,C,H,W]."""
    x, y = img1.to(dtype), img2.to(dtype)
    C = x.shape[-3]
    w = window_2d(window_size).to(device=x.device, dtype=dtype).expand(C, 1, window_size, window_size).contiguous()

    def blur(t):
        return F.conv2d(t, w, padding=window_size // 2, groups=C)

    mu_x, mu_y = blur(x), blur(y)
    mu_xx, mu_yy, mu_xy = mu_x.pow(2), mu_y.pow(2), mu_x * mu_y
    var_x = blur(x * x) - mu_xx
    var_y = blur(y * y) - mu_yy
    cov_xy = blur(x * y) - mu_xy
    smap = ((2 * mu_xy + C1) * (2 * cov_xy + C2)) / ((mu_xx + mu_yy + C1) * (var_x + var_y + C2))
    return smap.mean() if size_average else smap.mean(-3)


def ssim_and_grad(img1, img2, dL_dmap, dtype: torch.dtype = torch.float64):
    """(map, mean, dL/dimg1) for L = sum(map * dL_dmap): the quantities the goldens and the GPU tests compare."""
    x = img1.detach().to(dtype).requires_grad_(True)
    with torch.enable_grad():
        smap = ssim(x, img2.detach(), size_average=False, dtype=dtype)
        (smap * dL_dmap.to(device=smap.device, dtype=dtype)).sum().backward()
    mean = ssim(img1.detach(), img2.detach(), size_average=True, dtype=dtype)
    return smap.detach(), mean.detach(), x.grad
