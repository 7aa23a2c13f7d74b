"""Fused SSIM of wild-gaussians' photometric loss: host side of ``csrc/ssim.cu``.

``ssim(img1, img2, window_size=11, size_average=True)`` has the signature, output shapes and reductions of
``wildgaussians/method.py:644-673`` -- an 11-tap Gaussian window (sigma 1.5), zero padding, ``C1 = 0.01^2``,
``C2 = 0.03^2``, the map averaged over the 3 channels -- and runs as ONE kernel per direction instead of 5 depthwise
convolutions forward, 3 backward and ~60 elementwise launches.  The convolutions are plain fp32 (the reference's run in
TF32 under PyTorch's default ``cudnn.allow_tf32``).

* ``img1``, ``img2``: ``[3,H,W]`` or ``[B,3,H,W]`` fp32 CUDA tensors of the same shape; any size, including images
  smaller than the window.
* ``size_average=False`` returns the map, ``[H,W]`` or ``[B,H,W]``; ``True`` returns its mean (a 0-d tensor).
* The gradient flows to ``img1`` only; the backward's per-pixel factors (36 B per pixel) are kept only when ``img1``
  requires a gradient.  Nothing synchronises with the host.

There is no PyTorch fallback: unsupported input raises (``supported`` tells beforehand).
``wildgaussians_fused.enable(model, ssim=True)`` routes the reference's own ``ssim`` here where the input allows it.
"""
from __future__ import annotations

import torch

from diff_gaussian_rasterization import _C

__all__ = ["ssim", "supported"]

_lib = _C._lib


def _unsupported(img1, img2, window_size) -> str | None:
    if not (isinstance(img1, torch.Tensor) and isinstance(img2, torch.Tensor)):
        return "expects tensors"
    if not (img1.is_cuda and img2.is_cuda) or img1.device != img2.device:
        return "needs both images as CUDA tensors on one device; there is no CPU path"
    if img1.dtype != torch.float32 or img2.dtype != torch.float32:
        return "supports fp32 images only"
    if window_size != 11:
        return "supports window_size 11 only"
    if img1.dim() not in (3, 4) or img1.shape != img2.shape or img1.shape[-3] != 3:
        return f"expects two [3,H,W] or [B,3,H,W] images of the same shape, got {tuple(img1.shape)} and {tuple(img2.shape)}"
    if min(img1.shape) == 0:
        return "expects non-empty images"
    if img2.requires_grad:
        return "computes no gradient for img2; img2 must not require one"
    return None


def supported(img1, img2, window_size=11) -> bool:
    """True when ``ssim`` accepts these inputs."""
    return _unsupported(img1, img2, window_size) is None


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


class _FusedSSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img1, img2, want_grad):
        x, y = img1.detach().contiguous(), img2.detach().contiguous()
        B, _, H, W = x.shape
        dev = x.device
        with torch.cuda.device(dev):
            ssim_map = torch.empty((B, H, W), dtype=torch.float32, device=dev)
            partials = torch.empty((B, 9, H, W), dtype=torch.float32, device=dev) if want_grad else None
            _C._check(_lib.gsr_ssim_forward(B, H, W, x.data_ptr(), y.data_ptr(), ssim_map.data_ptr(),
                                            partials.data_ptr() if want_grad else None, _stream(dev)), "gsr_ssim_forward")
        if want_grad:
            ctx.save_for_backward(x, y, partials)
        return ssim_map

    @staticmethod
    def backward(ctx, dL_dmap):
        x, y, partials = ctx.saved_tensors
        B, _, H, W = x.shape
        dev = x.device
        g = dL_dmap.to(dtype=torch.float32).contiguous()
        with torch.cuda.device(dev):
            dL_dimg1 = torch.empty_like(x)
            _C._check(_lib.gsr_ssim_backward(B, H, W, x.data_ptr(), y.data_ptr(), partials.data_ptr(), g.data_ptr(),
                                             dL_dimg1.data_ptr(), _stream(dev)), "gsr_ssim_backward")
        return dL_dimg1, None, None


def ssim(img1, img2, window_size=11, size_average=True):
    """Drop-in for ``ssim`` of method.py:644-673 on supported input (see the module docstring); raises otherwise."""
    why = _unsupported(img1, img2, window_size)
    if why is not None:
        raise RuntimeError("fused_ssim.ssim " + why)
    batched = img1.dim() == 4
    x, y = (img1, img2) if batched else (img1.unsqueeze(0), img2.unsqueeze(0))
    want_grad = bool(img1.requires_grad and torch.is_grad_enabled())
    ssim_map = _FusedSSIM.apply(x, y, want_grad)
    if not batched:
        ssim_map = ssim_map.squeeze(0)
    return ssim_map.mean() if size_average else ssim_map
