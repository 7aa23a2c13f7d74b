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

``msssim(x, y, max_size=None, min_size=200)`` and ``ssim_down(x, y, max_size=None)`` are the image-quality statistics of
the uncertainty loss (``method.py:126-187``), forward only (``csrc/msssim.cu``): ``[B,3,H,W]`` fp32 CUDA inputs that
want no gradient, ``[B,H,W]`` output, about 10 and 3 launches at 1080p instead of ~260 PyTorch launches and five
blocking host-to-device copies of the window.

There is no PyTorch fallback: unsupported input raises (``supported``, ``supported_msssim`` and ``supported_ssim_down``
tell beforehand).  ``wildgaussians_fused.enable(model, ssim=True)`` routes the reference's own ``ssim`` here where the
input allows it, ``enable(model, msssim=True)`` its ``msssim`` and ``ssim_down``.
"""
from __future__ import annotations

import math

import torch

from diff_gaussian_rasterization import _C

__all__ = ["ssim", "supported", "msssim", "ssim_down", "supported_msssim", "supported_ssim_down"]

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


# ---- msssim / ssim_down of the uncertainty loss (forward only) --------------------------------------------------------

def _is_number(v) -> bool:
    return isinstance(v, (int, float)) and not isinstance(v, bool) and math.isfinite(v)


def _resized(H: int, W: int, max_size, clamp: bool):
    """The (h, w) that ``F.interpolate(x, scale_factor=s, mode='area')`` produces in method.py:126-135 / :171-176."""
    if max_size is None:
        return H, W
    s = max(max_size / H, max_size / W)
    if clamp:
        s = min(1, s)
    return int(H * s), int(W * s)


def _unsupported_stats(x, y, max_size, min_size, clamp) -> str | None:
    if not (isinstance(x, torch.Tensor) and isinstance(y, torch.Tensor)):
        return "expects tensors"
    if not (x.is_cuda and y.is_cuda) or x.device != y.device:
        return "needs both images as CUDA tensors on one device; there is no CPU path"
    if x.dtype != torch.float32 or y.dtype != torch.float32:
        return "supports fp32 images only"
    if x.dim() != 4 or x.shape != y.shape or x.shape[1] != 3:
        return f"expects two [B,3,H,W] images of the same shape, got {tuple(x.shape)} and {tuple(y.shape)}"
    if min(x.shape) == 0:
        return "expects non-empty images"
    if torch.is_grad_enabled() and (x.requires_grad or y.requires_grad):
        return "computes no gradient; neither image may require one"
    if max_size is not None and not _is_number(max_size):
        return "expects max_size None or a number"
    if min_size is not None and not (isinstance(min_size, int) and not isinstance(min_size, bool) and min_size >= 1):
        return "expects an integer min_size >= 1"
    B, _, H, W = x.shape
    h, w = _resized(H, W, max_size, clamp)
    if h < 1 or w < 1:
        return f"resizes {H}x{W} to an empty {h}x{w} image"
    if B > 65535 or (h + 15) // 16 > 65535 or max(H, W, h, w) >= 2 ** 31:
        return "batch or image size too large"
    return None


def supported_msssim(x, y, max_size=None, min_size=200) -> bool:
    """True when ``msssim`` accepts these inputs."""
    return _unsupported_stats(x, y, max_size, min_size, True) is None


def supported_ssim_down(x, y, max_size=None) -> bool:
    """True when ``ssim_down`` accepts these inputs."""
    return _unsupported_stats(x, y, max_size, None, False) is None


def msssim(x, y, max_size=None, min_size=200):
    """Drop-in for ``msssim`` of method.py:171-187 on supported input: the [B,H,W] map (level-0 size when max_size is
    None); raises otherwise."""
    why = _unsupported_stats(x, y, max_size, min_size, True)
    if why is not None:
        raise RuntimeError("fused_ssim.msssim " + why)
    x, y = x.detach().contiguous(), y.detach().contiguous()
    B, _, H, W = x.shape
    h, w = _resized(H, W, max_size, True)
    dev = x.device
    with torch.cuda.device(dev):
        nbytes = _lib.gsr_msssim_scratch_bytes(B, h, w, min_size)
        scratch = torch.empty(((nbytes + 3) // 4,), dtype=torch.float32, device=dev)
        out = torch.empty((B, H, W), dtype=torch.float32, device=dev)
        _C._check(_lib.gsr_msssim_forward(B, H, W, h, w, min_size, x.data_ptr(), y.data_ptr(), out.data_ptr(),
                                          scratch.data_ptr(), _stream(dev)), "gsr_msssim_forward")
    return out


def ssim_down(x, y, max_size=None):
    """Drop-in for ``ssim_down`` of method.py:126-135 on supported input: the [B,H,W] SSIM map of the area-resized
    images, bilinearly upsampled back; raises otherwise."""
    why = _unsupported_stats(x, y, max_size, None, False)
    if why is not None:
        raise RuntimeError("fused_ssim.ssim_down " + why)
    x, y = x.detach().contiguous(), y.detach().contiguous()
    B, _, H, W = x.shape
    h, w = _resized(H, W, max_size, False)
    dev = x.device
    with torch.cuda.device(dev):
        nbytes = _lib.gsr_ssim_down_scratch_bytes(B, h, w) if (h, w) != (H, W) else 0
        scratch = torch.empty(((nbytes + 3) // 4,), dtype=torch.float32, device=dev) if nbytes else None
        out = torch.empty((B, H, W), dtype=torch.float32, device=dev)
        _C._check(_lib.gsr_ssim_down_forward(B, H, W, h, w, x.data_ptr(), y.data_ptr(), out.data_ptr(),
                                             None if scratch is None else scratch.data_ptr(), _stream(dev)),
                  "gsr_ssim_down_forward")
    return out
