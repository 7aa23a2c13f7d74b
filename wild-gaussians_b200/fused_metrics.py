"""``compute_metrics`` of wildgaussians/evaluation.py:331-352 (PSNR, MSE, MAE, SSIM, LPIPS) on the GPU.

The reference computes the SSIM with one ``np.convolve`` per image row and column in a Python loop, and MSE / MAE as
float32 numpy means; it then copies both images to the device again for LPIPS.  Here one host-to-device copy per image
feeds ``gsr_metrics_forward`` (``csrc/metrics.cu``): two launches give every image's sums of the squared and absolute
differences (fp64 sums of the fp32 terms) and of the dm_pix SSIM map (filtered in fp64), and write the LPIPS inputs
``x * 2 - 1`` of both images on the device.  The reference's own LPIPS network (from, and cached in, the evaluation
module's ``_LPIPS_CACHE``) runs on those tensors through the same ``permute(0, 3, 1, 2)`` view the reference gives it.
The sums and the LPIPS values are copied into pinned memory, after which the call synchronises once.

Results keep the reference's keys, order, shapes and dtypes: psnr, mse, mae and lpips are float32, ssim is float64;
``reduce=True`` returns Python floats through the same ``.mean().item()``.  MSE and MAE are the fp64 means rounded to
float32 once, which is at least as close to the exact mean as the reference's float32 ``np.mean``; PSNR is
``-10 * np.log10`` of that float32 MSE, as the reference computes it.  The SSIM matches the reference's float64 value up
to summation order (about 1e-16).

uint8 and float32 images are staged as they are; other float dtypes go through the reference's ``convert_image_dtype``
first.  Calls the kernel does not cover -- no CUDA device, H or W below the 11-pixel window (where ``np.convolve``
swaps its operands), other dtypes, mismatched shapes -- run the reference's ``compute_metrics`` unchanged;
``supported(pred, gt)`` tells beforehand which path a call takes.
"""
from __future__ import annotations

import ctypes
import importlib
import math

import numpy as np
import torch

WINDOW = 11
MAX_IMAGES_X_CHANNELS = 65535          # gsr_metrics_forward: B * C <= 65535
LAUNCHES = 2                           # kernel launches of one call (the LPIPS network's own are not counted)


def dmpix_taps(kernel_size: int = WINDOW, sigma: float = 1.5) -> np.ndarray:
    """The dm_pix Gaussian window in float64, with the numpy operations (and so the bits) of the reference's filter."""
    hw = kernel_size // 2
    f = ((np.arange(kernel_size) - hw + (2 * hw - kernel_size + 1) / 2) / sigma) ** 2
    filt = np.exp(-0.5 * f)
    return filt / np.sum(filt)


_TAPS = dmpix_taps()
_C1, _C2 = (0.01 * 1.0) ** 2, (0.03 * 1.0) ** 2       # (k1 max_val)^2, (k2 max_val)^2 with dm_pix's defaults


def _evaluation():
    return importlib.import_module("wildgaussians.evaluation")


def _original(evaluation):
    f = evaluation.compute_metrics
    return getattr(f, "__wrapped__", f)


def why_unsupported(pred, gt):
    """None when ``compute_metrics(pred, gt)`` takes the fused path, else the reason it runs the reference."""
    if not (isinstance(pred, np.ndarray) and isinstance(gt, np.ndarray)):
        return "inputs are not numpy arrays"
    if gt.ndim < 3 or pred.ndim != gt.ndim or pred.shape[:-1] + (min(pred.shape[-1], gt.shape[-1]),) != gt.shape:
        return f"shapes {pred.shape} and {gt.shape} do not give [..., H, W, C] pairs"
    for x in (pred, gt):
        if x.dtype != np.uint8 and x.dtype.kind != "f":
            return f"dtype {x.dtype} is neither uint8 nor floating point"
    H, W, C = gt.shape[-3:]
    if H < WINDOW or W < WINDOW:
        return f"image {H}x{W} is smaller than the {WINDOW}-pixel SSIM window"
    B = math.prod(gt.shape[:-3])
    if B < 1 or C < 1 or B * C > MAX_IMAGES_X_CHANNELS:
        return f"{B} images of {C} channels (1 <= B * C <= {MAX_IMAGES_X_CHANNELS})"
    if not torch.cuda.is_available():
        return "no CUDA device"
    return None


def supported(pred, gt) -> bool:
    return why_unsupported(pred, gt) is None


class _Buffers:
    """Per-device pinned staging, device inputs, LPIPS inputs, sums and scratch; grown on demand, reused across calls
    (every call ends in a synchronisation, so no transfer is in flight when the next one refills them)."""

    def __init__(self, device):
        self.device = device
        self.t = {}

    def get(self, name, n, dtype, pinned=False):
        t = self.t.get(name)
        if t is None or t.numel() < n or t.dtype != dtype:
            t = self.t[name] = (torch.empty((n,), dtype=dtype, pin_memory=True) if pinned
                                else torch.empty((n,), dtype=dtype, device=self.device))
        return t[:n]


_buffers: dict = {}


def _stage(k, x, buf):
    """One host-to-device copy of ``x`` (uint8 or float32, any strides) through pinned memory, on the current stream."""
    host = buf.get(f"host{k}", x.nbytes, torch.uint8, pinned=True)
    np.copyto(host.numpy().view(x.dtype).reshape(x.shape), x)
    dev = buf.get(f"dev{k}", x.nbytes, torch.uint8)
    dev.copy_(host, non_blocking=True)
    return dev


def _lpips(evaluation, net, a, b):
    """The reference's ``_lpips`` (evaluation.py:255-291) from its second statement on: the network got or created in the
    module's ``_LPIPS_CACHE``, the module's ``_LPIPS_GPU_AVAILABLE`` probe, ``lp_net.to(device).forward(a, b)`` -- on
    inputs already normalised on the device.  Returns the network's output tensor."""
    lp_net = evaluation._LPIPS_CACHE.get(net)
    if lp_net is None:
        LPIPS = importlib.import_module("._metrics_lpips", evaluation.__package__).LPIPS
        lp_net = LPIPS(net=net, version="0.1")
        evaluation._LPIPS_CACHE[net] = lp_net
    device = torch.device("cpu")
    if evaluation._LPIPS_GPU_AVAILABLE is None:
        evaluation._LPIPS_GPU_AVAILABLE = torch.cuda.is_available()
        if evaluation._LPIPS_GPU_AVAILABLE:
            try:
                lp_net.cuda()
                torch.zeros((1,), device="cuda").cpu()
            except Exception:
                evaluation._LPIPS_GPU_AVAILABLE = False
    if evaluation._LPIPS_GPU_AVAILABLE:
        device = torch.device("cuda")
    with torch.no_grad():
        return lp_net.to(device).forward(a.to(device), b.to(device))


def compute_metrics(pred, gt, *, reduce: bool = True, run_lpips_vgg: bool = False, evaluation=None):
    """Drop-in for the reference's ``compute_metrics`` (same arguments, keys, shapes and dtypes).  ``evaluation``: the
    reference's evaluation module whose LPIPS cache and fallback are used (default ``wildgaussians.evaluation``)."""
    if evaluation is None:
        evaluation = _evaluation()
    if not supported(pred, gt):
        return _original(evaluation)(pred, gt, reduce=reduce, run_lpips_vgg=run_lpips_vgg)
    from diff_gaussian_rasterization import _C

    def reduction(x):
        return x.mean().item() if reduce else x

    pred = pred[..., :gt.shape[-1]]
    pred, gt = (x if x.dtype in (np.uint8, np.float32) else evaluation.convert_image_dtype(x, np.float32) for x in (pred, gt))
    batch = gt.shape[:-3]
    H, W, C = gt.shape[-3:]
    B, N = math.prod(batch), gt.size
    device = torch.device("cuda", torch.cuda.current_device())
    buf = _buffers.get(device)
    if buf is None:
        buf = _buffers[device] = _Buffers(device)
    stream = torch.cuda.current_stream(device)

    a = _stage(0, gt, buf)                     # the reference's ssim(gt, pred), lpips(gt, pred)
    b = _stage(1, pred, buf)
    lp = buf.get("lpips_in", 2 * N, torch.float32).view(2, B, H, W, C)
    sums = buf.get("sums", 3 * B, torch.float64)
    scratch = buf.get("scratch", (_C._lib.gsr_metrics_scratch_bytes(B, H, W, C) + 7) // 8, torch.float64)
    args = _C.GsrMetricsArgs(B=B, H=H, W=W, C=C, a_u8=int(gt.dtype == np.uint8), b_u8=int(pred.dtype == np.uint8),
                             a=a.data_ptr(), b=b.data_ptr(), c1=_C1, c2=_C2, lpips_a=lp[0].data_ptr(),
                             lpips_b=lp[1].data_ptr(), sums=sums.data_ptr(), scratch=scratch.data_ptr())
    args.taps[:] = _TAPS.tolist()
    with torch.cuda.device(device):
        _C._check(_C._lib.gsr_metrics_forward(ctypes.byref(args), stream.cuda_stream), "gsr_metrics_forward")
        nets = ["alex", "vgg"] if run_lpips_vgg else ["alex"]
        lp_out = [_lpips(evaluation, net, lp[0].permute(0, 3, 1, 2), lp[1].permute(0, 3, 1, 2)) for net in nets]
        host_sums = buf.get("host_sums", 3 * B, torch.float64, pinned=True)
        host_lp = buf.get("host_lpips", len(nets) * B, torch.float32, pinned=True).view(len(nets), B)
        host_sums.copy_(sums, non_blocking=True)
        for i, out in enumerate(lp_out):
            host_lp[i].copy_(out.reshape(B), non_blocking=True)
        stream.synchronize()

    s = host_sums.numpy().reshape(B, 3)
    n_ssim = (H - WINDOW + 1) * (W - WINDOW + 1) * C
    # float32 of the fp64 mean; [()] gives the numpy scalar the reference's np.mean returns when there is no batch shape
    mse_ = (s[:, 0] / (H * W * C)).astype(np.float32).reshape(batch)[()]
    mae_ = (s[:, 1] / (H * W * C)).astype(np.float32).reshape(batch)[()]
    out = {
        "psnr": reduction(-10 * np.log10(mse_)),
        "ssim": reduction(np.reshape(s[:, 2] / n_ssim, batch)),
        "mae": reduction(mae_),
        "mse": reduction(mse_),
        "lpips": reduction(host_lp[0].numpy().copy().reshape(batch)),
    }
    if run_lpips_vgg:
        out["lpips_vgg"] = reduction(host_lp[1].numpy().copy().reshape(batch))
    return out
