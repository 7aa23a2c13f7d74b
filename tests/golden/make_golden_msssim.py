"""Golden vectors of the uncertainty loss's image-quality statistics, produced by the REFERENCE ITSELF.

Runs where the reference checkout can be read (CPU torch is enough):
    python tests/golden/make_golden_msssim.py
imports wildgaussians/method.py unmodified (as make_golden_ssim.py does) and evaluates its ``msssim`` (:171-187) and
``ssim_down`` (:126-135) in float64 on the CPU.  The inputs are fp32 values (what the fp32 kernels see), quantised to
8 bits like decoded photographs so that the files stay small.  The parameters are scaled down from production
(max_size 400, min_size 80 at 1080p) so that small images reach the same branches: an area downsample with three coarse
levels and the final upsample, no resize (the ``dino+mssim`` call), an area upsample in ``ssim_down`` while ``msssim``
clamps its scale to 1, a batch with odd sizes and levels smaller than the window, and a near-flat pair.  Each file
holds img1, img2, max_size (-1 for None), min_size and both outputs ([B,H,W] float64).  The largest case stores the
outputs on every other row and column (``stride``), which keeps each file near 100 KB.
"""
import os

import numpy as np
import torch
import torch.nn.functional as F

from make_golden_colors import import_reference


def textured(shape, g):
    """A smooth random image with edges in [0, 1] (blurred noise plus a few steps), and a noisy copy, both 8-bit."""
    base = torch.rand(shape, generator=g, dtype=torch.float64)
    flat = base.reshape(-1, 1, *shape[-2:])
    smooth = F.avg_pool2d(flat, 3, 1, 1, count_include_pad=False).reshape(shape)
    steps = (torch.arange(shape[-1], dtype=torch.float64) % 13 < 6).to(torch.float64) * 0.3
    img2 = ((smooth * 0.7 + steps) * 255).round().clamp(0, 255) / 255
    img1 = ((img2 + 0.05 * torch.randn(shape, generator=g, dtype=torch.float64)) * 255).round().clamp(0, 255) / 255
    return img1, img2


def make_case(m, kind, shape, seed, max_size, min_size, stride):
    g = torch.Generator().manual_seed(seed)
    if kind == "flat":
        img2 = torch.full(shape, 0.5, dtype=torch.float64)
        img1 = img2 + 1e-3 * torch.randn(shape, generator=g, dtype=torch.float64)
    else:
        img1, img2 = textured(shape, g)
    img1, img2 = img1.float(), img2.float()                 # the inputs the fp32 kernels see
    x, y = img1.double(), img2.double()
    ms = m.msssim(x, y, max_size=max_size, min_size=min_size)
    sd = m.ssim_down(x, y, max_size=max_size)
    return dict(img1=img1.numpy(), img2=img2.numpy(), max_size=np.int64(-1 if max_size is None else max_size),
                min_size=np.int64(min_size), stride=np.int64(stride),
                msssim=ms[:, ::stride, ::stride].numpy(), ssim_down=sd[:, ::stride, ::stride].numpy())


CASES = {
    # name: (kind, shape, seed, max_size, min_size, output stride)
    "msssim_resize": ("textured", (1, 3, 68, 120), 31, 50, 10, 2),
    "msssim_noresize": ("textured", (1, 3, 56, 84), 32, None, 20, 1),
    "msssim_upsample": ("textured", (1, 3, 60, 90), 33, 100, 20, 1),
    "msssim_batched": ("textured", (2, 3, 37, 51), 34, None, 5, 1),
    "msssim_flat": ("flat", (1, 3, 48, 64), 35, 40, 10, 1),
}

if __name__ == "__main__":
    m, _ = import_reference()
    here = os.path.dirname(os.path.abspath(__file__))
    for name, (kind, shape, seed, max_size, min_size, stride) in CASES.items():
        case = make_case(m, kind, shape, seed, max_size, min_size, stride)
        path = os.path.join(here, name + ".npz")
        np.savez_compressed(path, **case)
        print(name, shape, "msssim mean", float(case["msssim"].mean()), f"{os.path.getsize(path) / 1024:.0f} KB")
