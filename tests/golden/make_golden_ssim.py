"""Golden vectors of the SSIM in wild-gaussians' photometric loss, produced by the REFERENCE ITSELF.

Runs where the reference checkout can be read (CPU torch is enough):
    python tests/golden/make_golden_ssim.py
imports wildgaussians/method.py unmodified (as make_golden_colors.py does) and evaluates its ``ssim`` (:644-673) in
float64 on the CPU.  The inputs are fp32 values (what the fp32 kernels see); ``img2`` plays the ground truth and is
quantised to 8 bits like a decoded photograph.  Each file holds img1, img2, the map (size_average=False), the mean
(size_average=True), a seeded upstream map ``dL_dmap`` and dL/dimg1 of sum(map * dL_dmap).
"""
import os

import numpy as np
import torch
import torch.nn.functional as F

from make_golden_colors import import_reference


def textured(shape, g):
    """A smooth random image with edges in [0, 1] (blurred noise plus a few steps), and a noisy copy of it."""
    base = torch.rand(shape, generator=g, dtype=torch.float64)
    flat = base.reshape(-1, 1, *shape[-2:])
    smooth = F.avg_pool2d(flat, 3, 1, 1, count_include_pad=False).reshape(shape)
    steps = (torch.arange(shape[-1], dtype=torch.float64) % 13 < 6).to(torch.float64) * 0.3
    img2 = ((smooth * 0.7 + steps) * 255).round().clamp(0, 255) / 255
    img1 = (img2 + 0.05 * torch.randn(shape, generator=g, dtype=torch.float64)).clamp(0, 1)
    return img1, img2


def make_case(m, kind, shape, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "flat":
        img2 = torch.full(shape, 0.5, dtype=torch.float64)
        img1 = img2 + 1e-3 * torch.randn(shape, generator=g, dtype=torch.float64)
    else:
        img1, img2 = textured(shape, g)
    img1, img2 = img1.float(), img2.float()                 # the inputs the fp32 kernels see
    map_shape = shape[:-3] + shape[-2:]
    dL = torch.randn(map_shape, generator=g, dtype=torch.float64).float()
    x = img1.double().requires_grad_(True)
    smap = m.ssim(x, img2.double(), size_average=False)
    (smap * dL.double()).sum().backward()
    mean = m.ssim(img1.double(), img2.double(), size_average=True)
    return dict(img1=img1.numpy(), img2=img2.numpy(), dL_dmap=dL.numpy(), map=smap.detach().numpy(),
                mean=np.float64(mean.item()), grad=x.grad.numpy())


CASES = {
    "ssim_textured": ("textured", (3, 37, 53), 21),
    "ssim_small": ("textured", (3, 7, 5), 22),
    "ssim_batched": ("textured", (2, 3, 24, 40), 23),
    "ssim_flat": ("flat", (3, 32, 48), 24),
}

if __name__ == "__main__":
    m, _ = import_reference()
    here = os.path.dirname(os.path.abspath(__file__))
    for name, (kind, shape, seed) in CASES.items():
        case = make_case(m, kind, shape, seed)
        path = os.path.join(here, name + ".npz")
        np.savez_compressed(path, **case)
        print(name, shape, "mean", float(case["mean"]), f"{os.path.getsize(path) / 1024:.0f} KB")
