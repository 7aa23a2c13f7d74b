"""Golden vectors of wild-gaussians' evaluation metrics, produced by the REFERENCE ITSELF.

Runs where the reference checkout can be read (CPU is enough):
    python tests/golden/make_golden_metrics.py
imports wildgaussians/evaluation.py unmodified and calls its ``compute_metrics(pred, gt, reduce=False)`` with the LPIPS
network replaced by one that returns zeros (a ``_LPIPS_CACHE`` entry; the pretrained weights would need a download).
Each ``metrics_<case>.npz`` holds ``pred``, ``gt``, ``half`` (1: the inputs are the NeRF-W protocol's right-half slices
``x[:, w // 2:]`` of the stored images, which are not contiguous) and the reference's ``psnr``, ``ssim``, ``mae`` and
``mse``.
"""
import os
import sys

import numpy as np
import torch

from make_golden_colors import REF

HERE = os.path.dirname(os.path.abspath(__file__))


class ZeroLPIPS(torch.nn.Module):
    def forward(self, a, b):
        return a.new_zeros((a.shape[0], 1, 1, 1))


def import_evaluation():
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import wildgaussians.evaluation as ev
    ev._LPIPS_CACHE["alex"] = ZeroLPIPS()
    return ev


def textured_u8(rng, shape):
    """A smooth random uint8 image with edges, and a noisy copy of it."""
    y, x = np.meshgrid(np.arange(shape[0]), np.arange(shape[1]), indexing="ij")
    base = 0.5 + 0.3 * np.sin(x[..., None] / 5.0 + np.arange(shape[2])) * np.cos(y[..., None] / 7.0) + 0.2 * ((x // 9) % 2)[..., None]
    gt = np.clip(base * 255 + rng.normal(0, 4, shape), 0, 255).round().astype(np.uint8)
    pred = np.clip(gt.astype(np.float64) + rng.normal(0, 12, shape), 0, 255).round().astype(np.uint8)
    return pred, gt


def cases(rng):
    pred, gt = textured_u8(rng, (40, 74, 3))
    yield "nerfw_half_u8", pred, gt, 1
    g = rng.random((2, 3, 23, 31, 3), dtype=np.float32)
    yield "batch_f32", (g + rng.normal(0, 0.08, g.shape)).astype(np.float32), g, 0
    g = rng.random((1, 19, 27, 3), dtype=np.float32)
    p = np.concatenate([(g + rng.normal(0, 0.05, g.shape)).astype(np.float32), rng.random((1, 19, 27, 1), dtype=np.float32)], -1)
    yield "rgba_pred", p, g, 0
    g = rng.uniform(-0.5, 1.5, (1, 21, 24, 3)).astype(np.float32)
    p = rng.uniform(-0.5, 1.5, (1, 21, 24, 3)).astype(np.float32)
    p[0, 3, 4] = [np.inf, -np.inf, -0.0]
    yield "out_of_range", p, g, 0
    const = np.stack([np.full((16, 18, 3), v, np.uint8) for v in (128, 128, 0, 255)]).reshape(2, 2, 16, 18, 3)
    yield "constant_u8", const[::-1].copy(), const, 0
    pred, gt = textured_u8(rng, (11, 11, 3))
    yield "tiny_11x11", pred, gt, 0
    pred, gt = textured_u8(rng, (37, 13, 3))
    yield "odd_37x13", pred, gt, 0
    pred, gt = textured_u8(rng, (12, 45, 3))
    yield "odd_12x45", pred.astype(np.float32) / 255, gt, 0


def main():
    ev = import_evaluation()
    rng = np.random.default_rng(2024)
    for name, pred, gt, half in cases(rng):
        p, g = (pred[:, pred.shape[1] // 2:], gt[:, gt.shape[1] // 2:]) if half else (pred, gt)
        out = ev.compute_metrics(p, g, reduce=False)
        np.savez_compressed(os.path.join(HERE, f"metrics_{name}.npz"), pred=pred, gt=gt, half=half,
                            **{k: np.asarray(out[k]) for k in ("psnr", "ssim", "mae", "mse")})
        print(name, p.shape, p.dtype, g.dtype, {k: np.asarray(out[k]).ravel()[:2] for k in ("ssim", "mse")})


if __name__ == "__main__":
    main()
