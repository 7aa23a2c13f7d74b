"""Float64 oracle of the evaluation metrics of wild-gaussians (``compute_metrics``, wildgaussians/evaluation.py:331-352):
MSE, MAE and the dm_pix SSIM, stated independently in vectorised numpy.

* Inputs as the metric sees them: ``pred`` sliced to the ground truth's channels; uint8 becomes ``v / 255`` rounded to
  fp32, other floats are rounded to fp32; both are clipped to [0, 1] (NaN passes through).
* MSE / MAE: the fp32 terms ``(a - b)^2`` and ``|a - b|``, summed exactly (``math.fsum``) and divided once in fp64.
* SSIM: a separable Gaussian window of 11 taps (sigma 1.5, normalised to sum 1) applied in fp64 without padding to
  a, b and the fp32 products a^2, b^2, ab; per output mu_a mu_b, the local (co)variances, variances floored at 2^-46
  (the square of fp32's machine epsilon), the covariance's magnitude capped at sqrt(var_a var_b), and
  ``(2 mu_a mu_b + C1) (2 cov + C2) / ((mu_a^2 + mu_b^2 + C1) (var_a + var_b + C2))`` with C1 = 0.01^2, C2 = 0.03^2;
  the image's value is the mean over the valid outputs and the channels.

``metrics(pred, gt)`` returns float64 arrays of the batch shape under the keys ``mse``, ``mae`` and ``ssim``.
"""
from __future__ import annotations

import math

import numpy as np

WINDOW = 11
SIGMA = 1.5
C1, C2 = 0.01 ** 2, 0.03 ** 2
VAR_FLOOR = 2.0 ** -46


def gaussian_taps(size: int = WINDOW, sigma: float = SIGMA) -> np.ndarray:
    r = (np.arange(size) - size // 2) / sigma
    g = np.exp(-0.5 * r ** 2)
    return g / g.sum()


def as_unit_f32(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x)
    x = x.astype(np.float32) / np.float32(255) if x.dtype == np.uint8 else x.astype(np.float32)
    return np.clip(x, np.float32(0), np.float32(1))


def _blur(z: np.ndarray, taps: np.ndarray) -> np.ndarray:
    """Valid-mode separable filter of [N, H, W, C] in float64 over W, then H."""
    win = np.lib.stride_tricks.sliding_window_view
    z = win(z.astype(np.float64), len(taps), axis=2) @ taps[::-1]
    return win(z, len(taps), axis=1) @ taps[::-1]


def ssim(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Per-image SSIM of fp32 [N, H, W, C] images already in [0, 1]."""
    t = gaussian_taps()
    mu_a, mu_b = _blur(a, t), _blur(b, t)
    var_a = np.maximum(VAR_FLOOR, _blur(a * a, t) - mu_a * mu_a)
    var_b = np.maximum(VAR_FLOOR, _blur(b * b, t) - mu_b * mu_b)
    cov = _blur(a * b, t) - mu_a * mu_b
    cov = np.sign(cov) * np.minimum(np.sqrt(var_a * var_b), np.abs(cov))
    s = (2 * mu_a * mu_b + C1) * (2 * cov + C2) / ((mu_a * mu_a + mu_b * mu_b + C1) * (var_a + var_b + C2))
    return s.mean(axis=(1, 2, 3))


def _exact_means(terms: np.ndarray) -> np.ndarray:
    flat = terms.reshape(terms.shape[0], -1).astype(np.float64)
    return np.array([math.fsum(row) / row.size for row in flat])


def metrics(pred: np.ndarray, gt: np.ndarray) -> dict:
    pred = np.asarray(pred)[..., :np.shape(gt)[-1]]
    a, b = as_unit_f32(gt), as_unit_f32(pred)
    assert a.shape == b.shape and a.ndim >= 3, (a.shape, b.shape)
    batch = a.shape[:-3]
    a, b = a.reshape(-1, *a.shape[-3:]), b.reshape(-1, *b.shape[-3:])
    d = a - b
    return {"mse": _exact_means(d * d).reshape(batch), "mae": _exact_means(np.abs(d)).reshape(batch),
            "ssim": ssim(a, b).reshape(batch)}
