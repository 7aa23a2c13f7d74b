"""TEST INFRASTRUCTURE -- CPU restatement of ``distCUDA2`` (submodules/simple-knn/spatial.cu:15-26 ->
``SimpleKNN::knn``, simple_knn.cu:185-220): per point the mean of the squared distances to its 3 nearest OTHER points.

The reference's search (Morton sort, 1024-point boxes, simple_knn.cu:147-183) is exact -- a box is skipped only when it
cannot contain a closer point -- so its result is a function of the point set alone: the three smallest values of
``fma(dz, dz, fma(dx, dx, dy * dy))`` (the contraction nvcc applies to ``d.x*d.x + d.y*d.y + d.z*d.z``, simple_knn.cu:134-135,
in the reference build: read off its SASS and pinned by the goldens -- any other nesting changes ~10 % of the last bits),
summed smallest first and divided by 3.0f (:182).  This file evaluates exactly that, by brute force for small P and through
a k-d tree candidate search (scipy) for larger P.  Pinned on the GPU box against the compiled, unmodified reference
(oracle/_ref/libsimpleknn_ref.so, tests/test_knn.py) and here against tests/golden/knn_*.npz made by that library on a GPU.
Only tests / smoke / bench may import it."""
from __future__ import annotations

import numpy as np

f32 = np.float32
FLT_MAX = np.finfo(np.float32).max


def _dist(p, q):
    """fp32 fma(dz, dz, fma(dx, dx, dy * dy)) for p [..., 3], q [..., 3] (float64 holds every product exactly; each
    fused step is one rounding to fp32)."""
    d = (q.astype(f32) - p.astype(f32)).astype(f32).astype(np.float64)
    s = (d[..., 1] * d[..., 1]).astype(f32).astype(np.float64)
    s = (d[..., 0] * d[..., 0] + s).astype(f32).astype(np.float64)
    return (d[..., 2] * d[..., 2] + s).astype(f32)


def _finish(best):
    """best: [P, 3] ascending -> (b0 + b1) + b2 then / 3.0f, fp32 (overflow to inf like the device code when P < 4)."""
    with np.errstate(over="ignore"):
        s = (best[:, 0] + best[:, 1]).astype(f32)
        s = (s + best[:, 2]).astype(f32)
        return (s / f32(3.0)).astype(f32)


def mean_dist2_bruteforce(points):
    pts = np.asarray(points, dtype=f32)
    P = pts.shape[0]
    best = np.full((P, 3), FLT_MAX, dtype=f32)
    for i in range(P):
        d = _dist(pts[i][None, :], pts)
        d[i] = np.inf
        d = d[~np.isnan(d)]
        k = min(3, P - 1, d.size)
        if k > 0:
            best[i, :k] = np.sort(d)[:k]
    return _finish(best)


def mean_dist2(points, candidates=12):
    """k-d tree candidates (float64 metric), exact fp32 distances over them, three smallest."""
    pts = np.asarray(points, dtype=f32)
    P = pts.shape[0]
    if P <= 2000:
        return mean_dist2_bruteforce(pts)
    from scipy.spatial import cKDTree
    k = min(P, candidates)
    _, idx = cKDTree(pts.astype(np.float64)).query(pts.astype(np.float64), k=k)
    d = _dist(pts[:, None, :], pts[idx])                       # [P, k]
    d[idx == np.arange(P)[:, None]] = np.inf                   # the point itself is excluded by identity, duplicates stay
    d.sort(axis=1)
    return _finish(d[:, :3].astype(f32))
