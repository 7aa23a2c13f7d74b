"""TEST INFRASTRUCTURE -- numpy/ctypes front end of ``oracle/bwd_bound.c``: the fp64 value of every slot of the
backward composite's per-Gaussian accumulator (csrc/render_bwd.cu) and an a-priori bound on how far the kernel's fp32
value can be from it.  The error model is described in the header of bwd_bound.c.  Only tests/ may import this.

``bound(...)`` takes the kernel's own forward artefacts (``records`` [P, 8] = {x, y, hx, hy, A, B, C, o} as
``debug_views`` returns them, colours, ``point_list``, ``ranges``, ``n_contrib``) and the backward's inputs, and returns
``S`` [P, 10], ``B`` [P, 10], ``M`` [P, 10] (magnitude scale), ``und`` [P] (1: a pair of the Gaussian is undetermined,
2: its bound is infinite) and counts.  ``check(acc, res)`` compares a kernel accumulator against it.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from ctypes import c_double, c_int, c_longlong, c_void_p

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

ALPHA_MAX = float(np.float32(0.99))            # the kernel's 0.99f
ALPHA_MIN = float(np.float32(1.0) / np.float32(255.0))   # the kernel's 1.0f / 255.0f
SLOTS = ("dmean2D.x", "dmean2D.y", "|dmean2D|", "dconic.x", "dconic.y", "dconic.w", "dopacity", "dcolor.r",
         "dcolor.g", "dcolor.b")


def lib_path() -> str:
    return os.path.join(_HERE, "_ref", "libbwd_bound.so")


def build() -> None:
    """Compile bwd_bound.c (gcc); cheap, so done on demand."""
    subprocess.run(["make", "-C", _HERE, "all"], check=True, capture_output=True)


def _lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(lib_path()):
            build()
        lib = ctypes.CDLL(lib_path())
        lib.bwd_bound.restype = c_longlong
        _LIB = lib
    return _LIB


def _np(x, dtype):
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(np.asarray(x), dtype=dtype)


def _p(a):
    return a.ctypes.data_as(c_void_p)


def bound(records, colors, point_list, ranges, n_contrib, subpixel_offset, bg, dL_dpix, W, H, tile_rows=(0, 0),
          alpha_max=ALPHA_MAX, alpha_min=ALPHA_MIN, colour_walk=False) -> dict:
    """Exact accumulator and its bound.  Every float input is read as float64 (fp32 values are exact in it).
    ``alpha_max`` / ``alpha_min``: the clamp and the blend threshold (the kernel's fp32 constants by default).
    ``colour_walk``: bound slots 7..9 for the colour-only walk of ``gsr_backward_colors`` (one atomic per warp) instead
    of render_bwd.cu's one flush per tile."""
    rec = _np(records, np.float64).reshape(-1, 8)
    P = rec.shape[0]
    col = _np(colors, np.float64).reshape(P, 3)
    pl = _np(point_list, np.int64).astype(np.uint32)
    rg = _np(ranges, np.int64).astype(np.uint32).reshape(-1, 2)
    nc = _np(n_contrib, np.int64).astype(np.uint32).reshape(H, W)
    so = _np(subpixel_offset, np.float64).reshape(H, W, 2)
    bgv = _np(bg, np.float64).reshape(3)
    dp = _np(dL_dpix, np.float64).reshape(3, H, W)
    if pl.size == 0:
        pl = np.zeros(1, np.uint32)
    S = np.zeros((P, 10)); B = np.zeros((P, 10)); M = np.zeros((P, 10))
    und = np.zeros(P, np.uint8)
    stats = np.zeros(2)
    over = 0
    if P:
        over = _lib().bwd_bound(c_int(P), c_int(W), c_int(H), c_int(tile_rows[0]), c_int(tile_rows[1]), _p(rg), _p(pl),
                                _p(so), _p(bgv), _p(rec), _p(col), _p(nc), _p(dp), c_double(alpha_max),
                                c_double(alpha_min), c_int(6 if colour_walk else 9),
                                c_int(4 if colour_walk else 1), _p(S), _p(B), _p(M), _p(und), _p(stats))
    return dict(S=S, B=B, M=M, und=und, overflow_pixels=int(over), undetermined_pairs=int(stats[0]),
                blended_pairs=int(stats[1]))


def check(acc, res, mask=None) -> dict:
    """Compare a kernel accumulator (``[P, 12]`` or ``[P, 10]``) against ``bound``'s result.

    Returns ``ratio`` (per slot, the worst |acc - S| / B over the rows with a finite, non-zero bound), ``violations``
    (row indices with |acc - S| > B in some slot), ``nonzero_where_zero`` (rows with S = B = 0 in a slot but a non-zero
    entry) and ``padding_nonzero`` (rows whose slots 10, 11 are not zero)."""
    a = np.asarray(acc, np.float64)
    a = a.reshape(a.shape[0], -1)
    S, B = res["S"], res["B"]
    d = np.abs(a[:, :10] - S)
    rows = np.ones(S.shape[0], bool) if mask is None else np.asarray(mask, bool)
    finite = np.isfinite(B)
    bad = (~(d <= B) & finite & rows[:, None]) | (~np.isfinite(a[:, :10]) & rows[:, None])
    zero = (S == 0) & (B == 0)
    nz = zero & (a[:, :10] != 0) & rows[:, None]
    ratio = {}
    for s, name in enumerate(SLOTS):
        m = rows & finite[:, s] & (B[:, s] > 0)
        ratio[name] = float((d[m, s] / B[m, s]).max()) if m.any() else 0.0
    pad = np.zeros(0, np.int64)
    if a.shape[1] >= 12:
        pad = np.nonzero(rows & np.any(a[:, 10:12] != 0, axis=1))[0]
    return dict(ratio=ratio, violations=np.nonzero(bad.any(axis=1))[0], nonzero_where_zero=np.nonzero(nz.any(axis=1))[0],
                padding_nonzero=pad)
