"""TEST INFRASTRUCTURE -- numpy/ctypes front end of ``oracle/fwd_bound.c``: the fp64 value of every output of the
training composite (csrc/render_fwd.cu, ``render_fwd_packed_kernel<false, false>``) along the kernel's own fp32
decisions, and an a-priori bound on how far the kernel's fp32 value can be from it.  The error model is described in
the header of fwd_bound.c.  Only tests/ may import this.

``bound(...)`` takes the kernel's own artefacts (``records`` [P, 8] = {x, y, hx, hy, A, B, C, o} as ``debug_views``
returns them, colours, ``point_list``, ``ranges``, the sub-pixel offsets, bg) and returns ``S`` [4, H, W] (colour
channels and final_T), ``B`` [4, H, W], ``nc_nom`` [H, W], ``und`` [H, W] (1: a decision is undetermined, 2: the
bound is infinite), the blend-mask words ``mbits`` / ``msure`` [T, 4, 32], counts and -- for a tested ``n_contrib`` --
``nc_ok`` [H, W].  ``check(...)`` compares kernel outputs against it; ``pair_power(...)`` exposes the oracle's fp32 power.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from ctypes import c_double, c_int, c_longlong, c_void_p

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

ALPHA_MAX = float(np.float32(0.99))                       # the kernel's 0.99f
ALPHA_MIN = float(np.float32(1.0) / np.float32(255.0))    # the kernel's 1.0f / 255.0f
T_MIN = float(np.float32(0.0001))                         # the kernel's 0.0001f
MASK_K = 1024
MASK_WORDS = MASK_K // 32
CHANNELS = ("r", "g", "b", "final_T")


def lib_path() -> str:
    return os.path.join(_HERE, "_ref", "libfwd_bound.so")


def build() -> None:
    """Compile fwd_bound.c (gcc); cheap, so done on demand."""
    subprocess.run(["make", "-C", _HERE, "all"], check=True, capture_output=True)


def _lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(lib_path()):
            build()
        lib = ctypes.CDLL(lib_path())
        lib.fwd_bound.restype = c_longlong
        _LIB = lib
    return _LIB


def _np(x, dtype):
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(np.asarray(x), dtype=dtype)


def _p(a):
    return a.ctypes.data_as(c_void_p)


def bound(records, colors, point_list, ranges, subpixel_offset, bg, W, H, tile_rows=(0, 0), alpha_max=ALPHA_MAX,
          alpha_min=ALPHA_MIN, t_min=T_MIN, debug_f64=False, n_contrib=None) -> dict:
    """Exact outputs and their bounds.  Every float input is read as float64 (fp32 values are exact in it).
    ``alpha_max`` / ``alpha_min`` / ``t_min``: the clamp and the two thresholds (the kernel's fp32 constants by default).
    ``debug_f64``: compute px and power in fp64 (oracle.c's fp64 expression) instead of emulating the kernel's fp32.
    ``n_contrib`` [H, W]: a tested n_contrib; ``nc_ok`` [H, W] then says, per pixel, whether it is the n_contrib of one
    of the evaluated decision combinations (``check`` needs it)."""
    rec = _np(records, np.float64).reshape(-1, 8)
    P = rec.shape[0]
    col = _np(colors, np.float64).reshape(P, 3)
    pl = _np(point_list, np.int64).astype(np.uint32)
    rg = _np(ranges, np.int64).astype(np.uint32).reshape(-1, 2)
    so = _np(subpixel_offset, np.float64).reshape(H, W, 2)
    bgv = _np(bg, np.float64).reshape(3)
    if pl.size == 0:
        pl = np.zeros(1, np.uint32)
    if rec.size == 0:
        rec = np.zeros((1, 8)); col = np.zeros((1, 3))
    T = rg.shape[0]
    S = np.zeros((4, H, W)); B = np.zeros((4, H, W))
    S[3] = 1.0
    S[:3] = bgv[:, None, None]
    nc_nom = np.zeros((H, W), np.uint32)
    nc_test = None if n_contrib is None else _np(n_contrib, np.int64).reshape(H, W).astype(np.uint32)
    nc_ok = np.zeros((H, W), np.uint8)
    und = np.zeros((H, W), np.uint8)
    mbits = np.zeros((T, 4, MASK_WORDS), np.uint32)
    msure = np.zeros((T, 4, MASK_WORDS), np.uint32)
    stats = np.zeros(3)
    over = _lib().fwd_bound(c_int(W), c_int(H), c_int(tile_rows[0]), c_int(tile_rows[1]), _p(rg), _p(pl), _p(so),
                            _p(bgv), _p(rec), _p(col), c_double(alpha_max), c_double(alpha_min), c_double(t_min),
                            c_int(int(bool(debug_f64))), _p(S), _p(B), _p(nc_nom),
                            None if nc_test is None else _p(nc_test), _p(nc_ok), _p(und), _p(mbits), _p(msure),
                            _p(stats))
    return dict(S=S, B=B, nc_nom=nc_nom, nc_test=nc_test, nc_ok=nc_ok.astype(bool), und=und, mbits=mbits, msure=msure,
                overflow_pixels=int(over), undetermined_pixels=int(stats[0]), blended_pairs=int(stats[1]),
                undetermined_alpha=int(stats[2]), W=W, H=H, tile_rows=tuple(tile_rows))


def pair_power(records, g, ux, uy, so) -> np.ndarray:
    """The fp32 power the oracle evaluates for the pairs (record g[i], pixel (ux[i], uy[i]), sub-pixel offset so[i])."""
    rec = _np(records, np.float64).reshape(-1, 8)
    g = _np(g, np.int64).astype(np.uint32)
    ux, uy = _np(ux, np.int32), _np(uy, np.int32)
    so = _np(so, np.float64).reshape(-1, 2)
    out = np.zeros(g.size, np.float32)
    _lib().fwd_pair_power(c_longlong(g.size), _p(rec), _p(g), _p(ux), _p(uy), _p(so), _p(out))
    return out


def band_rows(res):
    """Pixel rows [y0, y1) the oracle evaluated."""
    ty0, ty1 = res["tile_rows"]
    H = res["H"]
    if ty0 == 0 and ty1 == 0:
        return 0, H
    return 16 * ty0, min(16 * ty1, H)


def block_last(n_contrib, W, H):
    """[T, 4] largest n_contrib of each 8x8 block (block k = bx + 2 by of the tile)."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    nc = np.zeros((gy * 16, gx * 16), np.int64)
    nc[:H, :W] = np.asarray(n_contrib, np.int64).reshape(H, W)
    b = nc.reshape(gy, 2, 8, gx, 2, 8).max(axis=(2, 5))
    return b.transpose(0, 2, 1, 3).reshape(gy * gx, 4)


def check(res, out_color, final_T, n_contrib, masks=None) -> dict:
    """Compare the kernel's outputs (``out_color`` [3, H, W], ``final_T`` / ``n_contrib`` [H, W], optionally the blend
    masks [T, 4, 32]) with ``bound``'s result, over the rows the oracle evaluated.

    Returns ``ratio`` (per channel, the worst |kernel - S| / B over pixels with a finite, non-zero bound), ``ratio_det``
    (the same over determined pixels), ``violations`` (pixel indices, flattened, with |kernel - S| > B in a channel or a
    non-finite output), ``nc_outside`` (pixels whose n_contrib is not that of any evaluated decision combination: the
    single nominal value where the pixel is determined), ``mask_differ`` ((tile, block, position) triples where a sure mask
    bit differs, positions below min(MASK_K, the block's largest kernel n_contrib)) and ``mask_compared``.
    ``res`` must come from ``bound(..., n_contrib=n_contrib)`` with the same n_contrib."""
    y0, y1 = band_rows(res)
    H, W = res["H"], res["W"]
    assert res["nc_test"] is not None and np.array_equal(res["nc_test"], np.asarray(n_contrib).reshape(H, W)), \
        "bound() was not given this n_contrib"
    got = np.concatenate([np.asarray(out_color, np.float64).reshape(3, H, W),
                          np.asarray(final_T, np.float64).reshape(1, H, W)])[:, y0:y1]
    S, B = res["S"][:, y0:y1], res["B"][:, y0:y1]
    d = np.abs(got - S)
    bad = (~(d <= B) & np.isfinite(B)) | ~np.isfinite(got)
    det = res["und"][y0:y1] == 0
    ratio, ratio_det = {}, {}
    for c, name in enumerate(CHANNELS):
        m = np.isfinite(B[c]) & (B[c] > 0)
        ratio[name] = float((d[c][m] / B[c][m]).max()) if m.any() else 0.0
        md = m & det
        ratio_det[name] = float((d[c][md] / B[c][md]).max()) if md.any() else 0.0
    out = dict(ratio=ratio, ratio_det=ratio_det, violations=np.flatnonzero(bad.any(axis=0)),
               nc_outside=np.flatnonzero(~res["nc_ok"][y0:y1]))
    if masks is not None:
        last = np.minimum(block_last(np.asarray(n_contrib).reshape(H, W), W, H), MASK_K)
        gx = (W + 15) // 16
        ty0, ty1 = (y0 // 16, (y1 + 15) // 16)
        tiles = np.arange(ty0 * gx, ty1 * gx)
        pos = np.arange(MASK_K)
        unpack = lambda m: ((np.asarray(m, np.uint32)[..., :, None] >> np.arange(32, dtype=np.uint32)) & 1).astype(bool) \
            .reshape(*np.shape(m)[:-1], MASK_K)
        kb, sb, eb = unpack(masks[tiles]), unpack(res["msure"][tiles]), unpack(res["mbits"][tiles])
        live = pos[None, None, :] < last[tiles][:, :, None]
        differ = (kb != eb) & sb & live
        out["mask_differ"] = np.argwhere(differ)
        out["mask_differ"][:, 0] += tiles[0] if tiles.size else 0
        out["mask_compared"] = int((sb & live).sum())
        out["mask_unsure"] = int((~sb & live).sum())
    return out
