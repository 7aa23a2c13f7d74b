"""TEST INFRASTRUCTURE -- numpy/ctypes front end of ``oracle/oracle.c`` (the CPU restatement of the
reference rasterizer path; see the header of that file).

``forward(scene)`` / ``backward(state, dL_dpix)`` take and return plain numpy arrays.  ``scene`` is a dict
with the keys produced by ``synthetic.make_scene`` (numpy or torch CPU values).  ``dtype=np.float64`` runs
the fp64 build of the same algorithm (used for finite-difference checks of the backward restatement).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py`` may import this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from ctypes import POINTER, c_double, c_float, c_int, c_longlong, c_void_p

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBS = {}


def lib_path(dtype=np.float32) -> str:
    name = "liboracle.so" if np.dtype(dtype) == np.float32 else "liboracle_f64.so"
    return os.path.join(_HERE, "_ref", name)


def build() -> None:
    """Compile the C restatement (gcc); cheap, so done on demand."""
    subprocess.run(["make", "-C", _HERE, "all"], check=True, capture_output=True)


def _lib(dtype):
    dt = np.dtype(dtype)
    if dt not in _LIBS:
        path = lib_path(dt)
        if not os.path.exists(path):
            build()
        lib = ctypes.CDLL(path)
        lib.oracle_preprocess.restype = c_longlong
        lib.oracle_bin.restype = c_int
        lib.oracle_num_threads.restype = c_int
        assert lib.oracle_real_bytes() == dt.itemsize
        _LIBS[dt] = lib
    return _LIBS[dt]


def num_threads() -> int:
    return _lib(np.float32).oracle_num_threads()


def set_num_threads(n: int) -> None:
    for dt in (np.float32, np.float64):
        if os.path.exists(lib_path(dt)):
            _lib(dt).oracle_set_num_threads(int(n))


def _np(x, dtype):
    if x is None:
        return None
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    x = np.ascontiguousarray(np.asarray(x), dtype=dtype)
    return x if x.size else None


def _p(a):
    return None if a is None else a.ctypes.data_as(c_void_p)


def forward(scene: dict, dtype=np.float32, tile_rows=(0, 0), stages=("preprocess", "bin", "render")) -> dict:
    """Run the restated forward.  Returns every intermediate the reference keeps in its geom / binning /
    image buffers plus the outputs (``out_color``, ``radii``, ``final_T``, ``n_contrib``)."""
    lib = _lib(dtype)
    real = c_float if np.dtype(dtype) == np.float32 else c_double
    g = lambda k: _np(scene.get(k), dtype)
    means3D, shs, colors = g("means3D"), g("shs"), g("colors_precomp")
    opac, scales, rots, cov3Dp = g("opacities"), g("scales"), g("rotations"), g("cov3D_precomp")
    view, proj, campos = g("viewmatrix"), g("projmatrix"), g("campos")
    bg, subpix = g("bg"), g("subpixel_offset")
    W, H = int(scene["image_width"]), int(scene["image_height"])
    P = 0 if means3D is None else means3D.shape[0]
    D = int(scene.get("sh_degree", 0))
    M = 0 if shs is None else shs.shape[1]
    N = W * H
    gx, gy = (W + 15) // 16, (H + 15) // 16
    T = gx * gy
    st = dict(P=P, D=D, M=M, W=W, H=H, dtype=np.dtype(dtype), tile_rows=tuple(tile_rows), scene=scene)
    st["radii"] = np.zeros(P, np.int32)
    st["depths"] = np.zeros(P, dtype)
    st["means2D"] = np.zeros((P, 2), dtype)
    st["cov3D"] = np.zeros((P, 6), dtype)
    st["conic_opacity"] = np.zeros((P, 4), dtype)
    st["rgb"] = np.zeros((P, 3), dtype)
    st["clamped"] = np.zeros((P, 3), np.uint8)
    st["tiles_touched"] = np.zeros(P, np.uint32)
    st["rect"] = np.zeros((P, 4), np.int32)
    st["out_color"] = np.zeros((3, H, W), dtype)
    st["final_T"] = np.ones((H, W), dtype)
    st["n_contrib"] = np.zeros((H, W), np.uint32)
    st["ranges"] = np.zeros((T, 2), np.uint32)
    st["point_list"] = np.zeros(0, np.uint32)
    st["tile_of"] = np.zeros(0, np.uint32)
    st["num_rendered"] = 0
    if P == 0:
        return st
    if cov3Dp is not None:
        st["cov3D"] = cov3Dp.reshape(P, 6).copy()
    R = lib.oracle_preprocess(
        c_int(P), c_int(D), c_int(M), c_int(W), c_int(H), _p(means3D), _p(shs), _p(colors), _p(opac), _p(scales),
        real(float(scene.get("scale_modifier", 1.0))), _p(rots), _p(cov3Dp), _p(view), _p(proj), _p(campos),
        real(float(scene["tanfovx"])), real(float(scene["tanfovy"])), real(float(scene["kernel_size"])),
        c_int(int(bool(scene.get("prefiltered", False)))), c_int(tile_rows[0]), c_int(tile_rows[1]),
        _p(st["radii"]), _p(st["depths"]), _p(st["means2D"]), _p(st["cov3D"]), _p(st["conic_opacity"]), _p(st["rgb"]),
        _p(st["clamped"]), _p(st["tiles_touched"]), _p(st["rect"]))
    if R < 0:
        raise RuntimeError("Point is filtered although prefiltered is set. This shouldn't happen!")
    st["num_rendered"] = int(R)
    st["colors"] = colors if colors is not None else st["rgb"]
    if "bin" not in stages:
        return st
    st["point_list"] = np.zeros(int(R), np.uint32)
    st["tile_of"] = np.zeros(int(R), np.uint32)
    rc = lib.oracle_bin(c_int(P), c_int(W), c_int(H), c_longlong(int(R)), _p(st["radii"]), _p(st["depths"]),
                        _p(st["rect"]), _p(st["point_list"]), _p(st["tile_of"]), _p(st["ranges"]))
    if rc != 0:
        raise RuntimeError(f"oracle_bin failed ({rc})")
    if "render" not in stages:
        return st
    lib.oracle_render(c_int(W), c_int(H), c_int(tile_rows[0]), c_int(tile_rows[1]), _p(st["ranges"]),
                      _p(st["point_list"]), _p(subpix), _p(st["means2D"]), _p(st["colors"]), _p(st["conic_opacity"]),
                      _p(bg), _p(st["final_T"]), _p(st["n_contrib"]), _p(st["out_color"]))
    return st


def backward(st: dict, dL_dpix, acc=None) -> dict:
    """Restated backward on the state returned by ``forward``.  Returns the 8 gradients of the reference's
    ``rasterize_gaussians_backward`` (plus ``dL_dconic``).  ``acc`` ([P, 10]): run only the per-Gaussian chain rule,
    on these accumulator rows instead of the composite's (``dL_dpix`` is then not read)."""
    dtype = st["dtype"]
    lib = _lib(dtype)
    real = c_float if dtype == np.float32 else c_double
    scene = st["scene"]
    P, D, M, W, H = st["P"], st["D"], st["M"], st["W"], st["H"]
    g = lambda k: _np(scene.get(k), dtype)
    out = dict(
        dL_dmeans2D=np.zeros((P, 3), dtype), dL_dconic=np.zeros((P, 4), dtype), dL_dopacity=np.zeros((P, 1), dtype),
        dL_dcolors=np.zeros((P, 3), dtype), dL_dmeans3D=np.zeros((P, 3), dtype), dL_dcov3D=np.zeros((P, 6), dtype),
        dL_dsh=np.zeros((P, M, 3), dtype), dL_dscales=np.zeros((P, 3), dtype), dL_drotations=np.zeros((P, 4), dtype))
    if P == 0:
        return out
    if acc is None:
        dpix = _np(dL_dpix, dtype)
        acc = np.zeros((P, 10), np.float64)
        tr = st["tile_rows"]
        lib.oracle_render_backward(c_int(P), c_int(W), c_int(H), c_int(tr[0]), c_int(tr[1]), _p(st["ranges"]),
                                   _p(st["point_list"]), _p(g("subpixel_offset")), _p(g("bg")), _p(st["means2D"]),
                                   _p(st["conic_opacity"]), _p(st["colors"]), _p(st["final_T"]), _p(st["n_contrib"]),
                                   _p(dpix), _p(acc))
    else:
        acc = np.ascontiguousarray(acc, np.float64)
    out["acc"] = acc
    shs, scales, rots = g("shs"), g("scales"), g("rotations")
    lib.oracle_preprocess_backward(
        c_int(P), c_int(D), c_int(M), c_int(W), c_int(H), _p(g("means3D")), _p(st["radii"]), _p(shs),
        _p(st["clamped"]), _p(scales), real(float(scene.get("scale_modifier", 1.0))), _p(rots), _p(st["cov3D"]),
        _p(g("viewmatrix")), _p(g("projmatrix")), _p(g("campos")), real(float(scene["tanfovx"])),
        real(float(scene["tanfovy"])), real(float(scene["kernel_size"])), _p(st["conic_opacity"]), _p(acc),
        _p(out["dL_dmeans2D"]), _p(out["dL_dconic"]), _p(out["dL_dopacity"]), _p(out["dL_dcolors"]),
        _p(out["dL_dmeans3D"]), _p(out["dL_dcov3D"]), _p(out["dL_dsh"]), _p(out["dL_dscales"]),
        _p(out["dL_drotations"]))
    return out


def mark_visible(means3D, viewmatrix, dtype=np.float32):
    lib = _lib(dtype)
    m, v = _np(means3D, dtype), _np(viewmatrix, dtype)
    P = 0 if m is None else m.shape[0]
    present = np.zeros(P, np.uint8)
    if P:
        lib.oracle_mark_visible(c_int(P), _p(m), _p(v), _p(present))
    return present.astype(bool)
