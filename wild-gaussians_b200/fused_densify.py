"""Fused densification: ``GaussianModel.densify_and_prune`` (wildgaussians/method.py:1420-1468) and ``reset_opacity``
(:1249-1278) as sm_90a kernels (``csrc/densify.cu``).

``densify_and_prune(model, max_grad, min_opacity, extent, enable_size_pruning)`` leaves the model and its optimizer in
the state the reference's method leaves them in, from the same state and the same RNG state:

* the same clone / split / prune decisions, on the reference's fp32 arithmetic.  ``Q = torch.quantile(grads_abs,
  1 - ratio)`` is found by a radix select on the GPU, with torch's rank arithmetic and ``lerp``, so it equals torch's
  value bit for bit where torch accepts the input, and the same formula holds above the 2^24 elements torch refuses;
* the same row order (survivors of the rows not split, clones, split copy 1, split copy 2), written by ONE gather
  kernel straight into final-size tensors -- parameters, both Adam moments and the densification buffers -- instead of
  two ``torch.cat`` rounds and two rounds of boolean-mask indexing;
* the split children's samples from the same draw (``normal_(0, 1)`` of a ``[2S, 3]`` tensor on the default generator,
  which is what ``torch.normal(mean, std)`` draws), so the generator ends in the same state.  The children's ``xyz`` are
  computed in the kernel: they differ from the reference's cuBLAS ``bmm`` in the last bits;
* the same optimizer surgery: fresh ``nn.Parameter`` objects registered on the model, each group's state dict moved to
  the new key with ``step`` kept and zero moments for new rows, no ``.grad``;
* the same return tuple and, with ``enable_size_pruning``, the same printed line.

It makes one host synchronisation: the read-back of the counts (which also sizes the normal draw and the new tensors).
``reset_opacity(model)`` is one elementwise kernel and no synchronisation.  Anything ``supported`` refuses runs the
class's own method.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch
from torch import nn

from diff_gaussian_rasterization import _C

__all__ = ["densify_and_prune", "reset_opacity", "supported"]

PARAM_NAMES = ("xyz", "features_dc", "features_rest", "scales", "rotations", "opacities", "embeddings")
BUFFER_NAMES = ("xyz_grad", "denom", "filter_3D", "max_radii2D", "xyz_gradient_accum_abs", "xyz_gradient_accum_abs_max")
_pinned: dict = {}


def _fused_adam_cls():
    import fused_adam
    return fused_adam.FusedAdam


def _fp32_rows(t, P, dev) -> bool:
    return (isinstance(t, torch.Tensor) and t.device == dev and t.dtype == torch.float32 and t.is_contiguous() and t.dim() >= 1
            and int(t.shape[0]) == P)


def supported(model) -> bool:
    """The models the fused path covers: fp32 contiguous CUDA tensors, ``torch.optim.Adam`` or ``FusedAdam`` with one
    parameter per dynamically sized group, only the names method.py declares, and ``config.debug`` off."""
    opt = getattr(model, "optimizer", None)
    if opt is None or type(opt) not in (torch.optim.Adam, _fused_adam_cls()):
        return False
    if bool(getattr(model.config, "debug", False)):
        return False
    props = list(getattr(model, "_dynamically_sized_props", ()))
    if any(n not in PARAM_NAMES and n not in BUFFER_NAMES for n in props) or len(set(props)) != len(props):
        return False
    xyz = getattr(model, "xyz", None)
    if not isinstance(xyz, torch.Tensor) or not xyz.is_cuda:
        return False
    P, dev = int(xyz.shape[0]), xyz.device
    if not 1 <= P <= _C.DENSIFY_MAX_P:
        return False
    groups = {g.get("name"): g for g in opt.param_groups}
    for n in props:
        t = getattr(model, n, None)
        if t is None:
            if n in ("xyz", "scales", "rotations", "opacities", "xyz_grad", "denom"):
                return False
            continue
        if not _fp32_rows(t, P, dev):
            return False
        is_param = n in PARAM_NAMES
        if isinstance(t, nn.Parameter) != is_param or (n in groups) != is_param:
            return False
        if is_param:
            g = groups[n]
            if len(g["params"]) != 1 or g["params"][0] is not t:
                return False
            st = opt.state.get(t, None)
            if st is not None and not all(k in st and _fp32_rows(st[k], P, dev) and st[k].shape == t.shape
                                          for k in ("exp_avg", "exp_avg_sq")):
                return False
    if bool(model.config.use_gof_abs_gradient) and getattr(model, "xyz_gradient_accum_abs", None) is None:
        return False
    return True


def _counts_host(dev):
    key = str(dev)
    t = _pinned.get(key)
    if t is None:
        t = _pinned[key] = torch.empty((_C.DENSIFY_COUNTS,), dtype=torch.int32, pin_memory=True)
    return t


def _f32(x) -> float:
    return float(np.float32(x))


def plan(model, max_grad, min_opacity, extent, enable_size_pruning):
    """Runs the plan kernels and reads the counts back (one synchronisation).  Returns (counts dict, args, scratch)."""
    xyz = model.xyz
    dev, P = xyz.device, int(xyz.shape[0])
    use_abs = bool(model.config.use_gof_abs_gradient)
    a = _C.GsrDensifyArgs()
    a.P = P
    a.xyz_grad, a.denom = model.xyz_grad.data_ptr(), model.denom.data_ptr()
    a.accum_abs = model.xyz_gradient_accum_abs.data_ptr() if use_abs else None
    a.xyz, a.scales, a.rotations, a.opacities = (getattr(model, n).data_ptr() for n in ("xyz", "scales", "rotations", "opacities"))
    # torch compares a float tensor with a Python scalar after rounding the scalar to fp32
    a.max_grad = _f32(max_grad)
    a.clone_max_scale = _f32(model.config.percent_dense * extent)
    a.min_opacity = _f32(min_opacity)
    a.prune_max_scale = _f32(0.1 * extent)
    a.size_pruning = int(bool(enable_size_pruning))
    # `scales / (0.8 * N)` with a Python scalar is evaluated by torch's CUDA kernel as scales * fp32(1 / fp32(0.8 N))
    a.split_scale_mul = float(np.float32(1.0) / np.float32(0.8 * 2))
    scratch = torch.empty((_C._lib.gsr_densify_scratch_bytes(P),), dtype=torch.uint8, device=dev)
    counts = torch.empty((_C.DENSIFY_COUNTS,), dtype=torch.int32, device=dev)
    a.scratch, a.counts = scratch.data_ptr(), counts.data_ptr()
    stream = torch.cuda.current_stream(dev)
    _C._check(_C._lib.gsr_densify_plan(ctypes.byref(a), stream.cuda_stream), "gsr_densify_plan")
    host = _counts_host(dev)
    host.copy_(counts, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record(stream)
    ev.synchronize()
    c = host.tolist()
    q = np.array([c[6]], dtype=np.int32).view(np.float32)[0]
    res = dict(clones=c[0], splits=c[1], rows=c[2], big=c[3], kept_splits=c[4], n_ge=c[5], Q=float(q))
    return res, a, scratch


def densify_and_prune(model, max_grad, min_opacity, extent, enable_size_pruning, skyradius=None):
    """Drop-in for ``GaussianModel.densify_and_prune`` (method.py:1420-1468); see the module docstring."""
    if not supported(model):
        return type(model).densify_and_prune(model, max_grad, min_opacity, extent, enable_size_pruning, skyradius=skyradius)
    del skyradius  # unused, as in the reference
    with torch.no_grad(), torch.cuda.device(model.xyz.device):
        counts, a, scratch = plan(model, max_grad, min_opacity, extent, enable_size_pruning)
        dev, P = model.xyz.device, int(model.xyz.shape[0])
        C, S, P2 = counts["clones"], counts["splits"], counts["rows"]
        # torch.normal(mean=zeros(2S, 3), std=stds) draws normal_(0, 1) into a [2S, 3] tensor on the default generator
        normals = torch.empty((2 * S, 3), dtype=torch.float32, device=dev).normal_(0, 1)
        a.normals = normals.data_ptr() if S else None
        opt = model.optimizer
        groups = {g["name"]: g for g in opt.param_groups if g.get("name") in model._dynamically_sized_props}
        segs, new_params, new_buffers = [], {}, {}

        def seg(src, dst, kind):
            s = _C.GsrDensifySegment()
            s.src, s.dst, s.width, s.kind = src.data_ptr(), dst.data_ptr(), int(src.numel() // P), kind
            segs.append(s)

        for name in model._dynamically_sized_props:
            t = getattr(model, name, None)
            if t is None:
                continue
            new = torch.empty((P2, *t.shape[1:]), dtype=t.dtype, device=dev)
            if name in groups:
                kind = {"xyz": _C.DENSIFY_XYZ, "scales": _C.DENSIFY_SCALES}.get(name, _C.DENSIFY_COPY)
                seg(t, new, kind)
                st = opt.state.get(t, None)
                moments = None
                if st is not None:
                    moments = (torch.empty_like(new), torch.empty_like(new))
                    seg(st["exp_avg"], moments[0], _C.DENSIFY_ZERO_NEW)
                    seg(st["exp_avg_sq"], moments[1], _C.DENSIFY_ZERO_NEW)
                new_params[name] = (new, moments)
            else:
                seg(t, new, _C.DENSIFY_ZERO_NEW)
                new_buffers[name] = new
        if P2 > 0:
            arr = (_C.GsrDensifySegment * len(segs))(*segs)
            _C._check(_C._lib.gsr_densify_apply(ctypes.byref(a), arr, len(segs), torch.cuda.current_stream(dev).cuda_stream),
                      "gsr_densify_apply")
        del scratch     # back to the stream-ordered caching allocator, after the kernels that read it

        for group in opt.param_groups:
            name = group.get("name")
            if name not in new_params:
                continue
            new, moments = new_params[name]
            old = group["params"][0]
            param = nn.Parameter(new.requires_grad_(True))
            st = opt.state.get(old, None)
            if st is not None:
                st["exp_avg"], st["exp_avg_sq"] = moments
                del opt.state[old]
                opt.state[param] = st
            group["params"][0] = param
            setattr(model, name, param)
        for name, new in new_buffers.items():
            model.register_buffer(name, new)

    if enable_size_pruning:
        print(f"pruning ws points {counts['big']} -> {counts['big']}")
    return C, S, (P + C + S) - P2


def reset_opacity(model):
    """Drop-in for ``GaussianModel.reset_opacity`` (method.py:1249-1278): one kernel, a new ``opacities`` Parameter with
    zeroed moments under the new key, ``step`` kept."""
    assert model.optimizer is not None, "Not set up for training"
    if not supported(model):
        return type(model).reset_opacity(model)
    dev, P = model.xyz.device, int(model.xyz.shape[0])
    with torch.no_grad(), torch.cuda.device(dev):
        out = torch.empty_like(model.opacities)
        _C._check(_C._lib.gsr_reset_opacity(P, model.opacities.data_ptr(), model.scales.data_ptr(), model.filter_3D.data_ptr(),
                                            out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), "gsr_reset_opacity")
    for group in model.optimizer.param_groups:
        if group["name"] == "opacities":
            stored_state = model.optimizer.state.get(group["params"][0], None)
            stored_state["exp_avg"] = torch.zeros_like(out)
            stored_state["exp_avg_sq"] = torch.zeros_like(out)
            del model.optimizer.state[group["params"][0]]
            group["params"][0] = nn.Parameter(out.requires_grad_(True))
            model.register_parameter("opacities", group["params"][0])
            model.optimizer.state[group["params"][0]] = stored_state
