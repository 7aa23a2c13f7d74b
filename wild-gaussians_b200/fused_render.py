"""Inference render on one composite: a drop-in for ``WildGaussians.render`` (wildgaussians/method.py:1832-1866), the call
every evaluation protocol, ``train.py``'s evaluation and video loops and a viewer make once per image.

With ``wildgaussians_fused.enable_method(method)`` alone that call still composites the raw colours nobody reads, runs
a third full composite for depth on a distance built from PyTorch statements, writes the backward state of the training
composite, and copies colour, accumulation and depth back in separate pageable copies.  Here:

* one colour pass, toned only (``fused_colors(..., want_raw=False)``), or the SH colours for models without appearance;
* one geometry pass (``gsr_forward_geometry``: its instance-count read-back is the first host synchronisation);
* one display composite (``gsr_forward_display``): the training composite's walk and arithmetic, so colour and
  accumulation are the bits of today's fused path; no blend masks or ``n_contrib``; the depth channel composited
  alongside the colours from the per-Gaussian camera distance; an epilogue that writes ``clamp(0, 1)`` then NaN -> 0 in
  HWC, ``1 - T`` and the depth into one contiguous device block;
* one device-to-host copy of that block into pinned memory from torch's caching host allocator, and one synchronisation.

The returned arrays are views of that pinned block, a fresh one per call: a caller may keep them (``eval_all`` collects
them) and no later call overwrites them.  While they are alive the block stays pinned; once they are dropped torch's
host cache hands the block to a later call.  The only difference a caller can see is the layout of ``color``: the
reference returns a permuted (non-contiguous) view, this path a C-contiguous HWC array with the same values.

    import fused_render
    out = fused_render.render(method, camera, options)                   # same arguments and result as the method
    wildgaussians_fused.enable_method(method, render=True)              # or: route method.render here

Anything outside the accelerated configuration (see ``supported``) runs the method's own ``render``.
"""
from __future__ import annotations

import sys
from ctypes import byref

import numpy as np
import torch

import wildgaussians_fused as wgf
from diff_gaussian_rasterization import _C
from fused_colors import fused_activations, fused_colors, fused_sh_colors

_lib = _C._lib


def _method_module(method):
    return sys.modules[type(method.model).__module__]


def _wants_depth(options) -> bool:
    return options is not None and "depth" in options.get("outputs", ())


def supported(method, camera, options=None) -> bool:
    """True when ``render`` takes the fused path for this call: a configuration ``wildgaussians_fused`` accelerates
    (``_supported`` / ``_supported_sh``, which also exclude ``config.debug``), a pinhole camera, fp32 CUDA parameters,
    no tile-row shard, at least one Gaussian, and for models with appearance a float32 embedding of the configured size
    (or none).  A model without appearance ignores the embedding, as the reference does."""
    model, config = method.model, method.config
    appearance = wgf._supported(model, config)
    if not (appearance or wgf._supported_sh(model, config)):
        return False
    tens = [model.xyz, model.features_dc, model.features_rest, model.scales, model.opacities, model.rotations,
            model.filter_3D]
    if appearance:
        tens += [model.embeddings, model.appearance_embeddings] + list(model.appearance_mlp.mlp.parameters())
    if not all(t.is_cuda and t.dtype == torch.float32 for t in tens):
        return False
    if int(model.xyz.shape[0]) == 0:
        return False
    emb = (options or {}).get("embedding", None)
    if emb is not None:
        if not isinstance(emb, np.ndarray):
            return False
        if appearance and not (emb.dtype == np.float32 and emb.shape == (int(config.appearance_embedding_dim),)):
            return False
    if _C.get_tile_row_shard() != (0, 0):
        return False
    return camera.item().camera_models == _method_module(method).camera_model_to_int("pinhole")


def _reference(method):
    cls = type(method)
    if not hasattr(cls, "render"):            # e.g. a namespace holding (model, config)
        cls = _method_module(method).WildGaussians
    return cls.render


def display_composite(bg, means3D, colors, opacities, scales, rotations, viewmatrix, projmatrix, campos, tanfovx, tanfovy,
                      kernel_size, subpixel_offset, H, W, *, depth=False, depth_values=None, sh_degree=0):
    """Geometry pass + ``gsr_forward_display`` on the current stream: one fp32 device block holding the colour [H,W,3]
    (``clamp(0, 1)`` then NaN -> 0), the accumulation ``1 - T`` [H,W] and, with ``depth``, the depth channel [H,W],
    composited from ``depth_values`` [P] or, when it is None, from the camera distance ``|means3D - campos|``.  Every
    tensor is contiguous fp32 on one device; one host synchronisation (the instance-count read-back)."""
    dev = means3D.device
    P, HW = int(means3D.shape[0]), H * W
    f32 = dict(dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    out = torch.empty(((5 if depth else 4) * HW,), **f32)       # colour [H,W,3] | accumulation [H,W] | depth [H,W]
    radii = torch.empty((P,), dtype=torch.int32, device=dev)
    fa = _C.forward_args(background=bg, means3D=means3D, colors=colors, opacities=opacities, scales=scales,
                         rotations=rotations, viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos,
                         tan_fovx=tanfovx, tan_fovy=tanfovy, kernel_size=kernel_size, subpixel_offset=subpixel_offset,
                         H=H, W=W, radii=radii, degree=sh_degree,
                         out_color=out)     # out_color: only checked for NULL, not written
    geom, img, binning, scratch, R, N1 = _C._forward_geometry(fa, dev, stream)
    da = _C.GsrDisplayArgs()
    da.out_color, da.out_accum = out.data_ptr(), out[3 * HW:].data_ptr()
    dist = None
    if depth:
        da.depth, da.out_depth = 1, out[4 * HW:].data_ptr()
        if depth_values is not None:
            da.depth_values = depth_values.data_ptr()
        else:
            dist = torch.empty((P,), **f32)
            da.depth_scratch = dist.data_ptr()
    _C._check(_lib.gsr_forward_display(byref(fa), byref(da), geom.data_ptr(), img.data_ptr(), binning.data_ptr(),
                                       scratch.data_ptr(), R, N1, stream), "gsr_forward_display")
    # the buffers go back to torch's stream-ordered caching allocator: later allocations on this stream follow the kernels
    return out


def render(method, camera, options=None, **kwargs):
    """Drop-in for ``WildGaussians.render``: same arguments, same keys, shapes, dtypes and values.  Reads only
    ``method.model`` and ``method.config``; unsupported calls run the method's own implementation."""
    if not supported(method, camera, options):
        return _reference(method)(method, camera, options=options, **kwargs)
    del kwargs
    model, config = method.model, method.config
    cam = camera.item()
    m = _method_module(method)
    dev = model.xyz.device
    depth = _wants_depth(options)
    appearance = wgf._supported(model, config)
    model.eval()
    with torch.no_grad(), torch.cuda.device(dev):
        np_emb = (options or {}).get("embedding", None)
        embedding = None
        if appearance:
            # through pinned memory: a pageable upload would synchronise the stream
            embedding = (torch.from_numpy(np_emb).pin_memory().to(dev, non_blocking=True) if np_emb is not None
                         else model.get_embedding(None))
        cc = wgf._camera_constants(m, cam, dev)
        H, W = cc["height"], cc["width"]
        deg = wgf._active_degree(model)
        scales, opacity, rotations = fused_activations(model.scales, model.opacities, model.rotations, model.filter_3D)
        if appearance:
            colors = fused_colors(model.features_dc, model.features_rest, model.embeddings, embedding,
                                  model.appearance_mlp.mlp, model.xyz, cc["cam_center"], deg, want_raw=False)[1]
        else:
            colors = fused_sh_colors(model.features_dc, model.features_rest, model.xyz, cc["cam_center"], deg)

        out = display_composite(wgf._zeros((3,), dev), model.xyz, colors, opacity, scales, rotations, cc["world_view"],
                                cc["full_proj"], cc["cam_center"], cc["tanfovx"], cc["tanfovy"], float(config.kernel_size),
                                wgf._zeros((H, W, 2), dev), H, W, depth=depth, sh_degree=deg)
        host = torch.empty(out.shape, dtype=torch.float32, pin_memory=True)
        host.copy_(out, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()

    HW = H * W
    ret = {"color": host[:3 * HW].view(H, W, 3).numpy(),
           "accumulation": host[3 * HW:4 * HW].view(H, W).squeeze(-1).numpy()}
    if depth:
        ret["depth"] = host[4 * HW:].view(H, W).numpy()
    return ret
