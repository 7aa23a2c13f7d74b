"""Fused per-Gaussian colour op of wild-gaussians (SURVEY.md 8f-2): host side of ``csrc/appearance.cu``.

``fused_colors(...)`` returns the two colour sets ``GaussianModel._render_internal`` feeds the rasterizer -- the raw
SH colours (method.py:1571-1579) and the appearance-toned colours (method.py:1586-1598, ``EmbeddingModel.forward``
:889-900, ``eval_sh`` :493-548) -- from the model's raw parameters, with full autograd support, in ONE kernel per
direction: the 59 -> 128 -> 128 -> 6 MLP runs on wgmma tensor cores (bf16 operands, fp32 accumulation),
the activations never leave the SM.  Opt-in: ``wildgaussians/method.py`` itself is untouched;
``wildgaussians_fused.enable(model)`` swaps the caller.

Shapes are those of the reference's default config (config.py:16,49,59): SH degree 3 storage (3 + 45 features),
24 per-Gaussian embedding features (6 x appearance_n_fourier_freqs), 32-d image embedding, hidden width 128.
``fused_sh_colors(...)`` is the colour op of models without appearance (method.py:1555-1565, ``csrc/sh_colors.cu``):
the raw SH colours alone, one bandwidth-bound kernel per direction.  ``fused_activations(...)`` is ``get_gaussians``
without its features part (``csrc/activations.cu``).
There is no PyTorch fallback: other shapes raise.
"""
from __future__ import annotations

from ctypes import byref

import torch

from diff_gaussian_rasterization import _C

_lib = _C._lib


_last_status = {"fwd": None, "bwd": None}


def last_status_ok() -> bool:
    """False if a barrier wait inside the most recent fused colour kernels timed out (synchronises)."""
    return all(t is None or int(t.item()) == 0 for t in _last_status.values())


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def _f32c(t):
    return t if (t.dtype == torch.float32 and t.is_contiguous()) else t.float().contiguous()


class _FusedColors(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features_dc, features_rest, embeddings, app_embedding, W1, b1, W2, b2, W3, b3, means3D, campos,
                active_sh_degree, want_raw):
        dev = features_dc.device
        P = int(features_dc.shape[0])
        if not features_dc.is_cuda:
            raise RuntimeError("fused_colors needs CUDA tensors; there is no CPU path")
        if (tuple(features_dc.shape) != (P, 3) or tuple(features_rest.shape) != (P, 45) or tuple(embeddings.shape) != (P, 24)
                or app_embedding.numel() != 32 or tuple(W1.shape) != (128, 59) or tuple(W2.shape) != (128, 128)
                or tuple(W3.shape) != (6, 128) or tuple(means3D.shape) != (P, 3)):
            raise RuntimeError("fused_colors supports the reference's default shapes only: features 3 + 45, embeddings 24, "
                               "image embedding 32, MLP 59 -> 128 -> 128 -> 6")
        tens = [_f32c(t.detach()) for t in (features_dc, features_rest, embeddings, app_embedding, W1, b1, W2, b2, W3, b3,
                                            means3D, campos)]
        (fdc, frest, gemb, aemb, w1, bb1, w2, bb2, w3, bb3, means, cam) = tens
        frest, gemb = _aligned16(frest), _aligned16(gemb)         # the kernels read them as 16-byte vectors
        with torch.cuda.device(dev):
            blob = torch.empty((_lib.gsr_appearance_packed_weight_bytes(),), dtype=torch.uint8, device=dev)
            _C._check(_lib.gsr_appearance_pack_weights(w1.data_ptr(), bb1.data_ptr(), w2.data_ptr(), bb2.data_ptr(), w3.data_ptr(),
                                                       bb3.data_ptr(), aemb.data_ptr(), blob.data_ptr(), _stream(dev)),
                      "gsr_appearance_pack_weights")
            raw = torch.empty((P, 3), dtype=torch.float32, device=dev) if want_raw else None
            toned = torch.empty((P, 3), dtype=torch.float32, device=dev)
            status = torch.zeros((1,), dtype=torch.int32, device=dev)
            a = _C.GsrAppearanceArgs()
            a.P, a.sh_degree = P, int(active_sh_degree)
            a.features_dc, a.features_rest, a.embeddings = fdc.data_ptr(), frest.data_ptr(), gemb.data_ptr()
            a.means3D, a.campos, a.packed_weights = means.data_ptr(), cam.data_ptr(), blob.data_ptr()
            a.colors_raw = raw.data_ptr() if want_raw else None
            a.colors_toned = toned.data_ptr()
            a.status = status.data_ptr()
            _C._check(_lib.gsr_appearance_colors_forward(byref(a), _stream(dev)), "gsr_appearance_colors_forward")
            _last_status["fwd"] = status
        ctx.save_for_backward(fdc, frest, gemb, aemb, w1, means, cam, blob, status)
        ctx.deg, ctx.want_raw = int(active_sh_degree), bool(want_raw)
        if want_raw:
            return raw, toned
        return toned.new_empty((0, 3)), toned

    @staticmethod
    def backward(ctx, g_raw, g_toned):
        fdc, frest, gemb, aemb, w1, means, cam, blob, status = ctx.saved_tensors
        dev = fdc.device
        P = int(fdc.shape[0])
        with torch.cuda.device(dev):
            f32 = dict(dtype=torch.float32, device=dev)
            g_toned = _f32c(g_toned) if g_toned is not None else torch.zeros((P, 3), **f32)
            use_raw = ctx.want_raw and g_raw is not None
            g_raw = _f32c(g_raw) if use_raw else None
            d_dc, d_rest = torch.empty((P, 3), **f32), torch.empty((P, 45), **f32)
            d_gemb, d_means = torch.empty((P, 24), **f32), torch.empty((P, 3), **f32)
            pack = torch.empty((_lib.gsr_appearance_grad_pack_bytes() // 4,), **f32)
            a = _C.GsrAppearanceArgs()
            a.P, a.sh_degree = P, ctx.deg
            a.features_dc, a.features_rest, a.embeddings = fdc.data_ptr(), frest.data_ptr(), gemb.data_ptr()
            a.means3D, a.campos, a.packed_weights = means.data_ptr(), cam.data_ptr(), blob.data_ptr()
            a.dL_dcolors_raw = g_raw.data_ptr() if use_raw else None
            a.dL_dcolors_toned = g_toned.data_ptr()
            a.dL_dfeatures_dc, a.dL_dfeatures_rest = d_dc.data_ptr(), d_rest.data_ptr()
            a.dL_dembeddings, a.dL_dmeans3D = d_gemb.data_ptr(), d_means.data_ptr()
            a.grad_pack, a.status = pack.data_ptr(), status.data_ptr()
            _C._check(_lib.gsr_appearance_colors_backward(byref(a), _stream(dev)), "gsr_appearance_colors_backward")
            _last_status["bwd"] = status
            dW1, db1 = torch.empty((128, 59), **f32), torch.empty((128,), **f32)
            dW2, db2 = torch.empty((128, 128), **f32), torch.empty((128,), **f32)
            dW3, db3 = torch.empty((6, 128), **f32), torch.empty((6,), **f32)
            d_aemb = torch.empty((32,), **f32)
            _C._check(_lib.gsr_appearance_unpack_grads(pack.data_ptr(), w1.data_ptr(), aemb.data_ptr(), dW1.data_ptr(),
                                                       db1.data_ptr(), dW2.data_ptr(), db2.data_ptr(), dW3.data_ptr(),
                                                       db3.data_ptr(), d_aemb.data_ptr(), _stream(dev)),
                      "gsr_appearance_unpack_grads")
        return (d_dc, d_rest, d_gemb, d_aemb.view_as(aemb), dW1, db1, dW2, db2, dW3, db3, d_means, None, None, None)


class _FusedActivations(torch.autograd.Function):
    """``GaussianModel.get_gaussians`` (method.py:1060-1086) without its features part: one kernel per direction."""

    @staticmethod
    def forward(ctx, scales_raw, opacities_raw, rotations_raw, filter_3D):
        dev = scales_raw.device
        P = int(scales_raw.shape[0])
        if not scales_raw.is_cuda:
            raise RuntimeError("fused_activations needs CUDA tensors; there is no CPU path")
        s, o, r, f = (_f32c(t.detach()) for t in (scales_raw, opacities_raw, rotations_raw, filter_3D))
        if tuple(s.shape) != (P, 3) or o.numel() != P or tuple(r.shape) != (P, 4) or f.numel() != P:
            raise RuntimeError("fused_activations: expected scales [P,3], opacities [P,1], rotations [P,4], filter_3D [P,1]")
        with torch.cuda.device(dev):
            so, oo, ro = torch.empty_like(s), torch.empty_like(o), torch.empty_like(r)
            _C._check(_lib.gsr_gaussian_activations_forward(P, s.data_ptr(), o.data_ptr(), r.data_ptr(), f.data_ptr(), so.data_ptr(),
                                                            oo.data_ptr(), ro.data_ptr(), _stream(dev)),
                      "gsr_gaussian_activations_forward")
        ctx.save_for_backward(s, o, r, f)
        return so, oo, ro

    @staticmethod
    def backward(ctx, g_s, g_o, g_r):
        s, o, r, f = ctx.saved_tensors
        dev = s.device
        P = int(s.shape[0])
        with torch.cuda.device(dev):
            g_s, g_o, g_r = (None if g is None else _f32c(g) for g in (g_s, g_o, g_r))
            ds, do, dr = torch.empty_like(s), torch.empty_like(o), torch.empty_like(r)
            ptr = lambda t: None if t is None else t.data_ptr()
            _C._check(_lib.gsr_gaussian_activations_backward(P, s.data_ptr(), o.data_ptr(), r.data_ptr(), f.data_ptr(), ptr(g_s),
                                                             ptr(g_o), ptr(g_r), ds.data_ptr(), do.data_ptr(), dr.data_ptr(),
                                                             _stream(dev)), "gsr_gaussian_activations_backward")
        return ds, do, dr, None


def _aligned16(t):
    return t if t.data_ptr() % 16 == 0 else t.clone()


class _FusedSHColors(torch.autograd.Function):
    """The SH colours of a model without appearance (method.py:1555-1565, ``csrc/sh_colors.cu``): one kernel per direction."""

    @staticmethod
    def forward(ctx, features_dc, features_rest, means3D, campos, active_sh_degree):
        dev = features_dc.device
        P = int(features_dc.shape[0])
        if not all(t.is_cuda for t in (features_dc, features_rest, means3D, campos)):
            raise RuntimeError("fused_sh_colors needs CUDA tensors; there is no CPU path")
        if (tuple(features_dc.shape) != (P, 3) or tuple(features_rest.shape) != (P, 45) or tuple(means3D.shape) != (P, 3)
                or campos.numel() != 3 or not 0 <= int(active_sh_degree) <= 3):
            raise RuntimeError("fused_sh_colors supports SH degree 3 storage only: features_dc [P,3], features_rest [P,45], "
                               "means3D [P,3], campos [3], active degree 0..3")
        fdc, frest, means, cam = (_f32c(t.detach()) for t in (features_dc, features_rest, means3D, campos))
        frest = _aligned16(frest)
        deg = int(active_sh_degree)
        with torch.cuda.device(dev):
            colors = torch.empty((P, 3), dtype=torch.float32, device=dev)
            _C._check(_lib.gsr_sh_colors_forward(P, deg, fdc.data_ptr(), frest.data_ptr(), means.data_ptr(), cam.data_ptr(),
                                                 colors.data_ptr(), _stream(dev)), "gsr_sh_colors_forward")
        ctx.save_for_backward(fdc, frest, means, cam)
        ctx.deg = deg
        return colors

    @staticmethod
    def backward(ctx, g_colors):
        fdc, frest, means, cam = ctx.saved_tensors
        dev = fdc.device
        P = int(fdc.shape[0])
        with torch.cuda.device(dev):
            g = None if g_colors is None else _f32c(g_colors)
            d_dc, d_rest, d_means = torch.empty_like(fdc), torch.empty_like(frest), torch.empty_like(means)
            _C._check(_lib.gsr_sh_colors_backward(P, ctx.deg, fdc.data_ptr(), frest.data_ptr(), means.data_ptr(), cam.data_ptr(),
                                                  None if g is None else g.data_ptr(), d_dc.data_ptr(), d_rest.data_ptr(),
                                                  d_means.data_ptr(), _stream(dev)), "gsr_sh_colors_backward")
        return d_dc, d_rest, d_means, None, None


def fused_activations(scales_raw, opacities_raw, rotations_raw, filter_3D):
    """``(scales, opacities, rotations)`` as ``GaussianModel.get_gaussians`` returns them (method.py:1060-1086)."""
    return _FusedActivations.apply(scales_raw, opacities_raw, rotations_raw, filter_3D)


def fused_sh_colors(features_dc, features_rest, means3D, campos, active_sh_degree):
    """``colors [P,3]`` as ``GaussianModel._render_internal`` computes them for a model without appearance
    (method.py:1555-1565): ``clamp_min(eval_sh(deg, clamp_max(cat(dc, rest), 1), normalize(means3D - campos)) + 0.5, 0)``.
    The arguments are the model's raw parameters (unclamped, storage degree 3) and the camera centre; the gradient
    reaches ``features_dc``, ``features_rest`` (zero above the active degree) and ``means3D``."""
    return _FusedSHColors.apply(features_dc, features_rest, means3D, campos, int(active_sh_degree))


def fused_colors(features_dc, features_rest, embeddings, app_embedding, mlp, means3D, campos, active_sh_degree,
                 want_raw=True):
    """``(colors_raw [P,3] or None, colors_toned [P,3])``.  ``mlp`` is ``EmbeddingModel.mlp`` (nn.Sequential of
    Linear(59,128), ReLU, Linear(128,128), ReLU, Linear(128,6)); the other arguments are the model's raw parameters
    (``features_dc`` / ``features_rest`` unclamped) and the camera centre."""
    lin = [m for m in mlp if isinstance(m, torch.nn.Linear)]
    if len(lin) != 3:
        raise RuntimeError("fused_colors expects the reference's 3-layer appearance MLP")
    raw, toned = _FusedColors.apply(features_dc, features_rest, embeddings, app_embedding, lin[0].weight, lin[0].bias,
                                    lin[1].weight, lin[1].bias, lin[2].weight, lin[2].bias, means3D, campos,
                                    int(active_sh_degree), bool(want_raw))
    return (raw if want_raw else None), toned

