"""Fused attention and early exit for the DINOv2 backbone of wild-gaussians' uncertainty model: host side of
``csrc/attention.cu``.

``attention(qkv, num_heads)`` is the core of ``Attention.forward`` (``wildgaussians/dinov2.py:224-233``) from the ``qkv``
Linear's output to the input of ``proj``: ``qkv`` is ``[B, N, 3 * num_heads * 64]`` fp32 on the GPU, read in place as
``[B, N, 3, H, 64]``; the result is ``[B, N, num_heads * 64]``.  The kernel is exact softmax attention with 3xTF32
tensor-core products and an online softmax, so nothing of size N^2 is allocated: at 1080p (N = 10769 tokens) the
reference's two dense fp32 ``[B, 6, N, N]`` tensors take 2.8 GB each, at 4K (N = 45420) 49.5 GB each.

``get_intermediate_layers(backbone, x, n, reshape, return_class_token, norm)`` has the signature and return structure
of ``DinoVisionTransformer.get_intermediate_layers`` (dinov2.py:789-813), but runs only blocks 0..max(n) (the reference
runs all of them; later blocks cannot change earlier outputs) and uses the kernel for each block's attention core.  The
token-wise layers are the backbone's own modules, called in the reference's order: ``prepare_tokens_with_masks``,
``norm1``, ``attn.qkv``, ``attn.proj``, ``attn.proj_drop``, ``ls1``, ``norm2``, ``mlp``, ``ls2``, the residual adds and the
final ``norm``.

With ``blocks=True`` the token-wise layers run on ``csrc/vit.cu`` too, so the whole call is this project's kernels:
one launch for the token assembly (patch convolution as a GEMM, class, register and position embedding), per block
the fused ``norm1`` + ``qkv``, the attention (two launches), ``proj`` + ``ls1`` + residual, ``norm2`` + ``fc1`` + GELU and
``fc2`` + ``ls2`` + residual, and one launch per taken block for the final ``norm`` in the layout asked for
(``reshape=True`` writes ``[B, C, h, w]`` directly).  Products are 3xTF32; the result does not depend on torch's TF32
switches.  The interpolated position embedding is the backbone's own ``interpolate_pos_encoding``, computed once per
grid size and ``pos_embed`` version.

There is no PyTorch fallback: unsupported input raises (``supported`` tells beforehand).
``wildgaussians_fused.enable(model, dino=True)`` routes the uncertainty backbone's own ``get_intermediate_layers`` here
where the input allows it, and ``enable(model, dino_blocks=True)`` with ``blocks=True`` first.
"""
from __future__ import annotations

import sys

import torch

from diff_gaussian_rasterization import _C

__all__ = ["attention", "get_intermediate_layers", "supported"]

_lib = _C._lib
HEAD_DIM = 64


def _unsupported_qkv(qkv, num_heads) -> str | None:
    if not isinstance(qkv, torch.Tensor):
        return "expects a tensor"
    if not qkv.is_cuda:
        return "needs a CUDA tensor; there is no CPU path"
    if qkv.dtype != torch.float32:
        return "supports fp32 only"
    if not (isinstance(num_heads, int) and not isinstance(num_heads, bool) and num_heads >= 1):
        return "expects an integer num_heads >= 1"
    if qkv.dim() != 3 or qkv.shape[2] != 3 * num_heads * HEAD_DIM:
        return f"expects [B, N, 3 * {num_heads} * {HEAD_DIM}], got {tuple(qkv.shape)}"
    if qkv.shape[0] < 1 or qkv.shape[1] < 1:
        return "expects B >= 1 and N >= 1"
    if qkv.shape[0] > 65535 or num_heads > 65535 or qkv.shape[1] >= 2 ** 31:
        return "batch, token or head count too large"
    if torch.is_grad_enabled() and qkv.requires_grad:
        return "computes no gradient; qkv must not require one"
    return None


def attention(qkv, num_heads):
    """softmax((q / 8) k^T) v of every head, heads concatenated: ``[B, N, num_heads * 64]``; raises on unsupported input."""
    why = _unsupported_qkv(qkv, num_heads)
    if why is not None:
        raise RuntimeError("fused_dino.attention " + why)
    qkv = qkv.detach().contiguous()
    if qkv.data_ptr() % 16:
        qkv = qkv.clone()
    B, N, _ = qkv.shape
    dev = qkv.device
    with torch.cuda.device(dev):
        nbytes = _lib.gsr_attention_scratch_bytes(B, N, num_heads)
        scratch = torch.empty(((nbytes + 3) // 4,), dtype=torch.float32, device=dev)
        out = torch.empty((B, N, num_heads * HEAD_DIM), dtype=torch.float32, device=dev)
        _C._check(_lib.gsr_attention_forward(B, N, num_heads, qkv.data_ptr(), out.data_ptr(), scratch.data_ptr(),
                                             torch.cuda.current_stream(dev).cuda_stream), "gsr_attention_forward")
    return out


def _blocks_to_take(backbone, n):
    """The block indices the reference collects for ``n``, in block order; None where the reference's own assertion
    would fail (an index out of range, a repeated index) or it would collect nothing."""
    total = len(backbone.blocks)
    try:
        wanted = range(total - n, total) if isinstance(n, int) else n
        take = [i for i in range(total) if i in wanted]
        if len(take) != len(wanted):
            return None
    except TypeError:
        return None
    return take or None


def _unsupported(backbone, x, n) -> str | None:
    if not isinstance(x, torch.Tensor) or x.dim() != 4:
        return "expects a [B, 3, H, W] tensor"
    if not x.is_cuda:
        return "needs a CUDA tensor; there is no CPU path"
    if x.dtype != torch.float32:
        return "supports fp32 only"
    if getattr(backbone, "chunked_blocks", True):
        return "does not support chunked blocks"
    if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in backbone.parameters())):
        return "computes no gradient"
    take = _blocks_to_take(backbone, n)
    if take is None:
        return f"n={n!r} selects no valid set of blocks"
    m = sys.modules.get(type(backbone).__module__)
    attn_types = tuple(getattr(m, k) for k in ("Attention", "MemEffAttention") if hasattr(m, k))
    block_types = tuple(getattr(m, k) for k in ("Block", "NestedTensorBlock") if hasattr(m, k))
    for blk in backbone.blocks[:take[-1] + 1]:
        if type(blk) not in block_types or type(blk.attn) not in attn_types:
            return "supports the reference's Block and Attention / MemEffAttention only"
        a = blk.attn
        if a.qkv.in_features != HEAD_DIM * a.num_heads or a.qkv.out_features != 3 * a.qkv.in_features:
            return f"supports head dimension {HEAD_DIM} only"
        if blk.training and (blk.sample_drop_ratio > 0 or
                             any(isinstance(d, torch.nn.Dropout) and d.p > 0 for d in blk.modules())):
            return "does not support active dropout or drop-path"
    return None


def _unsupported_blocks(backbone, x, n) -> str | None:
    """What ``blocks=True`` needs beyond ``_unsupported``: the reference's ViT-S/B/L layout, with or without registers."""
    m = sys.modules.get(type(backbone).__module__)
    mlp_type, ls_type = getattr(m, "Mlp", None), getattr(m, "LayerScale", None)
    C = getattr(backbone, "embed_dim", None)
    if not isinstance(C, int) or C % 64 or not 64 <= C <= MAX_C:
        return f"supports embedding widths that are multiples of 64 up to {MAX_C} only"
    pe = getattr(backbone, "patch_embed", None)
    p = getattr(backbone, "patch_size", None)
    conv = getattr(pe, "proj", None)
    if (not isinstance(conv, torch.nn.Conv2d) or not isinstance(pe.norm, torch.nn.Identity) or conv.bias is None
            or conv.in_channels != 3 or conv.out_channels != C or conv.kernel_size != (p, p) or conv.stride != (p, p)
            or conv.padding != (0, 0) or conv.dilation != (1, 1) or conv.groups != 1 or p % 2):
        return "supports a bias-carrying p x p stride-p patch convolution (p even) without a patch-embed norm only"
    if x.shape[1] != 3 or x.shape[2] % p or x.shape[3] % p:
        return f"expects a [B, 3, H, W] input with H and W multiples of the patch size {p}"
    if x.shape[0] > 65535 or x.shape[0] * (1 + backbone.num_register_tokens + (x.shape[2] // p) * (x.shape[3] // p)) >= 2 ** 31:
        return "batch or token count too large"
    norms = [backbone.norm]
    linears = [conv]
    for blk in backbone.blocks[:_blocks_to_take(backbone, n)[-1] + 1]:
        mlp = blk.mlp
        if type(mlp) is not mlp_type or type(mlp.act) is not torch.nn.GELU or mlp.act.approximate != "none":
            return "supports the reference's Mlp with exact GELU only"
        if mlp.fc1.out_features != 4 * C or mlp.fc1.in_features != C or mlp.fc2.out_features != C:
            return "supports an Mlp of hidden width 4C only"
        for ls in (blk.ls1, blk.ls2):
            if not (type(ls) is ls_type or isinstance(ls, torch.nn.Identity)):
                return "supports LayerScale or Identity as ls1 / ls2 only"
        norms += [blk.norm1, blk.norm2]
        linears += [blk.attn.qkv, blk.attn.proj, mlp.fc1, mlp.fc2]
    for ln in norms:
        if type(ln) is not torch.nn.LayerNorm or not ln.elementwise_affine or ln.bias is None or \
                tuple(ln.normalized_shape) != (C,) or not ln.eps > 0:
            return "supports affine nn.LayerNorm over the embedding only"
    if any(lin.bias is None for lin in linears):
        return "supports Linear layers with a bias only"
    params = [backbone.cls_token, backbone.pos_embed] + \
        ([backbone.register_tokens] if backbone.num_register_tokens else []) + \
        [t for mod in norms + linears for t in (mod.weight, mod.bias)] + \
        [ls.gamma for blk in backbone.blocks[:_blocks_to_take(backbone, n)[-1] + 1] for ls in (blk.ls1, blk.ls2)
         if type(ls) is ls_type]
    if any(t.dtype != torch.float32 or t.device != x.device for t in params):
        return "supports fp32 weights on the input's device only"
    return None


# Above this many tokens per call (B * (1 + R + patches)) the token-wise GEMMs of ``blocks=True`` are slower than
# cuBLAS's fp32 GEMMs.  On one H100 80GB HBM3 at 700 W, with the random ViT-S/14 with registers of tools/bench_vit.py,
# ``blocks=True`` took 3.36 ms against 4.08 ms with ``blocks=False`` at 2455 tokens and 8.28 ms against 6.67 ms at
# 4905 tokens (DESIGN.md section 6).  The difference is linear in the token count (the attention is the same kernel on
# both paths) and crosses zero near 3200 tokens between those two measurements.
BLOCKS_MAX_TOKENS = 3072


def blocks_preferred(backbone, x) -> bool:
    """True where ``blocks=True`` measured faster than ``blocks=False`` for this input's token count."""
    p = backbone.patch_size
    return x.shape[0] * (1 + backbone.num_register_tokens + (x.shape[2] // p) * (x.shape[3] // p)) <= BLOCKS_MAX_TOKENS


def supported(backbone, x, n=1, *, blocks=False) -> bool:
    """True when ``get_intermediate_layers(backbone, x, n, ..., blocks=blocks)`` accepts these inputs."""
    why = _unsupported(backbone, x, n)
    if why is None and blocks:
        why = _unsupported_blocks(backbone, x, n)
    return why is None


def _attention_block(blk, x):
    """``Block.forward`` of dinov2.py:328-353 without drop-path, with the fused attention core."""
    a = blk.attn
    y = blk.norm1(x)
    y = a.proj_drop(a.proj(attention(a.qkv(y), a.num_heads)))
    x = x + blk.ls1(y)
    return x + blk.ls2(blk.mlp(blk.norm2(x)))


def get_intermediate_layers(backbone, x, n=1, reshape=False, return_class_token=False, norm=True, *, blocks=False):
    """Drop-in for ``backbone.get_intermediate_layers`` (dinov2.py:789-813) on supported input; raises otherwise.  With
    ``blocks``, every layer runs on this project's kernels (``csrc/vit.cu`` and the attention)."""
    why = _unsupported(backbone, x, n)
    if why is None and blocks:
        why = _unsupported_blocks(backbone, x, n)
    if why is not None:
        raise RuntimeError("fused_dino.get_intermediate_layers " + why)
    take = _blocks_to_take(backbone, n)
    if blocks:
        return _vit_layers(backbone, x, take, reshape, return_class_token, norm)
    tokens = backbone.prepare_tokens_with_masks(x)
    layers = []
    for i in range(take[-1] + 1):
        tokens = _attention_block(backbone.blocks[i], tokens)
        if i in take:
            layers.append(tokens)
    if norm:
        layers = [backbone.norm(t) for t in layers]
    cls = [t[:, 0] for t in layers]
    layers = [t[:, 1 + backbone.num_register_tokens:] for t in layers]
    if reshape:
        B, _, w, h = x.shape
        p = backbone.patch_size
        layers = [t.reshape(B, w // p, h // p, -1).permute(0, 3, 1, 2).contiguous() for t in layers]
    if return_class_token:
        return tuple(zip(layers, cls))
    return tuple(layers)


# ---------------------------------------------------------------------------------------------------- blocks=True

MAX_C = 1024
_LN_BIAS, _LN_GELU, _RESIDUAL = 0, 1, 2          # gsr_vit_linear ops (include/gsrast.h)
_LAYOUT_TOKENS, _LAYOUT_CHANNELS = 0, 1
_pos_cache: dict = {}


def _ptr(t):
    return None if t is None else t.data_ptr()


def _dev(t):
    """``t`` as the kernels read it: detached, contiguous and 16-byte aligned (a copy only where it is not).  Keep the
    result in a variable until the launch that reads it is enqueued: a dropped copy returns to the caching allocator at
    once, and the next copy on the stream may take its memory before the kernel runs."""
    t = t.detach().contiguous()
    return t.clone() if t.data_ptr() % 16 else t


def _pos_embed(backbone, gh, gw):
    """``interpolate_pos_encoding`` for a gh x gw grid, [1 + gh * gw, C], computed by the backbone itself once per grid
    size and ``pos_embed`` tensor and version (an in-place edit or ``load_state_dict`` bumps the version)."""
    pe = backbone.pos_embed
    key = (id(backbone), gh, gw)
    hit = _pos_cache.get(key)
    if hit is not None and hit[0] is pe and hit[1] == pe._version:
        return hit[2]
    p = backbone.patch_size
    like = pe.new_zeros(()).expand(1, 1 + gh * gw, pe.shape[-1])       # only its shape and dtype are read
    with torch.no_grad():
        pos = _dev(backbone.interpolate_pos_encoding(like, gh * p, gw * p).reshape(1 + gh * gw, -1))
        if pos.data_ptr() == pe.data_ptr():
            pos = pos.clone()                                            # the cache keeps its own copy
    if len(_pos_cache) >= 64:
        _pos_cache.clear()
    _pos_cache[key] = (pe, pe._version, pos)
    return pos


def _vit_layers(backbone, x, take, reshape, return_class_token, norm):
    B, _, H, W = x.shape
    p, C, R = backbone.patch_size, backbone.embed_dim, backbone.num_register_tokens
    gh, gw = H // p, W // p
    P = gh * gw
    T = 1 + R + P
    M = B * T
    dev = x.device
    f32 = dict(dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream(dev).cuda_stream
        pos = _pos_embed(backbone, gh, gw)
        conv = backbone.patch_embed.proj
        tokens = torch.empty((B, T, C), **f32)
        xd, cw, cb, cls_tok = _dev(x), _dev(conv.weight), _dev(conv.bias), _dev(backbone.cls_token)
        reg = _dev(backbone.register_tokens) if R else None
        _C._check(_lib.gsr_vit_tokens(B, H, W, C, p, R, xd.data_ptr(), cw.data_ptr(), cb.data_ptr(), cls_tok.data_ptr(),
                                      _ptr(reg), pos.data_ptr(), tokens.data_ptr(), st), "gsr_vit_tokens")
        del xd, cw, cb, cls_tok, reg

        def linear(op, src, mod, out, ln=None, gamma=None, resid=None):
            lw, lb, eps = (_dev(ln.weight), _dev(ln.bias), float(ln.eps)) if ln is not None else (None, None, 0.0)
            w, b = _dev(mod.weight), _dev(mod.bias)
            _C._check(_lib.gsr_vit_linear(op, M, mod.in_features, mod.out_features, src.data_ptr(), _ptr(lw), _ptr(lb), eps,
                                          w.data_ptr(), b.data_ptr(), _ptr(gamma), _ptr(resid), out.data_ptr(), st),
                      "gsr_vit_linear")

        layers = []
        for i in range(take[-1] + 1):
            blk = backbone.blocks[i]
            a = blk.attn
            g1, g2 = (_dev(ls.gamma) if hasattr(ls, "gamma") else None for ls in (blk.ls1, blk.ls2))
            qkv = torch.empty((B, T, 3 * C), **f32)
            linear(_LN_BIAS, tokens, a.qkv, qkv, ln=blk.norm1)
            att = attention(qkv, a.num_heads)
            del qkv
            nxt = torch.empty((B, T, C), **f32)
            linear(_RESIDUAL, att, a.proj, nxt, gamma=g1, resid=tokens)
            del att
            hidden = torch.empty((B, T, blk.mlp.fc1.out_features), **f32)
            linear(_LN_GELU, nxt, blk.mlp.fc1, hidden, ln=blk.norm2)
            linear(_RESIDUAL, hidden, blk.mlp.fc2, nxt, gamma=g2, resid=nxt)          # in place
            del hidden
            tokens = nxt
            if i in take:
                layers.append(tokens)

        nw = _dev(backbone.norm.weight) if norm else None
        nb = _dev(backbone.norm.bias) if norm else None
        eps = float(backbone.norm.eps) if norm else 0.0
        outs, cls = [], []
        for t in layers:
            feat = torch.empty((B, C, gh, gw) if reshape else (B, P, C), **f32)
            c = torch.empty((B, C), **f32) if return_class_token else None
            _C._check(_lib.gsr_vit_output(B, T, C, R, _LAYOUT_CHANNELS if reshape else _LAYOUT_TOKENS, t.data_ptr(),
                                          _ptr(nw), _ptr(nb), eps, feat.data_ptr(), _ptr(c), st), "gsr_vit_output")
            outs.append(feat)
            cls.append(c)
    if return_class_token:
        return tuple(zip(outs, cls))
    return tuple(outs)
