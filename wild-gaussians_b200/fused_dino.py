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

There is no PyTorch fallback: unsupported input raises (``supported`` tells beforehand).
``wildgaussians_fused.enable(model, dino=True)`` routes the uncertainty backbone's own ``get_intermediate_layers`` here
where the input allows it.
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


def supported(backbone, x, n=1) -> bool:
    """True when ``get_intermediate_layers(backbone, x, n, ...)`` accepts these inputs."""
    return _unsupported(backbone, x, n) is None


def _attention_block(blk, x):
    """``Block.forward`` of dinov2.py:328-353 without drop-path, with the fused attention core."""
    a = blk.attn
    y = blk.norm1(x)
    y = a.proj_drop(a.proj(attention(a.qkv(y), a.num_heads)))
    x = x + blk.ls1(y)
    return x + blk.ls2(blk.mlp(blk.norm2(x)))


def get_intermediate_layers(backbone, x, n=1, reshape=False, return_class_token=False, norm=True):
    """Drop-in for ``backbone.get_intermediate_layers`` (dinov2.py:789-813) on supported input; raises otherwise."""
    why = _unsupported(backbone, x, n)
    if why is not None:
        raise RuntimeError("fused_dino.get_intermediate_layers " + why)
    take = _blocks_to_take(backbone, n)
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
