"""TEST INFRASTRUCTURE -- float64 oracle of the DINOv2 backbone's attention core (wildgaussians/dinov2.py:224-233).

``attention(qkv, num_heads)`` restates, from the ``qkv`` Linear's output ``[B, N, 3 * H * D]`` to the input of ``proj``
``[B, N, H * D]``: split into q, k, v per head, ``q * D^-0.5``, ``q @ k^T``, ``softmax`` over the keys, ``@ v``, heads
concatenated.  It works in chunks of query rows, so its memory is O(chunk * N) rather than O(N^2) (45k tokens at 4K),
and ``rows`` restricts it to a subset of query rows.  ``dtype=torch.float32`` evaluates the same statements in fp32
(the reference's own rounding with TF32 off, the yardstick for the fused kernel's error).

``float64_backbone(backbone)`` is a float64 deep copy of a ``DinoVisionTransformer`` whose blocks use the chunked
oracle as their attention core: the reference's feature maps in float64 at 1080p and 4K with bounded memory.
"""
from __future__ import annotations

import copy
import types

import torch


def attention(qkv: torch.Tensor, num_heads: int, rows=None, chunk: int = 512, dtype=torch.float64) -> torch.Tensor:
    """[B, R, H * D] in ``dtype``: the attention output of query rows ``rows`` (all N when None)."""
    B, N, C3 = qkv.shape
    H = num_heads
    D = C3 // (3 * H)
    t = qkv.to(dtype).reshape(B, N, 3, H, D).permute(2, 0, 3, 1, 4)
    q, k, v = t[0] * D ** -0.5, t[1], t[2]
    idx = torch.arange(N, device=qkv.device) if rows is None else torch.as_tensor(rows, device=qkv.device)
    parts = []
    for i in range(0, idx.numel(), chunk):
        s = q[:, :, idx[i:i + chunk]] @ k.transpose(-2, -1)
        parts.append(s.softmax(dim=-1) @ v)
    o = torch.cat(parts, dim=2)                                   # [B, H, R, D]
    return o.transpose(1, 2).reshape(B, idx.numel(), H * D)


def _oracle_attention_forward(self, x):
    """``Attention.forward`` with the chunked oracle as its core (in the module's own dtype)."""
    y = attention(self.qkv(x), self.num_heads, dtype=x.dtype)
    return self.proj_drop(self.proj(y))


def float64_backbone(backbone):
    """A float64 copy of ``backbone`` whose attention modules run the chunked oracle."""
    b64 = copy.deepcopy(backbone).double()
    for blk in b64.blocks:
        blk.attn.forward = types.MethodType(_oracle_attention_forward, blk.attn)
    return b64
