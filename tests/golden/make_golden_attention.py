"""Golden vectors of the DINOv2 backbone's attention core, produced by the REFERENCE ITSELF.

Runs where the reference checkout can be read (CPU torch is enough):
    python tests/golden/make_golden_attention.py
imports wildgaussians/dinov2.py unmodified and runs its ``Attention`` module (:203-236) in float64 on the CPU.  Its
``qkv`` Linear is replaced by a module that returns the stored input and its ``proj`` by the identity, so the module's
own ``forward`` computes exactly the core: reshape and permute, ``q * scale``, ``q @ k^T``, ``softmax``, ``@ v``, heads
concatenated.  The inputs are fp32 values on a bf16 grid (what the fp32 kernel sees; the zero low bits keep the files
small).  Each file holds qkv [B, N, 3 * H * 64] fp32, num_heads, the query rows stored, and out [B, rows, H * 64]
float64: a few tokens, an odd N with B = 2, N = 200 with 6 heads (40 rows stored, first and last included), and a sharp
case whose scores reach about +-40 with the row maxima of some rows among the last tile's keys.
"""
import os
import sys

import numpy as np
import torch

from make_golden_colors import import_reference


def grid(t):
    return t.to(torch.bfloat16).to(torch.float32)


def make_case(dinov2, B, N, H, seed, rows=None, sharp=False):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, N, 3, H, 64, generator=g, dtype=torch.float64)
    if sharp:
        qkv[:, :, :2] *= 2.9                                       # q and k: |q.k / 8| up to about 40
        qkv[:, N - 7:, 1] *= 1.6                                   # the largest keys sit in the last 64-key tile
    qkv = grid(qkv.reshape(B, N, 3 * H * 64))
    attn = dinov2.Attention(H * 64, num_heads=H).double()

    class Fixed(torch.nn.Module):
        def forward(self, x):
            return qkv.double()

    attn.qkv, attn.proj = Fixed(), torch.nn.Identity()
    with torch.no_grad():
        out = attn(torch.zeros(B, N, H * 64, dtype=torch.float64))
    rows = np.arange(N) if rows is None else np.asarray(rows)
    return dict(qkv=qkv.numpy(), num_heads=np.int64(H), rows=rows.astype(np.int64), out=out[:, rows].numpy())


CASES = {
    # name: (B, N, H, seed, stored rows, sharp)
    "attention_tiny": (1, 5, 1, 41, None, False),
    "attention_odd": (2, 37, 2, 42, None, False),
    "attention_n200": (1, 200, 6, 43, [0, 1, 2, 63, 64, 65, 127, 128, 129] + list(range(170, 200)), False),
    "attention_sharp": (1, 150, 1, 44, None, True),
}

if __name__ == "__main__":
    import_reference()
    import wildgaussians.dinov2 as dinov2
    here = os.path.dirname(os.path.abspath(__file__))
    for name, (B, N, H, seed, rows, sharp) in CASES.items():
        case = make_case(dinov2, B, N, H, seed, rows, sharp)
        q = case["qkv"].reshape(B, N, 3, H, 64).astype(np.float64)
        smax = float(np.abs(np.einsum("bnhd,bmhd->bhnm", q[:, :, 0] * 0.125, q[:, :, 1])).max())
        path = os.path.join(here, name + ".npz")
        np.savez_compressed(path, **case)
        print(name, (B, N, H), f"max |score| {smax:.1f}", f"{os.path.getsize(path) / 1024:.0f} KB", file=sys.stderr)
