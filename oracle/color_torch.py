"""TEST INFRASTRUCTURE -- torch restatement (any dtype, autograd-capable) of wild-gaussians' per-Gaussian colour path,
the oracle of the fused colour op (SURVEY.md 8f-2).  Only tests/ and bench.py's comparison leg may import this module.

Statements restated (paths relative to /root/reference/wildgaussians/):
  method.py:1063-1066,1570   features = cat(features_dc, features_rest).clamp_max(1)
  method.py:1572             dir = normalize(means3D - campos)
  method.py:1574-1579        raw = clamp_min(eval_sh(deg, features.view(-1,16,3).transpose(1,2), dir) + 0.5, 0)
  method.py:889-900          EmbeddingModel.forward (appearance_model_sh = False)
  method.py:1589-1595        toned = clamp_min(eval_sh(deg, clamp_max(mlp_out,1).view(-1,16,3).transpose(1,2).clamp_max(1), dir) + 0.5, 0)
  method.py:493-548          eval_sh
Pinned by tests/golden/colors_*.npz (outputs and autograd gradients of the reference itself): tests/test_color_oracle.py.
"""
import torch

C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435)


def eval_sh(deg, sh, dirs):
    """sh [P, 3, 16], dirs [P, 3] -> [P, 3]"""
    res = C0 * sh[..., 0]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        res = res - C1 * y * sh[..., 1] + C1 * z * sh[..., 2] - C1 * x * sh[..., 3]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            res = (res + C2[0] * xy * sh[..., 4] + C2[1] * yz * sh[..., 5] + C2[2] * (2.0 * zz - xx - yy) * sh[..., 6]
                   + C2[3] * xz * sh[..., 7] + C2[4] * (xx - yy) * sh[..., 8])
            if deg > 2:
                res = (res + C3[0] * y * (3 * xx - yy) * sh[..., 9] + C3[1] * xy * z * sh[..., 10]
                       + C3[2] * y * (4 * zz - xx - yy) * sh[..., 11] + C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[..., 12]
                       + C3[4] * x * (4 * zz - xx - yy) * sh[..., 13] + C3[5] * z * (xx - yy) * sh[..., 14]
                       + C3[6] * x * (xx - 3 * yy) * sh[..., 15])
    return res


def _bf16(x):
    """Round to bfloat16 and back (straight-through gradient): how csrc/appearance.cu feeds the tensor cores."""
    return x.to(torch.bfloat16).to(x.dtype)


def mlp_bf16(color, embeddings, app_embedding, W1, b1, W2, b2, W3, b3):
    """The 59 -> 128 -> 128 -> 6 MLP with the OPERAND ROUNDING of csrc/appearance.cu (fp32 tensors): inputs, weights
    and hidden activations rounded to bf16, products exact and sums in fp32 (wgmma bf16), biases kept to
    ~2^-17 (bias_hi + bias_lo), the image embedding folded into the first bias in fp32.  Same function as the fp32 MLP
    up to that rounding -- but its ReLU masks are those of the rounded network, which is what a gradient check of the
    kernel needs (a mask flipped by rounding changes a gradient entry by O(1): the gradient of a network with kinks
    is not continuous in the weights' precision)."""
    nd = color.shape[-1] + embeddings.shape[-1]
    bias1 = b1 + W1[:, nd:] @ app_embedding
    x = _bf16(torch.cat((color, embeddings), dim=-1))
    h = _bf16(torch.relu(x @ _bf16(W1[:, :nd]).T + bias1))
    h = _bf16(torch.relu(h @ _bf16(W2).T + b2))
    return h @ _bf16(W3).T + b3


def colors(features_dc, features_rest, embeddings, app_embedding, W1, b1, W2, b2, W3, b3, means3D, campos, deg,
           emulate_bf16=False):
    """(raw [P,3], toned [P,3]) exactly as GaussianModel._render_internal computes them (emulate_bf16: with the MLP
    operand rounding of the CUDA kernel, see mlp_bf16)."""
    P = features_dc.shape[0]
    features = torch.cat((features_dc, features_rest), dim=-1).clamp_max(1.0)
    dirs = torch.nn.functional.normalize(means3D - campos[None].expand(P, 3), dim=1)
    raw = torch.clamp_min(eval_sh(deg, features.view(-1, 16, 3).transpose(1, 2), dirs) + 0.5, 0.0)
    if emulate_bf16:
        out = mlp_bf16(features[..., :3], embeddings, app_embedding, W1, b1, W2, b2, W3, b3) * 0.01
    else:
        inp = torch.cat((features[..., :3], embeddings, app_embedding[None].expand(P, -1)), dim=-1)
        h = torch.relu(inp @ W1.T + b1)
        h = torch.relu(h @ W2.T + b2)
        out = (h @ W3.T + b3) * 0.01
    offset, mul = out[:, :3], out[:, 3:]
    offset = torch.cat((offset / C0, torch.zeros_like(features[..., 3:])), dim=-1)
    toned_f = (features * mul.repeat(1, 16) + offset).clamp_max(1.0)
    sh = toned_f.view(-1, 16, 3).transpose(1, 2).contiguous().clamp_max(1.0)
    toned = torch.clamp_min(eval_sh(deg, sh, dirs) + 0.5, 0.0)
    return raw, toned
