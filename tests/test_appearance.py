"""GPU parity of the fused colour op (csrc/appearance.cu, wgmma) against (a) the golden vectors produced by the
reference itself (tests/golden/colors_*.npz: outputs + autograd gradients of wildgaussians' EmbeddingModel / eval_sh in
fp64) and (b) the torch restatement oracle/color_torch.py in fp32 on larger seeded inputs (raw + toned colours, every
gradient incl. the mean through the view direction, ragged last tile).

Bars.  The MLP runs with bf16 operands (fp32 accumulation); everything else is fp32.
  * colours: within 1e-3 absolute of the fp32 / fp64 reference (measured ~1e-5: the MLP output is scaled by 0.01);
    raw colours (no MLP involved) within 1e-5.
  * gradients: compared against the torch oracle evaluated WITH THE KERNEL'S OPERAND ROUNDING (oracle/color_torch.py,
    emulate_bf16=True): weight / bias / image-embedding gradients (sums over all Gaussians) entry-wise at 5e-2 of the
    tensor's largest magnitude and cosine >= 0.999; per-Gaussian gradients row-wise -- 99.5 % of the rows within 2e-2
    (a row is one Gaussian; the few rows beyond are Gaussians with a ReLU pre-activation within float rounding of zero,
    whose mask differs between the tensor core's and cuBLAS's summation order) and cosine >= 0.999.  A network with ReLU kinks has a gradient that
    is discontinuous in the precision of its weights: rounding flips ~0.3 % of the (Gaussian, neuron) masks and each
    flip changes a gradient entry by O(1), so the gradient OF THE ROUNDED NETWORK -- which is what the kernel computes,
    exactly like any bf16 autocast training step -- differs from the fp32 network's by ~5 % in max-norm while
    agreeing in direction.  Against the fp32 / fp64 reference the test therefore asserts direction and size (cosine
    >= 0.99, norm ratio within 3 %) instead of an entry-wise bound.
These bars pin the op to the reference goldens and to the fp32 network.  The entry-wise bars are in
tests/test_colour_op_exact.py: every colour and every per-Gaussian gradient of every row, and every weight, bias and
image-embedding gradient entry, within an a-priori bound of an fp64 oracle of the rounded network
(oracle/color_exact.py), on lattice, random and golden scenes, at the tile / warpgroup / CTA-boundary shapes.
"""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
COL_TOL, GRAD_TOL = 1e-3, 2e-2


def _mlp(W1, b1, W2, b2, W3, b3, dev):
    mlp = torch.nn.Sequential(torch.nn.Linear(59, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128), torch.nn.ReLU(),
                              torch.nn.Linear(128, 6)).to(dev)
    with torch.no_grad():
        for lin, W, b in ((mlp[0], W1, b1), (mlp[2], W2, b2), (mlp[4], W3, b3)):
            lin.weight.copy_(W); lin.bias.copy_(b)
    return mlp


def _cos_norm(a, b):
    a, b = a.detach().double().flatten(), b.detach().double().flatten()
    na, nb = float(a.norm()), float(b.norm())
    if nb == 0.0:
        return 1.0, (1.0 if na == 0.0 else float("inf"))
    return float(a @ b) / (na * nb + 1e-300), na / nb


def _rel(a, b):
    if b is None:                     # torch leaves an input that cannot influence the output without a gradient
        b = torch.zeros_like(a)
    a, b = a.detach(), b.detach()
    return float((a - b).abs().max()) / (float(b.abs().max()) + 1e-30)


@pytest.mark.parametrize("name", ["colors_deg3", "colors_deg1"])
def test_fused_colors_against_reference_golden(name):
    import fused_colors as fc
    dev = torch.device("cuda:0")
    d = dict(np.load(os.path.join(GOLD, name + ".npz")))
    T = lambda k: torch.tensor(d[k], dtype=torch.float32, device=dev)
    feats = T("features")
    dc, rest = feats[:, :3].contiguous().requires_grad_(True), feats[:, 3:].contiguous().requires_grad_(True)
    gemb, aemb = T("gembedding").requires_grad_(True), T("aembedding").requires_grad_(True)
    mlp = _mlp(T("W1"), T("b1"), T("W2"), T("b2"), T("W3"), T("b3"), dev)
    raw, toned = fc.fused_colors(dc, rest, gemb, aemb, mlp, T("means3D"), T("campos"), int(d["active_deg"]))
    err = float((toned.detach() - T("colors")).abs().max())
    assert err < COL_TOL, err
    (toned * T("dL_dcolors")).sum().backward()
    torch.cuda.synchronize()
    g_feat = torch.cat([dc.grad, rest.grad], dim=1)
    worst = {"features": _rel(g_feat, T("g_features")), "gembedding": _rel(gemb.grad, T("g_gembedding")),
             "aembedding": _rel(aemb.grad, T("g_aembedding"))}
    for i, lin in zip((1, 2, 3), (mlp[0], mlp[2], mlp[4])):
        worst[f"W{i}"] = _rel(lin.weight.grad, T(f"g_W{i}"))
        worst[f"b{i}"] = _rel(lin.bias.grad, T(f"g_b{i}"))
    pairs = {"features": (g_feat, T("g_features")), "gembedding": (gemb.grad, T("g_gembedding")),
             "aembedding": (aemb.grad, T("g_aembedding"))}
    for i, lin in zip((1, 2, 3), (mlp[0], mlp[2], mlp[4])):
        pairs[f"W{i}"] = (lin.weight.grad, T(f"g_W{i}")); pairs[f"b{i}"] = (lin.bias.grad, T(f"g_b{i}"))
    stats = {k: _cos_norm(a, b) for k, (a, b) in pairs.items()}
    print(name, "colour err", err, "max-norm rel err", worst, "(cosine, norm ratio)", stats)
    for k, (c, r) in stats.items():
        assert c >= 0.99 and abs(r - 1.0) <= 0.03, (k, c, r)
    for k in ("W3", "b3"):            # the last layer sees no ReLU mask downstream: entry-wise too
        assert worst[k] < GRAD_TOL, (k, worst[k])


@pytest.mark.parametrize("P,deg", [(100_037, 3), (4_096, 2), (77, 0)])
def test_fused_colors_against_torch_oracle(P, deg):
    import fused_colors as fc
    from oracle import color_torch as ct
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(1000 + P)
    R = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(dev)
    dc = ((torch.rand(P, 3, generator=g) * 1.6 - 0.9) / 0.28209479).to(dev)          # some colours clamp at 0, some features > 1
    rest, gemb, aemb = R(P, 45, scale=0.3), R(P, 24, scale=0.5), R(32, scale=0.5)
    means, campos = R(P, 3, scale=2.0), torch.tensor([0.1, -0.2, 0.3], device=dev)
    torch.manual_seed(P)
    mlp = torch.nn.Sequential(torch.nn.Linear(59, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128), torch.nn.ReLU(),
                              torch.nn.Linear(128, 6)).to(dev)
    with torch.no_grad():
        # a trained model has mul ~ 1 (tests/golden/make_golden_colors.py); 0.8 keeps `features * mul` of the features that
        # were clamped to exactly 1 away from the second clamp at 1 (a kink hit by construction would be a coin toss)
        mlp[4].bias[3:] = 80.0
    dLr, dLt = R(P, 3), R(P, 3)
    leaves = [t.clone().requires_grad_(True) for t in (dc, rest, gemb, aemb, means)]
    raw, toned = fc.fused_colors(leaves[0], leaves[1], leaves[2], leaves[3], mlp, leaves[4], campos, deg)
    ((raw * dLr).sum() + (toned * dLt).sum()).backward()
    ours = [t.grad.clone() for t in leaves] + [p.grad.clone() for p in mlp.parameters()]
    for p in mlp.parameters():
        p.grad = None
    leaves2 = [t.clone().requires_grad_(True) for t in (dc, rest, gemb, aemb, means)]
    lin = [mlp[0], mlp[2], mlp[4]]
    raw2, toned2 = ct.colors(leaves2[0], leaves2[1], leaves2[2], leaves2[3], lin[0].weight, lin[0].bias, lin[1].weight,
                             lin[1].bias, lin[2].weight, lin[2].bias, leaves2[4], campos, deg, emulate_bf16=True)
    ((raw2 * dLr).sum() + (toned2 * dLt).sum()).backward()
    ref = [t.grad for t in leaves2] + [p.grad for p in mlp.parameters()]
    # ... and the plain fp32 network, for the colour bar and the direction / size of the gradients
    for p in mlp.parameters():
        p.grad = None
    leaves3 = [t.clone().requires_grad_(True) for t in (dc, rest, gemb, aemb, means)]
    raw3, toned3 = ct.colors(leaves3[0], leaves3[1], leaves3[2], leaves3[3], lin[0].weight, lin[0].bias, lin[1].weight,
                             lin[1].bias, lin[2].weight, lin[2].bias, leaves3[4], campos, deg)
    ((raw3 * dLr).sum() + (toned3 * dLt).sum()).backward()
    ref32 = [t.grad for t in leaves3] + [p.grad for p in mlp.parameters()]
    torch.cuda.synchronize()
    assert float((toned - toned3).detach().abs().max()) < COL_TOL
    e_raw, e_toned = float((raw - raw2).detach().abs().max()), float((toned - toned2).detach().abs().max())
    assert e_raw < 1e-5, e_raw                                   # no MLP involved: fp32 on both sides
    assert e_toned < COL_TOL, e_toned
    names = ["features_dc", "features_rest", "embeddings", "app_embedding", "means3D", "W1", "b1", "W2", "b2", "W3", "b3"]
    worst = {n: _rel(a, b) for n, a, b in zip(names, ours, ref)}
    stats = {n: _cos_norm(a, torch.zeros_like(a) if b is None else b) for n, a, b in zip(names, ours, ref32)}
    print(P, deg, "raw", e_raw, "toned (vs rounded oracle)", e_toned, "max-norm rel err vs rounded oracle", worst,
          "(cosine, norm ratio) vs fp32", stats)
    for n, a, b in zip(names, ours, ref):
        b = torch.zeros_like(a) if b is None else b
        c, r = _cos_norm(a, b)
        assert c >= 0.999 and abs(r - 1.0) <= 0.01, (n, "vs rounded oracle", c, r)
        if a.dim() == 2 and a.shape[0] == P:                     # per-Gaussian tensor: row-wise
            rn = b.detach().norm(dim=1)
            row_err = (a.detach() - b.detach()).norm(dim=1) / (rn + 1e-3 * float(rn.max()) + 1e-30)
            q = float(torch.quantile(row_err.float().cpu(), 0.995)) if P >= 1000 else float(row_err.median())
            assert q < GRAD_TOL, (n, "row-wise 99.5 % quantile", q)
        else:
            assert worst[n] < 5e-2, (n, worst[n])
    for n, (c, r) in stats.items():
        assert c >= 0.99 and abs(r - 1.0) <= 0.03, (n, c, r)
    assert fc.last_status_ok()                        # no barrier wait timed out inside the kernels


def test_fused_colors_rejects_other_shapes_and_cpu():
    import fused_colors as fc
    dev = torch.device("cuda:0")
    mlp = torch.nn.Sequential(torch.nn.Linear(59, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128), torch.nn.ReLU(),
                              torch.nn.Linear(128, 6)).to(dev)
    z = lambda *s: torch.zeros(*s, device=dev)
    with pytest.raises(RuntimeError, match="default shapes"):
        fc.fused_colors(z(10, 3), z(10, 24), z(10, 24), z(32), mlp, z(10, 3), z(3), 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        fc.fused_colors(torch.zeros(10, 3), torch.zeros(10, 45), torch.zeros(10, 24), torch.zeros(32), mlp.cpu(),
                        torch.zeros(10, 3), torch.zeros(3), 3)


def test_fused_activations_against_torch_statements():
    """gsr_gaussian_activations_{forward,backward} against the statements of GaussianModel.get_gaussians
    (method.py:1060-1086) in torch fp32: outputs and gradients within 1e-5 / 1e-4 relative."""
    import fused_colors as fc
    dev = torch.device("cuda:0")
    P = 200_003
    g = torch.Generator().manual_seed(9)
    s = (torch.randn(P, 3, generator=g) * 0.7 - 3.0).to(dev)
    o = (torch.randn(P, 1, generator=g) * 2.0).to(dev)
    r = torch.randn(P, 4, generator=g).to(dev)
    f = (torch.rand(P, 1, generator=g) * 0.05).to(dev)
    gs, go, gr = (torch.randn(*t.shape, generator=g).to(dev) for t in (s, o, r))

    def ref(s, o, r):
        rot = torch.nn.functional.normalize(r)
        raw = torch.exp(s)
        scales = (torch.square(raw) + torch.square(f)).sqrt()
        coef = torch.sqrt(torch.square(raw).prod(dim=1) / (torch.square(raw) + torch.square(f)).prod(dim=1))
        return scales, torch.sigmoid(o) * coef[..., None], rot

    res = []
    for fn in (lambda a, b, c: fc.fused_activations(a, b, c, f), ref):
        L = [t.clone().requires_grad_(True) for t in (s, o, r)]
        out = fn(*L)
        torch.autograd.backward(list(out), [gs, go, gr])
        res.append(([x.detach() for x in out], [t.grad for t in L]))
    for a, b in zip(res[0][0], res[1][0]):
        assert float((a - b).abs().max()) < 1e-5 * max(1.0, float(b.abs().max()))
    for a, b in zip(res[0][1], res[1][1]):
        assert float((a - b).abs().max()) < 1e-4 * max(1.0, float(b.abs().max()))

    # Edge rows, against the same statements in float64 and row by row (their gradients reach 1e12):
    #  * quaternions below F.normalize's eps (|q| ~ 5.5e-13, and exactly 0): x / clamp_min(|x|, eps) has gradient g / eps
    #    there, the clamp passing nothing to the norm -- not the projected (g - n (n.g)) / |q|;
    #  * filter_3D == 0 with scale products in the fp32 denormal range (raw^2 ~ 1e-13 .. 1e-18): coef == 1 exactly, and
    #    its gradient is 0 (the fp32 torch statements give NaN and -inf there: prod^2 underflows);
    #  * saturated sigmoids (|opacity| = 40, 100).
    s_e = torch.tensor([[-15.0, -15.0, -15.0], [-20.0, -14.0, -16.0], [-1.0, -2.0, -3.0], [-15.0, -1.0, -2.0],
                        [-0.5, -0.7, -0.2], [-2.0, -2.0, -2.0]], device=dev)
    o_e = torch.tensor([[40.0], [-40.0], [-100.0], [100.0], [0.3], [-1.0]], device=dev)
    r_e = torch.tensor([[3e-13, -4e-13, 1e-13, 2e-13], [0.0, 0.0, 0.0, 0.0], [1.0, 2.0, 3.0, 4.0], [-1e-13, 0.0, 0.0, 0.0],
                        [3.0, -4.0, 1.0, 2.0], [0.0, 0.0, 0.0, 7e-13]], device=dev)
    f_e = torch.tensor([[0.0], [0.0], [0.0], [0.0], [1e-3], [0.0]], device=dev)
    g_e = [torch.randn(*t.shape, generator=g).to(dev) for t in (s_e, o_e, r_e)]

    def ref64(s, o, r):
        f64 = f_e.double()
        rot = torch.nn.functional.normalize(r)
        raw = torch.exp(s)
        scales = (torch.square(raw) + torch.square(f64)).sqrt()
        coef = torch.sqrt(torch.square(raw).prod(dim=1) / (torch.square(raw) + torch.square(f64)).prod(dim=1))
        return scales, torch.sigmoid(o) * coef[..., None], rot

    res = []
    for fn, dt in ((lambda a, b, c: fc.fused_activations(a, b, c, f_e), torch.float32), (ref64, torch.float64)):
        L = [t.to(dt).clone().requires_grad_(True) for t in (s_e, o_e, r_e)]
        out = fn(*L)
        torch.autograd.backward(list(out), [t.to(dt) for t in g_e])
        res.append(([x.detach().double() for x in out], [t.grad.double() for t in L]))
    for a, b in zip(res[0][0], res[1][0]):
        assert torch.isfinite(a).all()
        assert bool(((a - b).abs() <= 1e-5 * b.abs().amax(1, keepdim=True).clamp_min(1.0)).all()), (a, b)
    for a, b in zip(res[0][1], res[1][1]):
        assert torch.isfinite(a).all()
        assert bool(((a - b).abs() <= 1e-5 * b.abs().amax(1, keepdim=True) + 1e-12).all()), (a, b)
