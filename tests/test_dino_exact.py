"""The DINOv2 backbone kernels (csrc/vit.cu, csrc/attention.cu) under the fp64 oracle of ``oracle/vit_exact.py``: every
output entry of ``gsr_vit_linear`` (all three ops), ``gsr_vit_tokens``, ``gsr_attention_forward`` and ``gsr_vit_output``
within its a-priori bound, |kernel - S| <= B, at the tile edges and on adversarial inputs; the outputs that must be
exact (class and register tokens, ``norm=False`` copies, an attention row with one dominant key) bitwise.

CPU: S against the float64 module statements, an fp32 emulation of each kernel within B, and every corruption in
``MUTATIONS`` outside it.  GPU: the kernels themselves, the k-step premise of the model, and a replay of whole
backbones op by op, each op checked on its own fp32 input.  ``-s`` prints the worst |kernel - S| / B per op and family.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import attention_oracle as ao
from oracle import vit_exact as vx

WORST: dict = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if WORST:
        print("\nworst |kernel - S| / B per op and family:")
        for k in sorted(WORST):
            print(f"  {k[0]:<10} {k[1]:<34} {WORST[k]:.3f}")


def ratio(got, S, B):
    """max |got - S| / B; an entry with B = 0 must equal S exactly (else inf)."""
    d = (got.double() - S).abs()
    r = torch.where(B > 0, d / B, torch.where(d > 0, torch.full_like(d, math.inf), torch.zeros_like(d)))
    return float(r.max()) if r.numel() else 0.0


def check(op, family, got, S, B, what=""):
    assert got.shape == S.shape == B.shape, (op, family, what, got.shape, S.shape)
    assert bool(torch.isfinite(B).all()), (op, family, what)
    r = ratio(got, S, B)
    WORST[op, family] = max(WORST.get((op, family), 0.0), r)
    assert r <= 1.0, (op, family, what, r)
    return r


def inputs_linear(op, M, K, N, seed, dev="cpu", gamma=True):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    d = dict(x=r(M, K), w=r(N, K) * K ** -0.5, b=0.1 * r(N))
    if op == vx.RESIDUAL:
        d.update(gamma=r(N) if gamma else None, resid=r(M, N))
    else:
        d.update(ln_w=1 + 0.2 * r(K), ln_b=0.1 * r(K), eps=1e-6)
    return {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


# ---------------------------------------------------------------------------------------------------------------- CPU

def test_exact_value_is_the_float64_module_statements():
    """With every rounding term zero, B = 0 and S is nn.LayerNorm / nn.Linear / exact GELU / the patch convolution /
    softmax attention in float64, to 1e-12 relative."""
    torch.manual_seed(0)
    M, K, N = 37, 96, 128
    eps = float(torch.tensor(1e-6, dtype=torch.float32))
    ln = torch.nn.LayerNorm(K, eps=eps).double()
    lin = torch.nn.Linear(K, N).double()
    with torch.no_grad():
        ln.weight.normal_(1, 0.2)
        ln.bias.normal_(0, 0.1)
        lin2 = torch.nn.Linear(N, K).double()
        conv = torch.nn.Conv2d(3, 64, 14, 14).double()
        for mod in (ln, lin, lin2, conv):                     # fp32 values, as the kernels are given them
            for t in mod.parameters():
                t.copy_(t.float().double())
        x = torch.randn(M, K)
        f = lambda t: t.float()
        rel = lambda a, b: float((a - b).abs().max() / b.abs().max())
        for op, want in [(vx.LN_BIAS, lin(ln(x.double()))), (vx.LN_GELU, F.gelu(lin(ln(x.double()))))]:
            S, B = vx.linear(op, x, f(lin.weight), f(lin.bias), f(ln.weight), f(ln.bias), eps, scale=0)
            assert float(B.abs().max()) == 0 and rel(S, want) <= 1e-12, op
        h, resid, gam = torch.randn(M, N), torch.randn(M, K), torch.randn(K)
        S, B = vx.linear(vx.RESIDUAL, h, f(lin2.weight), f(lin2.bias), gamma=f(gam), resid=resid, scale=0)
        assert float(B.abs().max()) == 0 and rel(S, resid.double() + lin2(h.double()) * gam.double()) <= 1e-12
        img = torch.randn(2, 3, 42, 56)
        cls, reg, pos = torch.randn(1, 1, 64), torch.randn(1, 4, 64), torch.randn(1, 13, 64)
        S, B = vx.tokens(img, f(conv.weight), f(conv.bias), cls, reg[0], pos[0], 14, scale=0)
        pt = conv(img.double()).flatten(2).transpose(1, 2) + pos[:, 1:].double()
        want = torch.cat([(cls + pos[:, :1]).double().expand(2, -1, -1), reg.double().expand(2, -1, -1), pt], 1)
        assert float(B.abs().max()) == 0 and rel(S, want) <= 1e-12
        tok = torch.randn(2, 1 + 4 + 12, K)
        (sp, bp), (sc, bc) = vx.output(tok, 4, f(ln.weight), f(ln.bias), eps, vx.LAYOUT_CHANNELS, scale=0)
        want = ln(tok.double())
        assert float(bp.abs().max()) == 0 and rel(sp, want[:, 5:].transpose(1, 2)) <= 1e-12
        assert rel(sc, want[:, 0]) <= 1e-12
        qkv = torch.randn(2, 70, 3 * 2 * 64)
        S, B = vx.attention(qkv, 2, chunk=16, scale=0)
        assert float(B.abs().max()) == 0 and rel(S, ao.attention(qkv, 2)) <= 1e-12


@pytest.mark.parametrize("op", [vx.LN_BIAS, vx.LN_GELU, vx.RESIDUAL])
@pytest.mark.parametrize("M,K,N", [(1, 4, 64), (65, 36, 64), (70, 100, 128)])
def test_emulation_within_the_bound(op, M, K, N):
    d = inputs_linear(op, M, K, N, seed=M + K)
    for gamma in ((True, False) if op == vx.RESIDUAL else (True,)):
        if not gamma:
            d["gamma"] = None
        S, B = vx.linear(op, **d)
        for seed in range(2):
            check(f"linear{op}", "cpu emulation", vx.emulate_linear(op, **d, seed=seed), S, B)


def test_emulation_within_the_bound_tokens_output_attention():
    g = torch.Generator().manual_seed(3)
    img = torch.randn(2, 3, 28, 42, generator=g)
    w, b = 0.05 * torch.randn(64, 3, 14, 14, generator=g), 0.1 * torch.randn(64, generator=g)
    pos = torch.randn(7, 64, generator=g)
    S, B = vx.tokens(img, w, b, torch.randn(64), torch.randn(4, 64), pos, 14)
    got = (vx.emulate_gemm(vx.im2col(img, 14).float(), w.reshape(64, -1)) + b + pos[1:].repeat(2, 1)).reshape(2, 6, 64)
    check("tokens", "cpu emulation", got, S[:, 5:], B[:, 5:])
    tok = 3 + torch.randn(2, 40, 96, generator=g)
    nw, nb = 1 + 0.1 * torch.randn(96, generator=g), 0.1 * torch.randn(96, generator=g)
    for layout in (vx.LAYOUT_TOKENS, vx.LAYOUT_CHANNELS):
        (sp, bp), (sc, bc) = vx.output(tok, 4, nw, nb, 1e-6, layout)
        ep, ec = vx.emulate_output(tok, 4, nw, nb, 1e-6, layout)
        check("output", "cpu emulation", ep, sp, bp)
        check("output", "cpu emulation", ec, sc, bc)
    for N, H in [(1, 1), (65, 2), (130, 1)]:
        qkv = 1.5 * torch.randn(1, N, 3 * H * 64, generator=g)
        S, B = vx.attention(qkv, H, chunk=32)
        check("attention", "cpu emulation", vx.emulate_attention(qkv, H), S, B, N)
    for dom, H in [(5, 1), (64, 2)]:                          # determined rows: V passes through bitwise under P1
        qkv = dominant_qkv(70, dom, H)
        S, B = vx.attention(qkv, H, chunk=32)
        got = vx.emulate_attention(qkv, H)
        check("attention", "cpu emulation", got, S, B, dom)
        assert torch.equal(got[0], qkv[0, dom, 2 * H * 64:].expand(70, -1)), dom


def rising_max_qkv(N, H=1, step=3.0):
    """Key j's score is step * (tile of j) + small noise for every query: the running maximum rises at every tile."""
    g = torch.Generator().manual_seed(N)
    qkv = 0.3 * torch.randn(1, N, 3 * H * 64, generator=g)
    qkv[0, :, :H * 64] = 0.1 * torch.randn(N, H * 64, generator=g)
    qkv[0, :, 0::64][:, :H] = 8.0                                          # q dim 0 of every head
    qkv[0, :, H * 64::64][:, :H] = (step * (torch.arange(N) // 64)).unsqueeze(1).float()
    return qkv


def below_powers_of_two(n):
    """n fp32 values just below a power of two with the lowest bit set, +-2^e (1 - k 2^-24) for k = 1, 3: their
    tf32 hi part rounds up to 2^e, and v - hi = -+k 2^(e - 24) sits one bit below 2^e's 24-bit ulp."""
    i = torch.arange(n)
    e = (i % 13 - 6).double()
    k = torch.where(i % 2 == 0, 1.0, 3.0).double()
    sign = torch.where((i // 2) % 2 == 0, 1.0, -1.0).double()
    v = (sign * torch.exp2(e) * (1 - k * 2.0 ** -24)).float()
    assert torch.equal(v.double(), sign * torch.exp2(e) * (1 - k * 2.0 ** -24))
    assert torch.equal(vx._tf32(v).double().abs(), torch.exp2(e))
    return v


def dominant_qkv(N, dom, H=1):
    """Scores +-65 on key ``dom`` against every other: a gap of 130.  The first 32 dims of the dominant key's V row of
    every head are ``below_powers_of_two``, whose pass-through needs premise P1 of oracle/vit_exact.py."""
    g = torch.Generator().manual_seed(N + dom)
    qkv = torch.randn(1, N, 3 * H * 64, generator=g)
    qkv[0, :, :H * 64] = 0
    qkv[0, :, 0::64][:, :H] = 52.0
    qkv[0, :, H * 64:2 * H * 64] = 0
    qkv[0, :, H * 64::64][:, :H] = -10.0
    qkv[0, dom, H * 64::64][:H] = 10.0
    for h in range(H):
        qkv[0, dom, (2 * H + h) * 64:(2 * H + h) * 64 + 32] = below_powers_of_two(32)
    return qkv


def mutation_cases():
    """(mutation, evaluate -> (emulated, S, B)): each corruption on the input where it matters most."""
    def lin(op, d, mut):
        S, B = vx.linear(op, **d)
        return vx.emulate_linear(op, **d, mut=mut), S, B

    base = lambda op, M=65, K=36: inputs_linear(op, M, K, 64, seed=7)
    c = 1 + 2 ** -10 - 2 ** -23                                    # just below a tf32 boundary: RZ loses the most
    rz = dict(x=torch.full((1, 4), c), w=torch.full((64, 4), c), b=torch.zeros(64), gamma=None, resid=torch.zeros(1, 64))
    ln_big = base(vx.LN_BIAS, 3, 384)
    ln_big["x"] = 1000 + 0.5 * torch.randn(3, 384, generator=torch.Generator().manual_seed(1))
    gelu = base(vx.LN_GELU)
    gelu["b"] = torch.linspace(-3, 3, 64)
    att = lambda qkv, H, mut: (vx.emulate_attention(qkv, H, mut=mut),) + vx.attention(qkv, H, chunk=64)
    g = torch.Generator().manual_seed(5)
    return {
        "one_tf32": lambda: lin(vx.LN_BIAS, base(vx.LN_BIAS), "one_tf32"),
        "drop_corr_last": lambda: lin(vx.RESIDUAL, base(vx.RESIDUAL), "drop_corr_last"),
        "split_rz": lambda: lin(vx.RESIDUAL, rz, "split_rz"),
        "ln_fp32_stats": lambda: lin(vx.LN_BIAS, ln_big, "ln_fp32_stats"),
        "gelu_tanh": lambda: lin(vx.LN_GELU, gelu, "gelu_tanh"),
        "gamma_ignored": lambda: lin(vx.RESIDUAL, base(vx.RESIDUAL), "gamma_ignored"),
        "tail_rows_zero": lambda: lin(vx.LN_BIAS, base(vx.LN_BIAS), "tail_rows_zero"),
        "keys_unmasked": lambda: att(torch.randn(1, 65, 3 * 64, generator=g), 1, "keys_unmasked"),
        "no_rescale": lambda: att(rising_max_qkv(130), 1, "no_rescale"),
        "v_two_parts": lambda: att(dominant_qkv(70, 5), 1, "v_two_parts"),
        "heads_swapped": lambda: att(torch.randn(1, 20, 3 * 2 * 64, generator=g), 2, "heads_swapped"),
    }


def test_every_mutation_leaves_the_bound():
    cases = mutation_cases()
    assert sorted(cases) == sorted(vx.MUTATIONS)
    for name in vx.MUTATIONS:
        got, S, B = cases[name]()
        r = ratio(got, S, B)
        print(f"mutation {name}: worst |emulated - S| / B = {r:.3g}")
        assert r > 1.0, (name, r)


# ---------------------------------------------------------------------------------------------------------------- GPU

DEV = "cuda:0"


def lib():
    from diff_gaussian_rasterization import _C
    return _C


def _p(t):
    return None if t is None else t.data_ptr()


def k_linear(op, x, w, b, ln_w=None, ln_b=None, eps=1e-6, gamma=None, resid=None, out=None):
    C = lib()
    M, K = x.shape
    out = torch.full((M, w.shape[0]), math.nan, device=x.device) if out is None else out
    C._check(C._lib.gsr_vit_linear(op, M, K, w.shape[0], _p(x), _p(ln_w), _p(ln_b), eps, _p(w), _p(b), _p(gamma),
                                   _p(resid), _p(out), None), "gsr_vit_linear")
    return out


def k_tokens(x, w, b, cls, reg, pos, patch):
    C = lib()
    B, _, H, W = x.shape
    Cn = w.shape[0]
    R = 0 if reg is None else reg.shape[0]
    out = torch.full((B, 1 + R + (H // patch) * (W // patch), Cn), math.nan, device=x.device)
    C._check(C._lib.gsr_vit_tokens(B, H, W, Cn, patch, R, _p(x), _p(w), _p(b), _p(cls), _p(reg), _p(pos), _p(out), None),
             "gsr_vit_tokens")
    return out


def k_output(tok, R, nw, nb, eps, layout, want_cls):
    C = lib()
    B, T, Cn = tok.shape
    P = T - 1 - R
    pat = torch.full((B, P, Cn) if layout == vx.LAYOUT_TOKENS else (B, Cn, P), math.nan, device=tok.device)
    cls = torch.full((B, Cn), math.nan, device=tok.device) if want_cls else None
    C._check(C._lib.gsr_vit_output(B, T, Cn, R, layout, _p(tok), _p(nw), _p(nb), eps, _p(pat), _p(cls), None),
             "gsr_vit_output")
    return pat, cls


def k_attention(qkv, H):
    import fused_dino
    return fused_dino.attention(qkv, H)


M_EDGES = [1, 63, 64, 65, 127, 128, 129, 355, 10769]
KN = [(384, 1152), (384, 1536), (1536, 384), (768, 2304), (3072, 768), (1024, 4096), (4096, 1024), (36, 64), (4, 64)]


def run_linear(op, family, d, inplace=False):
    S, B = vx.linear(op, **d)
    if inplace:
        out = d["resid"].clone()
        got = k_linear(op, **{**d, "resid": out}, out=out)
        ref = k_linear(op, **d)
        assert torch.equal(got, ref), (family, "in place differs from out of place")
    else:
        got = k_linear(op, **d)
    check(f"linear{op}", family, got, S, B)
    return got, S, B


@pytest.mark.gpu
@pytest.mark.parametrize("op", [vx.LN_BIAS, vx.LN_GELU, vx.RESIDUAL])
def test_linear_rows_at_the_tile_edges(op):
    """Every M of the 64-row tile's edges, including 64k - 1, 64k and 64k + 1; the rows of the partial last tile are
    checked like every other row."""
    K, N = {vx.LN_BIAS: (384, 1152), vx.LN_GELU: (384, 1536), vx.RESIDUAL: (1536, 384)}[op]
    assert {m % 64 for m in M_EDGES} >= {0, 1, 63}
    for M in M_EDGES:
        got, S, B = run_linear(op, "rows M", inputs_linear(op, M, K, N, seed=M, dev=DEV))
        assert bool(torch.isfinite(got[(M - 1) // 64 * 64:]).all())        # the last tile was written (NaN-filled)


@pytest.mark.gpu
@pytest.mark.parametrize("op", [vx.LN_BIAS, vx.LN_GELU, vx.RESIDUAL])
def test_linear_widths_ragged_k_and_layer_scale(op):
    """ViT-S/B/L widths, K not a multiple of 32 on the LayerNorm path (K = 36 and 4: a zero-padded last chunk),
    gamma NULL and present, in place (out == resid) and out of place."""
    assert any(K % 32 for K, _ in KN) and any(N == 4096 for _, N in KN)
    for K, N in KN:
        for M in (129,) if K * N > 2 ** 20 else (65, 129):
            if op == vx.RESIDUAL:
                for gamma in (True, False):
                    for inplace in (False, True):
                        d = inputs_linear(op, M, K, N, seed=K + N, dev=DEV, gamma=gamma)
                        run_linear(op, f"K,N widths gamma={gamma}", d, inplace=inplace)
            else:
                run_linear(op, "K,N widths (ragged K)", inputs_linear(op, M, K, N, seed=K + N, dev=DEV))


@pytest.mark.gpu
@pytest.mark.parametrize("K", [384, 36])
def test_linear_adversarial_layer_norm_rows(K):
    """Rows with |mu| / sigma >= 1e3, constant rows (rstd = 1 / sqrt(eps)), one channel at ~1e3 (DINOv2's massive
    activations), and zero LayerNorm weights."""
    g = torch.Generator().manual_seed(K)
    M = 70
    x = torch.randn(M, K, generator=g)
    x[0:10] = 1000 + 0.5 * torch.randn(10, K, generator=g)
    x[10:20] = -3e3 + 1.0 * torch.randn(10, K, generator=g)
    x[20:30] = torch.linspace(-2, 2, 10).unsqueeze(1)                     # constant rows
    x[30:40, 3] = 1000.0
    xd = x.double()
    assert float((xd[0:20].mean(1).abs() / xd[0:20].std(1, unbiased=False)).min()) >= 1e3
    assert float(xd[20:30].std(1).max()) == 0
    for op in (vx.LN_BIAS, vx.LN_GELU):
        d = inputs_linear(op, M, K, 128, seed=K + 1)
        d["x"] = x
        for zero_w in (False, True):
            if zero_w:
                d["ln_w"] = d["ln_w"].clone()
                d["ln_w"][::2] = 0
            got, S, B = run_linear(op, "adversarial LN rows", {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v)
                                                               for k, v in d.items()})
            if op == vx.LN_BIAS and not zero_w:                 # constant rows: the LN output is ln_b exactly
                want = (d["ln_b"].double() @ d["w"].double().T + d["b"].double()).to(DEV)
                assert float((S[20:30] - want).abs().max()) <= 1e-9


@pytest.mark.gpu
def test_gelu_over_minus_ten_to_ten():
    """Pre-activations spread over [-10, 10], including v < -5 where 1 + erf cancels to below 1e-6."""
    M, K, N = 129, 384, 1536
    d = inputs_linear(vx.LN_GELU, M, K, N, seed=11)
    d["w"] = 0.02 * d["w"]
    d["b"] = torch.linspace(-10, 10, N)
    d = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}
    got, S, B = run_linear(vx.LN_GELU, "GELU in [-10, 10]", d)
    pre = vx.linear(vx.LN_BIAS, **d)[0]
    assert float(pre.min()) < -9.5 and float(pre.max()) > 9.5
    assert bool(((pre < -5) & (S.abs() < 1e-5)).any())


@pytest.mark.gpu
def test_tokens_patch_sizes_grids_and_widths():
    """Patch 14 (K = 588, ragged) and 16, B 1 and 3, grids 1x1, 3x5 and 78x138, R 0 and 4, C 64, 384 and 1024; class
    and register tokens bitwise."""
    g = torch.Generator().manual_seed(2)
    for patch, B, R in [(14, 1, 4), (14, 3, 0), (16, 1, 0), (16, 3, 4)]:
        for gh, gw in [(1, 1), (3, 5), (78, 138)]:
            for C in (64, 384, 1024):
                x = torch.randn(B, 3, gh * patch, gw * patch, generator=g)
                w = torch.randn(C, 3, patch, patch, generator=g) * (3 * patch * patch) ** -0.5
                b, cls = 0.1 * torch.randn(C, generator=g), torch.randn(C, generator=g)
                reg = torch.randn(R, C, generator=g) if R else None
                pos = torch.randn(1 + gh * gw, C, generator=g)
                t = [v.to(DEV) if v is not None else None for v in (x, w, b, cls, reg, pos)]
                got = k_tokens(*t, patch)
                S, Bd = vx.tokens(*t, patch)
                check("tokens", f"patch {patch}", got, S, Bd, (B, gh, gw, C, R))
                assert torch.equal(got[:, 0], (t[3] + t[5][0]).expand(B, C))
                if R:
                    assert torch.equal(got[:, 1:1 + R], t[4].expand(B, R, C))


def att_check(family, qkv, H):
    qkv = qkv.to(DEV).contiguous()
    got = k_attention(qkv, H)
    S, B = vx.attention(qkv, H)
    check("attention", family, got, S, B, (qkv.shape, H))
    return got, S, B


@pytest.mark.gpu
def test_attention_sizes():
    """N at the 64-key and 128-query tile edges, H 1, 6 and 16, B 1 and 3."""
    g = torch.Generator().manual_seed(9)
    for N in [1, 2, 63, 64, 65, 127, 128, 129, 192, 193, 355, 10769]:
        for H, B in ([(6, 1)] if N > 355 else [(6, 1), (1, 3), (16, 1)]):
            qkv = 1.5 * torch.randn(B, N, 3 * H * 64, generator=g)
            got, S, _ = att_check("N edges", qkv, H)
            if N == 1:
                assert torch.equal(got, qkv[:, :, 2 * H * 64:].to(DEV))


@pytest.mark.gpu
def test_attention_adversarial_families():
    g = torch.Generator().manual_seed(10)
    N, H = 193, 2
    # sharp scores, |s| ~ 40
    qkv = torch.randn(1, N, 3 * H * 64, generator=g)
    qkv[..., :2 * H * 64] *= 3.2
    s = (qkv[0, :, :64].double() / 8) @ qkv[0, :, H * 64:H * 64 + 64].double().T
    assert float(s.abs().max()) > 35
    att_check("sharp scores |s|~40", qkv, H)
    # every row's maximum in the partial last key tile
    qkv = torch.randn(1, N, 3 * H * 64, generator=g)
    qkv[0, :, 0::64][:, :H] = 8.0
    qkv[0, :, H * 64::64][:, :H] = 0.0
    qkv[0, 192:, H * 64::64][:, :H] = 10.0
    s = (qkv[0, :, :64].double() / 8) @ qkv[0, :, H * 64:H * 64 + 64].double().T
    assert bool((s.argmax(1) >= 192).all())
    att_check("max in the last key tile", qkv, H)
    # a maximum that rises at every tile
    qkv = rising_max_qkv(N, H)
    s = (qkv[0, :, :64].double() / 8) @ qkv[0, :, H * 64:H * 64 + 64].double().T
    tmax = torch.stack([s[:, i:i + 64].max(1).values for i in range(0, N, 64)], 1)
    assert bool((tmax[:, 1:] > tmax[:, :-1]).all())
    att_check("max rises at every tile", qkv, H)
    # uniform keys, zero q rows
    qkv = torch.randn(1, N, 3 * H * 64, generator=g)
    qkv[0, :, H * 64:2 * H * 64] = qkv[0, :1, H * 64:2 * H * 64]
    att_check("uniform keys", qkv, H)
    qkv = torch.randn(1, N, 3 * H * 64, generator=g)
    qkv[0, ::3, :H * 64] = 0
    att_check("zero q rows", qkv, H)
    # one dominant key, gap >= 120: the output row is that key's V row, bitwise
    for dom in (0, 100, 192):
        qkv = dominant_qkv(N, dom, H)
        got, _, _ = att_check("dominant key (bitwise)", qkv, H)
        v = qkv[0, dom, 2 * H * 64:].to(DEV)
        assert torch.equal(got[0], v.expand(N, -1)), dom


@pytest.mark.gpu
def test_output_sizes_layouts_and_copies():
    g = torch.Generator().manual_seed(12)
    R = 4
    for P in [1, 31, 32, 33, 10764]:
        for C in [32, 96, 384, 1024]:
            tok = (2 + torch.randn(2 if P < 10000 else 1, 1 + R + P, C, generator=g)).to(DEV)
            nw, nb = (1 + 0.2 * torch.randn(C, generator=g)).to(DEV), (0.1 * torch.randn(C, generator=g)).to(DEV)
            for layout in (vx.LAYOUT_TOKENS, vx.LAYOUT_CHANNELS):
                for want_cls in (False, True):
                    pat, cls = k_output(tok, R, nw, nb, 1e-6, layout, want_cls)
                    (sp, bp), (sc, bc) = vx.output(tok, R, nw, nb, 1e-6, layout)
                    check("output", "P, C, layout", pat, sp, bp, (P, C, layout))
                    if want_cls:
                        check("output", "class token", cls, sc, bc)
                    pat, cls = k_output(tok, R, None, None, 0.0, layout, want_cls)
                    want = tok[:, 1 + R:]
                    assert torch.equal(pat, want.transpose(1, 2) if layout else want)
                    if want_cls:
                        assert torch.equal(cls, tok[:, 0])


@pytest.mark.gpu
def test_k_step_premise():
    """One k-step alone: ``gsr_vit_linear(op=RESIDUAL)`` with K = 8 or 16, tf32-exact operands (their lo parts are
    zero, so the correction steps add zeros), zero bias and resid, NULL gamma.  Every other operation is then exact, so
    the output is the tensor cores' sum.  The exponents are spread so that the exact 8-product sums need more than 24
    bits; each result must lie within 2^-23 (n M + |result|) of the exact sum (one step; two for K = 16)."""
    g = torch.Generator().manual_seed(13)
    for K in (8, 16):
        x = vx._tf32(torch.randn(64, K, generator=g) * torch.exp2(torch.randint(-12, 1, (64, K), generator=g).float()))
        w = vx._tf32(torch.randn(128, K, generator=g) * torch.exp2(torch.randint(-12, 1, (128, K), generator=g).float()))
        assert bool((vx.split(x)[1] == 0).all()) and bool((vx.split(w)[1] == 0).all())
        got = k_linear(vx.RESIDUAL, x.to(DEV), w.to(DEV), torch.zeros(128, device=DEV),
                       resid=torch.zeros(64, 128, device=DEV)).cpu().double()
        p = x.double().unsqueeze(1) * w.double().unsqueeze(0)              # [64, 128, K] exact products
        exact = p.sum(-1)
        f32 = exact.float()
        assert float((f32.double() - exact).abs().max()) > 0                # the sums need more than 24 bits
        bound = torch.zeros_like(exact)
        acc = torch.zeros_like(exact)
        for s in range(K // 8):
            ps = p[..., 8 * s:8 * s + 8]
            n = ((ps != 0).sum(-1) + (acc != 0).long() - 1).clamp(min=0)
            mx = torch.maximum(ps.abs().amax(-1), acc.abs())
            acc = acc + ps.sum(-1)
            bound = bound + vx.TRUNC * (n * (mx + bound) + acc.abs() + bound)
        err = got - exact
        r = float((err.abs() / bound).max())
        rn = float((got == f32.double()).double().mean())
        rz = float((got == vx._rz32(exact).double()).double().mean())
        toward0 = float(((err * exact.sign()) < 0).double().mean())
        print(f"k-step premise K={K}: worst |err| / model bound {r:.3f}; results equal to RN {rn:.3f}, to RZ {rz:.3f}, "
              f"below the exact sum in magnitude {toward0:.3f}")
        WORST["premise", f"K={K} per-step bound"] = r
        assert r <= 1.0, (K, r)


@pytest.mark.gpu
def test_alignment_bit_premise_p1():
    """Premise P1 of oracle/vit_exact.py: a k-step keeps an alignment bit beyond the 24.  Two steps of
    ``gsr_vit_linear(op=RESIDUAL)`` (K = 16, tf32-exact operands, zero bias and resid): the first leaves the accumulator
    at -+k 2^(e - 24) (k = 1, 3), the second adds +-2^e.  The exact sum 2^e (1 - k 2^-24) is an fp32 number, so under P1
    the output is that sum bitwise; a 24-bit alignment would return 2^e.  This is the step that passes a V entry just
    below a power of two through a determined attention row."""
    M, N = 64, 64
    i = torch.arange(M)
    e = (i % 21 - 10).double()
    k = torch.where(i % 2 == 0, 1.0, 3.0).double()
    sign = torch.where((i // 2) % 2 == 0, 1.0, -1.0).double()
    x = torch.zeros(M, 16, dtype=torch.float64)
    x[:, 0] = -sign * k * torch.exp2(e - 24)
    x[:, 8] = sign * torch.exp2(e)
    w = torch.zeros(N, 16)
    w[:, 0] = w[:, 8] = torch.where(torch.arange(N) % 2 == 0, 1.0, -1.0)
    x = x.float()
    assert torch.equal(vx._tf32(x), x)
    want = x.double() @ w.double().T                                        # exact, and an fp32 number
    assert torch.equal(want.float().double(), want)
    got = k_linear(vx.RESIDUAL, x.to(DEV), w.to(DEV), torch.zeros(N, device=DEV),
                   resid=torch.zeros(M, N, device=DEV)).cpu().double()
    lost = float((got != want).double().mean())
    print(f"alignment-bit premise P1: {lost:.3f} of the crafted sums not returned exactly")
    assert lost == 0, got[got != want][:8]


# ------------------------------------------------------------------------------------------------- backbone replay

def replay(bb, x, blocks):
    """Each op of ``fused_dino._vit_layers`` in its order, on the kernel's own fp32 input of that op."""
    p, C, R = bb.patch_size, bb.embed_dim, bb.num_register_tokens
    B, _, H, W = x.shape
    import fused_dino
    pos = fused_dino._pos_embed(bb, H // p, W // p)
    conv = bb.patch_embed.proj
    cw, cb = conv.weight.detach().contiguous(), conv.bias.detach()
    reg = bb.register_tokens.detach()[0].contiguous() if R else None
    cls = bb.cls_token.detach().reshape(C).contiguous()
    tok = k_tokens(x, cw, cb, cls, reg, pos, p)
    check("tokens", "backbone replay", tok, *vx.tokens(x, cw, cb, cls, reg, pos, p))
    M = tok.shape[0] * tok.shape[1]
    for i in range(blocks):
        blk = bb.blocks[i]
        g1, g2 = (ls.gamma.detach() if hasattr(ls, "gamma") else None for ls in (blk.ls1, blk.ls2))
        lw = lambda m: dict(w=m.weight.detach(), b=m.bias.detach())
        ln = lambda n: dict(ln_w=n.weight.detach(), ln_b=n.bias.detach(), eps=float(n.eps))
        t2 = tok.reshape(M, C)
        d = dict(x=t2, **lw(blk.attn.qkv), **ln(blk.norm1))
        qkv = run_linear(vx.LN_BIAS, "backbone replay", d)[0]
        att = k_attention(qkv.reshape(B, -1, 3 * C), blk.attn.num_heads)
        check("attention", "backbone replay", att, *vx.attention(qkv.reshape(B, -1, 3 * C), blk.attn.num_heads))
        nxt = run_linear(vx.RESIDUAL, "backbone replay", dict(x=att.reshape(M, C), **lw(blk.attn.proj), gamma=g1,
                                                                resid=t2))[0]
        hid = run_linear(vx.LN_GELU, "backbone replay", dict(x=nxt, **lw(blk.mlp.fc1), **ln(blk.norm2)))[0]
        tok = run_linear(vx.RESIDUAL, "backbone replay", dict(x=hid, **lw(blk.mlp.fc2), gamma=g2, resid=nxt),
                         inplace=True)[0].reshape(B, -1, C)
    for layout in (vx.LAYOUT_TOKENS, vx.LAYOUT_CHANNELS):
        pat, c = k_output(tok, R, bb.norm.weight.detach(), bb.norm.bias.detach(), float(bb.norm.eps), layout, True)
        (sp, bp), (sc, bc) = vx.output(tok, R, bb.norm.weight.detach(), bb.norm.bias.detach(), float(bb.norm.eps), layout)
        check("output", "backbone replay", pat, sp, bp)
        check("output", "backbone replay", c, sc, bc)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(196, 350), (1092, 1932)])
def test_backbone_replay_vit_s14_registers(H, W):
    from test_fused_dino import dino_input, sharpened_backbone
    _, bb = sharpened_backbone(torch.device(DEV))
    with torch.no_grad():
        replay(bb, dino_input(H, W, 5, torch.device(DEV)), 6)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["vit_base", "vit_large"])
def test_backbone_replay_vit_b_and_l(variant):
    from test_fused_dino import dino_input, import_method
    m, _ = import_method()
    torch.manual_seed(4)
    bb = getattr(m.dinov2, variant)(patch_size=14, num_register_tokens=4, img_size=518, init_values=1.0, block_chunks=0)
    bb = bb.to(DEV).eval()
    with torch.no_grad():
        for blk in bb.blocks:
            blk.ls1.gamma.normal_(1.0, 0.2)
            blk.ls2.gamma.normal_(1.0, 0.2)
        replay(bb, dino_input(196, 350, 13, torch.device(DEV)), 2)
