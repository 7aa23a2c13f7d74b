"""TEST INFRASTRUCTURE -- fp64 oracle of the DINOv2 backbone kernels (csrc/vit.cu, csrc/attention.cu) AS THE KERNELS
ROUND THEM, with an a-priori bound B on how far the kernel's value of every output entry can be from the exact value S
of the operation on the kernel's own fp32 inputs.  Only tests/ may import this.

Entry points (each returns ``(S, B)``, float64, the shape of the kernel's output, on the inputs' device):
``linear`` (``gsr_vit_linear``, all three ops), ``tokens`` (``gsr_vit_tokens``), ``attention``
(``gsr_attention_forward``) and ``output`` (``gsr_vit_output``).  ``scale=0`` sets every rounding term to zero, so
B = 0 and S alone is the plain float64 statement.  ``emulate_*`` evaluate the kernels in fp32 as the model allows them
to round, with optional corruptions (``MUTATIONS``) for the self-tests.

The model (u = 2^-24, the fp32 round-to-nearest unit; every fp32 RN operation adds u |result|):

1. tf32 split, ``cvt.rna.tf32.f32``.  hi = rna(x) keeps 11 significant bits, |x - hi| <= 2^-11 |x|; x - hi is exact in
   fp32; lo = rna(x - hi), so |x - hi - lo| <= 2^-22 |x|, |hi| <= (1 + 2^-11) |x|, |lo| <= 2^-11 (1 + 2^-11) |x|.  A
   product of two tf32 values has at most 22 significant bits and is exact.  3xTF32 computes
   ahi bhi + ahi blo + alo bhi and drops alo blo, ahi eb, alo eb and ea b (e: the split residuals), together at most
   2^-22 (3 + 2^-9) |a| |b| per product.  V in the attention is split exactly (hi + mid + lo cover fp32's 24 bits); P is
   split in two, and the products dropped there are plo (vmid + vlo) and (p - phi - plo) v: 2^-22 (2 + 2^-10) p |v|.

2. One tensor-core k-step (``wgmma.m64n64k8.f32.tf32``) adds 8 exact products to the fp32 accumulator as one fused
   sum: the addends (the accumulator and the products) are aligned to the largest exponent among them, every addend
   other than the largest is truncated there to the accumulator's 24 significant bits, the aligned sum is formed and
   normalised back to fp32 (truncated or rounded).  An addend truncated at the largest one's ulp loses less than
   2^-23 M (M the largest magnitude), and the normalisation less than 2^-23 |result|.  With n the number of non-zero
   addends besides the largest (at most the number of non-zero products, nz <= 8):
       |err| <= 2^-23 (n M + |result|) <= 2^-23 (nz + [nz > 0]) (|acc| + sum |p|),
   a step of zero products is exact, and the first step of a fresh accumulator (acc = 0) has n <= nz - 1, so its
   weight is nz.  Hardware that keeps extra alignment bits, or rounds instead of truncating, stays inside this.

   Premise P1, a measured property of the H100 rather than a consequence of the above: a step keeps at least one
   alignment bit beyond the 24, i.e. an addend is truncated no coarser than 2^-24 of the largest addend's leading bit.
   So a step whose addends are all multiples of 2^(E - 24) (2^E <= M < 2^(E + 1)) and whose exact sum is an fp32
   number returns that sum exactly; under item 2 alone, 2^E plus an accumulator of -2^(E - 24) may return 2^E.  The
   bounds B never use P1.  Only two exactness claims do: the pass-through of a determined attention row (item 5),
   where v just below a power of two has vhi = 2^E and v - vhi an odd multiple of 2^(E - 24), and with it the
   bitwise assertion of that row and the catch of the two-part V split.
   tests/test_dino_exact.py::test_alignment_bit_premise_p1 asserts P1 with crafted steps of exactly that form, on both
   signs and several exponents, and the dominant-key tests put such V entries through the attention.  ``kstep``, the emulation, realises the model under P1.
  nz is taken as the number of k inside the operation's K (padding is zero), so data zeros only make
   the bound looser.  The premise test of tests/test_dino_exact.py holds the hardware to this per-step bound with
   crafted operands whose 8-product sums need more than 24 bits.  With C_t the running sum of |products| that reached
   an accumulator by step t, its error is sum_t 2^-23 (nz_t + [nz_t > 0]) C_t: a fixed weight per product.  Every
   bound below is therefore linear in |a_k| |w_k|, and a GEMM's B is one matmul (|A| diag(kappa)) |W|^T.

   vit.cu, per 32-wide K chunk: 8 correction steps (lo hi, then hi lo, per 8-wide k block) into a fresh ``corr`` and 4
   hi hi steps into a fresh ``hh``; then ``acc += hh + corr``: two fp32 RN additions (u |hh + corr| and u |acc|).
   attention.cu, per 64-key tile: ``sa`` takes 16 correction steps (lo hi, hi lo per 8 dims) and the hi hi steps of
   dims 0..31, ``sb`` (fresh) those of dims 32..63, then ``sc = sa + sb`` (u).  P V: one fresh accumulator ``ot``
   takes, per 8-key block, plo vhi, phi vlo, phi vmid (24 steps) and then phi vhi of every block (8), merged into O by
   ``o = fmaf(o, a, ot)`` (one rounding, u |o|).  An fp32 addition into a zero accumulator is exact: ``acc += hh +
   corr`` of the first chunk and the first tile's merge into O add no rounding.

3. LayerNorm (prologue and final norm): mean and variance in double, one pass, ``q/K - mu^2``, clamped at 0.  The
   double sums are bounded by the usual gamma_K = K 2^-53 / (1 - K 2^-53) terms; the cancellation term is
   gamma_{K+1} q/K + 2 |mu| dmu + dmu^2 + 2^-52 (q/K + mu^2), which for |mu| >> sigma is of the order 2^-53 mu^2 and
   dominates var.  mu and rstd are then rounded to fp32 (u each; rstd also carries the relative error dvar / (var +
   eps) of the double statistics).  ``(v - mu) * rs * w + b`` in fp32: v - mu, * rs and * w round once each, + b once
   more; the last two are the site nvcc may contract into an FMA, modelled as two roundings, which covers the fused
   and the unfused evaluation.  The exact S uses the fp32 ``eps`` the kernel is passed.

4. Epilogues.  ``acc + b`` (u; exact where b = 0).  ``resid + v`` likewise exact where resid = 0.  GELU: ``0.5f * v * (1.f + erff(v * (float)M_SQRT1_2))``: the fp32 constant and the
   product give z = v / sqrt(2) (1 + 2u), erff is within 2 ulp (CUDA Math API), ``1 + erf`` rounds once, 0.5 v is
   exact and the last product rounds once.  The erff error is absolute where 1 + erf cancels (v << 0), so the bound
   there is of the order |v| 2^-24 rather than relative to the tiny result.  The propagated GEMM error is multiplied by
   max |gelu'| < 1.13.  LayerScale: v * gamma then resid + v, again a contractible site (two roundings); gamma NULL: one
   rounding.  In place (out == resid) each element is read before it is written by the same thread, so the result is
   that of the out-of-place call (the tests assert it bitwise).  Tokens: ``acc + b`` then ``+ pos`` (u each); the class
   token ``cls + pos[0]`` is one fp32 addition and the register tokens are copies (asserted bitwise).

5. Attention.  The score error Es_j follows from the GEMM model of (q/8) k (the scaling by 1/8 is exact).  The kernel's
   weight of key j, expf(fl(sc_j - m_t)) times the later rescale factors expf(fl(m_t' - m_t'')), is
   exp(s_j - m_final) up to a relative perturbation exp(+-eta_j): the running maxima cancel exactly, what is left is
   Es_j, the rounding of every subtraction (u |sc - m| <= u (smax - s_j + 2 max Es), and the rescale subtractions sum
   to at most the same over the row since m is non-decreasing) and 2 ulp of expf per factor (2^-22 each, at most
   ceil(N/64) - t_j + 1 factors).  With eps_j = exp(eta_j) - 1, perturbed weights move the output by at most
       sum_j p_j eps_j |v_j - o| / (sum p (1 - max eps)),
   (the eta / (1 - eta) sum p |v - o| / sum p form per key).  Then the P V products and steps (item 2), the fp32 merge
   of every tile's partial sum into O (u per later tile), the fp32 sum l (16 sequential adds per thread and tile, one
   FMA per tile, two shuffle adds: (17 + ceil(N/64)) u relative) and the final division (u).  Subnormal weights and
   flushed products are covered by an absolute (N + 64 ceil(N/64)) 2^-124 max |v| (the kernel's weights are <= 1 and
   its l >= 1).  A row whose largest score exceeds every other by more than 110 + 2 max Es is determined: from the
   dominant key's tile on, every other weight is expf(< -104) = 0 in fp32, the rescale factor there is expf(< -104) = 0
   (what earlier tiles put into O and l is dropped by the FMA exactly) and 1 after it, the dominant weight is
   expf(0) = 1 with phi = 1 and plo = 0, and V's split is exact.  P V then adds vlo, vmid (together v - vhi, at most
   13 significant bits) and vhi: exact under P1.  So the kernel returns that key's V row unchanged, l = 1, and B on
   such a row is |S - v_max| (of the order e^-110 |v|).
   The oracle evaluates row chunks, so its memory stays O(chunk N), as oracle/attention_oracle.py does.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24                    # fp32 round-to-nearest unit
TRUNC = 2.0 ** -23                # per-addend and normalisation loss of one tensor-core k-step
Q = 1.0 + 2.0 ** -11              # |hi| <= Q |x|
RLO = 2.0 ** -11 * Q              # |lo| <= RLO |x|
SPLIT3 = 2.0 ** -22 * (3 + 2.0 ** -9)      # 3xTF32 product error per |a| |b|
SPLIT_PV = 2.0 ** -22 * (2 + 2.0 ** -10)   # P (two parts) times V (three exact parts)
ERF_ULP, EXP_ULP = 2, 2           # CUDA Math API maximum ulp errors of erff and expf
GELU_LIP = 1.13                   # max |gelu'(x)| = 1.1289, at x = sqrt(2)
SECOND = 1.0 + 2.0 ** -16         # slack for the products of first-order terms the bounds drop
VK, VB, ATT_BN, ATT_D = 32, 64, 64, 64
LN_BIAS, LN_GELU, RESIDUAL = 0, 1, 2
LAYOUT_TOKENS, LAYOUT_CHANNELS = 0, 1


def _gamma(n):
    e = n * 2.0 ** -53
    return e / (1 - e)


# ======================================================================================================================
# accumulator chains (item 2)
# ======================================================================================================================
def _chain(steps, nblocks, scale):
    """One fresh accumulator fed by ``steps`` = [(block, factor, nz)] in order, where block b's products are bounded
    by factor * g_b.  Returns (err, mag): |error| <= sum err[b] g_b, |result| <= sum mag[b] g_b."""
    err, mag = [0.0] * nblocks, [0.0] * nblocks
    nu = [scale * TRUNC * (nz + (nz > 0 and i > 0)) for i, (_, _, nz) in enumerate(steps)]   # step 0: acc = 0
    suffix = 0.0
    for i in range(len(steps) - 1, -1, -1):
        suffix += nu[i]
        b, f, _ = steps[i]
        err[b] += f * suffix
        mag[b] += f
    return torch.tensor(err, dtype=torch.float64), torch.tensor(mag, dtype=torch.float64)


def gemm_kappa(K, scale=1.0):
    """Per-k weight of vit_gemm_kernel: |kernel dot - sum a_k w_k| <= sum_k kappa_k |a_k| |w_k|."""
    chunks = (K + VK - 1) // VK
    nb = 4 * chunks
    nz = [max(0, min(8, K - 8 * s)) for s in range(nb)]
    kap = torch.full((nb,), scale * SPLIT3, dtype=torch.float64)
    for c in range(chunks):
        blocks = range(4 * c, 4 * c + 4)
        corr = [(s, f, nz[s]) for s in blocks for f in (RLO * Q, Q * RLO)]
        e1, m1 = _chain(corr, nb, scale)
        e2, m2 = _chain([(s, Q * Q, nz[s]) for s in blocks], nb, scale)
        mag = (m1 + m2) * SECOND
        kap += (e1 + e2) * SECOND + scale * U * mag * (1 + chunks - max(c, 1))   # hh + corr, acc (0 + t is exact)
    return kap.repeat_interleave(8)[:K]


def score_kappa(scale=1.0):
    """Per-dim weight of the attention scores: |sc - (q/8) k| <= sum_d kappa_d |q_d / 8| |k_d|."""
    nb = ATT_D // 8
    sa = [(c, f, 8) for c in range(nb) for f in (RLO * Q, Q * RLO)] + [(c, Q * Q, 8) for c in range(4)]
    e1, m1 = _chain(sa, nb, scale)
    e2, m2 = _chain([(c, Q * Q, 8) for c in range(4, 8)], nb, scale)
    return ((scale * SPLIT3 + (e1 + e2) * SECOND + scale * U * (m1 + m2) * SECOND)).repeat_interleave(8)


def pv_kappa(scale=1.0):
    """Per key position in a 64-key tile: |ot - sum_j p_j v_j| <= sum_j kappa_j p_j |v_j| (P's and V's parts bounded by
    |phi| <= Q p, |plo| <= RLO p, |vmid| <= 2^-11 Q |v|, |vlo| <= 2^-22 Q |v|)."""
    nb = ATT_BN // 8
    vm, vl = 2.0 ** -11 * Q, 2.0 ** -22 * Q
    st = [(j, f, 8) for j in range(nb) for f in (RLO * Q, Q * vl, Q * vm)] + [(j, Q * Q, 8) for j in range(nb)]
    e, m = _chain(st, nb, scale)
    return (scale * SPLIT_PV + e * SECOND).repeat_interleave(8), (m * SECOND).repeat_interleave(8)


def gemm_bound(a_abs, w, K, a_err=None, scale=1.0):
    """B of the kernel's dot products [M, N] for operands bounded by ``a_abs`` [M, K] (plus ``a_err``, an error the
    operand itself carries) and the weight ``w`` [N, K]."""
    wa = w.double().abs()
    kap = gemm_kappa(K, scale).to(a_abs.device)
    if a_err is None:
        return (a_abs * kap) @ wa.T
    return ((a_abs + a_err) * kap) @ wa.T + a_err @ wa.T


# ======================================================================================================================
# LayerNorm (item 3)
# ======================================================================================================================
def layer_norm(x, w, b, eps, scale=1.0):
    """(y, e): the exact fp64 LayerNorm of the fp32 rows ``x`` [M, K] with the fp32 ``eps``, and a bound on the
    kernel's fp32 value of each element."""
    xd = x.double()
    K = xd.shape[-1]
    eps = float(torch.tensor(eps, dtype=torch.float32))
    mu = xd.mean(-1, keepdim=True)
    var = ((xd - mu) ** 2).mean(-1, keepdim=True)
    rho = 1.0 / torch.sqrt(var + eps)
    wd, bd = w.double(), b.double()
    y = (xd - mu) * rho * wd + bd
    if scale == 0:
        return y, torch.zeros_like(y)
    qk = (xd * xd).mean(-1, keepdim=True)
    dmu = _gamma(K + 2) * xd.abs().mean(-1, keepdim=True)
    dvar = _gamma(K + 2) * qk + 2 * mu.abs() * dmu + dmu ** 2 + 2.0 ** -52 * (qk + mu * mu)
    rr = dvar / (var + eps)
    rrho = torch.where(rr < 0.25, rr + 2.0 ** -50, torch.full_like(rr, math.inf))
    e_mu = dmu + U * (mu.abs() + dmu)
    e_rho = rho * (rrho + U * (1 + rrho))
    dv = (xd - mu).abs()
    ed = e_mu + U * (dv + e_mu)
    rf = rho + e_rho
    e1 = ed * rf + dv * e_rho + U * (dv + ed) * rf
    t1 = dv * rho + e1
    e2 = e1 * wd.abs() + U * t1 * wd.abs()
    e = (e2 + U * (y.abs() + e2)) * SECOND
    return y, e


# ======================================================================================================================
# entry points
# ======================================================================================================================
def _bias_add(d, bg, bias, scale):
    """acc + b: S and B of the rounded sum, from the dot's exact value ``d`` and bound ``bg``."""
    s = d + bias.double()
    return s, bg + scale * U * (s.abs() + bg) * (bias != 0)            # x + 0 is exact


def linear(op, x, w, b, ln_w=None, ln_b=None, eps=1e-6, gamma=None, resid=None, scale=1.0):
    """``gsr_vit_linear``: x [M, K], w [N, K], b [N]; ``resid`` [M, N] for RESIDUAL."""
    K = x.shape[-1]
    if op in (LN_BIAS, LN_GELU):
        a, ae = layer_norm(x, ln_w, ln_b, eps, scale)
        d = a @ w.double().T
        bg = gemm_bound(a.abs(), w, K, ae, scale)
    else:
        a = x.double()
        d = a @ w.double().T
        bg = gemm_bound(a.abs(), w, K, None, scale)
    v, bv = _bias_add(d, bg, b, scale)
    if op == LN_BIAS:
        return v, bv
    if op == LN_GELU:
        s = 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))
        vm = v.abs() + bv
        z = vm / math.sqrt(2)
        zmin = torch.clamp(v.abs() - bv, min=0) * (1 - 4 * U) / math.sqrt(2)
        derf = 2 / math.sqrt(math.pi) * z * torch.exp(-zmin ** 2) * 2 * U * (1 + 2 * U)
        erf_ulp = ERF_ULP * TRUNC * torch.erf(z)                   # ulp(y) <= 2^-23 |y|
        ee = (derf + erf_ulp) * scale
        one = (1 + torch.erf(v / math.sqrt(2))).abs() + ee + bv
        ev = 0.5 * vm * (ee + scale * U * one)
        bo = GELU_LIP * bv + ev + scale * U * (s.abs() + GELU_LIP * bv + ev)
        return s, bo * SECOND
    g = gamma.double() if gamma is not None else torch.ones_like(b, dtype=torch.float64)
    vg = v * g
    s = resid.double() + vg
    bo = bv * g.abs()
    if gamma is not None:
        bo = bo + scale * U * (vg.abs() + bo)
    bo = bo + scale * U * (s.abs() + bo) * (resid != 0)                 # 0 + v is exact
    return s, bo * SECOND


def im2col(x, patch):
    """[B * P, 3 p^2] rows of the image, columns (channel, ky, kx) as the patch convolution's weight is laid out."""
    cols = F.unfold(x.double(), patch, stride=patch)                  # [B, 3 p^2, P]
    return cols.transpose(1, 2).reshape(-1, cols.shape[1])


def tokens(x, weight, bias, cls, reg, pos, patch, scale=1.0):
    """``gsr_vit_tokens``: [B, T, C] with T = 1 + R + P.  Class and register rows of S are the kernel's fp32 values
    (B = 0 there); the tests also assert them bitwise."""
    B, _, H, W = x.shape
    C = weight.shape[0]
    P = (H // patch) * (W // patch)
    R = 0 if reg is None else reg.shape[0]
    wm = weight.reshape(C, -1)
    a = im2col(x, patch)
    d = a @ wm.double().T
    v, bv = _bias_add(d, gemm_bound(a.abs(), wm, wm.shape[1], None, scale), bias, scale)
    pd = pos.double()[1:1 + P].repeat(B, 1)
    s = v + pd
    bo = (bv + scale * U * (s.abs() + bv)) * SECOND
    S = torch.zeros(B, 1 + R + P, C, dtype=torch.float64, device=x.device)
    Bd = torch.zeros_like(S)
    S[:, 0] = (cls.reshape(C) + pos[0]).double()
    if R:
        S[:, 1:1 + R] = reg.reshape(R, C).double()
    S[:, 1 + R:] = s.reshape(B, P, C)
    Bd[:, 1 + R:] = bo.reshape(B, P, C)
    return S, Bd


def output(tok, R, norm_w, norm_b, eps, layout=LAYOUT_TOKENS, scale=1.0):
    """``gsr_vit_output``: (S, B) of the patch tokens in ``layout`` and (S, B) of the class token [B, C]."""
    Bn, T, C = tok.shape
    if norm_w is None:
        y, e = tok.double(), torch.zeros(tok.shape, dtype=torch.float64, device=tok.device)
    else:
        y, e = layer_norm(tok.reshape(-1, C), norm_w, norm_b, eps, scale)
        y, e = y.reshape(Bn, T, C), e.reshape(Bn, T, C)
    sp, bp = y[:, 1 + R:], e[:, 1 + R:]
    if layout == LAYOUT_CHANNELS:
        sp, bp = sp.transpose(1, 2), bp.transpose(1, 2)
    return (sp.contiguous(), bp.contiguous()), (y[:, 0].contiguous(), e[:, 0].contiguous())


def attention(qkv, H, chunk=256, sub=32, scale=1.0):
    """``gsr_attention_forward``: qkv [B, N, 3 H 64] fp32 -> (S, B) [B, N, H 64]."""
    Bn, N, _ = qkv.shape
    dev = qkv.device
    t = qkv.reshape(Bn, N, 3, H, ATT_D).permute(2, 0, 3, 1, 4).double()
    q, k, v = t[0] * 0.125, t[1], t[2]                                 # [B, H, N, 64]
    T = (N + ATT_BN - 1) // ATT_BN
    ks = score_kappa(scale).to(dev)
    kp, _ = pv_kappa(scale)
    key = torch.arange(N, device=dev)
    tile = key // ATT_BN
    kkey = kp.to(dev)[key % ATT_BN] + scale * U * (T - tile.clamp(min=1)).double()   # P V steps + merges into O
    nexp = (T - tile + 1).double()
    rho_l = scale * U * (17 + T + 1)
    S = torch.empty(Bn, H, N, ATT_D, dtype=torch.float64, device=dev)
    Bd = torch.empty_like(S)
    for b in range(Bn):
        for h in range(H):
            kk, vv = k[b, h], v[b, h]
            ka, va = kk.abs(), vv.abs()
            vmax = float(va.max())
            for r0 in range(0, N, chunk):
                qc = q[b, h, r0:r0 + chunk]
                s = qc @ kk.T
                es = (qc.abs() * ks) @ ka.T * SECOND
                smax, am = s.max(-1, keepdim=True)
                esm = es.max(-1, keepdim=True).values
                p = torch.exp(s - smax)
                L = p.sum(-1, keepdim=True)
                o = (p @ vv) / L
                eta = es + scale * (2 * U * (smax - s + 2 * esm) + EXP_ULP * TRUNC * nexp)
                ep = torch.expm1(eta * SECOND)
                emax = ep.max(-1, keepdim=True).values
                den = L * (1 - emax)
                num = torch.empty_like(o)
                for i0 in range(0, qc.shape[0], sub):
                    dv = (vv.unsqueeze(0) - o[i0:i0 + sub].unsqueeze(1)).abs()          # [sub, N, 64]
                    num[i0:i0 + sub] = ((p[i0:i0 + sub] * ep[i0:i0 + sub]).unsqueeze(-1) * dv).sum(1)
                t1 = num / den
                eo = ((p * (1 + ep) * kkey) @ va) * SECOND
                bo = t1 + eo / den / (1 - rho_l) + (o.abs() + t1) * rho_l / (1 - rho_l)
                bo = bo + scale * U * (o.abs() + bo) + scale * (N + 64 * T) * 2.0 ** -124 * vmax
                # determined rows: one key above every other by more than 110 + 2 max Es
                s2 = s.scatter(-1, am, -math.inf)
                det = (s2.max(-1, keepdim=True).values - smax + 2 * esm < -110).squeeze(-1)
                if bool(det.any()):
                    vdom = vv[am.squeeze(-1)]
                    bo[det] = (o[det] - vdom[det]).abs() * (1 + 2.0 ** -40)
                S[b, h, r0:r0 + chunk] = o
                Bd[b, h, r0:r0 + chunk] = bo * SECOND
    return S.transpose(1, 2).reshape(Bn, N, H * ATT_D), Bd.transpose(1, 2).reshape(Bn, N, H * ATT_D)


# ======================================================================================================================
# fp32 emulation of the kernels, as the model lets them round (CPU self-tests)
# ======================================================================================================================
MUTATIONS = ["one_tf32", "drop_corr_last", "split_rz", "ln_fp32_stats", "gelu_tanh", "gamma_ignored",
             "tail_rows_zero", "keys_unmasked", "no_rescale", "v_two_parts", "heads_swapped"]


def _tf32(x, rz=False):
    bits = x.contiguous().view(torch.int32)
    if not rz:
        bits = bits + 0x1000                                  # sign-magnitude: adding half an ulp rounds half away
    return (bits & ~0x1FFF).view(torch.float32)


def split(x, mut=None):
    hi = _tf32(x, mut == "split_rz")
    lo = _tf32(x - hi, mut == "split_rz")
    return hi, lo


def _rz32(s):
    f = s.float()
    over = f.double().abs() > s.abs()
    return torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)


def kstep(acc, prods):
    """One k-step at the model's worst under premise P1: each addend truncated at 2^-24 of the largest one's leading
    bit, the exact aligned sum truncated to fp32.  acc [...] fp32, prods [..., k] exact products in float64."""
    terms = torch.cat([acc.double().unsqueeze(-1), prods], -1)
    mx = terms.abs().amax(-1, keepdim=True).clamp_min(2.0 ** -1000)
    ulp = torch.exp2(torch.floor(torch.log2(mx)) - 24)                    # 24 bits + the alignment bit of P1
    return _rz32((torch.trunc(terms / ulp) * ulp).sum(-1))


def _prod(a, b):
    """[M, N, k] exact products of a [M, k] and b [N, k] (fp32 -> float64)."""
    return a.double().unsqueeze(1) * b.double().unsqueeze(0)


def emulate_gemm(a, w, mut=None):
    """vit_gemm_kernel's dot products: a [M, K], w [N, K] fp32 -> [M, N] fp32."""
    M, K = a.shape
    Kp = (K + VK - 1) // VK * VK
    a = F.pad(a, (0, Kp - K))
    w = F.pad(w, (0, Kp - K))
    ah, al = split(a, mut)
    wh, wl = split(w, mut)
    if mut == "one_tf32":
        wl = torch.zeros_like(wl)
    acc = torch.zeros(M, w.shape[0])
    chunks = Kp // VK
    for c in range(chunks):
        corr = torch.zeros_like(acc)
        hh = torch.zeros_like(acc)
        for j in range(4):
            ks = slice(c * VK + 8 * j, c * VK + 8 * j + 8)
            if not (mut == "drop_corr_last" and c == chunks - 1):
                corr = kstep(corr, _prod(al[:, ks], wh[:, ks]))
                corr = kstep(corr, _prod(ah[:, ks], wl[:, ks]))
            hh = kstep(hh, _prod(ah[:, ks], wh[:, ks]))
        acc = acc + (hh + corr)
    return acc


def _fma_or_not(a, b, c, gen):
    """a * b + c in fp32, fused or not at random per element."""
    fused = (a.double() * b.double() + c.double()).float()
    return torch.where(torch.rand(fused.shape, generator=gen) < 0.5, fused, a * b + c)


def emulate_ln(x, w, b, eps, gen, mut=None):
    xd = x.double()
    K = x.shape[-1]
    if mut == "ln_fp32_stats":
        mu32 = x.mean(-1, keepdim=True)
        var32 = torch.clamp((x * x).mean(-1, keepdim=True) - mu32 * mu32, min=0)
        mu, rs = mu32, 1 / torch.sqrt(var32 + eps)
    else:
        s, q = xd.sum(-1, keepdim=True), (xd * xd).sum(-1, keepdim=True)
        mud = s / K
        var = torch.clamp(q / K - mud * mud, min=0)
        mu, rs = mud.float(), (1 / torch.sqrt(var + float(torch.tensor(eps, dtype=torch.float32)))).float()
    return _fma_or_not((x - mu) * rs, w, b, gen)


def emulate_linear(op, x, w, b, ln_w=None, ln_b=None, eps=1e-6, gamma=None, resid=None, seed=0, mut=None):
    gen = torch.Generator().manual_seed(seed)
    a = emulate_ln(x, ln_w, ln_b, eps, gen, mut) if op != RESIDUAL else x
    v = emulate_gemm(a, w, mut) + b
    if op == LN_GELU:
        if mut == "gelu_tanh":
            v = F.gelu(v, approximate="tanh")
        else:
            v = 0.5 * v * (1 + torch.erf(v * torch.tensor(math.sqrt(0.5), dtype=torch.float32)))
    elif op == RESIDUAL:
        if gamma is not None and mut != "gamma_ignored":
            v = _fma_or_not(v, gamma.expand_as(v), resid, gen)
        else:
            v = resid + v
    if mut == "tail_rows_zero":
        M = v.shape[0]
        start = (M - 1) // VB * VB                                # the last row tile: its second half (or its row)
        v[start + (M - start) // 2:] = 0
    return v


def emulate_output(tok, R, norm_w, norm_b, eps, layout=LAYOUT_TOKENS, seed=0, mut=None):
    gen = torch.Generator().manual_seed(seed)
    Bn, T, C = tok.shape
    y = tok if norm_w is None else emulate_ln(tok.reshape(-1, C), norm_w, norm_b, eps, gen, mut).reshape(Bn, T, C)
    p = y[:, 1 + R:]
    return (p.transpose(1, 2) if layout == LAYOUT_CHANNELS else p).contiguous(), y[:, 0].contiguous()


def emulate_attention(qkv, H, mut=None):
    """attention_fwd_kernel in fp32: per (batch, head), 64-key tiles, the kernel's accumulator order, online softmax,
    P split in registers, the per-thread partial sums of l."""
    Bn, N, _ = qkv.shape
    T = (N + ATT_BN - 1) // ATT_BN
    Np = T * ATT_BN
    t = qkv.reshape(Bn, N, 3, H, ATT_D).permute(2, 0, 3, 1, 4)
    q, k, v = t[0] * 0.125, t[1], t[2]
    if mut == "heads_swapped" and H > 1:
        v = v[:, [1, 0] + list(range(2, H))]
    out = torch.empty(Bn, H, N, ATT_D)
    for b in range(Bn):
        for h in range(H):
            qh, ql = split(q[b, h])
            kk = F.pad(k[b, h], (0, 0, 0, Np - N))
            vv = F.pad(v[b, h], (0, 0, 0, Np - N))
            kh, kl = split(kk)
            vh = _tf32(vv)
            vm, vlo = split(vv - vh)                                 # exact: hi + mid + lo = v
            if mut == "v_two_parts":
                vlo = torch.zeros_like(vlo)
            m = torch.full((N, 1), -math.inf)
            o = torch.zeros(N, ATT_D)
            lt = torch.zeros(N, 4)                                   # the four threads' partial sums
            for i in range(T):
                js = slice(i * ATT_BN, (i + 1) * ATT_BN)
                sa = torch.zeros(N, ATT_BN)
                for c in range(8):
                    d = slice(8 * c, 8 * c + 8)
                    sa = kstep(sa, _prod(ql[:, d], kh[js, d]))
                    sa = kstep(sa, _prod(qh[:, d], kl[js, d]))
                sb = torch.zeros_like(sa)
                for c in range(8):
                    d = slice(8 * c, 8 * c + 8)
                    if c < 4:
                        sa = kstep(sa, _prod(qh[:, d], kh[js, d]))
                    else:
                        sb = kstep(sb, _prod(qh[:, d], kh[js, d]))
                sc = sa + sb
                if mut != "keys_unmasked":
                    sc[:, max(0, N - i * ATT_BN):] = -math.inf
                mx = torch.maximum(m, sc.max(-1, keepdim=True).values)
                a = torch.exp(m - mx)
                m = mx
                p = torch.exp(sc - m)
                pt = p.reshape(N, 8, 4, 2).permute(0, 2, 1, 3).reshape(N, 4, 16)   # thread t: keys 8j + 2t + e
                ls = torch.zeros(N, 4)
                for e in range(16):
                    ls = ls + pt[:, :, e]
                lt = ((lt.double() * a.double() + ls.double()).float())
                ph, pl = split(p)
                ot = torch.zeros(N, ATT_D)
                for j in range(8):
                    ky = slice(i * ATT_BN + 8 * j, i * ATT_BN + 8 * j + 8)
                    kj = slice(8 * j, 8 * j + 8)
                    ot = kstep(ot, _prod(pl[:, kj], vh[ky].T))
                    ot = kstep(ot, _prod(ph[:, kj], vlo[ky].T))
                    ot = kstep(ot, _prod(ph[:, kj], vm[ky].T))
                for j in range(8):
                    ky = slice(i * ATT_BN + 8 * j, i * ATT_BN + 8 * j + 8)
                    ot = kstep(ot, _prod(ph[:, 8 * j:8 * j + 8], vh[ky].T))
                if mut == "no_rescale":
                    o = o + ot
                else:
                    o = (o.double() * a.double() + ot.double()).float()
            l = (lt[:, 0] + lt[:, 1]) + (lt[:, 2] + lt[:, 3])
            out[b, h] = o / l.unsqueeze(-1)
    return out.transpose(1, 2).reshape(Bn, N, H * ATT_D)
