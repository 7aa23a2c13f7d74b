"""TEST INFRASTRUCTURE -- fp64 oracle of the fused colour op (csrc/appearance.cu) AS THE KERNEL ROUNDS IT, with an
a-priori bound on how far the kernel's value of every entry can be from the oracle's.  Only tests/ may import this.

What is modelled (appearance.cu):
  * bf16 operands, rounded to nearest even: X = [min(dc, 1), gemb], W1[:, :27], W2, W3, H1, H2 (forward) and
    dO, dZ2, dZ1 (backward);
  * the folded layer-1 bias b1 + W1[:, 27:] . aemb (fp32 fma chain) and the bias_hi + bias_lo bf16 split of every
    bias (|hi + lo - b| <= 2^-17 |b|);
  * fp32 where the kernel is fp32: the colour stage (view direction, SH basis, tone map, clamps and their backward),
    db3 from the fp32 dOut, and the unpack products dW1[:, 27:] = db1 * aemb and daemb = W1[:, 27:]^T db1.
Everything is evaluated in float64 on the inputs' device, in row chunks, so it runs at millions of Gaussians on a GPU
and at 10^5 on a CPU.

Every value is an interval, centre +- radius (midpoint-radius interval arithmetic), that contains the kernel's value:
  * fp32 arithmetic (IEEE, round to nearest): unit roundoff U32 = 2^-24, a k-term fp32 sum gets gamma_k * sum |term|.
  * Tensor-core (wgmma) fp32 accumulation is not IEEE: it aligns the products of a K = 16 group to the largest exponent
    of the group and the accumulator and keeps a limited number of bits.  Assumed: each aligned product loses at most
    one fp32 ulp of the group's largest magnitude.  That gives an error <= n * 2^-22 * sum |term| for an n-term chain
    (U_TC = 2^-22, twice the fp32 unit roundoff, to also cover the normalisation of every group).  The weight-gradient
    sums chain the 128 rows of every tile a CTA owns, then the CTAs' fp32 atomics: n = 128 * tiles per CTA + CTAs + 64.
  * A bf16 rounding of a value known only to within +-e is the interval [bf16(v - e), bf16(v + e)] (rounding is
    monotone).  When that interval holds two bf16 values the entry is FLAGGED; its one-ulp ambiguity then flows into
    every bound downstream through |weights|.
  * A ReLU mask or colour-stage clamp whose argument's interval straddles the kink is UNDETERMINED: the mask is the
    interval [0, 1], so the downstream values allow either choice, and the row is reported as undetermined.  Interval
    products keep both choices inside every bound that depends on them, the weight gradients included.
With ``exact_mlp=True`` (lattice scenes, see ``lattice_scene``) the forward GEMM sums carry no accumulation error: the
scene's operands sit on dyadic grids on which every partial sum is an fp32 number in any order, which
``check_lattice_premise`` asserts.  The colour stage is then the only rounding in the forward.
"""
from __future__ import annotations

import math

import torch

U32 = 2.0 ** -24
U_TC = 2.0 ** -22
F32_001 = float(torch.tensor(0.01, dtype=torch.float32))           # the kernel's 0.01f
F32_C0 = float(torch.tensor(0.28209479177387814, dtype=torch.float32))
E_DIR = 16 * U32             # |fp32 view direction - exact| per component (difference, sum of squares, sqrt, 1/x, x)
TILE = 128
N_IN1 = 27                   # dc 3 + gemb 24: the K of layer 1 besides the bias columns

C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435)


def gamma(n, u=U32):
    return n * u / (1.0 - n * u)


class Iv:
    """An interval centre +- radius of float64 tensors."""
    __slots__ = ("c", "r")

    def __init__(self, c, r=None):
        self.c = c
        self.r = torch.zeros_like(c) if r is None else r

    @staticmethod
    def hull(lo, hi):
        return Iv((lo + hi) * 0.5, (hi - lo) * 0.5)

    @property
    def lo(self):
        return self.c - self.r

    @property
    def hi(self):
        return self.c + self.r

    def mag(self):
        return self.c.abs() + self.r

    def __add__(self, o):
        o = _iv(o)
        return Iv(self.c + o.c, self.r + o.r)

    __radd__ = __add__

    def __sub__(self, o):
        o = _iv(o)
        return Iv(self.c - o.c, self.r + o.r)

    def __neg__(self):
        return Iv(-self.c, self.r)

    def __mul__(self, o):
        o = _iv(o)
        return Iv(self.c * o.c, self.c.abs() * o.r + o.c.abs() * self.r + self.r * o.r)

    __rmul__ = __mul__

    def __getitem__(self, idx):
        return Iv(self.c[idx], self.r[idx])

    def exact(self):
        return self.r == 0

    def widen(self, e):
        return Iv(self.c, self.r + e)


def _iv(x):
    if isinstance(x, Iv):
        return x
    if not torch.is_tensor(x):
        x = torch.tensor(float(x), dtype=torch.float64)
    return Iv(x, torch.zeros_like(x))


def cat(ivs, dim):
    return Iv(torch.cat([v.c for v in ivs], dim), torch.cat([v.r for v in ivs], dim))


def stack(ivs, dim):
    return Iv(torch.stack([v.c for v in ivs], dim), torch.stack([v.r for v in ivs], dim))


# ---- roundings ----------------------------------------------------------------------------------------------------
def bf16(x):
    return x.to(torch.bfloat16).to(torch.float64)


def f32(x):
    return x.to(torch.float32).to(torch.float64)


def round_bf16(v: Iv):
    """(interval of the kernel's bf16 rounding of a value in v, flagged entries)"""
    lo, hi = bf16(v.lo), bf16(v.hi)
    return Iv.hull(lo, hi), lo != hi


def fp32_op(v: Iv, exact_value=None):
    """One fp32 rounding of the result interval v.  ``exact_value`` (where given) is the fp32 result the kernel
    computes when every operand is an exactly known fp32 number; those entries keep radius 0."""
    out = v.widen(U32 * v.mag())
    if exact_value is None:
        return out
    ex = v.exact()
    return Iv(torch.where(ex, exact_value, out.c), torch.where(ex, torch.zeros_like(out.r), out.r))


def mul32(a: Iv, b: Iv):
    a, b = _iv(a), _iv(b)
    return fp32_op(a * b, (a.c.float() * b.c.float()).double() if _all_f32(a.c, b.c) else None)


def div32(a: Iv, d: float):
    a = _iv(a)
    af = a.c.float()
    ex = (af / torch.full_like(af, d)).double() if _all_f32(a.c) else None      # IEEE division, as the kernel's `/`
    return fp32_op(Iv(a.c / d, a.r / abs(d)), ex)


def fma32(a: Iv, b: Iv, c: Iv):
    """fmaf(a, b, c): exact where every operand is exact and a*b + c is an fp32 number (then no rounding happens)."""
    a, b, c = _iv(a), _iv(b), _iv(c)
    p = a * b + c
    out = p.widen(U32 * p.mag())
    ab = a.c * b.c                                    # exact in fp64 for fp32 operands
    s = ab + c.c
    bb = s - ab
    err = (ab - (s - bb)) + (c.c - bb)                # TwoSum: s + err == ab + c exactly
    ok = a.exact() & b.exact() & c.exact() & (err == 0) & (f32(s) == s)
    return Iv(torch.where(ok, s, out.c), torch.where(ok, torch.zeros_like(out.r), out.r))


def fsum(terms, extra_ops=0):
    """An fp32 sum / fma chain of the given intervals (any order)."""
    c = sum(t.c for t in terms)
    r = sum(t.r for t in terms)
    m = sum(t.mag() for t in terms)
    return Iv(c, r + gamma(len(terms) + extra_ops) * m)


def _all_f32(*xs):
    return all(bool((f32(x) == x).all()) for x in xs)


# ---- kinks ---------------------------------------------------------------------------------------------------------
class Mask:
    """A predicate on an interval: ``sure`` where it holds for every value of the interval, ``maybe`` where it holds for
    some.  ``undetermined = maybe & ~sure``."""
    __slots__ = ("sure", "maybe")

    def __init__(self, sure, maybe):
        self.sure, self.maybe = sure, maybe

    @property
    def undetermined(self):
        return self.maybe & ~self.sure

    def apply(self, v: Iv):
        """v where the predicate holds, 0 where it does not, the hull of both where undetermined"""
        v = _iv(v)
        z = torch.zeros_like(v.c)
        und = Iv.hull(torch.minimum(v.lo, z), torch.maximum(v.hi, z))
        c = torch.where(self.sure, v.c, torch.where(self.maybe, und.c, z))
        r = torch.where(self.sure, v.r, torch.where(self.maybe, und.r, z))
        return Iv(c, r)


def ge0(v: Iv):
    return Mask(v.lo >= 0, v.hi >= 0)


def le(v: Iv, t):
    return Mask(v.hi <= t, v.lo <= t)


def relu_mask(z: Iv, rounded=True):
    """the kernel's mask: the stored activation bf16(relu(z)) is positive"""
    f = bf16 if rounded else (lambda x: x)
    return Mask(f(z.lo.clamp_min(0)) > 0, f(z.hi.clamp_min(0)) > 0)


def iv_min(v: Iv, t):
    return Iv.hull(v.lo.clamp_max(t), v.hi.clamp_max(t))


def iv_max(v: Iv, t):
    return Iv.hull(v.lo.clamp_min(t), v.hi.clamp_min(t))


# ---- SH basis --------------------------------------------------------------------------------------------------------
def sh_basis(deg, x, y, z, absval=False):
    """[..., 16] basis values (0 above the degree).  absval: the same polynomials with |coefficients| and every
    difference turned into a sum -- evaluated at |x|, |y|, |z| it dominates |b_k| and |grad b_k|, and
    absbasis(|d| + e) - absbasis(|d|) bounds |b_k(d') - b_k(d)| for |d' - d| <= e."""
    A = (lambda c: abs(c)) if absval else (lambda c: c)
    S = (lambda a, b: a + b) if absval else (lambda a, b: a - b)
    zero = torch.zeros_like(x)
    b = [zero + A(C0)] + [zero] * 15
    if deg > 0:
        b[1], b[2], b[3] = A(-C1) * y, A(C1) * z, A(-C1) * x
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b[4], b[5], b[6] = A(C2[0]) * xy, A(C2[1]) * yz, A(C2[2]) * S(S(2.0 * zz, xx), yy)
        b[7], b[8] = A(C2[3]) * xz, A(C2[4]) * S(xx, yy)
        if deg > 2:
            b[9] = A(C3[0]) * y * S(3.0 * xx, yy)
            b[10] = A(C3[1]) * xy * z
            b[11] = A(C3[2]) * y * S(S(4.0 * zz, xx), yy)
            b[12] = A(C3[3]) * z * S(S(2.0 * zz, 3.0 * xx), 3.0 * yy)
            b[13] = A(C3[4]) * x * S(S(4.0 * zz, xx), yy)
            b[14] = A(C3[5]) * z * S(xx, yy)
            b[15] = A(C3[6]) * x * S(xx, 3.0 * yy)
    return torch.stack(b, dim=-1)


def _basis_grad(deg, d, g, absval):
    """sum_k g[..., k] grad b_k(d) -> [..., 3] (autograd of the polynomial, as sh_basis_grad_dot differentiates it)"""
    if deg == 0:                                      # the basis is constant
        return torch.zeros_like(d)
    with torch.enable_grad():
        d = d.detach().clone().requires_grad_(True)
        b = sh_basis(deg, d[..., 0], d[..., 1], d[..., 2], absval)
        (gd,) = torch.autograd.grad((b * g).sum(), d)
    return gd.detach()


def basis_iv(deg, d):
    """the kernel's fp32 basis values at the fp32 direction (|d_kernel - d| <= E_DIR per component)"""
    b = sh_basis(deg, d[..., 0], d[..., 1], d[..., 2])
    a = d.abs()
    ba0 = sh_basis(deg, a[..., 0], a[..., 1], a[..., 2], True)
    a1 = a + E_DIR
    ba1 = sh_basis(deg, a1[..., 0], a1[..., 1], a1[..., 2], True)
    return Iv(b, (ba1 - ba0) + 12 * U32 * ba1)


def basis_grad_iv(deg, d, g: Iv):
    c = _basis_grad(deg, d, g.c, False)
    a, ga = d.abs(), g.c.abs()
    lo = _basis_grad(deg, a, ga, True)
    hi = _basis_grad(deg, a + E_DIR, ga + g.r, True)
    return Iv(c, (hi - lo) + 24 * U32 * hi)


def through_normalize_iv(d, inv_len, g: Iv):
    """(g - d (d . g)) * inv_len with the kernel's fp32 d (E_DIR) and inv_len (relative 4 U32)"""
    dg = (g.c * d).sum(-1, keepdim=True)
    c = g.c - d * dg
    a, ga = d.abs(), g.c.abs()
    n_lo = ga + a * (ga * a).sum(-1, keepdim=True)
    a1, ga1 = a + E_DIR, ga + g.r
    n_hi = ga1 + a1 * (ga1 * a1).sum(-1, keepdim=True)
    n = Iv(c, (n_hi - n_lo) + 8 * U32 * n_hi)
    il = Iv(inv_len, 4 * U32 * inv_len)
    out = n * il
    return out.widen(U32 * out.mag())


# ---- the op ----------------------------------------------------------------------------------------------------------
def effective_biases(W1, b1, W2, b2, W3, b3, aemb, bf16_operands=True, exact_fold=False):
    """the biases the kernel's GEMMs add: (layer-1 bias interval incl. the folded image embedding, b2, b3 intervals)"""
    W1, b1, b2, b3, aemb = (t.double() for t in (W1, b1, b2, b3, aemb))
    terms = W1[:, N_IN1:] * aemb[None]
    fold = b1 + terms.sum(1)
    fold_err = 0.0 if exact_fold else gamma(terms.shape[1] + 1) * (b1.abs() + terms.abs().sum(1))

    def split(b):                                     # bias_hi + bias_lo of an fp32 value, as appearance_pack_kernel
        hi = bf16(b)
        return hi + bf16(b - hi)

    if not bf16_operands:
        return Iv(fold, torch.full_like(fold, 0.0) + fold_err), Iv(b2), Iv(b3)
    if exact_fold:
        return Iv(split(fold)), Iv(split(b2)), Iv(split(b3))
    e1 = fold_err + 2.0 ** -17 * (fold.abs() + fold_err)
    return Iv(fold, e1 + torch.zeros_like(fold)), Iv(split(b2)), Iv(split(b3))


def _gemm(a: Iv, W, K, acc=True):
    """a [R, k] @ W^T (W exact [n, k]): centre, operand radius and an n-term tensor-core accumulation bound"""
    Wa = W.abs()
    c = a.c @ W.T
    r = a.r @ Wa.T
    if acc:
        r = r + K * U_TC * (a.mag() @ Wa.T)
    return Iv(c, r)


def _plus_bias(z: Iv, b: Iv, K, acc=True):
    return Iv(z.c + b.c, z.r + b.r + ((K * U_TC) * b.c.abs() if acc else 0.0))


def colour_op(dc, rest, gemb, aemb, W1, b1, W2, b2, W3, b3, means, campos, deg, dL_toned=None, dL_raw=None, *,
              exact_mlp=False, bf16_operands=True, bf16_backward=True, chunk=None):
    """Forward and backward of the fused colour op.  Returns a dict:
      raw, toned, g_dc, g_rest, g_gemb, g_means  -- Iv per row entry ([P, 3], [P, 45], [P, 24], [P, 3])
      undetermined                               -- bool [P]: a ReLU mask or colour-stage clamp of the row is undetermined
      sums                                       -- weight-gradient sums over the rows (see weight_grads)
      stats                                      -- counts of flagged roundings and undetermined masks per kind
    With dL_toned None only the forward is evaluated.  bf16_operands / bf16_backward False drop the bf16 roundings
    (of the forward operands / of dO, dZ2 and dZ1): the fp64 network with the kernel's fp32 bounds."""
    dev = dc.device
    d64 = lambda t: None if t is None else t.detach().to(dev, torch.float64)
    dc, rest, gemb, aemb, W1, b1, W2, b2, W3, b3, means, campos = (
        d64(t) for t in (dc, rest, gemb, aemb, W1, b1, W2, b2, W3, b3, means, campos))
    dL_toned, dL_raw = d64(dL_toned), d64(dL_raw)
    P = dc.shape[0]
    chunk = chunk or (1 << 18 if dev.type == "cuda" else 1 << 14)
    rb_f = bf16 if bf16_operands else (lambda x: x)
    W1b, W2b, W3b = rb_f(W1[:, :N_IN1]), rb_f(W2), rb_f(W3)
    bias1, bias2, bias3 = effective_biases(W1, b1, W2, b2, W3, b3, aemb, bf16_operands, exact_fold=exact_mlp)
    acc = not exact_mlp
    rnd_fwd = (lambda v: round_bf16(v)) if bf16_operands else (lambda v: (v, torch.zeros_like(v.c, dtype=torch.bool)))
    rnd_bwd = (lambda v: round_bf16(v)) if bf16_backward else (lambda v: (v, torch.zeros_like(v.c, dtype=torch.bool)))
    bwd = dL_toned is not None

    out = {k: [] for k in ("raw", "toned", "g_dc", "g_rest", "g_gemb", "g_means", "undetermined")}
    stats = {k: 0 for k in ("H1 flagged", "H2 flagged", "dO flagged", "dZ2 flagged", "dZ1 flagged",
                            "layer-1 masks undetermined", "layer-2 masks undetermined", "colour clamps undetermined")}
    sums = {}

    def acc_sum(name, A: Iv, B: Iv):
        c, r, m = A.c.T @ B.c, A.c.abs().T @ B.r + A.r.T @ (B.c.abs() + B.r), A.mag().T @ B.mag()
        if name in sums:
            c0, r0, m0 = sums[name]
            c, r, m = c0 + c, r0 + r, m0 + m
        sums[name] = (c, r, m)

    for s0 in range(0, P, chunk):
        sl = slice(s0, min(P, s0 + chunk))
        R = sl.stop - sl.start
        fdc = dc[sl]
        feats = torch.cat((fdc, rest[sl]), 1).view(R, 16, 3)                 # [R, k, c]
        fv = feats.clamp_max(1.0)
        # ---- MLP forward ------------------------------------------------------------------------------------------
        X = rb_f(torch.cat((fv[:, 0, :], gemb[sl]), 1))                       # [R, 27]
        Z1 = _plus_bias(_gemm(Iv(X), W1b, 32, acc), bias1, 32, acc)
        m1 = relu_mask(Z1, bf16_operands)
        H1, fl = rnd_fwd(iv_max(Z1, 0.0))
        stats["H1 flagged"] += int(fl.sum())
        Z2 = _plus_bias(_gemm(H1, W2b, 144, acc), bias2, 144, acc)
        m2 = relu_mask(Z2, bf16_operands)
        H2, fl = rnd_fwd(iv_max(Z2, 0.0))
        stats["H2 flagged"] += int(fl.sum())
        O = _plus_bias(_gemm(H2, W3b, 144, acc), bias3, 144, acc)             # [R, 6]
        und = m1.undetermined.any(1) | m2.undetermined.any(1)
        stats["layer-1 masks undetermined"] += int(m1.undetermined.sum())
        stats["layer-2 masks undetermined"] += int(m2.undetermined.sum())
        # ---- colour stage (fp32) ----------------------------------------------------------------------------------
        v = means[sl] - campos[None]
        nrm = v.norm(dim=1, keepdim=True).clamp_min(1e-12)
        inv_len = 1.0 / nrm
        d = v * inv_len
        b = basis_iv(deg, d)                                                   # [R, 16]
        bk = b[:, :, None]                                                     # [R, 16, 1]
        fvi = Iv(fv)
        rr = fsum([bk[:, k] * fvi[:, k] for k in range(16)])                   # [R, 3]
        rp = fp32_op(rr + 0.5)
        mul = mul32(Iv(torch.full_like(O.c[:, 3:], F32_001)), O[:, 3:])          # [R, 3]
        off = div32(mul32(Iv(torch.full_like(O.c[:, :3], F32_001)), O[:, :3]), F32_C0)
        t0p = fma32(fvi[:, 0], mul, off)
        tp = [t0p] + [mul32(fvi[:, k], mul) for k in range(1, 16)]
        tc = [iv_min(t, 1.0) for t in tp]
        ss = fsum([bk[:, k] * tc[k] for k in range(16)])
        sp = fp32_op(ss + 0.5)
        out["raw"].append(iv_max(rp, 0.0))
        out["toned"].append(iv_max(sp, 0.0))
        if not bwd:
            out["undetermined"].append(und)
            continue
        # ---- colour stage backward ----------------------------------------------------------------------------------
        mr, mt = ge0(rp), ge0(sp)
        dLr = mr.apply(Iv(dL_raw[sl])) if dL_raw is not None else Iv(torch.zeros_like(rp.c))
        dLt = mt.apply(Iv(dL_toned[sl]))
        masks = [le(t, 1.0) for t in tp]
        cu = (mt.undetermined.any(1) | (mr.undetermined.any(1) if dL_raw is not None else False))
        for k, m in enumerate(masks):
            if k <= (deg + 1) ** 2 - 1:
                cu = cu | m.undetermined.any(1)
        stats["colour clamps undetermined"] += int(cu.sum())
        und = und | cu
        dt = [m.apply(mul32(bk[:, k], dLt)) for k, m in enumerate(masks)]   # [R, 3] each
        dmul = fsum([dt[k] * fvi[:, k] for k in range(16)])
        dOut = cat([div32(mul32(Iv(torch.full_like(dt[0].c, F32_001)), dt[0]), F32_C0),
                    mul32(Iv(torch.full_like(dmul.c, F32_001)), dmul)], 1)        # [R, 6] fp32
        g_dc_col = fma32(dt[0], mul, mul32(bk[:, 0], dLr))
        g_rest = [Mask(feats[:, k] <= 1.0, feats[:, k] <= 1.0).apply(fma32(dt[k], mul, mul32(bk[:, k], dLr)))
                  for k in range(1, 16)]
        gk = stack([fsum([dLr * fvi[:, k], dLt * tc[k]], extra_ops=0) for k in range(16)], 1)   # [R, 16, 3]
        gk = Iv(gk.c.sum(2), gk.r.sum(2) + gamma(7) * gk.mag().sum(2))                        # the 3 channels
        dd = basis_grad_iv(deg, d, gk)
        out["g_means"].append(through_normalize_iv(d, inv_len, dd))
        # ---- MLP backward -----------------------------------------------------------------------------------------
        dO, fl = rnd_bwd(dOut)
        stats["dO flagged"] += int(fl.sum())
        dH2 = Iv(dO.c @ W3b, dO.r @ W3b.abs() + 16 * U_TC * (dO.mag() @ W3b.abs()))
        dZ2r, fl = rnd_bwd(dH2)
        stats["dZ2 flagged"] += int((fl & m2.maybe).sum())
        dZ2 = m2.apply(dZ2r)
        dH1 = Iv(dZ2.c @ W2b, dZ2.r @ W2b.abs() + 128 * U_TC * (dZ2.mag() @ W2b.abs()))
        dZ1r, fl = rnd_bwd(dH1)
        stats["dZ1 flagged"] += int((fl & m1.maybe).sum())
        dZ1 = m1.apply(dZ1r)
        dX = Iv(dZ1.c @ W1b, dZ1.r @ W1b.abs() + 128 * U_TC * (dZ1.mag() @ W1b.abs()))   # [R, 27]
        gdc = fp32_op(g_dc_col + dX[:, :3])
        out["g_dc"].append(Mask(fdc <= 1.0, fdc <= 1.0).apply(gdc))
        g_rest = stack(g_rest, 1)                                               # [R, 15, 3]
        out["g_rest"].append(Iv(g_rest.c.reshape(R, 45), g_rest.r.reshape(R, 45)))
        out["g_gemb"].append(dX[:, 3:])
        out["undetermined"].append(und)
        # ---- weight-gradient sums -----------------------------------------------------------------------------------
        one = Iv(torch.ones((R, 1), dtype=torch.float64, device=dev))
        acc_sum("W3", dO, H2)
        acc_sum("b3", dOut, one)
        acc_sum("W2", dZ2, H1)
        acc_sum("b2", dZ2, one)
        acc_sum("W1", dZ1, Iv(X))
        acc_sum("b1", dZ1, one)

    res = {}
    for k, parts in out.items():
        if not parts:
            continue
        res[k] = torch.cat(parts) if k == "undetermined" else cat(parts, 0)
    res["stats"] = stats
    res["P"] = P
    if bwd:
        res["sums"] = {k: tuple(t if k.startswith("W") else t.reshape(-1) for t in v) for k, v in sums.items()}
        res["W1"], res["aemb"] = W1, aemb
    return res


def sum_chain(P, ctas_per_sm, num_sms):
    """number of terms chained into one weight-gradient entry: the rows of every tile of one CTA, then the CTAs"""
    tiles = (P + TILE - 1) // TILE
    grid = min(tiles, ctas_per_sm * num_sms)
    return TILE * ((tiles + grid - 1) // grid) + grid + 64


def weight_grads(res, ctas_per_sm=1, num_sms=132):
    """parameter gradients as the unpack kernel returns them: W1 [128, 59], b1, W2, b2, W3, b3, aemb.
    ctas_per_sm = 1 for gsr_appearance_colors_backward, 2 for gsr_appearance_embedding_backward."""
    n = sum_chain(res["P"], ctas_per_sm, num_sms)
    g = {k: Iv(c, r + n * U_TC * m) for k, (c, r, m) in res["sums"].items()}
    W1, aemb = res["W1"], res["aemb"]
    db1 = g["b1"]
    g_w1e = mul32(Iv(db1.c[:, None].expand(-1, aemb.numel()).contiguous(), db1.r[:, None].expand(-1, aemb.numel()).contiguous()),
                  Iv(aemb[None].expand(db1.c.shape[0], -1).contiguous()))
    g["W1"] = cat([g["W1"], g_w1e], 1)
    Wa = W1[:, N_IN1:]
    g["aemb"] = Iv(Wa.T @ db1.c, Wa.abs().T @ db1.r + gamma(128) * (Wa.abs().T @ db1.mag()))
    return g


# ---- comparison ------------------------------------------------------------------------------------------------------
def excess(kernel, ref: Iv):
    """|kernel - centre| - radius per entry (> 0: outside the bound); a 1e-12 relative slack covers the oracle's fp64"""
    k = kernel.detach().to(ref.c.device, torch.float64)
    return (k - ref.c).abs() - ref.r - 1e-12 * ref.mag() - 1e-300


def ratio(kernel, ref: Iv):
    """largest |kernel - centre| / radius (inf where an exact entry differs)"""
    k = kernel.detach().to(ref.c.device, torch.float64)
    e = (k - ref.c).abs()
    r = ref.r + 1e-12 * ref.mag() + 1e-300
    return float((e / r).max()) if e.numel() else 0.0


def check(name, kernel, ref: Iv, rows=None):
    """assert every entry (or every entry of the selected rows) of `kernel` lies within the oracle's bound"""
    ex = excess(kernel, ref)
    if rows is not None:
        ex = ex[rows.to(ex.device)]
    bad = ex > 0
    if bool(bad.any()):
        idx = bad.nonzero()[:5].tolist()
        raise AssertionError(f"{name}: {int(bad.sum())} entries outside the bound, first {idx}, worst excess "
                             f"{float(ex.max()):.3e}")


def check_row_grads(kernel: dict, res: dict):
    for k in ("g_dc", "g_rest", "g_gemb", "g_means"):
        check(k, kernel[k], res[k])


def check_weight_grads(kernel: dict, g: dict, names=("W1", "b1", "W2", "b2", "W3", "b3", "aemb")):
    for k in names:
        check("d" + k, kernel[k], g[k])


# ---- lattice scenes --------------------------------------------------------------------------------------------------
def lattice_scene(P, seed, device="cpu"):
    """Inputs on dyadic grids on which every forward GEMM sum of the kernel is exact in fp32 in any order (span of
    the largest partial sum over the grid step <= 2^20, checked by check_lattice_premise):
      features k/4 in [-1, 1.5] (so some equal 1 and some clamp), gemb and aemb k/4 in [-1, 1];
      W1, W2 k/8 with |k| <= 3, W3 k/8 with |k| <= 1, b1 k/32, b2 k/32, b3 = (k/8, ..., 100 + k/8, ...);
    output channel 2 of the tone map is the identity (W3 rows 2 and 5 zero, b3 = (.., 0, .., 100)): mul = 1, offset 0,
    so t == f exactly and the clamps `t <= 1` are hit exactly where a feature is 1.  Many layer-1 pre-activations are
    exactly 0.  Means and camera are random (the colour stage is fp32 either way)."""
    g = torch.Generator().manual_seed(seed)
    K = lambda lo, hi, *s: torch.randint(lo, hi + 1, s, generator=g).double()
    feats = K(-4, 6, P, 48) / 4
    gemb = K(-4, 4, P, 24) / 4
    aemb = K(-4, 4, 32) / 4
    W1 = K(-3, 3, 128, 59) / 8
    W2 = K(-3, 3, 128, 128) / 8
    W3 = K(-1, 1, 6, 128) / 8
    W3[2] = 0.0
    W3[5] = 0.0
    b1 = K(-32, 32, 128) / 32
    b2 = K(-32, 32, 128) / 32
    b3 = K(-8, 8, 6) / 8
    b3[3:] += 100.0
    b3[2], b3[5] = 0.0, 100.0
    means = torch.randn(P, 3, generator=g, dtype=torch.float64) * 2.0
    campos = torch.tensor([0.1, -0.2, 0.3], dtype=torch.float64)
    f = lambda t: t.float().to(device)
    return dict(dc=f(feats[:, :3]), rest=f(feats[:, 3:]), gemb=f(gemb), aemb=f(aemb), W1=f(W1), b1=f(b1), W2=f(W2),
                b2=f(b2), W3=f(W3), b3=f(b3), means=f(means), campos=f(campos))


def _grid_exact(x, step):
    return bool((torch.remainder(x.double() / step, 1.0) == 0).all())


def check_lattice_premise(s, span_bits=20):
    """Assert the lattice premise for scene `s`: every forward GEMM's terms lie on a grid of step 2^-e, the sum of
    their magnitudes is below 2^span_bits steps, and evaluating the sums in fp32 in two different orders and in fp64
    gives identical values.  Returns the worst span in bits per layer."""
    W1, W2, W3, aemb = (s[k].double().cpu() for k in ("W1", "W2", "W3", "aemb"))
    b1, b2, b3 = (s[k].double().cpu() for k in ("b1", "b2", "b3"))
    fold_terms = torch.cat((b1[:, None], W1[:, N_IN1:] * aemb[None]), 1)
    bias1 = fold_terms.sum(1)
    assert bool((fold_terms.float().sum(1).double() == bias1).all()) and bool(
        (fold_terms.flip(1).float().cumsum(1)[:, -1].double() == bias1).all()), "layer-1 bias fold is not exact"
    for b in (bias1, b2, b3):
        hi = bf16(b)
        assert bool((hi + bf16(b - hi) == b).all()), "a bias is not exact as bias_hi + bias_lo"
    X = torch.cat((s["dc"].double().cpu().clamp_max(1.0), s["gemb"].double().cpu()), 1)
    assert bool((bf16(X) == X).all()), "X is not bf16-exact"
    for W in (W1[:, :N_IN1], W2, W3):
        assert bool((bf16(W) == W).all()), "a weight is not bf16-exact"
    spans = []
    A = X
    for W, b, step in ((W1[:, :N_IN1], bias1, 2.0 ** -5), (W2, b2, 2.0 ** -8), (W3, b3, 2.0 ** -11)):
        terms_abs = A.abs() @ W.abs().T + b.abs()
        assert _grid_exact(A, step / 2.0 ** -3) and _grid_exact(W, 2.0 ** -3) and _grid_exact(b, step), "off the grid"
        spans.append(math.log2(float(terms_abs.max()) / step))
        assert spans[-1] <= span_bits, ("span", spans)
        z = A @ W.T + b
        Af, Wf = A.float(), W.float()
        z32a = b.float().expand(A.shape[0], -1).clone()                   # fp32, k ascending
        z32b = torch.zeros_like(z32a)                                     # fp32, k descending, bias last
        for j in range(A.shape[1]):
            z32a = z32a + Af[:, j:j + 1] * Wf[None, :, j]
            jj = A.shape[1] - 1 - j
            z32b = z32b + Af[:, jj:jj + 1] * Wf[None, :, jj]
        z32b = z32b + b.float()
        assert bool((z32a.double() == z).all()) and bool((z32b.double() == z).all()), "fp32 sums are not exact"
        A = bf16(z.clamp_min(0.0))
    return spans
