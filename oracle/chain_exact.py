"""TEST INFRASTRUCTURE -- fp64 oracle of the per-Gaussian chain rule (csrc/preprocess_bwd.cu, DESIGN.md 3.3) AS THE
KERNEL ROUNDS IT, with an a-priori bound on how far the kernel's value of every output entry can be from the oracle's.
Only tests/ may import this.

The chain rule is written once, in ``chain``, as the kernel's expression tree over an arithmetic back end:
  * ``IvArith``  -- midpoint-radius intervals in float64 (``color_exact.Iv``).  The centre is the exact value S of the
    formulas on the kernel's fp32 inputs; the radius B bounds the kernel's fp32 value.  Every fp32 operation adds
    u |result| (u = 2^-24) and an absolute 2^-149 (a product or quotient can land in the subnormal range); every
    ``a * b + c`` site that nvcc may contract is modelled as two roundings, which covers the fused and the unfused
    evaluation.  ``__fmaf_rn`` sites (quat_to_mat) are one rounding.  A result whose magnitude can reach the fp32
    overflow threshold gets an infinite radius.  With ``u = 0`` the same code is the plain fp64 evaluation.
  * ``F32Arith`` -- an fp32 emulation with torch float32 tensors, contracting each candidate fma site or not
    at random per entry (tests/test_chain_rule_exact.py: the bound must hold for it, and corruptions of it must not).
Decisions (the guard-band masks, the N != 0 branch of the conic backward, the det clamps of the opacity compensation,
the colour clamp bits) are ``color_exact.Mask`` objects in the interval back end: where an interval straddles the
threshold the decision is UNDETERMINED, both branches are kept (the hull), and the row is reported in ``und``.

Semantics kept from the reference (what S is): the ``det^2 + 1e-7`` regulariser and the branch on its fp32 reciprocal
being non-zero (decided the way fp32 decides it: ``det^2`` rounds to +inf from 2^128 - 2^103 on); ``det1^2 + 1e-6`` in
dL/ddet1; dL/dopacity zeroed when det0 or det1 is at the 1e-6 clamp, and left unscaled by coef in the N == 0 branch;
dL/dscale without a modifier factor; the raw quaternion (not normalised, note N5).  The kernel's fp32 constants are
the default; ``F64`` holds the fp64 ones (the CPU oracle's), used to pin S to ``cpu_oracle``.

The clamp bits are not an input of the ABI: the forward stores rgb = max(raw, 0), so rgb > 0 means not clamped and
rgb == 0 means clamped unless raw was exactly +0.  ``clamp_bits_from_rgb`` settles the second case with an interval of
the forward's raw colour (``color_exact.basis_iv``) and leaves a channel undetermined only where that interval
reaches 0.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from oracle.color_exact import Iv, Mask, U32, basis_iv, fsum, fp32_op

ETA = 2.0 ** -149                 # absolute error of one fp32 rounding in the subnormal range (twice the half ulp)
F32_OVF = 2.0 ** 128 - 2.0 ** 103  # exact values from here on round to +inf in fp32
INF = float("inf")


def _f32(x):
    return float(np.float32(x))


@dataclass(frozen=True)
class Consts:
    lim: float          # the guard band, 1.3 tan_fov
    k7: float           # det^2 regulariser
    k6: float           # the opacity compensation's eps and clamp
    ovf: float          # where det^2 overflows
    sh: tuple           # SH constants C0, C1, C2[5], C3[7]
    f32: bool           # scalar set-up (focal, limits) in fp32


_SH64 = (0.28209479177387814, 0.4886025119029199, 1.0925484305920792, -1.0925484305920792, 0.31539156525252005,
         -1.0925484305920792, 0.5462742152960396, -0.5900435899266435, 2.890611442640554, -0.4570457994644658,
         0.3731763325901154, -0.4570457994644658, 1.445305721320277, -0.5900435899266435)
F32 = Consts(_f32(1.3), _f32(1e-7), _f32(1e-6), F32_OVF, tuple(_f32(c) for c in _SH64), True)
F64 = Consts(1.3, 1e-7, 1e-6, INF, _SH64, False)


# ======================================================================================================================
# arithmetic back ends
# ======================================================================================================================
def _mask_not(m):
    return Mask(~m.maybe, ~m.sure)


class IvArith:
    """Intervals: centre = exact value, radius = bound on the fp32 evaluation's distance from it."""

    def __init__(self, u=U32, eta=ETA, ovf=F32_OVF, device="cpu"):
        self.u, self.eta, self.ovf, self.device = u, eta, ovf, torch.device(device)

    def v(self, x):
        x = torch.as_tensor(x, dtype=torch.float64, device=self.device)
        return Iv(x, torch.zeros_like(x))

    def _r(self, v: Iv):
        c, r = v.c, v.r
        bad = ~torch.isfinite(c) | torch.isnan(r)
        c = torch.where(bad, torch.zeros_like(c), c)
        r = torch.where(bad, torch.full_like(r, INF), r)
        if self.u == 0:
            return Iv(c, r)
        m = c.abs() + r
        r = r + self.u * m + self.eta
        return Iv(c, torch.where(m >= self.ovf, torch.full_like(r, INF), r))

    def add(self, a, b):
        return self._r(a + b)

    def sub(self, a, b):
        return self._r(a - b)

    def mul(self, a, b):
        return self._r(a * b)

    def div(self, a, b):
        c = a.c / b.c
        den = b.c.abs() - b.r
        r = (a.r + c.abs() * b.r) / den
        r = torch.where(den > 0, r, torch.full_like(r, INF))
        return self._r(Iv(c, r))

    def sqrt(self, a):
        c = a.c.clamp_min(0).sqrt()
        lo, hi = a.lo.clamp_min(0).sqrt(), a.hi.clamp_min(0).sqrt()
        r = torch.maximum(hi - c, c - lo)
        r = torch.where(a.c < 0, torch.full_like(r, INF), r)
        return self._r(Iv(c, r))

    def fma(self, a, b, c):                      # a contraction candidate: covers fused and unfused
        return self._r(self._r(a * b) + c)

    def fma_rn(self, a, b, c):                   # __fmaf_rn
        return self._r(a * b + c)

    def neg(self, a):
        return -a

    def clamp(self, x, lo, hi):                  # fminf / fmaxf against exact fp32 limits (no rounding)
        cc = x.c.clamp(lo, hi)
        r = torch.maximum((x.hi.clamp(lo, hi) - cc).abs(), (cc - x.lo.clamp(lo, hi)).abs())
        return Iv(cc, r)

    def lt(self, x, t):
        return Mask(x.hi < t, x.lo < t)

    def le(self, x, t):
        return Mask(x.hi <= t, x.lo <= t)

    def gt(self, x, t):
        return Mask(x.lo > t, x.hi > t)

    Not = staticmethod(_mask_not)

    @staticmethod
    def Or(a, b):
        return Mask(a.sure | b.sure, a.maybe | b.maybe)

    def sel(self, m, a, b):
        """a where the predicate holds, b where it does not, the hull of both where it is undetermined"""
        a, b = (x if isinstance(x, Iv) else self.v(x) for x in (a, b))
        lo, hi = torch.minimum(a.lo, b.lo), torch.maximum(a.hi, b.hi)
        hc, hr = (lo + hi) * 0.5, (hi - lo) * 0.5
        bad = torch.isnan(hc) | torch.isnan(hr)
        hc = torch.where(bad, torch.zeros_like(hc), hc)
        hr = torch.where(bad, torch.full_like(hr, INF), hr)
        shape = torch.broadcast_shapes(a.c.shape, b.c.shape, m.sure.shape)
        c = torch.where(m.sure, a.c, torch.where(m.maybe, hc, b.c)).expand(shape)
        r = torch.where(m.sure, a.r, torch.where(m.maybe, hr, b.r)).expand(shape)
        return Iv(c, r)

    @staticmethod
    def overflows(x: Iv, extra, ovf):
        """Mask: x^2 + extra rounds to +inf in fp32 (x an interval of the fp32 operand)"""
        lo2, hi2 = x.lo * x.lo, x.hi * x.hi
        sq_lo = torch.where((x.lo <= 0) & (x.hi >= 0), torch.zeros_like(lo2), torch.minimum(lo2, hi2))
        sq_hi = torch.maximum(lo2, hi2)
        return Mask(sq_lo + extra >= ovf, sq_hi + extra >= ovf)

    @staticmethod
    def und(m):
        return m.undetermined

    @staticmethod
    def stack(xs, dim=-1):
        shape = torch.broadcast_shapes(*(x.c.shape for x in xs))
        return Iv(torch.stack([x.c.expand(shape) for x in xs], dim), torch.stack([x.r.expand(shape) for x in xs], dim))


class F32Arith:
    """fp32 evaluation with torch float32 tensors; every contraction candidate fused or not at random per entry."""

    def __init__(self, gen: torch.Generator, p_fuse=0.5):
        self.gen, self.p = gen, p_fuse

    @staticmethod
    def v(x):
        return torch.as_tensor(x).float()

    def add(self, a, b):
        return a + b

    def sub(self, a, b):
        return a - b

    def mul(self, a, b):
        return a * b

    def div(self, a, b):
        return a / b

    def sqrt(self, a):
        return torch.sqrt(a)

    def fma_rn(self, a, b, c):
        return (a.double() * b.double() + c.double()).float()

    def fma(self, a, b, c):
        fused = self.fma_rn(a, b, c)
        plain = a * b + c
        pick = torch.rand(fused.shape, generator=self.gen) < self.p
        return torch.where(pick, fused, plain)

    def neg(self, a):
        return -a

    def clamp(self, x, lo, hi):
        return x.clamp(lo, hi)

    def lt(self, x, t):
        return x < t

    def le(self, x, t):
        return x <= t

    def gt(self, x, t):
        return x > t

    @staticmethod
    def Not(m):
        return ~m

    @staticmethod
    def Or(a, b):
        return a | b

    @staticmethod
    def sel(m, a, b):
        return torch.where(m, torch.as_tensor(a, dtype=torch.float32), torch.as_tensor(b, dtype=torch.float32))

    @staticmethod
    def overflows(x, extra, ovf):
        return torch.isinf(x * x + extra)

    @staticmethod
    def und(m):
        return torch.zeros_like(m)

    @staticmethod
    def stack(xs, dim=-1):
        shape = torch.broadcast_shapes(*(x.shape for x in xs))
        return torch.stack([x.expand(shape) for x in xs], dim)


# ======================================================================================================================
# the kernel's expression tree
# ======================================================================================================================
def _dot3(A, a0, b0, a1, b1, a2, b2):
    """a0*b0 + a1*b1 + a2*b2 (nvcc fuses the second and third products into the sums)"""
    return A.fma(a2, b2, A.fma(a1, b1, A.mul(a0, b0)))


def _fms(A, a, b, c, d):
    """a*b - c*d"""
    return A.fma(a, b, A.neg(A.mul(c, d)))


def _quat_to_mat(A, q):
    """R.m[col][row] as gaussian_math.cuh's quat_to_mat (explicit __fmaf_rn / __fmul_rn)"""
    r, x, y, z = q
    xz, rx, rz, yy, zz = A.mul(x, z), A.mul(r, x), A.mul(r, z), A.mul(y, y), A.mul(z, z)
    two = lambda t: A.mul(A.v(2.0), t)
    one = A.v(1.0)
    return [[A.sub(one, two(A.add(yy, zz))), two(A.fma_rn(x, y, A.neg(rz))), two(A.fma_rn(r, y, xz))],
            [two(A.fma_rn(x, y, rz)), A.sub(one, two(A.fma_rn(x, x, zz))), two(A.fma_rn(y, z, A.neg(rx)))],
            [two(A.fma_rn(A.neg(r), y, xz)), two(A.fma_rn(y, z, rx)), A.sub(one, two(A.fma_rn(x, x, yy)))]]


def _cov3d(A, sc, mod, q):
    """Sigma = (S R)^T (S R) upper triangle; (S R).m[c][r] = s_r R.m[c][r] (S diagonal: the zero products are exact)"""
    R = _quat_to_mat(A, q)
    s = [A.mul(mod, sc[i]) for i in range(3)]
    M = [[A.mul(s[r], R[c][r]) for r in range(3)] for c in range(3)]
    sig = lambda c, r: _dot3(A, M[r][0], M[c][0], M[r][1], M[c][1], M[r][2], M[c][2])
    return [sig(0, 0), sig(0, 1), sig(0, 2), sig(1, 1), sig(1, 2), sig(2, 2)]


def _sh_basis(A, K, deg, x, y, z):
    zero = A.v(0.0)
    b = [A.v(K[0])] + [zero] * 15
    if deg > 0:
        b[1], b[2], b[3] = A.mul(A.v(-K[1]), y), A.mul(A.v(K[1]), z), A.mul(A.v(-K[1]), x)
    if deg > 1:
        xx, yy, zz, xy, yz, xz = A.mul(x, x), A.mul(y, y), A.mul(z, z), A.mul(x, y), A.mul(y, z), A.mul(x, z)
        c = lambda k: A.v(K[k])
        b[4], b[5] = A.mul(c(2), xy), A.mul(c(3), yz)
        b[6] = A.mul(c(4), A.sub(A.fma(A.v(2.0), zz, A.neg(xx)), yy))
        b[7], b[8] = A.mul(c(5), xz), A.mul(c(6), A.sub(xx, yy))
        if deg > 2:
            b[9] = A.mul(A.mul(c(7), y), A.fma(A.v(3.0), xx, A.neg(yy)))
            b[10] = A.mul(A.mul(c(8), xy), z)
            b[11] = A.mul(A.mul(c(9), y), A.sub(A.fma(A.v(4.0), zz, A.neg(xx)), yy))
            b[12] = A.mul(A.mul(c(10), z), A.fma(A.v(-3.0), yy, A.fma(A.v(-3.0), xx, A.mul(A.v(2.0), zz))))
            b[13] = A.mul(A.mul(c(11), x), A.sub(A.fma(A.v(4.0), zz, A.neg(xx)), yy))
            b[14] = A.mul(A.mul(c(12), z), A.sub(xx, yy))
            b[15] = A.mul(A.mul(c(13), x), A.fma(A.v(-3.0), yy, xx))
    return b


def _sumprod(A, terms):
    """t0 + t1 + ... of products (coef, g): each product fused into the running sum or not"""
    acc = A.mul(*terms[0])
    for a, b in terms[1:]:
        acc = A.fma(a, b, acc)
    return acc


def _sh_grad_dot(A, C, deg, x, y, z, g):
    """sum_k g[k] grad b_k(x, y, z), in sh_math.cuh's grouping.  Products of literals (SHK3_0 * 6.f) are folded by the
    compiler with one fp32 rounding: that rounded constant is the kernel's exact operand."""
    zero = A.v(0.0)
    if deg == 0:
        return [zero, zero, zero]
    K = C.sh
    c = lambda k, *f: A.v(_f32(K[k] * math.prod(f)) if C.f32 else K[k] * math.prod(f))
    rx, ry, rz = A.mul(c(1, -1), g[3]), A.mul(c(1, -1), g[1]), A.mul(c(1), g[2])
    if deg > 1:
        rx = A.add(rx, _sumprod(A, [(A.mul(c(2), y), g[4]), (A.mul(c(4, -2), x), g[6]), (A.mul(c(5), z), g[7]),
                                    (A.mul(c(6, 2), x), g[8])]))
        ry = A.add(ry, _sumprod(A, [(A.mul(c(2), x), g[4]), (A.mul(c(3), z), g[5]), (A.mul(c(4, -2), y), g[6]),
                                    (A.mul(c(6, -2), y), g[8])]))
        rz = A.add(rz, _sumprod(A, [(A.mul(c(3), y), g[5]), (A.mul(c(4, 4), z), g[6]), (A.mul(c(5), x), g[7])]))
    if deg > 2:
        xx, yy, zz, xy, yz, xz = A.mul(x, x), A.mul(y, y), A.mul(z, z), A.mul(x, y), A.mul(y, z), A.mul(x, z)
        four_zz = A.mul(A.v(4.0), zz)
        rx = A.add(rx, _sumprod(A, [
            (A.mul(c(7, 6), xy), g[9]), (A.mul(c(8), yz), g[10]), (A.mul(c(9, -2), xy), g[11]),
            (A.mul(c(10, -6), xz), g[12]),
            (A.mul(c(11), A.sub(A.fma(A.v(-3.0), xx, four_zz), yy)), g[13]), (A.mul(c(12, 2), xz), g[14]),
            (A.mul(c(13, 3), A.sub(xx, yy)), g[15])]))
        ry = A.add(ry, _sumprod(A, [
            (A.mul(c(7, 3), A.sub(xx, yy)), g[9]), (A.mul(c(8), xz), g[10]),
            (A.mul(c(9), A.fma(A.v(-3.0), yy, A.sub(four_zz, xx))), g[11]), (A.mul(c(10, -6), yz), g[12]),
            (A.mul(c(11, -2), xy), g[13]), (A.mul(c(12, -2), yz), g[14]), (A.mul(c(13, -6), xy), g[15])]))
        rz = A.add(rz, _sumprod(A, [
            (A.mul(c(8), xy), g[10]), (A.mul(c(9, 8), yz), g[11]),
            (A.mul(c(10), A.fma(A.v(-3.0), yy, A.fma(A.v(-3.0), xx, A.mul(A.v(6.0), zz)))), g[12]),
            (A.mul(c(11, 8), xz), g[13]), (A.mul(c(12), A.sub(xx, yy)), g[14])]))
    return [rx, ry, rz]


MUTATIONS = ("swap_xy_masks", "cov_offdiag_no_2", "db_not_halved", "fx_for_fy", "clamp_wrong_channel",
             "opacity_without_coef", "det1_plus_eps_squared", "modifier_in_dscale", "quat_normalised",
             "no_sh_direction_term", "no_proj_w_terms")


def chain(A, x, C: Consts, mut=None):
    """The kernel's chain rule for every row of ``x`` (see ``lift``).  Returns {output: [components]} in back end A.
    ``mut`` names a corruption of the kernel (``MUTATIONS``; only meaningful with F32Arith)."""
    acc = x["acc"]
    dm2 = acc[0:3]
    gx, gy, gz = acc[3], acc[4], acc[5]
    dop = acc[6]
    dcol = acc[7:10]
    mean = x["mean"]
    view, proj = x["view"], x["proj"]
    fx, fy, limx, limy = x["fx"], x["fy"], x["limx"], x["limy"]
    if x["cov3D"] is not None:
        cov3D = x["cov3D"]
    else:
        q = x["rot"]
        if mut == "quat_normalised":
            n = A.sqrt(_dot3(A, q[0], q[0], q[1], q[1], A.fma(q[2], q[2], A.mul(q[3], q[3])), A.v(1.0)))
            q = [A.div(t, n) for t in q]
        cov3D = _cov3d(A, x["scale"], x["mod"], q)

    # ---- ewa_project ----
    t = [A.add(_dot3(A, view[r], mean[0], view[r + 4], mean[1], view[r + 8], mean[2]), view[r + 12]) for r in range(3)]
    tz = t[2]
    txtz, tytz = A.div(t[0], tz), A.div(t[1], tz)
    tx, ty = A.mul(A.clamp(txtz, -limx, limx), tz), A.mul(A.clamp(tytz, -limy, limy), tz)
    tz2 = A.mul(tz, tz)
    J00, J11 = A.div(fx, tz), A.div(fy, tz)
    J02, J12 = A.neg(A.div(A.mul(fx, tx), tz2)), A.neg(A.div(A.mul(fy, ty), tz2))
    # T.m[0][r] = view[4r] J00 + view[4r+2] J02, T.m[1][r] = view[4r+1] J11 + view[4r+2] J12 (J's zeros are exact)
    t0 = [A.fma(view[4 * r + 2], J02, A.mul(view[4 * r], J00)) for r in range(3)]
    t1 = [A.fma(view[4 * r + 2], J12, A.mul(view[4 * r + 1], J11)) for r in range(3)]
    V = [[cov3D[0], cov3D[1], cov3D[2]], [cov3D[1], cov3D[3], cov3D[4]], [cov3D[2], cov3D[4], cov3D[5]]]
    sym = lambda v: [_dot3(A, v[0], V[0][k], v[1], V[1][k], v[2], V[2][k]) for k in range(3)]
    u0, u1 = sym(t0), sym(t1)
    ca0 = _dot3(A, u0[0], t0[0], u0[1], t0[1], u0[2], t0[2])
    b = _dot3(A, u1[0], t0[0], u1[1], t0[1], u1[2], t0[2])
    cc0 = _dot3(A, u1[0], t1[0], u1[1], t1[1], u1[2], t1[2])
    a, c = A.add(ca0, x["ks"]), A.add(cc0, x["ks"])

    # ---- (1) conic -> cov2D ----
    det = _fms(A, a, c, b, b)
    nz = A.Not(A.overflows(det, C.k7, C.ovf))                 # N = 1 / (det^2 + 1e-7) != 0
    N = A.div(A.v(1.0), A.fma(det, det, A.v(C.k7)))
    r0x, r0y = _fms(A, c, gx, b, gy), _fms(A, c, gy, b, gz)
    r1x, r1y = _fms(A, a, gy, b, gx), _fms(A, a, gz, b, gy)
    da = A.mul(A.neg(N), _fms(A, r0x, c, r0y, b))
    db = A.mul(A.mul(A.v(-2.0), N), _fms(A, r0y, a, r0x, b))
    dc = A.mul(A.neg(N), _fms(A, r1y, a, r1x, b))
    # ---- (2) opacity compensation ----
    det0r, det1r = _fms(A, ca0, cc0, b, b), _fms(A, a, c, b, b)
    clampd = A.Or(A.le(det0r, C.k6), A.le(det1r, C.k6))
    det0, det1 = A.clamp(det0r, C.k6, INF), A.clamp(det1r, C.k6, INF)
    inv1 = A.div(A.v(1.0), A.add(det1, A.v(C.k6)))
    coef = A.sqrt(A.fma(det0, inv1, A.v(C.k6)))
    inv_c = A.div(A.v(1.0), A.add(coef, A.v(C.k6)))
    half = A.mul(A.mul(A.mul(A.v(0.5), dop), A.mul(x["opac"], inv_c)), inv_c)
    d0 = A.mul(half, inv1)
    if mut == "det1_plus_eps_squared":
        e1 = A.add(det1, A.v(C.k6))
        d1den = A.mul(e1, e1)
    else:
        d1den = A.fma(det1, det1, A.v(C.k6))
    d1 = A.div(A.mul(A.neg(half), det0), d1den)
    da_c = A.add(da, A.fma(d1, c, A.mul(d0, cc0)))
    db_c = A.fma(A.neg(A.mul(A.v(2.0), b)), A.add(d0, d1), db)
    dc_c = A.add(dc, A.fma(d1, a, A.mul(d0, ca0)))
    dop_c = dop if mut == "opacity_without_coef" else A.mul(dop, coef)
    zero = A.v(0.0)
    dL_da = A.sel(nz, A.sel(clampd, da, da_c), zero)
    dL_db = A.sel(nz, A.sel(clampd, db, db_c), zero)
    dL_dc = A.sel(nz, A.sel(clampd, dc, dc_c), zero)
    o_op = A.sel(nz, A.sel(clampd, zero, dop_c), dop)

    # ---- (3) cov2D -> Sigma ----
    two = A.v(2.0)
    g0 = [A.fma(dL_db, u1[k], A.mul(A.mul(two, dL_da), u0[k])) for k in range(3)]
    g1 = [A.fma(dL_db, u0[k], A.mul(A.mul(two, dL_dc), u1[k])) for k in range(3)]

    def diag(i):
        return A.fma(A.mul(dL_dc, t1[i]), t1[i], A.fma(A.mul(dL_db, t0[i]), t1[i], A.mul(A.mul(dL_da, t0[i]), t0[i])))

    def off(i, j):
        inner = A.fma(A.mul(dL_dc, t1[i]), t1[j], A.mul(A.mul(dL_da, t0[i]), t0[j]))
        cross = A.fma(t0[j], t1[i], A.mul(t0[i], t1[j]))
        f = inner if mut == "cov_offdiag_no_2" and (i, j) == (0, 1) else A.mul(two, inner)
        return A.fma(dL_db, cross, f)

    o_cov = [A.sel(nz, v, zero) for v in (diag(0), off(0, 1), off(0, 2), diag(1), off(1, 2), diag(2))]

    # ---- (4) projection rows -> view-space mean ----
    w0, w1, w2 = (view[0], view[4], view[8]), (view[1], view[5], view[9]), (view[2], view[6], view[10])
    dot = lambda w, g: _dot3(A, w[0], g[0], w[1], g[1], w[2], g[2])
    dJ00, dJ02, dJ11, dJ12 = dot(w0, g0), dot(w2, g0), dot(w1, g1), dot(w2, g1)
    iz = A.div(A.v(1.0), tz)
    iz2 = A.mul(iz, iz)
    iz3 = A.mul(iz2, iz)
    fyb = fx if mut == "fx_for_fy" else fy
    xf = A.Not(A.Or(A.lt(txtz, -limx), A.gt(txtz, limx)))
    yf = A.Not(A.Or(A.lt(tytz, -limy), A.gt(tytz, limy)))
    if mut == "swap_xy_masks":
        xf, yf = yf, xf
    gvx = A.sel(xf, A.mul(A.mul(A.neg(fx), iz2), dJ02), zero)
    gvy = A.sel(yf, A.mul(A.mul(A.neg(fyb), iz2), dJ12), zero)
    s1 = A.fma(fyb, dJ11, A.mul(fx, dJ00))
    s2 = A.fma(A.mul(fyb, ty), dJ12, A.mul(A.mul(fx, tx), dJ02))
    gvz = A.fma(A.neg(iz2), s1, A.mul(A.mul(two, iz3), s2))
    dmc = [A.fma(gvz, w2[k], A.fma(gvy, w1[k], A.mul(gvx, w0[k]))) for k in range(3)]

    # ---- (5) projective divide ----
    mh = [A.add(_dot3(A, proj[r], mean[0], proj[r + 4], mean[1], proj[r + 8], mean[2]), proj[r + 12]) for r in (0, 1, 3)]
    iw = A.div(A.v(1.0), A.add(mh[2], A.v(C.k7)))
    nx, ny = A.mul(mh[0], iw), A.mul(mh[1], iw)
    qx, qy = A.mul(dm2[0], iw), A.mul(dm2[1], iw)
    qw = A.neg(A.fma(qy, ny, A.mul(qx, nx)))
    if mut == "no_proj_w_terms":
        dmp = [A.fma(proj[4 * k + 1], qy, A.mul(proj[4 * k], qx)) for k in range(3)]
    else:
        dmp = [_dot3(A, proj[4 * k], qx, proj[4 * k + 1], qy, proj[4 * k + 3], qw) for k in range(3)]
    o_m3 = [A.add(dmc[k], dmp[k]) for k in range(3)]

    out = dict(dL_dopacity=[o_op], dL_dcov3D=o_cov)

    # ---- SH backward ----
    if x["sh"] is not None:
        deg, M = x["deg"], x["M"]
        used = (deg + 1) ** 2
        K = C.sh
        v = [A.sub(mean[k], x["campos"][k]) for k in range(3)]
        inv_len = A.div(A.v(1.0), A.sqrt(_dot3(A, v[0], v[0], v[1], v[1], v[2], v[2])))
        d = [A.mul(v[k], inv_len) for k in range(3)]
        clamp = list(x["clamp"])
        if mut == "clamp_wrong_channel":
            clamp = clamp[1:] + clamp[:1]
        g = [A.sel(clamp[ch], zero, dcol[ch]) for ch in range(3)]
        w = _sh_basis(A, K, deg, *d)
        sh = x["sh"]
        gk = [_dot3(A, g[0], sh[k][0], g[1], sh[k][1], g[2], sh[k][2]) if k < used else zero for k in range(16)]
        dsh = []
        for k in range(M):
            for ch in range(3):
                dsh.append(A.mul(w[k], g[ch]) if k < used else zero)
        out["dL_dsh"] = dsh
        gd = _sh_grad_dot(A, C, deg, d[0], d[1], d[2], gk)
        dd = _dot3(A, gd[0], d[0], gd[1], d[1], gd[2], d[2])
        gm = [A.mul(A.fma(A.neg(d[k]), dd, gd[k]), inv_len) for k in range(3)]
        if mut != "no_sh_direction_term":
            o_m3 = [A.add(o_m3[k], gm[k]) for k in range(3)]
    out["dL_dmean3D"] = o_m3

    # ---- Sigma -> scale / rotation ----
    if x["cov3D"] is None:
        q = x["rot"]
        R = _quat_to_mat(A, q)
        sv = [A.mul(x["mod"], x["scale"][i]) for i in range(3)]
        half_db = dL_db if mut == "db_not_halved" else A.mul(A.v(0.5), dL_db)
        o_sc, h = [], []
        for i in range(3):
            r = (R[0][i], R[1][i], R[2][i])
            pi = _dot3(A, t0[0], r[0], t0[1], r[1], t0[2], r[2])
            qi = _dot3(A, t1[0], r[0], t1[1], r[1], t1[2], r[2])
            al = A.fma(half_db, qi, A.mul(dL_da, pi))
            be = A.fma(dL_dc, qi, A.mul(half_db, pi))
            s = A.mul(A.mul(two, sv[i]), A.fma(be, qi, A.mul(al, pi)))
            if mut == "modifier_in_dscale":
                s = A.mul(s, x["mod"])
            o_sc.append(s)
            f = A.mul(A.mul(two, sv[i]), sv[i])
            h.append([A.mul(f, A.fma(be, t1[k], A.mul(al, t0[k]))) for k in range(3)])
        ax, ay, az = A.sub(h[1][2], h[2][1]), A.sub(h[2][0], h[0][2]), A.sub(h[0][1], h[1][0])
        sxy, sxz, syz = A.add(h[0][1], h[1][0]), A.add(h[0][2], h[2][0]), A.add(h[1][2], h[2][1])
        qr, qx_, qy_, qz_ = q
        four = A.v(4.0)
        o_rot = [A.mul(two, _dot3(A, qx_, ax, qy_, ay, qz_, az)),
                 A.fma(A.neg(A.mul(four, qx_)), A.add(h[1][1], h[2][2]), A.mul(two, _dot3(A, qr, ax, qy_, sxy, qz_, sxz))),
                 A.fma(A.neg(A.mul(four, qy_)), A.add(h[0][0], h[2][2]), A.mul(two, _dot3(A, qr, ay, qx_, sxy, qz_, syz))),
                 A.fma(A.neg(A.mul(four, qz_)), A.add(h[0][0], h[1][1]), A.mul(two, _dot3(A, qr, az, qx_, sxz, qy_, syz)))]
        out["dL_dscale"], out["dL_drot"] = o_sc, o_rot

    und = A.und(xf) | A.und(yf) | A.und(nz) | (A.und(clampd) & (nz.maybe if isinstance(nz, Mask) else nz))
    if x["sh"] is not None:
        for m in x["clamp"]:
            und = und | A.und(m)
    out["und"] = und
    if isinstance(nz, Mask):                          # rows that surely reach each edge
        out["edges"] = dict(guard_band=~xf.maybe | ~yf.maybe, n_zero=~nz.maybe, det_clamp=nz.sure & clampd.sure,
                            clamped_channel=(x["clamp"][0].sure | x["clamp"][1].sure | x["clamp"][2].sure)
                            if x["sh"] is not None else torch.zeros_like(und))
    return out


# ======================================================================================================================
# inputs, clamp bits, front ends
# ======================================================================================================================
def scalars(W, H, tan_fovx, tan_fovy, C: Consts):
    """focal_x / focal_y as the host computes them (W / (2 tan)) and the guard band 1.3 tan, in fp32 or fp64"""
    if C.f32:
        f = np.float32
        tx, ty = f(tan_fovx), f(tan_fovy)
        return (float(f(W) / (f(2) * tx)), float(f(H) / (f(2) * ty)), float(f(C.lim) * tx), float(f(C.lim) * ty))
    return W / (2.0 * tan_fovx), H / (2.0 * tan_fovy), C.lim * tan_fovx, C.lim * tan_fovy


def clamp_bits_from_rgb(rgb, shs, deg, means, campos):
    """Mask per channel: the forward clamped it (raw < 0).  rgb > 0: no; rgb == 0: yes unless the forward's raw colour
    (interval: fp32 direction, basis and fma chain) can be >= 0."""
    rgb, shs, means, campos = (torch.as_tensor(t).double() for t in (rgb, shs, means, campos))
    v = means - campos[None]
    d = v / v.norm(dim=1, keepdim=True)
    bk = basis_iv(deg, d)                                               # [P, 16]
    used = (deg + 1) ** 2
    raw = fp32_op(fsum([bk[:, k:k + 1] * Iv(shs[:, k, :]) for k in range(used)]) + 0.5)
    zero = rgb == 0
    return [Mask(zero[:, ch] & (raw.hi[:, ch] < 0), zero[:, ch]) for ch in range(3)]


def lift(A, *, acc, means3D, view, proj, W, H, tan_fovx, tan_fovy, kernel_size, scale_modifier, opac, C: Consts,
         scales=None, rotations=None, cov3D_precomp=None, shs=None, deg=0, campos=None, clamp=None):
    """The chain rule's inputs in back end A.  ``clamp``: three per-channel masks (IvArith) or bool tensors."""
    col = lambda t, k: A.v(t[:, k])
    fx, fy, limx, limy = scalars(W, H, tan_fovx, tan_fovy, C)
    f32 = (lambda s: float(np.float32(s))) if C.f32 else float
    x = dict(acc=[col(acc, k) for k in range(10)], mean=[col(means3D, k) for k in range(3)],
             view=[A.v(view[k]) for k in range(16)], proj=[A.v(proj[k]) for k in range(16)],
             fx=A.v(fx), fy=A.v(fy), limx=limx, limy=limy, ks=A.v(f32(kernel_size)), mod=A.v(f32(scale_modifier)),
             opac=A.v(opac), cov3D=None, sh=None)
    if cov3D_precomp is not None:
        x["cov3D"] = [col(cov3D_precomp, k) for k in range(6)]
    else:
        x["scale"] = [col(scales, k) for k in range(3)]
        x["rot"] = [col(rotations, k) for k in range(4)]
    if shs is not None:
        x["sh"] = [[A.v(shs[:, k, ch]) for ch in range(3)] for k in range(shs.shape[1])]
        x["deg"], x["M"] = int(deg), int(shs.shape[1])
        x["campos"] = [A.v(campos[k]) for k in range(3)]
        x["clamp"] = clamp
    return x


OUTPUTS = ("dL_dmean2D", "dL_dconic", "dL_dopacity", "dL_dcolor", "dL_dmean3D", "dL_dcov3D", "dL_dsh", "dL_dscale",
           "dL_drot")


def _active(acc, radii):
    return (radii > 0) & (acc != 0).any(1)


def bound(*, acc, radii, C: Consts = F32, u=U32, device="cpu", **kw):
    """S, B, M and und for every output.  ``acc`` [P, 10] (the kernel's fp32 rows), ``radii`` [P]; the other keywords
    are ``lift``'s.  Rows of culled Gaussians (radii 0) and all-zero rows are exactly zero (S = B = 0).
    Returns {output: {"S", "B", "M"}} plus "und" (bool [P]) and "active" (bool [P]).  M = B / u is the magnitude
    scale of the entry (the sum of |terms| along its expression tree)."""
    dev = torch.device(device)
    t = lambda v: None if v is None else torch.as_tensor(np.asarray(v) if not torch.is_tensor(v) else v).to(dev).double()
    acc64 = t(acc)
    P = acc64.shape[0]
    radii = torch.as_tensor(np.asarray(radii) if not torch.is_tensor(radii) else radii).to(dev)
    active = _active(acc64, radii)
    A = IvArith(u=u, ovf=C.ovf, device=dev)
    kw = {k: (t(v) if k in ("means3D", "view", "proj", "opac", "scales", "rotations", "cov3D_precomp", "shs",
                             "campos") else v) for k, v in kw.items()}
    if kw.get("clamp") is not None:                   # Masks, or exact bits
        kw["clamp"] = [Mask(m.sure.to(dev), m.maybe.to(dev)) if isinstance(m, Mask) else
                       Mask(torch.as_tensor(np.asarray(m, bool)).to(dev), torch.as_tensor(np.asarray(m, bool)).to(dev))
                       for m in kw["clamp"]]
    x = lift(A, acc=acc64, C=C, **kw)
    o = chain(A, x, C)
    z = torch.zeros(P, dtype=torch.float64, device=dev)
    ex = lambda k: Iv(acc64[:, k], torch.zeros_like(acc64[:, k]))
    o["dL_dmean2D"] = [ex(0), ex(1), ex(2)]
    o["dL_dconic"] = [ex(3), ex(4), Iv(z, z), ex(5)]
    o["dL_dcolor"] = [ex(7), ex(8), ex(9)]
    res = {}
    for k in OUTPUTS:
        if k not in o:
            continue
        v = IvArith.stack(o[k], 1)
        c = torch.where(active[:, None], v.c, torch.zeros_like(v.c))
        r = torch.where(active[:, None], v.r, torch.zeros_like(v.r))
        res[k] = dict(S=c, B=r, M=r / u if u > 0 else torch.zeros_like(r))
    und = o["und"] & active
    for k in res:
        und = und | (torch.isinf(res[k]["B"]).any(1) & active)
    res["und"] = und
    res["active"] = active
    res["edges"] = {k: (v & active) for k, v in o["edges"].items()}
    return res


def emulate(*, acc, radii, gen, C: Consts = F32, mut=None, **kw):
    """The kernel's fp32 arithmetic (F32Arith, random contraction), optionally corrupted by ``mut``; same outputs as
    ``bound`` (float32 tensors; culled and all-zero rows zero)."""
    A = F32Arith(gen)
    accf = torch.as_tensor(np.asarray(acc, np.float32))
    radii = torch.as_tensor(np.asarray(radii))
    active = _active(accf, radii)
    t = lambda v: None if v is None else torch.as_tensor(np.asarray(v, np.float32))
    kw = {k: (t(v) if k in ("means3D", "view", "proj", "opac", "scales", "rotations", "cov3D_precomp", "shs",
                             "campos") else v) for k, v in kw.items()}
    if kw.get("clamp") is not None:
        kw["clamp"] = [torch.as_tensor(np.asarray(m, bool)) for m in kw["clamp"]]
    x = lift(A, acc=accf, C=C, **kw)
    o = chain(A, x, C, mut=mut)
    res = {}
    for k in OUTPUTS:
        if k in o:
            v = F32Arith.stack(o[k], 1)
            res[k] = torch.where(active[:, None], v, torch.zeros_like(v))
    return res


def ratios(kernel: dict, res: dict, rows=None):
    """worst |kernel - S| / B per output over the rows (default: all determined active rows; entries with B = inf
    skipped).  An entry with B = 0 counts as inf where it differs from S."""
    out = {}
    sel = (res["active"] & ~res["und"]) if rows is None else rows
    for k, v in kernel.items():
        if k not in res:
            continue
        S, B = res[k]["S"], res[k]["B"]
        kv = torch.as_tensor(v).to(S.device).double().reshape(S.shape)
        e = (kv - S).abs()
        slack = 1e-12 * res[k]["M"] + 1e-300           # the oracle's own fp64 evaluation
        r = torch.where(e == 0, torch.zeros_like(e), e / (B + slack))
        r = torch.where(torch.isinf(B), torch.zeros_like(r), r)
        r = torch.where(torch.isnan(kv) & ~torch.isinf(B), torch.full_like(r, INF), r)
        r = r[sel]
        out[k] = float(r.max()) if r.numel() else 0.0
    return out
