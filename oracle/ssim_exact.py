"""TEST INFRASTRUCTURE -- fp64 oracle of the SSIM kernels (csrc/ssim.cu, csrc/ssim_common.cuh), the training loss
block (csrc/train_loss.cu) and the multi-scale SSIM (csrc/msssim.cu) AS THE KERNELS ROUND THEM, with an a-priori
bound on how far the kernel's value of every output entry can be from the oracle's.  Only tests/ may import this.

Each kernel's expression tree is written once, over an arithmetic back end ``A``:
  * ``IvArith`` -- midpoint-radius intervals in float64 (``color_exact.Iv``).  The centre is the exact value S of the
    kernel's formulas on its fp32 inputs; the radius B is a running-error bound on the kernel's fp32 value:
      - every fp32 operation adds u |result| + 2^-149 (u = 2^-24; the absolute term covers the subnormal range);
      - every ``a * b + c`` site that nvcc may contract (the build uses -O3 with the default -fmad=true) is two
        roundings, the product's and the sum's, which covers the fused and the unfused evaluation;
      - explicit ``fmaf`` and the ``__f*_rn`` intrinsics are one rounding each; IEEE ``/`` and ``sqrtf`` are
        correctly rounded (no fast-math), so they are one rounding each too;
      - the oracle's own fp64 evaluation error is absorbed by 2^-50 |result| per rounded stage;
      - a result whose magnitude can reach the fp32 overflow threshold gets an infinite radius;
      - ``fmaxf(v, 0)`` before ``sqrtf`` is an interval clamp, and the square root of an interval is the hull of the
        square roots of its ends.
    With u = 0 (and no absolute term) the same code is the plain fp64 evaluation of the kernels' formulas.
  * ``F32Arith`` -- an fp32 emulation in torch float32.  Each contractible site is contracted or not at random, per
    entry; ``fmaf`` is emulated exactly (the fp32 product is exact in fp64, and a TwoSum residual settles the tie of
    the double rounding fp64 -> fp32).  ``MUTATIONS`` are corruptions of this emulation.

What S is:
  * Window.  The fp32 taps are ``ssim_oracle.window_1d`` (``ssim_window`` builds the same bits, which the tests
    assert), applied separably: the 2-D weight is the real product g_i g_j, as the kernels apply it.  The reference's
    2-D window is fl(g_i g_j), which differs from it by at most u g_i g_j per tap, so every 2-D blur of a value v
    differs by at most u blur(|v|) -- the definitional window term.  ``IvArith(u=0, defn_gap=True)`` evaluates the
    formulas with that term on every blur and with C1, C2, C3 as the hulls of the kernels' fp32 constants and the
    oracles' fp64 ones, and the tests hold the unmodified float64 oracles inside it.
  * Bilinear resampling (``lerp_at`` in msssim.cu).  Indices and weights are the ones PyTorch's fp32 kernels compute:
    scale = fl(in / out), src = max(scale (dst + 0.5) - 0.5, 0), i0 = floor(src), i1 = min(i0 + 1, in - 1),
    l1 = src - i0 (exact in fp32), l0 = 1 - l1 (real; the kernel rounds it).  nvcc may contract
    ``scale * (dst + 0.5f) - 0.5f``, so both outcomes are evaluated; where they give different (i0, l1), S is the hull
    of both.  With fp64 weights (``weights64=True``) the same code is ``F.interpolate`` in float64; the gap between the
    two definitions is ``bilinear_gap``.
  * Area resize.  Windows [floor(i H / h), ceil((i + 1) H / h)), exact integers; the kernel's row-major fp32 sum, then
    two IEEE divisions by the window's height and width.
  * ``avg_pool2``.  Floor-sized 2x2 windows, ((a + b) + c) + d, then / 4.
  * SSIM backward.  S is the analytic gradient written in ssim.cu's header, evaluated exactly:
    dL/dx_p = w*(g dS/dmu_x)_p + 2 x_p w*(g dS/dE_xx)_p + y_p w*(g dS/dE_xy)_p with g = dL/dmap / 3, and the optional
    per-pixel factors s0 then s1 (``__fmul_rn``, one rounding each).
  * The loss block.  raw_scaled, dL/dmap and dL/dtoned are chains of explicitly rounded intrinsics, so they are exact
    functions of the inputs: ``loss_exact_parts`` restates them in numpy fp32 (sign(0) = 0) and the tests compare them
    bitwise.  The loss and the eight metrics are sums, in double, of the kernel's fp32 per-pixel terms (its own
    ssim_map included) followed by a few double operations and one fp32 rounding: ``loss_values`` returns the exact
    value (``math.fsum`` of the terms) and the double evaluation's error, n 2^-53 sum |t| per n-term sum plus 2^-52
    relative per double operation (1 double ulp for ``log10``).  The kernel's output must be the round-to-nearest fp32
    of the exact value; the neighbouring fp32 value is accepted only where the exact value lies within that error of a
    rounding midpoint.  0/0 (no mask pixel) is NaN and mse = 0 gives psnr = +inf, exactly as the formulas give them.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle.color_exact import Iv, U32

ETA = 2.0 ** -149                  # absolute error of one fp32 rounding in the subnormal range
SLACK = 2.0 ** -50                 # the oracle's own fp64 evaluation error, per rounded stage
F32_OVF = 2.0 ** 128 - 2.0 ** 103  # exact values from here on round to +inf in fp32
INF = float("inf")
R = 5                              # window radius
K = 2 * R + 1
C1 = float(np.float32(0.01 * 0.01))          # SSIM_C1, SSIM_C2: Python doubles rounded to fp32
C2 = float(np.float32(0.03 * 0.03))
C3 = float(np.float32(C2) / np.float32(2))

# Corruptions of the fp32 emulation (F32Arith(mut=k)); each must leave the bound on some CPU family entry.
MUTATIONS = {
    1: "window taps shifted by one",
    2: "clamp-to-edge halo instead of zero padding",
    3: "C1 and C2 swapped",
    4: "dS/dE_xx with its sign flipped",
    5: "factor 2 missing on x_p d1",
    6: "g not divided by 3",
    7: "s0 applied twice, s1 ignored",
    8: "partials channel stride HW instead of 3 HW",
    9: "interp(c s) in the combine instead of interp(c) interp(s)",
    10: "area window end taken as floor instead of ceil",
    11: "avg_pool2 over ceil-sized windows",
    12: "bilinear without the upper-edge clamp",
    13: "mse_masked divided by 3 sum(m)",
    14: "sign(0) = 1",
}


def window_taps():
    """The kernels' fp32 taps (ssim_window in ssim_common.cuh): fp32(exp(.)), divided by fp32(double sum)."""
    t = np.array([np.float32(math.exp(-float((x - R) ** 2) / (2.0 * 1.5 * 1.5))) for x in range(K)], dtype=np.float32)
    s = np.float32(sum(float(v) for v in t))
    return torch.from_numpy(t / s)


# ======================================================================================================================
# arithmetic back ends
# ======================================================================================================================
def _ivmap(f, x):
    return Iv(f(x.c), f(x.r)) if isinstance(x, Iv) else f(x)


class IvArith:
    """Intervals: centre = exact value, radius = bound on the fp32 evaluation's distance from it."""

    def __init__(self, u=U32, device="cpu", defn_gap=False):
        self.u = u
        self.eta = ETA if u else 0.0
        self.slack = SLACK if u else 0.0
        self.device = torch.device(device)
        self.mut = None
        # defn_gap: the definitional terms against the unmodified float64 oracles -- the window term u blur(|v|) on
        # every 2-D blur, and C1, C2, C3 as the hull of the kernel's fp32 constants and the oracles' fp64 ones
        self.window_gap = U32 if defn_gap else 0.0
        self.consts = None
        if defn_gap:
            both = lambda a, b: Iv(torch.tensor((a + b) / 2, dtype=torch.float64, device=self.device),
                                   torch.tensor(abs(a - b) / 2, dtype=torch.float64, device=self.device))
            self.consts = (both(C1, 0.01 ** 2), both(C2, 0.03 ** 2), both(C3, 0.03 ** 2 / 2))

    def v(self, x):
        if isinstance(x, Iv):
            return x
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
        r = r + (self.u + self.slack) * m + self.eta
        return Iv(c, torch.where(m >= F32_OVF, torch.full_like(r, INF), r))

    def add(self, a, b):
        return self._r(self.v(a) + self.v(b))

    def sub(self, a, b):
        return self._r(self.v(a) - self.v(b))

    def mul(self, a, b):
        return self._r(self.v(a) * self.v(b))

    def scale(self, a, k):                       # multiplication by an exact power of two: no rounding
        a = self.v(a)
        return Iv(a.c * k, a.r * abs(k))

    def div(self, a, b):
        a, b = self.v(a), self.v(b)
        c = a.c / b.c
        den = b.c.abs() - b.r
        r = (a.r + c.abs() * b.r) / den
        r = torch.where(den > 0, r, torch.full_like(r, INF))
        return self._r(Iv(c, r))

    def sqrt0(self, a):                          # sqrtf(fmaxf(a, 0))
        a = self.v(a)
        lo, hi = a.lo.clamp_min(0).sqrt(), a.hi.clamp_min(0).sqrt()
        c = a.c.clamp_min(0).sqrt()
        return self._r(Iv(c, torch.maximum(hi - c, c - lo)))

    def fmaf(self, a, b, c):                     # explicit fmaf: one rounding
        return self._r(self.v(a) * self.v(b) + self.v(c))

    def fma(self, a, b, c):                      # a * b + c, contractible: two roundings
        return self.add(self.mul(a, b), c)

    def fms(self, a, b, c):                      # c - a * b, contractible
        return self.sub(c, self.mul(a, b))

    def dot2(self, a, b, c, d):                  # a * b + c * d, either product may be fused
        return self.add(self.mul(a, b), self.mul(c, d))

    def where(self, m, a, b):
        a, b = self.v(a), self.v(b)
        return Iv(torch.where(m, a.c, b.c), torch.where(m, a.r, b.r))

    def hull(self, a, b):
        lo, hi = torch.minimum(a.lo, b.lo), torch.maximum(a.hi, b.hi)
        return Iv((lo + hi) * 0.5, (hi - lo) * 0.5)

    def gap(self, blurred, absval_blur):          # the definitional window term on a 2-D blur
        if not self.window_gap:
            return blurred
        return blurred.widen(self.window_gap * absval_blur)

    def absv(self, a):
        return self.v(a).mag()


def _fmaf32(a, b, c):
    """fp32 fmaf(a, b, c) exactly: a b is exact in fp64, s + e == a b + c exactly (TwoSum), and a tie of the rounding
    of s to fp32 is settled by the sign of e."""
    a, b, c = (torch.as_tensor(t, dtype=torch.float32) for t in (a, b, c))
    p = a.double() * b.double()
    cc = c.double()
    s = p + cc
    bb = s - p
    e = (p - (s - bb)) + (cc - bb)
    r = s.float()
    toward = torch.where(s > r.double(), torch.full_like(r, INF), torch.full_like(r, -INF))
    nb = torch.nextafter(r, toward)
    tie = (r.double() != s) & ((r.double() + nb.double()) * 0.5 == s) & (e != 0)
    up = torch.maximum(r, nb)
    dn = torch.minimum(r, nb)
    fixed = torch.where(e > 0, up, dn)
    return torch.where(tie, fixed, r)


class F32Arith:
    """fp32 evaluation; every contraction candidate fused or not at random per entry.  ``mut``: a MUTATIONS key."""

    def __init__(self, gen: torch.Generator | None = None, p_fuse=0.5, mut=None, device="cpu"):
        self.gen = gen if gen is not None else torch.Generator().manual_seed(0)
        self.p, self.mut, self.device = p_fuse, mut, torch.device(device)
        self.window_gap = 0.0

    def v(self, x):
        return torch.as_tensor(x, dtype=torch.float32, device=self.device)

    def add(self, a, b):
        return self.v(a) + self.v(b)

    def sub(self, a, b):
        return self.v(a) - self.v(b)

    def mul(self, a, b):
        return self.v(a) * self.v(b)

    def scale(self, a, k):
        return self.v(a) * k

    def div(self, a, b):
        return self.v(a) / self.v(b)

    def sqrt0(self, a):
        return torch.sqrt(self.v(a).clamp_min(0))

    def fmaf(self, a, b, c):
        a, b, c = self.v(a), self.v(b), self.v(c)
        shape = torch.broadcast_shapes(a.shape, b.shape, c.shape)
        return _fmaf32(a.expand(shape), b.expand(shape), c.expand(shape))

    def _pick(self, shape, n=2):
        return torch.randint(0, n, shape, generator=self.gen).to(self.device)

    def fma(self, a, b, c):
        f, p = self.fmaf(a, b, c), self.mul(a, b) + self.v(c)
        return torch.where(self._pick(f.shape) == 0, f, p)

    def fms(self, a, b, c):
        return self.fma(-self.v(a), b, c)

    def dot2(self, a, b, c, d):
        ab, cd = self.mul(a, b), self.mul(c, d)
        plain = ab + cd
        f1, f2 = self.fmaf(a, b, cd), self.fmaf(c, d, ab)
        k = self._pick(plain.shape, 3)
        return torch.where(k == 0, plain, torch.where(k == 1, f1, f2))

    def where(self, m, a, b):
        return torch.where(m, self.v(a), self.v(b))

    def hull(self, a, b):                         # the emulation takes one outcome per entry
        return torch.where(self._pick(a.shape) == 0, a, b)

    def gap(self, blurred, absval_blur):
        return blurred

    def absv(self, a):
        return self.v(a).abs()


# ======================================================================================================================
# the window and the separable blur (ssim_common.cuh)
# ======================================================================================================================
def _pad_hw(x, pad_h, pad_w, A):
    """zero padding of the last two dims (clamp-to-edge under mutation 2)"""
    def f(t):
        if A.mut == 2:
            idx_h = torch.arange(-pad_h, t.shape[-2] + pad_h, device=t.device).clamp(0, t.shape[-2] - 1)
            idx_w = torch.arange(-pad_w, t.shape[-1] + pad_w, device=t.device).clamp(0, t.shape[-1] - 1)
            return t.index_select(-2, idx_h).index_select(-1, idx_w)
        return torch.nn.functional.pad(t, (pad_w, pad_w, pad_h, pad_h))
    return _ivmap(f, x)


def blur_rows(A, x, w):
    """The horizontal fmaf chain at every column: sum_k w_k x[q + k - R], zeros outside the image."""
    W = (x.c if isinstance(x, Iv) else x).shape[-1]
    xp = _pad_hw(x, 0, R + 1, A)                  # one extra column each side for the shifted-taps mutation
    off = 2 if A.mut == 1 else 1
    m = A.v(0.0)
    for k in range(K):
        m = A.fmaf(float(w[k]), _ivmap(lambda t: t[..., off + k:off + k + W], xp), m)
    return m


def blur_cols(A, h, w):
    """The vertical fmaf chain over horizontally blurred rows (zero rows outside the image)."""
    H = (h.c if isinstance(h, Iv) else h).shape[-2]
    hp = _pad_hw(h, R, 0, A) if A.mut != 2 else _ivmap(lambda t: torch.nn.functional.pad(t, (0, 0, R, R)), h)
    m = A.v(0.0)
    for k in range(K):
        m = A.fmaf(float(w[k]), _ivmap(lambda t: t[..., k:k + H, :], hp), m)
    return m


def blur(A, x, w):
    """The separable 2-D blur of the kernels, plus the definitional window term when the back end carries one."""
    out = blur_cols(A, blur_rows(A, x, w), w)
    if A.window_gap:
        a = A.absv(x)
        w64 = w.double().to(a.device)
        k2 = (w64[:, None] * w64[None, :])[None, None]
        ab = torch.nn.functional.conv2d(a.reshape(-1, 1, *a.shape[-2:]), k2, padding=R).reshape(a.shape)
        out = A.gap(out, ab)
    return out


def moments(A, x, y, w):
    """mu_x, mu_y, E_xx, E_yy, E_xy of one channel stack: x*x, y*y, x*y are fp32 products (one rounding each)."""
    return (blur(A, x, w), blur(A, y, w), blur(A, A.mul(x, x), w), blur(A, A.mul(y, y), w), blur(A, A.mul(x, y), w))


def _consts(A):
    if getattr(A, "consts", None) is not None:
        return A.consts[:2]
    return (C2, C1) if A.mut == 3 else (C1, C2)


# ======================================================================================================================
# ssim.cu
# ======================================================================================================================
def ssim_forward(A, x, y, w=None):
    """gsr_ssim_forward on [B,3,H,W]: (map [B,H,W], factors [B,3 (dS/dmu_x, dS/dE_xx, dS/dE_xy),3 (channel),H,W])."""
    w = window_taps() if w is None else w
    c1, c2 = _consts(A)
    mx, my, exx, eyy, exy = moments(A, x, y, w)
    mxx, myy, mxy = A.mul(mx, mx), A.mul(my, my), A.mul(mx, my)
    A1 = A.add(A.scale(mxy, 2.0), c1)
    A2 = A.add(A.scale(A.fms(mx, my, exy), 2.0), c2)
    B1 = A.add(A.dot2(mx, mx, my, my), c1)
    B2 = A.add(A.add(A.fms(mx, mx, exx), A.fms(my, my, eyy)), c2)
    D = A.mul(B1, B2)
    S = A.div(A.mul(A1, A2), D)
    acc = _ivmap(lambda t: t[:, 0], S)
    for c in (1, 2):
        acc = A.add(acc, _ivmap(lambda t: t[:, c], S))
    smap = A.div(acc, 3.0)
    invD = A.div(1.0, D)
    t2 = A.mul(A.scale(mx, 2.0), S)
    f0 = A.mul(A.dot2(A.scale(my, 2.0), A.sub(A2, A1), A.scale(t2, -1.0), A.sub(B2, B1)), invD)
    f1 = A.div(S, B2)
    f1 = A.scale(f1, -1.0) if A.mut != 4 else f1
    f2 = A.mul(A.scale(A1, 2.0), invD)
    st = lambda fs: Iv(torch.stack([f.c for f in fs], 1), torch.stack([f.r for f in fs], 1)) if isinstance(fs[0], Iv) \
        else torch.stack(fs, 1)
    return smap, st([f0, f1, f2])


def _plane(P, k, c, A):
    """factor k of channel c from [B,3,3,H,W] partials: stride 3 HW per factor (HW under mutation 8)"""
    idx = k * 3 + c if A.mut != 8 else k + c
    return _ivmap(lambda t: t.reshape(t.shape[0], 9, *t.shape[-2:])[:, idx], P)


def ssim_backward(A, x, y, P, G, s0=None, s1=None, w=None):
    """ssim_bwd_kernel: dL/dimg1 [B,3,H,W] from the factors P [B,3,3,H,W] and dL/dmap G [B,H,W], scaled per pixel by
    s0 then s1 ([B,H,W] or None)."""
    w = window_taps() if w is None else w
    g = A.div(G, 3.0) if A.mut != 6 else A.v(G)
    out = []
    for c in range(3):
        d = [blur(A, A.mul(g, _plane(P, k, c, A)), w) for k in range(3)]
        xc, yc = _ivmap(lambda t: t[:, c], x), _ivmap(lambda t: t[:, c], y)
        x2 = A.scale(xc, 2.0) if A.mut != 5 else xc
        v = A.fma(yc, d[2], A.fma(x2, d[1], d[0]))
        if A.mut == 7:
            v = A.mul(A.mul(v, s0), s0) if s0 is not None else v
        else:
            if s0 is not None:
                v = A.mul(v, s0)
            if s1 is not None:
                v = A.mul(v, s1)
        out.append(v)
    if isinstance(out[0], Iv):
        return Iv(torch.stack([o.c for o in out], 1), torch.stack([o.r for o in out], 1))
    return torch.stack(out, 1)


# ======================================================================================================================
# msssim.cu
# ======================================================================================================================
def msssim_parts(A, x, y, level0, w=None):
    """msssim_parts_kernel: level 0 -> l c s [B,3,h,w]; coarse -> (c, s) [B,3,2,h,w]."""
    w = window_taps() if w is None else w
    c1, c2 = _consts(A)
    c3 = C3 if A.mut != 3 else float(np.float32(C1) / np.float32(2))
    if getattr(A, "consts", None) is not None:
        c3 = A.consts[2]
    mx, my, exx, eyy, exy = moments(A, x, y, w)
    mxx, myy, mxy = A.mul(mx, mx), A.mul(my, my), A.mul(mx, my)
    vx, vy, cxy = A.fms(mx, mx, exx), A.fms(my, my, eyy), A.fms(mx, my, exy)
    sdx, sdy = A.sqrt0(vx), A.sqrt0(vy)
    cs = A.div(A.fma(A.scale(sdx, 2.0), sdy, c2), A.add(A.add(vx, vy), c2))
    st = A.div(A.add(cxy, c3), A.fma(sdx, sdy, c3))
    if level0:
        lum = A.div(A.add(A.scale(mxy, 2.0), c1), A.add(A.dot2(mx, mx, my, my), c1))
        return A.mul(A.mul(lum, cs), st)
    if isinstance(cs, Iv):
        return Iv(torch.stack([cs.c, st.c], 2), torch.stack([cs.r, st.r], 2))
    return torch.stack([cs, st], 2)


def area_windows(n_in, n_out, mut=None):
    i = np.arange(n_out, dtype=np.int64)
    lo = i * n_in // n_out
    hi = ((i + 1) * n_in + n_out - 1) // n_out if mut != 10 else ((i + 1) * n_in) // n_out
    return lo, np.maximum(hi, lo + (0 if mut == 10 else 1))


def area_resize(A, x, h, w):
    """area_resize_kernel: [B,3,H,W] -> [B,3,h,w], row-major fp32 window sums, then / kh / kw."""
    Hin, Win = (x.c if isinstance(x, Iv) else x).shape[-2:]
    y0, y1 = area_windows(Hin, h, A.mut)
    x0, x1 = area_windows(Win, w, A.mut)
    kh, kw = y1 - y0, x1 - x0
    dev = A.device
    s = A.v(torch.zeros((1, 1, h, w), dtype=torch.float64, device=dev))
    for dy in range(int(kh.max())):
        ry = torch.from_numpy(np.minimum(y0 + dy, Hin - 1)).to(dev)
        vy = torch.from_numpy(dy < kh).to(dev)
        rows = _ivmap(lambda t: t.index_select(-2, ry), x)
        for dx in range(int(kw.max())):
            rx = torch.from_numpy(np.minimum(x0 + dx, Win - 1)).to(dev)
            valid = vy[:, None] & torch.from_numpy(dx < kw).to(dev)[None, :]
            s = A.where(valid, A.add(s, _ivmap(lambda t: t.index_select(-1, rx), rows)), s)
    khf = torch.from_numpy(np.maximum(kh, 1).astype(np.float64)).to(dev)[:, None]
    kwf = torch.from_numpy(np.maximum(kw, 1).astype(np.float64)).to(dev)[None, :]
    return A.div(A.div(s, khf), kwf)


def avg_pool2(A, x):
    """avg_pool2_kernel: floor-sized 2x2 means, ((a + b) + c) + d, then / 4 (ceil-sized under mutation 11)."""
    hi, wi = (x.c if isinstance(x, Iv) else x).shape[-2:]
    if A.mut == 11:                               # ceil-sized windows: the mean of what lies inside the image
        ho, wo = (hi + 1) // 2, (wi + 1) // 2
        xp = _ivmap(lambda t: torch.nn.functional.pad(t, (0, 2 * wo - wi, 0, 2 * ho - hi)), x)
        cnt = torch.nn.functional.pad(torch.ones(1, 1, hi, wi, device=A.device), (0, 2 * wo - wi, 0, 2 * ho - hi))
        cnt = torch.nn.functional.avg_pool2d(cnt, 2) * 4
        q = lambda dy, dx: _ivmap(lambda t: t[..., dy::2, dx::2], xp)
        return A.div(A.add(A.add(A.add(q(0, 0), q(0, 1)), q(1, 0)), q(1, 1)), cnt.float())
    ho, wo = hi // 2, wi // 2
    q = lambda dy, dx: _ivmap(lambda t: t[..., dy:2 * ho:2, dx:2 * wo:2], x)
    return A.div(A.add(A.add(A.add(q(0, 0), q(0, 1)), q(1, 0)), q(1, 1)), 4.0)


def lerp_weights(n_in, n_out, fused, weights64=False):
    """(i0, i1, l1) of lerp_at for every output index; fused: scale * (dst + 0.5f) - 0.5f as one fmaf."""
    dst = np.arange(n_out, dtype=np.float32) + np.float32(0.5)
    if weights64:
        scale = n_in / n_out
        src = np.maximum(scale * dst.astype(np.float64) - 0.5, 0.0)
    else:
        scale = np.float32(n_in) / np.float32(n_out)
        if fused:
            src = _fmaf32(torch.full((n_out,), float(scale)), torch.from_numpy(dst),
                          torch.full((n_out,), -0.5)).numpy()
        else:
            src = np.float32(scale) * dst - np.float32(0.5)
        src = np.maximum(src, np.float32(0)).astype(np.float32)
    i0 = src.astype(np.int64)
    i1 = np.minimum(i0 + 1, n_in - 1)
    l1 = src.astype(np.float64) - i0
    return i0, i1, l1


def _lerp_one(A, p, ty, tx, clamp=True):
    (iy0, iy1, ly1), (ix0, ix1, lx1) = ty, tx
    dev = A.device
    n_in_h, n_in_w = (p.c if isinstance(p, Iv) else p).shape[-2:]
    if not clamp:                                 # mutation 12: the upper neighbour read past the edge (a zero)
        p = _ivmap(lambda t: torch.nn.functional.pad(t, (0, 1, 0, 1)), p)
        iy1, ix1 = iy0 + 1, ix0 + 1
    T = lambda a: torch.from_numpy(np.asarray(a)).to(dev)
    rows = lambda iy: _ivmap(lambda t: t.index_select(-2, T(iy)), p)
    g = lambda r, ix: _ivmap(lambda t: t.index_select(-1, T(ix)), r)
    ly1t, lx1t = T(ly1)[:, None], T(lx1)[None, :]
    if isinstance(A, F32Arith):
        ly1t, lx1t = ly1t.float(), lx1t.float()
    ly0, lx0 = A.sub(1.0, ly1t), A.sub(1.0, lx1t)
    r0, r1 = rows(iy0), rows(iy1)
    a0 = A.dot2(lx0, g(r0, ix0), lx1t, g(r0, ix1))
    a1 = A.dot2(lx0, g(r1, ix0), lx1t, g(r1, ix1))
    return A.dot2(ly0, a0, ly1t, a1)


def bilinear(A, p, h_out, w_out, weights64=False):
    """lerp2 of [..., h, w] at every output index of an (h_out, w_out) grid, both contraction outcomes of lerp_at."""
    h, w = (p.c if isinstance(p, Iv) else p).shape[-2:]
    clamp = A.mut != 12
    if weights64:
        return _lerp_one(A, p, lerp_weights(h, h_out, False, True), lerp_weights(w, w_out, False, True), clamp)
    ty = [lerp_weights(h, h_out, f) for f in (False, True)]
    tx = [lerp_weights(w, w_out, f) for f in (False, True)]
    out = _lerp_one(A, p, ty[0], tx[0], clamp)
    same = all(np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2]) for a, b in (ty, tx))
    if same:
        return out
    return A.hull(out, _lerp_one(A, p, ty[1], tx[1], clamp))


def msssim_combine(A, lcs0, levels, h, w, weights64=False):
    """msssim_combine_kernel: per level-0 pixel and channel, lcs0 times bilinear(c) times bilinear(s) of every coarse
    level, then ((v0 + v1) + v2) / 3 -> [B,h,w]."""
    v = lcs0
    for cs in levels:
        c = _ivmap(lambda t: t[:, :, 0], cs)
        s = _ivmap(lambda t: t[:, :, 1], cs)
        if A.mut == 9:
            v = A.mul(v, bilinear(A, A.mul(c, s), h, w, weights64))
        else:
            v = A.mul(v, bilinear(A, c, h, w, weights64))
            v = A.mul(v, bilinear(A, s, h, w, weights64))
    ch = lambda k: _ivmap(lambda t: t[:, k], v)
    return A.div(A.add(A.add(ch(0), ch(1)), ch(2)), 3.0)


def msssim_levels(h, w, min_size):
    n = 0
    while h > min_size and w > min_size:
        h //= 2
        w //= 2
        n += 1
    return n


def msssim(A, x, y, h, w, min_size, weights64=False, stages=None):
    """gsr_msssim_forward end to end.  Returns a dict of every stage: x0, y0 (resized), lcs0, per coarse level l: px{l},
    py{l} (pooled), cs{l}, mean0 and out.  ``stages``: the kernel's own intermediates (same keys, fp32 tensors) -- each stage is then
    evaluated on the kernel's fp32 input of that stage (the op replay) instead of on the oracle's previous stage."""
    H, W = (x.c if isinstance(x, Iv) else x).shape[-2:]
    take = (lambda k, v: A.v(stages[k].double()) if isinstance(A, IvArith) else stages[k]) if stages is not None \
        else (lambda k, v: v)
    o = {}
    resize = (h, w) != (H, W)
    if resize:
        o["x0"], o["y0"] = area_resize(A, x, h, w), area_resize(A, y, h, w)
        xs, ys = take("x0", o["x0"]), take("y0", o["y0"])
    else:
        xs, ys = x, y
    o["lcs0"] = msssim_parts(A, xs, ys, True)
    levels = []
    for l in range(msssim_levels(h, w, min_size)):
        o[f"px{l}"], o[f"py{l}"] = avg_pool2(A, xs), avg_pool2(A, ys)
        xs, ys = take(f"px{l}", o[f"px{l}"]), take(f"py{l}", o[f"py{l}"])
        o[f"cs{l}"] = msssim_parts(A, xs, ys, False)
        levels.append(take(f"cs{l}", o[f"cs{l}"]))
    o["mean0"] = msssim_combine(A, take("lcs0", o["lcs0"]), levels, h, w, weights64)
    o["out"] = bilinear(A, take("mean0", o["mean0"]), H, W, weights64) if resize else o["mean0"]
    return o


def ssim_down(A, x, y, h, w, stages=None, weights64=False):
    """gsr_ssim_down_forward: area resize, the SSIM map, bilinear up.  Stages x0, y0, map, out."""
    H, W = (x.c if isinstance(x, Iv) else x).shape[-2:]
    take = (lambda k, v: A.v(stages[k].double()) if isinstance(A, IvArith) else stages[k]) if stages is not None \
        else (lambda k, v: v)
    o = {}
    if (h, w) == (H, W):
        o["out"] = ssim_forward(A, x, y)[0]
        return o
    o["x0"], o["y0"] = area_resize(A, x, h, w), area_resize(A, y, h, w)
    o["map"] = ssim_forward(A, take("x0", o["x0"]), take("y0", o["y0"]))[0]
    o["out"] = bilinear(A, take("map", o["map"]), H, W, weights64)
    return o


def pad64(n):
    return (n + 63) // 64 * 64


def msssim_layout(B, h, w, min_size):
    """msssim_layout of msssim.cu, offsets in floats: x0, y0, per coarse level px, py, cs, then lcs0, mean0, total."""
    planes = B * 3
    off = 0
    L = {}
    L["x0"] = off; off += pad64(planes * h * w)
    L["y0"] = off; off += pad64(planes * h * w)
    hl, wl = h, w
    sizes = []
    for l in range(msssim_levels(h, w, min_size)):
        hl, wl = hl // 2, wl // 2
        sizes.append((hl, wl))
        L[f"px{l}"] = off; off += pad64(planes * hl * wl)
        L[f"py{l}"] = off; off += pad64(planes * hl * wl)
        L[f"cs{l}"] = off; off += pad64(2 * planes * hl * wl)
    L["lcs0"] = off; off += pad64(planes * h * w)
    L["mean0"] = off; off += pad64(B * h * w)
    L["total"] = off
    return L, sizes


def msssim_stages(scratch, B, h, w, min_size, out):
    """The kernel's intermediates read from its scratch (float32 tensor) by msssim_layout."""
    L, sizes = msssim_layout(B, h, w, min_size)
    s = {}
    cut = lambda k, shape: scratch[L[k]:L[k] + int(np.prod(shape))].view(shape)
    s["x0"], s["y0"] = cut("x0", (B, 3, h, w)), cut("y0", (B, 3, h, w))
    for l, (hl, wl) in enumerate(sizes):
        s[f"px{l}"], s[f"py{l}"] = cut(f"px{l}", (B, 3, hl, wl)), cut(f"py{l}", (B, 3, hl, wl))
        s[f"cs{l}"] = cut(f"cs{l}", (B, 3, 2, hl, wl))
    s["lcs0"] = cut("lcs0", (B, 3, h, w))
    s["mean0"] = cut("mean0", (B, h, w))
    s["out"] = out
    return s


# ======================================================================================================================
# train_loss.cu
# ======================================================================================================================
def _sg(v, s):
    """scale_grads_value: __fadd_rn(__fmul_rn(v, s), __fmul_rn(v, __fsub_rn(1, s))), in numpy fp32"""
    one = np.float32(1)
    return (v * s) + (v * (one - s))


def loss_exact_parts(toned, raw, gt, mask, weight, grad_scale, c_l1, c_ssim, dL_dloss, mut=None):
    """The bitwise part of the loss block in numpy fp32: raw_scaled [3,H,W] (None without mask and grad_scale),
    dL_dmap [H,W], d_toned [3,H,W], and the fp32 per-pixel terms T2 (scaled toned)."""
    f = lambda t: None if t is None else np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32))
    toned, raw, gt, mask, weight, gs = f(toned), f(raw), f(gt), f(mask), f(weight), f(grad_scale)
    H, W = gt.shape[-2:]
    mask, weight, gs = (None if t is None else t.reshape(H, W) for t in (mask, weight, gs))
    HW = H * W
    t, r = toned.copy(), raw.copy()
    if mask is not None:
        t, r = _sg(t, mask), _sg(r, mask)
    if gs is not None:
        t, r = _sg(t, gs), _sg(r, gs)
    raw_scaled = r if (mask is not None or gs is not None) else None
    g, c1, c2 = np.float32(dL_dloss), np.float32(c_l1), np.float32(c_ssim)
    gl = (g * c1) / np.float32(3 * HW)
    gsm = (g * c2) / np.float32(HW)
    gL = gl * weight if weight is not None else np.full((H, W), gl, np.float32)
    dmap = -(gsm * weight) if weight is not None else np.full((H, W), -gsm, np.float32)
    d = t - gt
    zero_sign = np.float32(1) if mut == 14 else np.float32(0)
    sgn = np.where(d > 0, np.float32(1), np.where(d < 0, np.float32(-1), zero_sign)).astype(np.float32)
    v = gL[None] * sgn
    if gs is not None:
        v = v * gs
    if mask is not None:
        v = v * mask
    return dict(raw_scaled=raw_scaled, dL_dmap=dmap, d_toned=v.astype(np.float32), T2=t, gt=gt, mask=mask,
                weight=weight)


METRICS = ("l1_loss", "ssim", "mse", "psnr", "mask_percentage", "ssim_masked", "mse_masked", "l1_loss_masked")


def _xsum(a):
    """(math.fsum of the terms, sum |t|, n)"""
    a = np.asarray(a, dtype=np.float64).ravel()
    return math.fsum(a.tolist()), float(np.abs(a).sum()), a.size


def loss_values(parts, ssim_map, c_l1, c_ssim, mut=None):
    """Exact values and double-evaluation errors of the loss and the eight metrics: {name: (S, E)} with the kernel's
    fp32 per-pixel terms (ssim_map: the kernel's map [H,W]).  S is NaN / +inf where the formulas give those."""
    T2, gt, m, w = parts["T2"], parts["gt"], parts["mask"], parts["weight"]
    S = np.asarray(ssim_map, dtype=np.float32)
    H, W = gt.shape[-2:]
    n1, n3 = float(H * W), float(3 * H * W)
    d = T2 - gt
    l1 = np.abs(d)
    e = d * d
    one = np.float32(1)
    sums = {"l1w": _xsum(l1 * w[None] if w is not None else l1), "l1": _xsum(l1), "e": _xsum(e),
            "sw": _xsum((one - S) * w if w is not None else one - S), "s": _xsum(S)}
    if m is not None:
        sums.update(l1m=_xsum(l1 * m[None]), em=_xsum(e * m[None]), m=_xsum(m), sm=_xsum(S * m))
    u = 2.0 ** -53

    def err(k):                                       # accumulation error of the kernel's double sum and fsum's own
        s, a, n = sums[k]
        return n * u * a + u * abs(s)

    def ratio(kn, d_, kd=None):                        # (S, E) of sum_n / d_ (d_ a count) or sum_n / sum_d
        sn, en = sums[kn][0], err(kn)
        if kd is None:
            v = sn / d_
            return v, (en / d_) + 4 * u * abs(v)
        sd, ed = sums[kd][0], err(kd)
        if sd == 0:
            return (math.nan if sn == 0 else math.copysign(INF, sn)), 0.0
        v = sn / sd
        return v, (en + abs(v) * ed) / max(abs(sd) - ed, 1e-300) + 4 * u * abs(v)

    out = {}
    l1w, El1w = ratio("l1w", n3)
    sw, Esw = ratio("sw", n1)
    a, b = float(np.float32(c_l1)) * l1w, float(np.float32(c_ssim)) * sw
    out["loss"] = (a + b, abs(float(np.float32(c_l1))) * El1w + abs(float(np.float32(c_ssim))) * Esw
                   + 4 * u * (abs(a) + abs(b)))
    out["l1_loss"] = ratio("l1", n3)
    out["ssim"] = ratio("s", n1)
    mse, Emse = ratio("e", n3)
    out["mse"] = (mse, Emse)
    if mse == 0:
        out["psnr"] = (INF, 0.0)
    else:
        p = -10.0 * math.log10(mse)
        out["psnr"] = (p, 10.0 * Emse / (mse * math.log(10)) + 8 * u * abs(p) + 1e-300)
    if m is not None:
        out["mask_percentage"] = ratio("m", n1)
        out["ssim_masked"] = ratio("sm", None, "m")
        out["mse_masked"] = ratio("em", None, "m")
        out["l1_loss_masked"] = ratio("l1m", None, "m")
        if mut == 13:
            v, E = out["mse_masked"]
            out["mse_masked"] = (v / 3.0, E / 3.0)
    else:
        for k in METRICS[4:]:
            out[k] = (0.0, 0.0)
    return out


def accepted_f32(S, E):
    """The fp32 values a kernel may return for exact value S with double-evaluation error E: rn32(S), and its
    neighbour where S lies within E of a rounding midpoint (NaN and inf: only themselves)."""
    if math.isnan(S) or math.isinf(S):
        return {np.float32(S)}
    E = 2 * E + 1e-300
    return {np.float32(S - E), np.float32(S), np.float32(S + E)}


def emulate_loss_values(parts, ssim_map, c_l1, c_ssim, mut=None):
    """The kernel's loss and metrics, emulated: the fp32 terms summed in float64 in torch's order, the kernel's double
    statements, one fp32 rounding."""
    T2, gt, m, w = parts["T2"], parts["gt"], parts["mask"], parts["weight"]
    S = np.asarray(ssim_map, dtype=np.float32)
    H, W = gt.shape[-2:]
    n1, n3 = float(H * W), float(3 * H * W)
    s = lambda t: float(torch.from_numpy(np.asarray(t, dtype=np.float64)).sum())
    d = T2 - gt
    l1, e = np.abs(d), d * d
    one = np.float32(1)
    t0 = s(l1 * w[None] if w is not None else l1)
    ts = s((one - S) * w if w is not None else one - S)
    mse = s(e) / n3
    o = {"loss": np.float32(float(np.float32(c_l1)) * (t0 / n3) + float(np.float32(c_ssim)) * (ts / n1)),
         "l1_loss": np.float32(s(l1) / n3), "ssim": np.float32(s(S) / n1), "mse": np.float32(mse)}
    with np.errstate(divide="ignore", invalid="ignore"):
        o["psnr"] = np.float32(-10.0 * np.log10(mse))
        if m is not None:
            sm = s(m)
            div = lambda a: np.float32(np.float64(a) / np.float64(sm))
            o["mask_percentage"] = np.float32(sm / n1)
            o["ssim_masked"] = div(s(S * m))
            o["mse_masked"] = div(s(e * m[None]) / (3.0 if mut == 13 else 1.0))
            o["l1_loss_masked"] = div(s(l1 * m[None]))
        else:
            for k in METRICS[4:]:
                o[k] = np.float32(0)
    return o


def window_gap_oracles():
    """The exact separable window as the 2-D window of ``ssim_oracle`` (float64 outer product of the fp32 taps)."""
    g = window_taps().double()
    return g[:, None] * g[None, :]


def bilinear_gap(h_in, w_in, maxabs):
    """Bound on |bilinear with fp32 weights - bilinear with fp64 weights| of an input with max |p| = maxabs: the fp32
    source coordinate is within 4 u (n_in + 1) of the fp64 one on either axis (fl(in / out), the product, the
    subtraction), the interpolant is continuous with slope at most 2 maxabs per unit of either coordinate, and the
    interval evaluation's centre leaves l0 = 1 - l1 unrounded."""
    return 2 * maxabs * 4 * U32 * ((h_in + 1) + (w_in + 1))
