"""The SSIM kernels (csrc/ssim.cu, csrc/ssim_common.cuh), the training loss block (csrc/train_loss.cu) and the
multi-scale SSIM (csrc/msssim.cu) under the fp64 oracle of ``oracle/ssim_exact.py``: every output entry within its
a-priori bound, |kernel - S| <= B, at the tile edges, image borders and on adversarial content; raw_scaled, dL/dmap
and dL/dtoned bitwise; the loss and the eight metrics the round-to-nearest fp32 of their exact values.

CPU: S against the float64 oracles (``ssim_oracle``, ``train_loss_oracle``, ``msssim_oracle``) under the same
definitions and within the definitional terms of the unmodified ones, an fp32 emulation of each kernel within B, and
every corruption in ``MUTATIONS`` outside it.  GPU: the kernels themselves, end to end from the images and as an op
replay on each stage's own fp32 input.  ``-s`` prints the worst |kernel - S| / B per op and family.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import msssim_oracle, ssim_oracle
from oracle import ssim_exact as sx
from oracle import train_loss_oracle as tlo

WORST: dict = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if WORST:
        print("\nworst |kernel - S| / B per op and family:")
        for k in sorted(WORST):
            print(f"  {k[0]:<16} {k[1]:<30} {WORST[k]:.3f}")


def ratio(got, S, B):
    """max |got - S| / B; an entry with B = 0 must equal S exactly (else inf); NaN in got is inf."""
    d = (got.to(S.device).double() - S).abs()
    r = torch.where(B > 0, d / B, torch.where(d > 0, torch.full_like(d, math.inf), torch.zeros_like(d)))
    r = torch.where(torch.isnan(d), torch.full_like(d, math.inf), r)
    return float(r.max()) if r.numel() else 0.0


def check(op, family, got, S, B=None, what=""):
    if B is None:
        S, B = S.c, S.r
    assert got.shape == S.shape == B.shape, (op, family, what, got.shape, S.shape)
    assert bool(torch.isfinite(B).all()), (op, family, what)
    r = ratio(got, S, B)
    WORST[op, family] = max(WORST.get((op, family), 0.0), r)
    assert r <= 1.0, (op, family, what, r)
    return r


# ------------------------------------------------------------------------------------------------------- content

def content(kind, shape, seed, dev="cpu"):
    """(x, y) of one content family, [B,3,H,W] fp32."""
    g = torch.Generator(device=dev).manual_seed(seed)
    r = lambda: torch.rand(shape, generator=g, device=dev)
    B, C, H, W = shape
    if kind == "uniform":
        return r(), r()
    if kind == "training":
        lo = torch.rand(B, C, H // 6 + 2, W // 6 + 2, generator=g, device=dev)
        sm = torch.nn.functional.interpolate(lo, size=(H, W), mode="bilinear", align_corners=False)
        return (sm + 0.05 * torch.randn(shape, generator=g, device=dev)).clamp(0, 1), sm
    if kind == "flat0":
        return 1e-3 * r(), 1e-3 * r()
    if kind == "flat1":
        return 1 - 1e-3 * r(), 1 - 1e-3 * r()
    if kind == "equal":
        x = r()
        return x, x.clone()
    if kind == "inverse":
        y = r()
        return 1 - y, y
    if kind == "checker":
        i = torch.arange(H, device=dev)[:, None] + torch.arange(W, device=dev)[None, :]
        c = (i % 2).float().expand(shape).contiguous()
        return c, 1 - c if seed % 2 else r()
    if kind == "render":
        return -0.5 + 2.5 * r(), -0.5 + 2.5 * r()
    if kind == "structured":                       # contrast ratio and correlation both varying along x
        t = torch.linspace(0, 1, W, device=dev)
        rho = torch.cos(6 * t)
        n1, n2 = r() - 0.5, r() - 0.5
        return 0.5 + (0.1 + 0.8 * t) * n1, 0.5 + (0.9 - 0.8 * t) * (rho * n1 + (1 - rho * rho).sqrt() * n2)
    if kind == "spike":
        x, y = 0.2 * r(), 0.2 * r()
        for (py, px) in [(0, 0), (H - 1, W - 1), (15, 31), (16, 32), (H - 1, 0), (0, W - 1)]:
            if py < H and px < W:
                x[..., py, px] = 1.0
        return x, y
    raise ValueError(kind)


CONTENT = ("uniform", "training", "flat0", "flat1", "equal", "inverse", "checker", "render", "spike", "structured")


def dmap(kind, shape, seed, dev="cpu"):
    """dL/dmap [B,H,W] of one family"""
    g = torch.Generator(device=dev).manual_seed(seed + 1000)
    if kind == "random":
        return torch.randn(shape, generator=g, device=dev)
    if kind == "ones":
        return torch.ones(shape, device=dev)
    if kind == "zeros":
        return torch.zeros(shape, device=dev)
    if kind == "magnitudes":                        # 2^e with e uniform in [-20, 20], random signs
        e = torch.randint(-20, 21, shape, generator=g, device=dev).float()
        s = torch.randint(0, 2, shape, generator=g, device=dev).float() * 2 - 1
        return s * torch.exp2(e)
    raise ValueError(kind)


# ---------------------------------------------------------------------------------------------------------------- CPU

@pytest.fixture()
def same_definitions(monkeypatch):
    """The float64 oracles under the kernels' definitions: the separable window (real products of the fp32 taps) and
    the fp32 constants."""
    w2 = sx.window_gap_oracles()
    for m in (ssim_oracle, msssim_oracle):
        monkeypatch.setattr(m, "window_2d", lambda *a, **k: w2)
        monkeypatch.setattr(m, "C1", sx.C1)
        monkeypatch.setattr(m, "C2", sx.C2)
    monkeypatch.setattr(msssim_oracle, "C3", sx.C3)


def test_window_taps_are_the_reference_bits():
    assert torch.equal(sx.window_taps().view(torch.int32), ssim_oracle.window_1d().view(torch.int32))


def _ssim_u0(x, y, G, A=None, s0=None, s1=None):
    A = A or sx.IvArith(u=0)
    smap, P = sx.ssim_forward(A, x, y)
    return smap, P, sx.ssim_backward(A, x, y, P, A.v(G.double()), s0, s1)


def test_exact_value_is_the_float64_ssim_oracle(same_definitions):
    g = torch.Generator().manual_seed(0)
    for shape in [(2, 3, 13, 17), (1, 3, 1, 1), (1, 3, 4, 40)]:
        x, y = torch.rand(shape, generator=g), torch.rand(shape, generator=g)
        G = torch.randn(shape[0], *shape[2:], generator=g)
        smap, P, dx = _ssim_u0(x, y, G)
        rm, _, rg = ssim_oracle.ssim_and_grad(x, y, G)
        assert float(smap.r.max()) == 0 and float((smap.c - rm).abs().max()) <= 1e-12, shape
        assert float((dx.c - rg).abs().max()) <= 1e-12 * max(1.0, float(rg.abs().max())), shape


def test_gap_to_the_unmodified_ssim_oracle_is_the_definitional_term():
    """fl(g_i g_j) against g_i g_j and fp64 against fp32 constants: the unmodified oracle lies within the
    definitional terms (u blur(|v|) per blur, the constants' hulls), evaluated without rounding."""
    g = torch.Generator().manual_seed(1)
    for kind in ("uniform", "flat0", "render"):
        x, y = content(kind, (1, 3, 12, 19), 1)
        G = torch.randn(1, 12, 19, generator=g)
        smap, P, dx = _ssim_u0(x, y, G, sx.IvArith(u=0, defn_gap=True))
        rm, _, rg = ssim_oracle.ssim_and_grad(x, y, G)
        check("ssim.map", "definitional gap", rm, smap)
        check("ssim.dimg", "definitional gap", rg, dx.widen(1e-12 * dx.mag()))


def test_exact_value_is_the_float64_train_loss_oracle(same_definitions):
    for branch, (mk, wk, sg) in BRANCHES.items():
        toned, raw, gt, mask, weight, gscale = loss_case("cpu", 11, 14, branch, 5)
        lam = 0.2
        want_loss, want_met, want_dT, want_dR = tlo.loss_and_grads(toned, raw, gt, lam, mask, weight, gscale)
        A = sx.IvArith(u=0)
        m = lambda t: None if t is None else t.double()
        T2, R2 = toned.double(), raw.double()
        for s in (m(mask), m(gscale)):                 # sg(v, s) = v s + v (1 - s) = v
            if s is not None:
                T2, R2 = T2 * s + T2 * (1 - s), R2 * s + R2 * (1 - s)
        smap, P = sx.ssim_forward(A, R2[None], gt[None].double())
        w = 1.0 if weight is None else weight[0].double()
        L1 = (T2 - gt.double()).abs()
        loss = (1 - lam) * (L1 * w).mean() + lam * ((1 - smap.c[0]) * w).mean()
        assert abs(float(loss) - float(want_loss)) <= 1e-12, branch
        dm = -lam / smap.c[0].numel() * (w if weight is not None else torch.ones_like(smap.c[0]))
        dR = sx.ssim_backward(A, R2[None], gt[None].double(), P, A.v(dm[None]), m(gscale), m(mask))
        assert float((dR.c[0] - want_dR).abs().max()) <= 1e-12 * float(want_dR.abs().max()), branch
        sgn = torch.sign(T2 - gt.double())
        dT = (1 - lam) / (3 * L1[0].numel()) * w * sgn
        for s in (m(gscale), m(mask)):
            if s is not None:
                dT = dT * s
        assert float((dT - want_dT).abs().max()) <= 1e-12 * float(want_dT.abs().max()), branch


MS_CPU = [  # (B, H, W, h, w, min_size): resize with non-integer ratios, odd levels, an upsample from h = 1
    (2, 23, 37, 15, 26, 5),
    (1, 17, 20, 17, 20, 3),
    (1, 9, 30, 1, 7, 1),
    (1, 6, 5, 13, 11, 4),
]


def test_exact_value_is_the_float64_msssim_oracle(same_definitions):
    g = torch.Generator().manual_seed(2)
    for B, H, W, h, w, mn in MS_CPU:
        x, y = torch.rand(B, 3, H, W, generator=g), torch.rand(B, 3, H, W, generator=g)
        A = sx.IvArith(u=0)
        o = sx.msssim(A, x, y, h, w, mn, weights64=True)
        want = _msssim_at(x, y, h, w, mn)
        assert float((o["out"].c - want).abs().max()) <= 1e-12, (H, W, h, w)
        sd = sx.ssim_down(A, x, y, h, w, weights64=True)
        want = _ssim_down_at(x, y, h, w)
        assert float((sd["out"].c - want).abs().max()) <= 1e-12, (H, W, h, w)


def _msssim_at(x, y, h, w, min_size, dtype=torch.float64):
    """msssim_oracle.msssim with the area-resize size given directly (the oracle derives it from max_size)."""
    H, W = x.shape[-2:]
    orig = msssim_oracle.resized_size
    msssim_oracle.resized_size = lambda *a, **k: (h, w)
    try:
        return msssim_oracle.msssim(x, y, max_size=0 if (h, w) != (H, W) else None, min_size=min_size, dtype=dtype)
    finally:
        msssim_oracle.resized_size = orig


def _ssim_down_at(x, y, h, w, dtype=torch.float64):
    H, W = x.shape[-2:]
    orig = msssim_oracle.resized_size
    msssim_oracle.resized_size = lambda *a, **k: (h, w)
    try:
        return msssim_oracle.ssim_down(x, y, max_size=0 if (h, w) != (H, W) else None, dtype=dtype)
    finally:
        msssim_oracle.resized_size = orig


def test_gap_to_the_unmodified_msssim_oracle_is_the_definitional_term():
    """The unmodified oracle (fp32-rounded 2-D window, fp64 constants, fp64 resampling weights) within the window and
    constant terms plus ``bilinear_gap`` per resampling."""
    g = torch.Generator().manual_seed(3)
    for B, H, W, h, w, mn in MS_CPU:
        x, y = torch.rand(B, 3, H, W, generator=g), torch.rand(B, 3, H, W, generator=g)
        A = sx.IvArith(u=0, defn_gap=True)
        o = sx.msssim(A, x, y, h, w, mn, weights64=True)
        want = _msssim_at(x, y, h, w, mn)
        check("msssim.out", "definitional gap", want, o["out"].widen(1e-12))
        o32 = sx.msssim(sx.IvArith(u=0), x, y, h, w, mn)
        o64 = sx.msssim(sx.IvArith(u=0), x, y, h, w, mn, weights64=True)
        n_lv = sx.msssim_levels(h, w, mn)
        maxabs = 4.0 ** (n_lv + 1)                     # |l c s| <= 4 per factor, so every resampled map is bounded
        gap = (n_lv * 2 + 1) * sx.bilinear_gap(max(H, h), max(W, w), maxabs) * maxabs
        assert float((o32["out"].c - o64["out"].c).abs().max()) <= gap, (H, W, h, w)


# ---- CPU families: the emulation inside B, every mutation outside it --------------------------------------------------

def loss_case(dev, H, W, branch, seed, mask_kind=None):
    g = torch.Generator(device=dev).manual_seed(seed)
    gt = torch.rand(3, H, W, generator=g, device=dev)
    toned = (gt + 0.08 * torch.randn(3, H, W, generator=g, device=dev)).clamp(0, 1)
    raw = (0.9 * gt + 0.05 + 0.05 * torch.randn(3, H, W, generator=g, device=dev)).clamp(0, 1)
    toned[:, : max(1, H // 5), : max(1, W // 5)] = gt[:, : max(1, H // 5), : max(1, W // 5)]     # sign(0) = 0
    u = torch.rand(1, H, W, generator=g, device=dev)
    binary = (u > 0.3).float()
    mk, wk, sg = BRANCHES[branch]
    mask = None if mk is None else (binary if mk == "binary" else torch.round(u * 255) / 255)
    if mask is not None and mask_kind == "zeros":
        mask = torch.zeros_like(mask)
    if mask is not None and mask_kind == "ones":
        mask = torch.ones_like(mask)
    w = {None: None, "binary": binary, "ramped": 1 + 0.37 * (binary - 1),
         "centred": binary.sub(binary.mean() - 1).clamp(0, 2)}[wk]
    return toned, raw, gt, mask, (None if sg else w), (w if sg else None)


BRANCHES = {   # (mask, weight, scale_grad), as in tests/test_fused_train.py
    "plain": (None, None, False),
    "mask": ("binary", None, False),
    "fractional_mask": ("fractional", None, False),
    "w_binary": (None, "binary", False),
    "w_ramped": (None, "ramped", False),
    "w_centred": (None, "centred", False),
    "scale_grad_ramped": (None, "ramped", True),
    "mask_scale_grad_centred": ("binary", "centred", True),
    "fractional_mask_w_ramped": ("fractional", "ramped", False),
}


def _cpu_ssim_families():
    fams = []
    for i, (kind, shape) in enumerate([("uniform", (2, 3, 13, 17)), ("training", (1, 3, 20, 35)),
                                       ("flat1", (1, 3, 7, 9)), ("inverse", (1, 3, 5, 12)), ("render", (3, 3, 6, 4))]):
        x, y = content(kind, shape, i)
        G = dmap(("random", "magnitudes", "ones", "random", "random")[i], (shape[0], *shape[2:]), i)
        g = torch.Generator().manual_seed(50 + i)
        s0 = torch.rand(shape[0], *shape[2:], generator=g) if i % 2 == 0 else None
        s1 = torch.rand(shape[0], *shape[2:], generator=g) if i in (0, 3) else None
        fams.append((f"{kind} {shape}", x, y, G, s0, s1))
    return fams


def _ssim_ops(A, x, y, G, s0, s1):
    smap, P = sx.ssim_forward(A, x, y)
    v = (lambda t: A.v(t.double())) if isinstance(A, sx.IvArith) else (lambda t: t)
    return {"ssim.map": smap, "ssim.factors": P,
            "ssim.dimg": sx.ssim_backward(A, x, y, P, v(G), None if s0 is None else v(s0), None if s1 is None else v(s1))}


def _ms_ops(A, x, y, h, w, mn):
    o = sx.msssim(A, x, y, h, w, mn)
    d = sx.ssim_down(A, x, y, h, w)
    return {"msssim." + k: v for k, v in o.items()} | {"ssim_down." + k: v for k, v in d.items()}


def _cpu_loss_family(A, branch, mut=None, H=12, W=15, mask_kind=None, lam=0.2, dL=0.37):
    toned, raw, gt, mask, weight, gscale = loss_case("cpu", H, W, branch, 7, mask_kind)
    c_l1, c_ssim = float(np.float32(1 - lam)), float(np.float32(lam))
    parts = sx.loss_exact_parts(toned, raw, gt, mask, weight, gscale, c_l1, c_ssim, dL, mut)
    r_in = torch.from_numpy(parts["raw_scaled"] if parts["raw_scaled"] is not None else raw.numpy())[None]
    ops = _ssim_ops(A, r_in, gt[None], torch.from_numpy(parts["dL_dmap"])[None], gscale, mask)
    return parts, ops, c_l1, c_ssim


@pytest.fixture(scope="module")
def cpu_bounds():
    A = sx.IvArith()
    ssim = [(name, _ssim_ops(A, x, y, G, s0, s1)) for name, x, y, G, s0, s1 in _cpu_ssim_families()]
    ms = []
    for i, (B, H, W, h, w, mn) in enumerate(MS_CPU):
        x, y = content(("uniform", "structured", "inverse", "training")[i], (B, 3, H, W), 9 + i)
        ms.append((f"{B}x{H}x{W}->{h}x{w} min {mn}", x, y, h, w, mn, _ms_ops(A, x, y, h, w, mn)))
    return ssim, ms


def _emulate_all(mut, seed, cpu_bounds):
    """{(op, family): (emulated, S, B)} over every CPU family"""
    ssim, ms = cpu_bounds
    out = {}
    E = sx.F32Arith(torch.Generator().manual_seed(seed), mut=mut)
    for (name, x, y, G, s0, s1), (_, b) in zip(_cpu_ssim_families(), ssim):
        for k, v in _ssim_ops(E, x, y, G, s0, s1).items():
            out[k, name] = (v, b[k])
    for name, x, y, h, w, mn, b in ms:
        try:
            got = _ms_ops(E, x, y, h, w, mn)
        except (RuntimeError, IndexError):          # a mutation that changes a stage's shape
            continue
        for k, v in got.items():
            if v.shape == b[k].c.shape:
                out[k, name] = (v, b[k])
    return out


@pytest.mark.parametrize("seed", [0, 1])
def test_emulation_within_the_bound(seed, cpu_bounds):
    for (op, fam), (got, iv) in _emulate_all(None, seed, cpu_bounds).items():
        check(op, "cpu emulation " + fam, got, iv)


def _loss_outputs_ok(parts_ref, parts, S_map, c_l1, c_ssim, mut):
    """bitwise parts equal and every loss value accepted"""
    for k in ("raw_scaled", "dL_dmap", "d_toned"):
        if parts_ref[k] is not None and not np.array_equal(parts_ref[k].view(np.uint32), parts[k].view(np.uint32)):
            return False
    want = sx.loss_values(parts_ref, S_map, c_l1, c_ssim)
    got = sx.emulate_loss_values(parts, S_map, c_l1, c_ssim, mut)
    return all(_accepted(got[k], *want[k]) for k in want)


def _accepted(v, S, E):
    v = np.float32(v)
    if np.isnan(v) or math.isnan(S):
        return bool(np.isnan(v)) and math.isnan(S)
    return v in sx.accepted_f32(S, E)


@pytest.mark.parametrize("branch", list(BRANCHES))
def test_loss_emulation_within_the_bound(branch):
    for mask_kind, lam, dL in ((None, 0.2, 1.0), ("zeros", 1.0, 2.0 ** -12), ("ones", 0.0, 0.37)):
        parts, ops, c_l1, c_ssim = _cpu_loss_family(sx.F32Arith(), branch, None, mask_kind=mask_kind, lam=lam, dL=dL)
        _, bnd, _, _ = _cpu_loss_family(sx.IvArith(), branch, None, mask_kind=mask_kind, lam=lam, dL=dL)
        for k in ops:
            check(k, "cpu loss " + branch, ops[k], bnd[k])
        assert _loss_outputs_ok(parts, parts, ops["ssim.map"][0].numpy(), c_l1, c_ssim, None), branch


@pytest.mark.parametrize("mut", sorted(sx.MUTATIONS))
def test_mutation_leaves_the_bound(mut, cpu_bounds):
    """Each corruption is at least 10x outside B on some entry of the CPU families (or, for the bitwise and rounded
    loss outputs, gives a value the exact model does not accept)."""
    if mut in (13, 14):
        for branch in ("mask", "mask_scale_grad_centred", "fractional_mask"):
            ref, ops, c_l1, c_ssim = _cpu_loss_family(sx.F32Arith(), branch)
            parts, _, _, _ = _cpu_loss_family(sx.F32Arith(), branch, mut)
            if not _loss_outputs_ok(ref, parts, ops["ssim.map"][0].numpy(), c_l1, c_ssim, mut):
                return
        pytest.fail(f"mutation {mut} ({sx.MUTATIONS[mut]}) was not detected")
    worst = 0.0
    for (op, fam), (got, iv) in _emulate_all(mut, 0, cpu_bounds).items():
        worst = max(worst, ratio(got, iv.c, iv.r))
    assert worst >= 10.0, (mut, sx.MUTATIONS[mut], worst)


# ---------------------------------------------------------------------------------------------------------------- GPU

def _lib():
    from diff_gaussian_rasterization import _C
    return _C


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nan(*shape, dev="cuda"):
    return torch.full(shape, math.nan, device=dev)


def kernel_ssim(x, y, G):
    """gsr_ssim_forward with partials, then gsr_ssim_backward (the plain backward; the scaled one runs through
    gsr_train_loss_backward in the loss tests)."""
    C = _lib()
    B, _, H, W = x.shape
    smap, P, dx = _nan(B, H, W), _nan(B, 3, 3, H, W), _nan(B, 3, H, W)
    C._check(C._lib.gsr_ssim_forward(B, H, W, x.data_ptr(), y.data_ptr(), smap.data_ptr(), P.data_ptr(), _stream()),
             "gsr_ssim_forward")
    C._check(C._lib.gsr_ssim_backward(B, H, W, x.data_ptr(), y.data_ptr(), P.data_ptr(), G.data_ptr(), dx.data_ptr(),
                                      _stream()), "gsr_ssim_backward")
    torch.cuda.synchronize()
    return smap, P, dx


def _check_ssim_gpu(family, x, y, G):
    dev = x.device
    smap, P, dx = kernel_ssim(x, y, G)
    A = sx.IvArith(device=dev)
    s_map, s_P = sx.ssim_forward(A, x, y)
    check("ssim.map", family, smap, s_map)
    check("ssim.factors", family, P, s_P)
    check("ssim.dimg", family + " end to end", dx, sx.ssim_backward(A, x, y, s_P, A.v(G.double())))
    check("ssim.dimg", family, dx, sx.ssim_backward(A, x, y, A.v(P.double()), A.v(G.double())))
    return dx


SSIM_H = (1, 5, 10, 11, 15, 16, 17, 31, 32, 33, 47, 48, 49)
SSIM_W = (1, 5, 11, 31, 32, 33, 63, 64, 65)


@pytest.mark.gpu
@pytest.mark.parametrize("H", SSIM_H)
def test_ssim_shapes_and_contents(H):
    dev = torch.device("cuda:0")
    for j, W in enumerate(SSIM_W):
        i = SSIM_H.index(H) * len(SSIM_W) + j
        B = 1 + i % 3
        kind = CONTENT[i % len(CONTENT)]
        gk = ("random", "ones", "zeros", "magnitudes")[i % 4]
        x, y = content(kind, (B, 3, H, W), i, dev)
        G = dmap(gk, (B, H, W), i, dev)
        _check_ssim_gpu(f"shape grid {kind}", x, y, G)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", CONTENT)
def test_ssim_contents_at_a_tiled_size(kind):
    dev = torch.device("cuda:0")
    for k, gk in enumerate(("random", "magnitudes")):
        x, y = content(kind, (2, 3, 70, 100), 3 + k, dev)
        _check_ssim_gpu(f"{kind} dmap {gk}", x, y, dmap(gk, (2, 70, 100), k, dev))


@pytest.mark.gpu
def test_ssim_one_hot_dmap_touches_only_the_window():
    """dL/dmap one-hot at tile and image corners: dL/dimg1 is zero outside the 11x11 neighbourhood, bitwise."""
    dev = torch.device("cuda:0")
    H, W = 40, 70
    x, y = content("training", (2, 3, H, W), 5, dev)
    for py, px in [(0, 0), (H - 1, W - 1), (15, 31), (16, 32), (31, 63), (32, 64), (0, W - 1), (H - 1, 0)]:
        G = torch.zeros(2, H, W, device=dev)
        G[1, py, px] = 0.75
        dx = _check_ssim_gpu("one-hot dmap", x, y, G)
        near = torch.zeros(2, 1, H, W, dtype=torch.bool, device=dev)
        near[1, :, max(0, py - 5):py + 6, max(0, px - 5):px + 6] = True
        assert bool((dx.masked_select(~near.expand_as(dx)) == 0).all()), (py, px)
        assert bool((dx[1].abs() > 0).any()), (py, px)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(1080, 1920), (2160, 4096)])
def test_ssim_image_sizes(H, W):
    dev = torch.device("cuda:0")
    x, y = content("training", (1, 3, H, W), 11, dev)
    _check_ssim_gpu(f"{H}x{W}", x, y, dmap("random", (1, H, W), 11, dev))


# ---- the loss block ---------------------------------------------------------------------------------------------------

def kernel_loss(toned, raw, gt, mask, weight, gscale, c_l1, c_ssim, dL):
    C = _lib()
    dev = gt.device
    H, W = gt.shape[-2:]
    ptr = lambda t: None if t is None else t.data_ptr()
    scaled = mask is not None or gscale is not None
    o = dict(raw_scaled=_nan(3, H, W) if scaled else None, ssim_map=_nan(H, W), ssim_partials=_nan(9, H, W),
             loss=_nan(1), metrics=_nan(8), dL_dmap=_nan(H, W), d_toned=_nan(3, H, W), d_raw=_nan(3, H, W))
    scratch = torch.zeros(C._lib.gsr_train_loss_scratch_bytes(), dtype=torch.uint8, device=dev)
    g = torch.tensor([dL], dtype=torch.float32, device=dev)
    a = C.GsrTrainLossArgs()
    a.H, a.W, a.c_l1, a.c_ssim = H, W, c_l1, c_ssim
    for k, t in dict(toned=toned, raw=raw, gt=gt, mask=mask, weight=weight, grad_scale=gscale, scratch=scratch,
                     dL_dloss=g, **o).items():
        setattr(a, k, ptr(t))
    C._check(C._lib.gsr_train_loss_forward(ctypes.byref(a), _stream()), "gsr_train_loss_forward")
    C._check(C._lib.gsr_train_loss_backward(ctypes.byref(a), _stream()), "gsr_train_loss_backward")
    torch.cuda.synchronize()
    return o


LOSS_CASES = ([("odd", b, (37, 53), None, 0.2, 1.0) for b in BRANCHES]
              + [(f"{H}x{W}", b, (H, W), mk, lam, dL) for (H, W), b, mk, lam, dL in [
                  ((511, 513), "mask_scale_grad_centred", None, 0.2, 0.37),
                  ((512, 512), "fractional_mask_w_ramped", None, 1.0, 2.0 ** -12),
                  ((1, 262145), "scale_grad_ramped", None, 0.0, 1.0),
                  ((1, 262145), "mask", "ones", 0.2, 0.37),
                  ((1080, 1920), "mask_scale_grad_centred", None, 0.2, 1.0),
                  ((37, 53), "mask", "zeros", 0.2, 1.0),
                  ((37, 53), "mask_scale_grad_centred", "zeros", 1.0, 0.37),
                  ((37, 53), "fractional_mask", "ones", 0.0, 2.0 ** -12),
                  ((512, 512), "plain", None, 0.2, 2.0 ** -12)]])


def _check_loss_gpu(family, toned, raw, gt, mask, weight, gscale, lam, dL):
    c_l1, c_ssim = float(np.float32(1 - lam)), float(np.float32(lam))
    o = kernel_loss(toned, raw, gt, mask, weight, gscale, c_l1, c_ssim, dL)
    parts = sx.loss_exact_parts(toned, raw, gt, mask, weight, gscale, c_l1, c_ssim, dL)
    for k in ("raw_scaled", "dL_dmap", "d_toned"):
        if parts[k] is None:
            assert o[k] is None
            continue
        got = o[k].cpu().numpy()
        assert np.array_equal(got.view(np.uint32), parts[k].view(np.uint32)), (family, k)
    smap = o["ssim_map"].cpu().numpy()
    want = sx.loss_values(parts, smap, c_l1, c_ssim)
    got = dict(zip(sx.METRICS, o["metrics"].cpu().numpy().tolist()), loss=float(o["loss"].cpu()))
    for k, (S, E) in want.items():
        assert _accepted(got[k], S, E), (family, k, got[k], S, E)
    # the SSIM forward on raw_scaled and the scaled backward, replayed on the kernel's own partials and dL/dmap
    dev = gt.device
    A = sx.IvArith(device=dev)
    r_in = (o["raw_scaled"] if o["raw_scaled"] is not None else raw)[None]
    s_map, s_P = sx.ssim_forward(A, r_in, gt[None])
    check("loss.ssim_map", family, o["ssim_map"][None], s_map)
    P = o["ssim_partials"].view(1, 3, 3, *gt.shape[-2:])
    check("loss.partials", family, P, s_P)
    v = lambda t: None if t is None else A.v(t.double())
    d = sx.ssim_backward(A, r_in, gt[None], A.v(P.double()), A.v(o["dL_dmap"][None].double()), v(gscale), v(mask))
    check("loss.d_raw", family, o["d_raw"][None], d)


@pytest.mark.gpu
@pytest.mark.parametrize("family,branch,size,mask_kind,lam,dL", LOSS_CASES)
def test_loss_block(family, branch, size, mask_kind, lam, dL):
    dev = torch.device("cuda:0")
    toned, raw, gt, mask, weight, gscale = loss_case(dev, *size, branch, 3, mask_kind)
    fam = f"{family} {branch}" + (f" mask {mask_kind}" if mask_kind else "")
    _check_loss_gpu(fam, toned, raw, gt, mask, weight, gscale, lam, dL)


@pytest.mark.gpu
def test_loss_block_toned_equals_gt():
    """toned == gt everywhere: mse = 0, psnr = +inf, every L1 sign 0."""
    dev = torch.device("cuda:0")
    for branch in ("plain", "mask"):
        toned, raw, gt, mask, weight, gscale = loss_case(dev, 37, 53, branch, 4)
        _check_loss_gpu(f"toned == gt {branch}", gt.clone(), raw, gt, mask, weight, gscale, 0.2, 1.0)


# ---- msssim and ssim_down ---------------------------------------------------------------------------------------------

def kernel_msssim(x, y, h, w, mn):
    C = _lib()
    B, _, H, W = x.shape
    nbytes = C._lib.gsr_msssim_scratch_bytes(B, h, w, mn)
    L, _ = sx.msssim_layout(B, h, w, mn)
    assert nbytes == L["total"] * 4
    scratch = _nan(L["total"], dev=x.device)
    out = _nan(B, H, W, dev=x.device)
    C._check(C._lib.gsr_msssim_forward(B, H, W, h, w, mn, x.data_ptr(), y.data_ptr(), out.data_ptr(), scratch.data_ptr(),
                                       _stream()), "gsr_msssim_forward")
    torch.cuda.synchronize()
    return sx.msssim_stages(scratch, B, h, w, mn, out)


def kernel_ssim_down(x, y, h, w):
    C = _lib()
    B, _, H, W = x.shape
    resize = (h, w) != (H, W)
    nbytes = C._lib.gsr_ssim_down_scratch_bytes(B, h, w)
    n = sx.pad64(B * 3 * h * w)
    assert nbytes == (2 * n + sx.pad64(B * h * w)) * 4
    scratch = _nan(nbytes // 4, dev=x.device)
    out = _nan(B, H, W, dev=x.device)
    C._check(C._lib.gsr_ssim_down_forward(B, H, W, h, w, x.data_ptr(), y.data_ptr(), out.data_ptr(),
                                          scratch.data_ptr() if resize else None, _stream()), "gsr_ssim_down_forward")
    torch.cuda.synchronize()
    st = {"out": out}
    if resize:
        st["x0"] = scratch[:B * 3 * h * w].view(B, 3, h, w)
        st["y0"] = scratch[n:n + B * 3 * h * w].view(B, 3, h, w)
        st["map"] = scratch[2 * n:2 * n + B * h * w].view(B, h, w)
    return st


MS_CASES = [  # (B, H, W, h, w, min_size): resize on / off, 0, 1, 2 and 4+ coarse levels, odd level sizes,
    # non-integer area ratios, upsampling from h = 1 and w = 1, 1 x N and N x 1
    (1, 64, 80, 64, 80, 100),
    (2, 45, 61, 45, 61, 30),
    (1, 99, 131, 71, 94, 20),
    (2, 200, 310, 150, 233, 8),
    (1, 1080, 1920, 400, 711, 80),
    (1, 1, 300, 1, 300, 1),
    (2, 300, 1, 300, 1, 1),
    (1, 3, 40, 1, 13, 1),
    (1, 40, 3, 9, 1, 1),
    (1, 17, 29, 5, 33, 2),
    (2, 37, 53, 23, 29, 2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,h,w,mn", MS_CASES)
def test_msssim_and_ssim_down(B, H, W, h, w, mn):
    dev = torch.device("cuda:0")
    kind = CONTENT[(H + W) % len(CONTENT)]
    x, y = content(kind, (B, 3, H, W), H * W, dev)
    fam = f"{B}x{H}x{W}->{h}x{w} min {mn} {kind}"
    st = kernel_msssim(x, y, h, w, mn)
    A = sx.IvArith(device=dev)
    ee = sx.msssim(A, x, y, h, w, mn)
    rp = sx.msssim(A, x, y, h, w, mn, stages=st)
    resize = (h, w) != (H, W)
    for k in ee:
        if k in ("x0", "y0") and not resize:
            continue
        got = st[k] if (k != "mean0" or resize) else st["out"]
        check("msssim." + k.rstrip("0123456789"), fam + " end to end", got, ee[k])
        check("msssim." + k.rstrip("0123456789"), fam, got, rp[k])
    sd = kernel_ssim_down(x, y, h, w)
    ee = sx.ssim_down(A, x, y, h, w)
    rp = sx.ssim_down(A, x, y, h, w, stages=sd)
    for k in ee:
        check("ssim_down." + k, fam + " end to end", sd[k], ee[k])
        check("ssim_down." + k, fam, sd[k], rp[k])
