"""Per-Gaussian chain rule (csrc/preprocess_bwd.cu) under an fp64 running-error oracle (``oracle/chain_exact.py``):
every entry of every output of ``gsr_backward_finalize`` is held to |kernel - S| <= B on accumulator rows the test
chooses, so a wrong term cannot hide behind the composite's atomics or a tensor-level tolerance.

GPU tests (``-m gpu``; no compiled reference needed): ``gsr_backward_finalize`` called through ``GsrBackwardArgs`` with
dL/dconic and dL/dcov3D requested, on the composite's own rows, log-uniform random rows (|slot| in 1e-6 .. 1e6),
single-slot rows (one slot per row, every slot in turn) and the composite's rows scaled by 1e-30 and 1e30.  Scenes:
posed (precomp, sh3, cov3d), the guard band, the depth span to the near plane, kernel size / scale modifier settings,
degenerate splats at kernel size 0 and 0.1, opaque stacks, the widest strip and huge splats whose det^2 overflows fp32
(the N == 0 branch); SH layouts M = 4 and 16 (vector path), M = 9 and M = 16 offset by 4 bytes (scalar path), a degree
below the tensor's and a scene without SH.  Also: culled and all-zero rows are exactly zero (dL_dsh included), SH
coefficients above the active degree are zero, consumed accumulator rows are zeroed and culled rows left alone, and
few rows are undetermined.  Each family asserts it reaches the edge it exists for.

CPU tests: with the fp64 constants S equals ``cpu_oracle``'s fp64 chain rule to 1e-12 of M; an fp32 emulation of the
kernel with random fma contraction stays within B; and each corruption of that emulation in ``chain_exact.MUTATIONS``
exceeds B on the row where it matters most.

The measured worst |kernel - S| / B per output and family is in DESIGN.md (3.3, numerics note).
"""
import ctypes

import numpy as np
import pytest
import torch

import synthetic
from oracle import chain_exact, cpu_oracle

UND_SHARE = 2e-3        # most undetermined rows a family may have (the degenerate family and the 1e30 rows excepted)
OUT_KEYS = {"dL_dmean2D": "dL_dmeans2D", "dL_dconic": "dL_dconic", "dL_dopacity": "dL_dopacity",
            "dL_dcolor": "dL_dcolors", "dL_dmean3D": "dL_dmeans3D", "dL_dcov3D": "dL_dcov3D", "dL_dsh": "dL_dsh",
            "dL_dscale": "dL_dscales", "dL_drot": "dL_drotations"}          # chain_exact -> cpu_oracle names


# ======================================================================================================================
# scenes and accumulator rows
# ======================================================================================================================
def scene_huge(seed=221, P=4000, W=160, H=120):
    """Ordinary splats plus 10 % whose scales (1e2 .. 1e5 times the depth) make det = |cov2D| so large that det^2
    overflows fp32 -- the kernel's N = 1 / (det^2 + 1e-7) is 0 there -- and some just below that."""
    from test_adversarial_scenes import _cloud, build_scene, posed_camera
    cam = posed_camera(W, H, seed)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, P, cam)
    n = P // 10
    s[:n] = xyz[:n, 2:3] * torch.exp(torch.log(torch.tensor(1e2)) + torch.rand(n, 1, generator=g, dtype=torch.float64)
                                     * float(np.log(1e3))) * torch.exp(0.2 * torch.randn(n, 3, generator=g,
                                                                                          dtype=torch.float64))
    op[:n] = 0.01
    return build_scene(cam, W, H, seed, xyz, s, rot, op)


def scene_of(name, small=False):
    from test_adversarial_scenes import (scene_degenerate, scene_depth_span, scene_guard_band, scene_opaque,
                                         scene_posed, scene_settings, scene_widest_strip)
    kw = dict(P=3000, W=70, H=50) if small else dict(P=20_000)
    table = {
        "posed_precomp": lambda: scene_posed("precomp", **kw),
        "posed_sh3": lambda: scene_posed("sh3", **kw),
        "posed_cov3d": lambda: scene_posed("cov3d", **kw),
        "guard_band": lambda: scene_guard_band(**kw),
        "depth_span": lambda: scene_depth_span(**kw),
        "settings_0_0.6": lambda: scene_settings(0.0, 0.6, **kw),
        "settings_0.3_1.7": lambda: scene_settings(0.3, 1.7, **kw),
        "settings_0_1.7": lambda: scene_settings(0.0, 1.7, **kw),
        "degenerate_0": lambda: scene_degenerate(0.0, **kw),
        "degenerate_0.1": lambda: scene_degenerate(0.1, **kw),
        "opaque": lambda: scene_opaque(**kw),
        "widest_strip": lambda: scene_widest_strip(P=kw["P"]),
        "huge": lambda: scene_huge(P=kw["P"] // 5 if not small else 3000),
    }
    return table[name]()


def log_uniform_rows(P, seed, single_slot=False):
    """[P, 10] fp32 rows, |slot| log-uniform in 1e-6 .. 1e6 with random signs; single_slot: row i has only slot i % 10"""
    g = np.random.default_rng(seed)
    a = (10.0 ** g.uniform(-6, 6, (P, 10)) * np.where(g.random((P, 10)) < 0.5, -1, 1)).astype(np.float32)
    if single_slot:
        a = np.where(np.arange(10)[None] == (np.arange(P) % 10)[:, None], a, np.float32(0))
    return a


def oracle_inputs(sc, opac, M=None, deg=None, clamp=None):
    """chain_exact keyword inputs of a scene (numpy / torch CPU or device values)"""
    kw = dict(means3D=sc["means3D"], view=sc["viewmatrix"].reshape(-1), proj=sc["projmatrix"].reshape(-1),
              W=int(sc["image_width"]), H=int(sc["image_height"]), tan_fovx=float(sc["tanfovx"]),
              tan_fovy=float(sc["tanfovy"]), kernel_size=float(sc["kernel_size"]),
              scale_modifier=float(sc["scale_modifier"]), opac=opac)
    if "cov3D_precomp" in sc:
        kw["cov3D_precomp"] = sc["cov3D_precomp"]
    else:
        kw["scales"], kw["rotations"] = sc["scales"], sc["rotations"]
    if "shs" in sc:
        shs = sc["shs"]
        kw.update(shs=shs[:, :M] if M else shs, deg=sc["sh_degree"] if deg is None else deg, campos=sc["campos"],
                  clamp=clamp)
    return kw


# ======================================================================================================================
# CPU tests
# ======================================================================================================================
CPU_SCENES = ["posed_sh3", "posed_cov3d", "guard_band", "settings_0.3_1.7", "settings_0_0.6", "degenerate_0",
              "degenerate_0.1"]


def _cpu_rows(st, seed):
    """the composite's rows for the first half of the Gaussians, log-uniform rows for the rest, every tenth single-slot"""
    P = st["P"]
    comp = cpu_oracle.backward(st, st["scene"]["dL_dpix"])["acc"].astype(np.float32)
    rnd = log_uniform_rows(P, seed)
    one = log_uniform_rows(P, seed + 1, single_slot=True)
    i = np.arange(P)[:, None]
    return np.where(i < P // 2, comp, np.where(i % 10 == 0, one, rnd))


@pytest.mark.parametrize("name", CPU_SCENES)
def test_oracle_value_is_the_fp64_cpu_oracle(name):
    """With the fp64 constants and decisions, S equals cpu_oracle's fp64 chain rule on the same rows to 1e-12 of M."""
    sc = scene_of(name, small=True)
    st = cpu_oracle.forward(sc, np.float64)
    acc = _cpu_rows(st, 3)
    ref = cpu_oracle.backward(st, None, acc=acc)
    kw = oracle_inputs(sc, st["conic_opacity"][:, 3], clamp=[st["clamped"][:, c] != 0 for c in range(3)])
    ex = chain_exact.bound(acc=acc, radii=st["radii"], C=chain_exact.F64, u=0.0, **kw)
    mag = chain_exact.bound(acc=acc, radii=st["radii"], C=chain_exact.F64, **kw)
    act = ex["active"].numpy()
    assert act.sum() > 1000
    for k, rk in OUT_KEYS.items():
        if k not in ex:
            continue
        S = ex[k]["S"].numpy()
        M = np.where(np.isfinite(mag[k]["M"].numpy()), mag[k]["M"].numpy(), np.inf)
        r = ref[rk].reshape(S.shape)
        err = np.abs(S - r)[act]
        bad = err > 1e-12 * M[act] + 1e-300
        assert not bad.any(), (name, k, int(bad.sum()), float((err / np.maximum(M[act], 1e-300)).max()))


def _emulation_case(name):
    sc = scene_of(name, small=True)
    st = cpu_oracle.forward(sc)
    acc = _cpu_rows(st, 5)
    clamp = [st["clamped"][:, c] != 0 for c in range(3)]
    kw = oracle_inputs(sc, st["conic_opacity"][:, 3], clamp=clamp)
    res = chain_exact.bound(acc=acc, radii=st["radii"], **kw)
    return sc, st, acc, kw, res


@pytest.mark.parametrize("name", ["posed_sh3", "guard_band", "degenerate_0", "settings_0.3_1.7"])
def test_bound_holds_for_an_fp32_emulation(name):
    sc, st, acc, kw, res = _emulation_case(name)
    for seed in range(3):
        em = chain_exact.emulate(acc=acc, radii=st["radii"], gen=torch.Generator().manual_seed(seed), **kw)
        r = chain_exact.ratios(em, res, rows=res["active"])
        print(f"{name} seed {seed}: worst |emulated - S| / B " + ", ".join(f"{k} {v:.2e}" for k, v in r.items()))
        assert max(r.values()) <= 1.0, (name, seed, r)


# the scene on which each corruption matters
MUTATION_SCENES = {
    "swap_xy_masks": "guard_band", "cov_offdiag_no_2": "posed_cov3d", "db_not_halved": "posed_sh3",
    "fx_for_fy": "posed_sh3", "clamp_wrong_channel": "posed_sh3", "opacity_without_coef": "settings_0.3_1.7",
    "det1_plus_eps_squared": "degenerate_0", "modifier_in_dscale": "settings_0.3_1.7",
    "quat_normalised": "degenerate_0.1", "no_sh_direction_term": "posed_sh3", "no_proj_w_terms": "posed_sh3"}
_CASES = {}


@pytest.mark.parametrize("mut", chain_exact.MUTATIONS)
def test_mutations_are_caught(mut):
    """Each corruption, applied to every row, takes some determined row beyond its bound: the worst row is the
    placement where the corruption matters most."""
    name = MUTATION_SCENES[mut]
    if name not in _CASES:
        _CASES[name] = _emulation_case(name)
    sc, st, acc, kw, res = _CASES[name]
    em = chain_exact.emulate(acc=acc, radii=st["radii"], gen=torch.Generator().manual_seed(0), mut=mut, **kw)
    r = chain_exact.ratios(em, res)
    worst = max(r.values())
    print(f"{mut} on {name}: worst |mutated - S| / B = {worst:.3g} ({max(r, key=r.get)})")
    assert worst > 1.0, (mut, r)


# ======================================================================================================================
# GPU helpers
# ======================================================================================================================
def _aligned(n, dev, offset_floats=0):
    """a float32 tensor of n entries whose first element sits offset_floats after a 256-byte boundary"""
    buf = torch.full((n + 128,), float("nan"), dtype=torch.float32, device=dev)
    off = (-buf.data_ptr()) % 256 // 4 + offset_floats
    return buf[off:off + n]


def gpu_forward(sc, M=None):
    """Forward through the C ABI; the composite's [P, 10] rows; the oracle's record inputs."""
    from diff_gaussian_rasterization import _C
    from make_golden import backward_args, call_args
    sc = dict(sc)
    if M is not None:
        sc["shs"] = sc["shs"][:, :M].contiguous()
    d = synthetic.to_device(sc, torch.device("cuda:0"))
    P, W, H = d["means3D"].shape[0], d["image_width"], d["image_height"]
    Mf = d["shs"].shape[1] if "shs" in d else 0
    _C.set_geometry_cache(False)
    try:
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(*call_args(d))
        v = _C.debug_views(geom, binning, img, P, Mf, W, H, R)
        acc = _C.rasterize_gaussians_backward_partials(*backward_args(d, radii, geom, R, binning, img))
        acc = acc[:P * 12].view(P, 12)[:, :10].clone()
        torch.cuda.synchronize()
    finally:
        _C.set_geometry_cache(True)
    return dict(sc=sc, d=d, P=P, M=Mf, R=R, radii=radii, geom=geom, acc=acc, rec=v["records"].clone(),
                rgb=v["rgb"].clone() if Mf else None)


def gpu_finalize(o, acc10, D=None, sh_offset=0):
    """gsr_backward_finalize on fixed rows acc10 [P, 10] (culled rows' accumulator entries set to 1: not read).
    Returns the nine outputs and the accumulator after the call."""
    from diff_gaussian_rasterization import _C
    d, P, M = o["d"], o["P"], o["M"]
    dev = d["means3D"].device
    acc = _aligned(P * 12, dev).view(P, 12)
    acc.zero_()
    acc[:, :10] = acc10
    acc[~o["radii"].gt(0)] = 1.0
    before = acc.clone()
    nan = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device=dev)
    outs = dict(dL_dmean2D=nan(P, 3), dL_dconic=nan(P, 4), dL_dopacity=nan(P, 1), dL_dcolor=nan(P, 3),
                dL_dmean3D=nan(P, 3), dL_dcov3D=nan(P, 6))
    e = torch.empty(0, device=dev)
    keep = {k: d[k].float().contiguous() for k in ("means3D", "viewmatrix", "projmatrix", "campos")}
    for k in ("scales", "rotations", "cov3D_precomp"):
        keep[k] = d[k].float().contiguous() if k in d else e
    a = _C.GsrBackwardArgs()
    a.P, a.D, a.M, a.R = P, int(d["sh_degree"] if D is None else D), M, int(o["R"])
    a.W, a.H = d["image_width"], d["image_height"]
    a.means3D = keep["means3D"].data_ptr()
    a.scales = keep["scales"].data_ptr() if keep["scales"].numel() else None
    a.rotations = keep["rotations"].data_ptr() if keep["rotations"].numel() else None
    a.cov3D_precomp = keep["cov3D_precomp"].data_ptr() if keep["cov3D_precomp"].numel() else None
    a.scale_modifier = float(d["scale_modifier"])
    a.viewmatrix = keep["viewmatrix"].data_ptr(); a.projmatrix = keep["projmatrix"].data_ptr()
    a.campos = keep["campos"].data_ptr()
    a.tan_fovx = float(d["tanfovx"]); a.tan_fovy = float(d["tanfovy"]); a.kernel_size = float(d["kernel_size"])
    radii = o["radii"].contiguous()
    a.radii = radii.data_ptr(); a.geom_buffer = o["geom"].data_ptr()
    a.accum_scratch = acc.data_ptr(); a.accum_is_zero = 1
    a.dL_dmean2D = outs["dL_dmean2D"].data_ptr(); a.dL_dconic = outs["dL_dconic"].data_ptr()
    a.dL_dopacity = outs["dL_dopacity"].data_ptr(); a.dL_dcolor = outs["dL_dcolor"].data_ptr()
    a.dL_dmean3D = outs["dL_dmean3D"].data_ptr(); a.dL_dcov3D = outs["dL_dcov3D"].data_ptr()
    if M:
        shs = _aligned(P * M * 3, dev, sh_offset)
        shs.copy_(d["shs"].reshape(-1))
        dsh = _aligned(P * M * 3, dev, sh_offset)
        a.shs, a.dL_dsh = shs.data_ptr(), dsh.data_ptr()
        outs["dL_dsh"] = dsh.view(P, M * 3)
        keep["shs"] = shs
    if a.scales:
        outs["dL_dscale"], outs["dL_drot"] = nan(P, 3), nan(P, 4)
        a.dL_dscale, a.dL_drot = outs["dL_dscale"].data_ptr(), outs["dL_drot"].data_ptr()
    _C._check(_C._lib.gsr_backward_finalize(ctypes.byref(a), torch.cuda.current_stream().cuda_stream),
              "gsr_backward_finalize")
    torch.cuda.synchronize()
    return outs, before, acc.clone()


def gpu_oracle(o, acc10, D=None):
    sc, d = o["sc"], o["d"]
    dev = d["means3D"].device
    deg = int(d["sh_degree"] if D is None else D)
    clamp = None
    if o["M"]:
        clamp = chain_exact.clamp_bits_from_rgb(o["rgb"], d["shs"], int(d["sh_degree"]), d["means3D"], d["campos"])
    kw = oracle_inputs(d, o["rec"][:, 7], deg=deg, clamp=clamp)
    return chain_exact.bound(acc=acc10, radii=o["radii"], device=dev, **kw)


def check_feed(name, o, acc10, D=None, sh_offset=0, und_share=UND_SHARE):
    outs, before, after = gpu_finalize(o, acc10, D, sh_offset)
    res = gpu_oracle(o, acc10, D)
    vis = o["radii"].gt(0)
    active = res["active"]
    # the accumulator contract: consumed rows are zero afterwards, rows of culled Gaussians untouched
    assert torch.equal(after[~vis], before[~vis]), name
    assert not after[active].any(), name
    assert torch.equal(after[vis & ~active], before[vis & ~active]), name
    r = {}
    for k, v in outs.items():
        assert not torch.isnan(v[~active]).any() and not v[~active].any(), (name, k, "inactive row not zero")
        S, B = res[k]["S"], res[k]["B"]
        kv = v.double().reshape(S.shape)
        e = (kv - S).abs()
        ok = (e <= B + 1e-12 * res[k]["M"] + 1e-300) | torch.isinf(B)
        bad = ~ok
        if bad.any():
            i = bad.any(1).nonzero()[:3, 0]
            raise AssertionError(f"{name} {k}: {int(bad.sum())} entries beyond their bound, rows {i.tolist()}: "
                                 f"kernel {kv[i].tolist()} S {S[i].tolist()} B {B[i].tolist()}")
        r[k] = chain_exact.ratios({k: v}, res)[k]
    if "dL_dsh" in outs:
        deg = int(o["d"]["sh_degree"] if D is None else D)
        used = (deg + 1) ** 2
        assert not outs["dL_dsh"][:, used * 3:].any(), (name, "dL_dsh above the active degree")
    n_und = int(res["und"].sum())
    n_act = int(active.sum())
    print(f"{name}: active {n_act} undetermined {n_und} edges " +
          " ".join(f"{k} {int(v.sum())}" for k, v in res["edges"].items()) +
          "; worst |k - S| / B: " + ", ".join(f"{k} {v:.2e}" for k, v in r.items()))
    if und_share is not None:
        assert n_und <= max(2, und_share * o["P"]), (name, "undetermined rows", n_und)
    return res, r


def check_scene(name, sc, M=None, D=None, sh_offset=0, und_share=UND_SHARE, feeds=("composite", "random", "single",
                                                                                     "tiny", "large")):
    o = gpu_forward(sc, M)
    P = o["P"]
    dev = o["acc"].device
    results = {}
    for f in feeds:
        if f == "composite":
            a, u = o["acc"], und_share
        elif f in ("random", "single"):
            a, u = torch.from_numpy(log_uniform_rows(P, 17, single_slot=f == "single")).to(dev), und_share
        else:
            a, u = o["acc"] * (1e-30 if f == "tiny" else 1e30), None
        assert a.any()
        results[f] = check_feed(f"{name}/{f}", o, a, D, sh_offset, u)
    return o, results


# ======================================================================================================================
# GPU tests
# ======================================================================================================================
FAMILIES = ["posed_precomp", "posed_sh3", "posed_cov3d", "guard_band", "depth_span", "settings_0_0.6",
            "settings_0.3_1.7", "settings_0_1.7", "opaque", "widest_strip"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", FAMILIES)
def test_families(name):
    sc = scene_of(name)
    o, res = check_scene(name, sc)
    e = res["random"][0]["edges"]
    if name == "guard_band":
        assert int(e["guard_band"].sum()) > 100, "no row beyond the guard band"
    if name == "posed_sh3":
        assert int(e["clamped_channel"].sum()) > 100, "no clamped colour channel"
    if name == "depth_span":
        from test_adversarial_scenes import view_space
        z = view_space(sc)[:, 2]
        assert int(((z < 0.21) & o["radii"].gt(0).cpu()).sum()) > 10, "nothing rendered at the near plane"
    if name.startswith("settings"):
        assert float(sc["scale_modifier"]) != 1.0
    if name == "opaque":
        assert int((o["rec"][:, 7] >= 0.99).sum()) > 100
    if name == "widest_strip":
        assert o["d"]["image_width"] == 65535 * 16


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["degenerate_0", "degenerate_0.1"])
def test_degenerate_splats(name):
    """Needles and sub-pixel splats: det0 = ca0 cc0 - b^2 cancels, so its a-priori interval often straddles the 1e-6
    clamp and such rows are undetermined (about 10 % here); their entries are still held to the hull of both branches."""
    o, res = check_scene(name, scene_of(name), und_share=None)
    e = res["random"][0]["edges"]
    assert int(e["det_clamp"].sum()) > 100, "no row at the det clamp"


@pytest.mark.gpu
def test_huge_splats_reach_the_overflow_branch():
    o, res = check_scene("huge", scene_of("huge"), und_share=None, feeds=("composite", "random", "single"))
    e = res["random"][0]["edges"]
    assert int(e["n_zero"].sum()) > 20, "no row with det^2 overflowing"


# (M, degree, byte offset of the SH and dL_dsh rows): vector path (M 4 / 16 aligned), scalar path (M 9, misaligned)
SH_LAYOUTS = [(4, 1, 0), (16, 3, 0), (9, 2, 0), (16, 3, 1), (16, 1, 0), (9, 1, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("M,D,off", SH_LAYOUTS)
def test_sh_layouts(M, D, off):
    from test_adversarial_scenes import scene_posed
    sc = scene_posed("sh3", P=20_000)
    sc["sh_degree"] = D
    check_scene(f"sh_M{M}_D{D}_off{off}", sc, M=M, D=D, sh_offset=off, feeds=("composite", "random", "single"))
