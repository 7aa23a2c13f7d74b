"""Backward composite (csrc/render_bwd.cu) under an fp64 running-error oracle (``oracle/bwd_exact.py``,
``oracle/bwd_bound.c``): every slot of every Gaussian's accumulator row is held to an a-priori bound.

GPU tests (``-m gpu``; no compiled reference needed): the raw [P, 12] accumulator of ``gsr_backward_partials`` satisfies
|acc - S| <= B entry by entry, rows with S = B = 0 and the padding slots 10, 11 are exactly zero, and few Gaussians are
undetermined (a blend decision within its error of a threshold).  Scenes: the ordinary SMALL scenes, a posed camera with
bg != 0, the DENSE scene (n_contrib beyond MASK_K, the footprint-box fallback), single-tile stacks whose n_contrib and
list length sit at MASK_K - 1 / MASK_K / MASK_K + 1, at round boundaries 64 r - 1 / 64 r / 64 r + 1 and at mask-word
multiples of 32, the image shapes 1x1, 1x37, 17x33 and 4095x3, a tile-row shard, opaque stacks at the 0.99 clamp and the
faint scene; upstream gradients random, one channel zero, constant, scaled by 1e-20 and 1e20, and a single non-zero
pixel.  ``gsr_backward`` (with dL/dconic), ``gsr_backward_finalize`` and ``gsr_backward_colors`` are held to the same
slots.

CPU tests: the oracle's value equals the fp64 CPU oracle's accumulator; a numpy fp32 emulation of the kernel's arithmetic,
summed in random pair / warp / tile / flush orders, stays within the bound; and corruptions of that emulation (a pair,
a warp block or the last walked position dropped, dL/dpix swapped within a pair, |.| after the warp sum, the background
term omitted, C for A in the flush, slots 3 and 4 swapped, a row flushed twice) are each caught.

The measured worst error / bound per scene is in DESIGN.md (3.2, numerics note).
"""
import ctypes

import numpy as np
import pytest
import torch

import synthetic
from oracle import bwd_exact, cpu_oracle

K = 1024                # MASK_K (common.cuh)
UND_SHARE = 2e-3        # most Gaussians with an undetermined pair a scene may have (the faint family excepted)


def records_of(st):
    """[P, 8] records {x, y, hx, hy, A, B, C, o} from a CPU-oracle forward state."""
    r = np.zeros((st["P"], 8), np.float64)
    r[:, 0:2] = st["means2D"]
    r[:, 4:8] = st["conic_opacity"]
    return r


# ======================================================================================================================
# scenes
# ======================================================================================================================
def scene_stack(n, seed=301, W=16, H=16, opacity=0.006):
    """One tile: n faint splats much wider than the image, so every pixel blends every one of them and n_contrib = the
    list length = n in every pixel (0.994^1025 > 1e-4: no pixel saturates)."""
    from test_adversarial_scenes import _cloud, build_scene, posed_camera
    cam = posed_camera(W, H, seed)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, n, cam, spread=0.05, opac_range=(opacity, opacity * 1.02))
    s = (xyz[:, 2] * 8.0)[:, None].expand(n, 3).contiguous()
    return build_scene(cam, W, H, seed, xyz, s, rot, op, subpixel_jitter=0.3)


def ordinary_scenes():
    from test_adversarial_scenes import scene_posed
    from test_blend_masks import SMALL, _scene
    return {"small_320x240": _scene(SMALL[0]), "small_300x200_jitter": _scene(SMALL[1]),
            "posed_bg": scene_posed("precomp")}


# ======================================================================================================================
# GPU helpers
# ======================================================================================================================
def _run(scene, dL=None, shard=None):
    """Forward and backward partials through the C ABI.  Returns the accumulator and the oracle's inputs."""
    from diff_gaussian_rasterization import _C
    from make_golden import backward_args, call_args
    d = synthetic.to_device(scene, torch.device("cuda:0"))
    if dL is not None:
        d["dL_dpix"] = torch.as_tensor(dL, dtype=torch.float32).to(d["means3D"].device).contiguous()
    W, H = d["image_width"], d["image_height"]
    P = d["means3D"].shape[0]
    M = d["shs"].shape[1] if "shs" in d else 0
    _C.set_geometry_cache(False)
    try:
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(*call_args(d))
        v = _C.debug_views(geom, binning, img, P, M, W, H, R)
        bargs = backward_args(d, radii, geom, R, binning, img)
        acc = _C.rasterize_gaussians_backward_partials(*bargs, shard=shard)[:P * 12].view(P, 12).clone()
        torch.cuda.synchronize()
    finally:
        _C.set_geometry_cache(True)
    colors = v["rgb"] if M > 0 else d["colors_precomp"]
    ins = dict(records=v["records"].cpu().numpy(), colors=colors.cpu().numpy(), point_list=v["point_list"].cpu().numpy(),
               ranges=v["ranges"].cpu().numpy(), n_contrib=v["n_contrib"].cpu().numpy(),
               subpixel_offset=d["subpixel_offset"].cpu().numpy(), bg=d["bg"].cpu().numpy(),
               dL_dpix=d["dL_dpix"].cpu().numpy(), W=W, H=H)
    return dict(d=d, acc=acc.cpu().numpy(), ins=ins, radii=radii, bufs=(R, geom, binning, img), P=P)


def _oracle(o, shard=None, **kw):
    return bwd_exact.bound(**o["ins"], tile_rows=shard or (0, 0), **kw)


def _assert_within(name, acc, res, slots=range(10), und_share=UND_SHARE):
    """Every entry within its bound; rows with S = B = 0 and the padding exactly zero; few undetermined."""
    full = res["S"].copy()
    a = np.asarray(acc, np.float64)
    for s in slots:
        full[:, s] = a[:, s]
    if a.shape[1] >= 12:
        full = np.concatenate([full, a[:, 10:12]], axis=1)
    c = bwd_exact.check(full, res)
    P = res["S"].shape[0]
    n_und = int((res["und"] > 0).sum())
    worst = ", ".join(f"{k} {v:.2e}" for k, v in c["ratio"].items())
    det = bwd_exact.check(full, res, mask=res["und"] == 0)["ratio"]
    print(f"{name}: P={P} blended pairs {res['blended_pairs']} undetermined pairs {res['undetermined_pairs']} "
          f"Gaussians {n_und} ({n_und / max(P, 1):.1e}) overflow pixels {res['overflow_pixels']}; worst error/B: {worst}; "
          f"without undetermined Gaussians: {max(det.values()):.2e}")
    assert c["violations"].size == 0, (name, "entries beyond their bound in rows", c["violations"][:10].tolist(),
                                       a[c["violations"][:3]], res["S"][c["violations"][:3]], res["B"][c["violations"][:3]])
    assert c["nonzero_where_zero"].size == 0, (name, "non-zero where nothing blends", c["nonzero_where_zero"][:10].tolist())
    assert c["padding_nonzero"].size == 0, (name, "padding slots written", c["padding_nonzero"][:10].tolist())
    if und_share is not None:
        assert n_und <= max(2, und_share * P), (name, "undetermined Gaussians", n_und)
    return c


def _check_scene(name, scene, dL=None, shard=None, und_share=UND_SHARE):
    o = _run(scene, dL, shard)
    res = _oracle(o, shard)
    _assert_within(name, o["acc"], res, und_share=und_share)
    return o, res


# ======================================================================================================================
# GPU tests
# ======================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small_320x240", "small_300x200_jitter", "posed_bg"])
def test_ordinary_scenes(name):
    o, res = _check_scene(name, ordinary_scenes()[name])
    assert res["blended_pairs"] > 100_000


@pytest.mark.gpu
def test_dense_beyond_mask_k():
    from test_blend_masks import DENSE, DENSE_OPACITY, _scene
    o, res = _check_scene("dense", _scene(DENSE, DENSE_OPACITY))
    assert int(o["ins"]["n_contrib"].max()) > K, "scene does not reach the positions beyond MASK_K"


# list lengths around MASK_K, the 64-entry staging rounds and the 32-bit mask words; each a single tile where every
# pixel's n_contrib equals the list length
STACKS = [K - 1, K, K + 1, 127, 128, 129, 191, 192, 193, 32, 96, 160, 1]


@pytest.mark.gpu
@pytest.mark.parametrize("n", STACKS)
def test_list_position_boundaries(n):
    o, res = _check_scene(f"stack_{n}", scene_stack(n))
    nc = o["ins"]["n_contrib"]
    assert int(nc.max()) == n and int(nc.min()) == n, (n, int(nc.min()), int(nc.max()))
    assert int(np.diff(o["ins"]["ranges"][0])[0]) == n


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", [(1, 1), (1, 37), (17, 33), (4095, 3)])
def test_image_shapes(W, H):
    from test_adversarial_scenes import scene_shape
    _check_scene(f"shape_{W}x{H}", scene_shape(W, H))


@pytest.mark.gpu
def test_tile_row_shard():
    from test_blend_masks import SMALL, _scene
    o, res = _check_scene("shard_3_9", _scene(SMALL[0]), shard=(3, 9))
    # rows of Gaussians that touch no tile of the shard stay zero; some do
    assert (np.abs(o["acc"]).sum(axis=1) == 0).sum() > 0 and res["blended_pairs"] > 0


@pytest.mark.gpu
def test_opaque_stacks_at_the_clamp():
    from test_adversarial_scenes import scene_opaque
    o, res = _check_scene("opaque", scene_opaque())
    rec = o["ins"]["records"]
    assert (rec[:, 7] >= 0.99).sum() > 100


@pytest.mark.gpu
def test_faint_scene():
    from test_adversarial_scenes import scene_faint
    o, res = _check_scene("faint", scene_faint(), und_share=None)
    assert res["blended_pairs"] == 0 and not np.any(o["acc"])


def _upstream(kind, H, W, seed=7):
    g = np.random.default_rng(seed)
    dL = g.standard_normal((3, H, W)).astype(np.float32)
    if kind == "channel_zero":
        dL[1] = 0
    elif kind == "constant":
        dL[:] = np.float32(0.37)
    elif kind == "tiny":
        dL *= np.float32(1e-20)
    elif kind == "huge":
        dL *= np.float32(1e20)
    elif kind == "one_pixel":
        y, x = H // 2 + 3, W // 3 + 5
        one = dL[:, y, x].copy()
        dL[:] = 0
        dL[:, y, x] = one
    return dL


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["random", "channel_zero", "constant", "tiny", "huge", "one_pixel"])
def test_upstream_gradients(kind):
    from test_adversarial_scenes import scene_posed
    sc = scene_posed("precomp", P=20_000, W=200, H=150)
    dL = _upstream(kind, 150, 200)
    o, res = _check_scene(f"upstream_{kind}", sc, dL=dL)
    if kind == "one_pixel":
        # only the Gaussians blended in that pixel have a non-zero row
        touched = np.any(o["acc"] != 0, axis=1)
        assert 0 < touched.sum() <= 400, int(touched.sum())


def _backward_with_conic(o):
    """gsr_backward through the C ABI with dL_dconic requested; returns (dL_dmeans2D, dL_dconic, dL_dcolors)."""
    from diff_gaussian_rasterization import _C
    d, P = o["d"], o["P"]
    R, geom, binning, img = o["bufs"]
    dev = d["means3D"].device
    f = dict(dtype=torch.float32, device=dev)
    m2, con, col, op, m3 = (torch.full((P, k), float("nan"), **f) for k in (3, 4, 3, 1, 3))
    cov = torch.full((P, 6), float("nan"), **f)
    acc = torch.zeros((P * 12 + 64,), **f)
    e = torch.empty(0, **f)
    keep = dict(bg=d["bg"], means3D=d["means3D"], colors=d.get("colors_precomp", e), scales=d.get("scales", e),
                rotations=d.get("rotations", e), cov3D=d.get("cov3D_precomp", e), view=d["viewmatrix"],
                proj=d["projmatrix"], so=d["subpixel_offset"], dL=d["dL_dpix"], campos=d["campos"])
    keep = {k: v.float().contiguous() for k, v in keep.items()}
    scl = torch.zeros((P, 3), **f)
    rot = torch.zeros((P, 4), **f)
    a = _C.GsrBackwardArgs()
    a.P, a.D, a.M, a.R, a.W, a.H = P, 0, 0, int(R), d["image_width"], d["image_height"]
    a.background = keep["bg"].data_ptr(); a.means3D = keep["means3D"].data_ptr(); a.shs = None
    a.colors_precomp = keep["colors"].data_ptr(); a.scales = keep["scales"].data_ptr()
    a.scale_modifier = float(d["scale_modifier"]); a.rotations = keep["rotations"].data_ptr()
    a.cov3D_precomp = keep["cov3D"].data_ptr() if keep["cov3D"].numel() else None
    a.viewmatrix = keep["view"].data_ptr(); a.projmatrix = keep["proj"].data_ptr(); a.campos = keep["campos"].data_ptr()
    a.tan_fovx = float(d["tanfovx"]); a.tan_fovy = float(d["tanfovy"]); a.kernel_size = float(d["kernel_size"])
    a.subpixel_offset = keep["so"].data_ptr(); a.radii = o["radii"].contiguous().data_ptr()
    a.geom_buffer = geom.data_ptr(); a.binning_buffer = binning.data_ptr(); a.img_buffer = img.data_ptr()
    a.dL_dpix = keep["dL"].data_ptr(); a.debug = 0
    a.tile_y0, a.tile_y1 = 0, 0
    a.accum_scratch = acc.data_ptr() + (-acc.data_ptr()) % 256
    a.accum_is_zero = 1
    a.dL_dmean2D = m2.data_ptr(); a.dL_dconic = con.data_ptr(); a.dL_dopacity = op.data_ptr()
    a.dL_dcolor = col.data_ptr(); a.dL_dmean3D = m3.data_ptr(); a.dL_dcov3D = cov.data_ptr()
    a.dL_dsh = None; a.dL_dscale = scl.data_ptr(); a.dL_drot = rot.data_ptr()
    _C._check(_C._lib.gsr_backward(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "gsr_backward")
    torch.cuda.synchronize()
    return m2.cpu().numpy(), con.cpu().numpy(), col.cpu().numpy()


@pytest.mark.gpu
def test_full_backward_finalize_and_colour_walk():
    """gsr_backward's dL/dmeans2D (with the |.| channel), dL/dconic and dL/dcolors are accumulator slots and get their
    bounds; gsr_backward_finalize copies those slots of a fixed accumulator bit for bit and leaves culled rows zero;
    gsr_backward_colors' dL/dcolor is held to slots 7..9 under the colour walk's summation."""
    from diff_gaussian_rasterization import _C
    from make_golden import backward_args
    from test_adversarial_scenes import scene_posed
    from test_fused_embedding import color_backward
    o = _run(scene_posed("precomp", P=20_000, W=200, H=150))
    res = _oracle(o)
    vis = (o["radii"] > 0).cpu().numpy()
    P = o["P"]

    m2, con, col = _backward_with_conic(o)
    acc = np.zeros((P, 10))
    acc[:, 0:3], acc[:, 3:5], acc[:, 5], acc[:, 7:10] = m2, con[:, 0:2], con[:, 3], col
    assert not np.isnan(acc).any() and not np.any(con[:, 2])
    _assert_within("gsr_backward", acc, res, slots=(0, 1, 2, 3, 4, 5, 7, 8, 9))

    d = o["d"]
    R, geom, binning, img = o["bufs"]
    fixed = torch.zeros((P * 12 + 64,), dtype=torch.float32, device=d["means3D"].device)
    off = (-fixed.data_ptr()) % 256 // 4
    view = fixed[off:off + P * 12]
    view.copy_(torch.from_numpy(o["acc"]).reshape(-1))
    view.view(P, 12)[~o["radii"].gt(0)] = 1.0          # rows of culled Gaussians are not read
    before = view.view(P, 12).cpu().numpy().copy()
    g = _C.rasterize_gaussians_backward_finalize(view, *backward_args(d, o["radii"], geom, R, binning, img))
    torch.cuda.synchronize()
    m2f, colf = g[0].cpu().numpy(), g[1].cpu().numpy()
    assert np.array_equal(m2f[vis].view(np.int32), before[vis][:, 0:3].view(np.int32))
    assert np.array_equal(colf[vis].view(np.int32), before[vis][:, 7:10].view(np.int32))
    assert not np.any(m2f[~vis]) and not np.any(colf[~vis])

    cw = color_backward(d, R, geom, binning, img, d["dL_dpix"]).cpu().numpy()
    acc_c = np.zeros((P, 10))
    acc_c[:, 7:10] = cw
    _assert_within("gsr_backward_colors", acc_c, _oracle(o, colour_walk=True), slots=(7, 8, 9))


# ======================================================================================================================
# CPU tests
# ======================================================================================================================
def cpu_cases():
    from test_adversarial_scenes import scene_guard_band, scene_posed
    return {"small": synthetic.make_scene(2000, 64, 48, seed=5, subpixel_jitter=0.3, bg=(0.2, 0.5, 0.1)),
            "posed": scene_posed("precomp", P=3000, W=70, H=50),
            "guard_band": scene_guard_band(P=3000, W=70, H=50)}


@pytest.mark.parametrize("name", ["small", "posed", "guard_band"])
def test_oracle_value_is_the_fp64_oracle_accumulator(name):
    """S equals cpu_oracle's fp64 accumulator (same decisions: the fp64 constants 0.99 and 1/255 are passed) to 1e-12
    of the slot's magnitude scale."""
    sc = cpu_cases()[name]
    st = cpu_oracle.forward(sc, np.float64)
    acc = cpu_oracle.backward(st, sc["dL_dpix"])["acc"]
    res = bwd_exact.bound(records_of(st), st["colors"], st["point_list"], st["ranges"], st["n_contrib"],
                          sc["subpixel_offset"], sc["bg"], sc["dL_dpix"], st["W"], st["H"], alpha_max=0.99,
                          alpha_min=1.0 / 255.0)
    assert res["blended_pairs"] > 1000
    err = np.abs(res["S"] - acc)
    assert np.all(err <= 1e-12 * res["M"]), (name, float((err / np.maximum(res["M"], 1e-300)).max()))
    assert not np.any((res["M"] == 0) & (acc != 0))


# ---- numpy fp32 emulation of render_bwd_packed_kernel -----------------------------------------------------------------
F32 = np.float32


def _fma(a, b, c):
    """fp32 fma (the exact product and sum in fp64, one rounding to fp32; a double rounding is at most 2^-29 ulp off)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def _tile_pixels(tx, ty):
    """Pixel i = 64 warp + 2 lane + k of a tile, mapped as PixelMap does (render_common.cuh): lane pairs are i, i ^ 1."""
    i = np.arange(256)
    w, lane, k = i // 64, (i // 2) % 32, i % 2
    return tx * 16 + (w % 2) * 8 + (lane & 7), ty * 16 + (w // 2) * 8 + (lane >> 3) * 2 + k


def emulate_tile(st, sc, t, rng, skip_last=False, swap=None, no_bg=None):
    """Per-pixel fp32 terms of one tile, in the kernel's operation order (render_bwd.cu:339-390).  Returns the list
    positions' Gaussian ids and terms [total, 256, 12]: the 10 slots, then the signed |.| parts u1 |o| W/2, u2 |o| H/2.
    expf is perturbed by up to one ulp either way (the bound allows two)."""
    W, H = st["W"], st["H"]
    gx = (W + 15) // 16
    ux, uy = _tile_pixels(t % gx, t // gx)
    inside = (ux < W) & (uy < H)
    cx, cy = np.minimum(ux, W - 1), np.minimum(uy, H - 1)
    so = np.asarray(sc["subpixel_offset"], F32)
    px = np.where(inside, ux.astype(F32) + so[cy, cx, 0], ux.astype(F32))
    py = np.where(inside, uy.astype(F32) + so[cy, cx, 1], uy.astype(F32))
    nc = np.where(inside, st["n_contrib"][cy, cx].astype(np.int64), 0)
    dL = np.where(inside[None], np.asarray(sc["dL_dpix"], F32)[:, cy, cx], F32(0))
    if swap is not None:
        dL[:, [swap, swap ^ 1]] = dL[:, [swap ^ 1, swap]]
    r0, r1 = (int(v) for v in st["ranges"][t])
    total = int(min(nc.max(initial=0), r1 - r0))
    ids = st["point_list"][r0:r0 + total].astype(np.int64)
    m = st["means2D"][ids].astype(F32)
    co = st["conic_opacity"][ids].astype(F32)
    col = np.asarray(st["colors"], F32)[ids]
    A, B, C, o = (co[:, c:c + 1] for c in range(4))
    dx = m[:, 0:1] + (-px)[None]
    dy = m[:, 1:2] + (-py)[None]
    power = _fma(_fma(dx, A * dx, dy * (C * dy)), F32(-0.5), dy * ((-B) * dx))
    G = np.exp(power.astype(np.float64)).astype(F32)
    G = np.nextafter(G, np.where(rng.integers(0, 2, G.shape) == 1, F32(np.inf), F32(0)).astype(F32), dtype=F32) \
        if total else G
    a = np.minimum(F32(0.99), o * G)
    act = (np.arange(total)[:, None] < nc[None]) & ~(power > 0) & ~(a < F32(1.0) / F32(255.0))
    alpha = np.where(act, a, F32(0))
    Gm = np.where(act, G, F32(0))
    oma = F32(1) + (-alpha)
    T = np.ones(256, F32)
    for p in range(total):                                     # the forward's test_T (render_fwd.cu:208)
        T = np.where(act[p], T * oma[p], T)
    bg = np.asarray(sc["bg"], F32)
    tb = -T * _fma(bg[2], dL[2], _fma(bg[1], dL[1], bg[0] * dL[0]))
    if no_bg is not None:
        tb[no_bg] = 0
    inv = (1.0 / oma.astype(np.float64)).astype(F32)
    bkz, bkw = np.abs(o) * F32(0.5 * W), np.abs(o) * F32(0.5 * H)
    terms = np.zeros((total, 256, 12), F32)
    rdot = lcd = la = np.zeros(256, F32)
    for p in range(total - 1 - int(skip_last), -1, -1):
        T = T * inv[p]
        aT = alpha[p] * T
        rdot = _fma(la, lcd + (-rdot), rdot)
        cd = _fma(col[p, 2], dL[2], _fma(col[p, 1], dL[1], col[p, 0] * dL[0]))
        lcd, la = cd, alpha[p]
        dLda = _fma(cd + (-rdot), T, tb * inv[p])
        w = Gm[p] * dLda
        wx, wy = w * dx[p], w * dy[p]
        u1 = _fma(A[p], wx, -((-B[p]) * wy))
        u2 = _fma(C[p], wy, -((-B[p]) * wx))
        v2 = _fma(np.abs(u2), bkw[p], np.abs(u1) * bkz[p])
        terms[p] = np.stack([wx, wy, v2, wx * dx[p], wx * dy[p], wy * dy[p], w, aT * dL[0], aT * dL[1], aT * dL[2],
                             u1 * bkz[p], u2 * bkw[p]], axis=1)
    return ids, terms


def _tree_sum(x, rng):
    """fp32 sum of the rows of x along a random binary tree of depth ceil(log2 n)."""
    x = x[rng.permutation(x.shape[0])]
    while x.shape[0] > 1:
        n = x.shape[0] // 2
        s = x[:n] + x[n:2 * n]
        x = np.concatenate([s, x[2 * n:]]) if x.shape[0] % 2 else s
    return x[0]


def emulate(st, sc, rng, tiles=None, mut=None):
    """Accumulator [P, 10] fp32 of the emulated kernel: per (tile, position) a random pair / butterfly tree over each warp's
    64 pixels, the warp rows in random order, the flush conversion (render_bwd.cu:403-409), and the tiles' rows added in a
    random order.  ``mut`` = (kind, tile, position, index) corrupts one step (see test_mutations_are_caught)."""
    P, W, H = st["P"], st["W"], st["H"]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    kind, mt, mp, mi = mut if mut else (None, -1, -1, -1)
    rows = {}
    for t in range(gx * gy):
        if tiles is not None and t in tiles and t != mt:
            ids, terms = tiles[t]
        else:
            ids, terms = emulate_tile(st, sc, t, rng, skip_last=kind == "skip_last" and t == mt,
                                      swap=mi if kind == "swap_dL" and t == mt else None,
                                      no_bg=mi if kind == "no_bg" and t == mt else None)
        for p in range(terms.shape[0]):
            tm = terms[p]
            if not np.any(tm[:, :10]):
                continue
            here = t == mt and p == mp
            if here and kind == "drop_pair":
                tm = tm.copy(); tm[mi] = 0
            if here and kind == "drop_warp":
                tm = tm.copy(); tm[64 * mi:64 * mi + 64] = 0
            ws = [_tree_sum(tm[64 * w:64 * w + 64, :10], rng) for w in range(4)]
            if here and kind == "abs_after_sum":
                blk = tm[64 * mi:64 * mi + 64]
                ws[mi][2] = np.abs(_tree_sum(blk[:, 10:11], rng)[0]) + np.abs(_tree_sum(blk[:, 11:12], rng)[0])
            s = np.zeros(10, F32)
            for w in range(4):                                 # PartRows: warp order
                s = s + ws[w]
            if not np.any(s):
                continue
            g = int(ids[p])
            A, B, C, o = (F32(v) for v in st["conic_opacity"][g])
            A_ = C if here and kind == "C_for_A" else A
            gxv = (-o * F32(0.5 * W)) * _fma(A_, s[0], B * s[1])
            gyv = (-o * F32(0.5 * H)) * _fma(C, s[1], B * s[0])
            h = F32(-0.5) * o
            row = np.array([gxv, gyv, s[2], h * s[3], h * s[4], h * s[5], s[6], s[7], s[8], s[9]], F32)
            if here and kind == "swap34":
                row[[3, 4]] = row[[4, 3]]
            rows.setdefault(g, []).extend([row] * (2 if here and kind == "twice" else 1))
    acc = np.zeros((P, 10), F32)
    for g, rs in rows.items():
        for k in rng.permutation(len(rs)):
            acc[g] = acc[g] + rs[k]
    return acc


def _emulation_case(name):
    from test_adversarial_scenes import scene_one_tile_crowd, scene_posed
    sc = {"small": lambda: synthetic.make_scene(2500, 40, 36, seed=9, subpixel_jitter=0.3, bg=(0.2, 0.5, 0.1)),
          "posed": lambda: scene_posed("precomp", P=3000, W=40, H=36),
          "crowd": lambda: scene_one_tile_crowd(P=1500)}[name]()
    st = cpu_oracle.forward(sc)
    res = bwd_exact.bound(records_of(st), st["colors"], st["point_list"], st["ranges"], st["n_contrib"],
                          sc["subpixel_offset"], sc["bg"], sc["dL_dpix"], st["W"], st["H"])
    return sc, st, res


def _excess(acc, res):
    """Largest |acc - S| / B over all entries (inf where B = 0 and acc != S)."""
    d = np.abs(np.asarray(acc, np.float64) - res["S"])
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0, 0.0, d / res["B"])
    return float(np.nan_to_num(r, nan=0.0, posinf=np.inf).max())


@pytest.mark.parametrize("name", ["small", "posed", "crowd"])
def test_bound_holds_for_an_fp32_emulation_in_random_orders(name):
    sc, st, res = _emulation_case(name)
    assert res["blended_pairs"] > 1000 and res["overflow_pixels"] == 0
    for seed in range(3):
        acc = emulate(st, sc, np.random.default_rng(seed))
        assert np.any(acc)
        e = _excess(acc, res)
        print(f"{name} seed {seed}: worst |emulated - S| / B = {e:.3f}")
        assert e <= 1.0, (name, seed, e)


MUTATIONS = ["drop_pair", "drop_warp", "skip_last", "swap_dL", "abs_after_sum", "no_bg", "C_for_A", "swap34", "twice"]


def _placements(kind, st, tiles, g, res, limit=6):
    """Candidate places for a corruption that touches Gaussian g, the most effective first."""
    out = []
    for t, (ids, terms) in tiles.items():
        hit = np.nonzero(ids == g)[0]
        if kind == "skip_last":
            if terms.shape[0]:
                out.append((0.0, (kind, t, -1, -1)))
            continue
        for p in hit:
            tm = terms[p]
            mag = (np.abs(tm[:, :10]) / np.maximum(res["B"][g], 1e-300)).max(axis=1)
            if kind in ("drop_pair", "swap_dL", "no_bg"):
                for i in np.argsort(-mag)[:limit]:
                    if mag[i] > 0:
                        out.append((mag[i], (kind, t, int(p), int(i))))
            elif kind in ("drop_warp", "abs_after_sum"):
                for w in range(4):
                    out.append((mag[64 * w:64 * w + 64].sum(), (kind, t, int(p), w)))
            else:
                out.append((mag.sum(), (kind, t, int(p), -1)))
    out.sort(key=lambda x: -x[0])
    return [m for _, m in out[:limit]]


@pytest.mark.parametrize("kind", MUTATIONS)
def test_mutations_are_caught(kind):
    """Each corruption of the emulated kernel, placed where it changes the chosen Gaussian most, breaks the bound."""
    sc, st, res = _emulation_case("small")
    gx, gy = (st["W"] + 15) // 16, (st["H"] + 15) // 16
    tiles = {t: emulate_tile(st, sc, t, np.random.default_rng(100 + t)) for t in range(gx * gy)}
    finite = np.all(np.isfinite(res["B"]), axis=1) & (res["und"] == 0)
    g = int(np.argmax(np.where(finite, res["M"][:, 6], -1)))          # the Gaussian with the largest sum |G dL/dalpha|
    best = 0.0
    for mut in _placements(kind, st, tiles, g, res):
        acc = emulate(st, sc, np.random.default_rng(7), tiles=tiles, mut=mut)
        best = max(best, _excess(acc, res))
        if best > 1.0:
            break
    print(f"{kind}: worst |mutated - S| / B = {best:.3g}")
    assert best > 1.0, (kind, best)
