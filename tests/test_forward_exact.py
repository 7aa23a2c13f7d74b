"""Forward composite (csrc/render_fwd.cu, ``render_fwd_packed_kernel<false, false>``) under an fp64 running-error oracle
(``oracle/fwd_exact.py``, ``oracle/fwd_bound.c``): every pixel's colour and final_T is held to an a-priori bound,
n_contrib to its admissible set and the blend masks to the oracle's bits wherever they are sure.  The oracle walks every
list position of every pixel without culling, so a pair the kernel's per-warp culling drops although it blends shows
up as a pixel beyond its bound.

GPU tests (``-m gpu``; no compiled reference needed): the ordinary SMALL scenes, a posed camera with bg != 0, the DENSE
scene (n_contrib beyond MASK_K: the culling alone, no masks); single-tile stacks whose list length sits at the forward's
128-instance rounds (128 r - 1 / 128 r / 128 r + 1), its 32-wide warp batches and mask words and MASK_K +- 1, stacks
that saturate at 128 r - 1 / 128 r / 128 r + 1; a tile where some 8x8 blocks saturate in round 0 while others run many
rounds; opaque stacks at the 0.99 clamp, the faint scene (T = 1 exactly, n_contrib = 0); the image shapes 1x1, 1x37,
17x33 and 4095x3, a tile-row band, the widest strip, kernel_size 0 and 0.1, degenerate splats; and the culling rim:
Gaussians whose largest alpha over a chosen warp block lies within 1e-3 above 1/255 (or just below), centred beyond an
edge or a corner of the block, at rotations and anisotropies on both sides of the preprocess's cdet gate, with sub-pixel
jitter 0 and 0.3 and on edge tiles partly outside the image, and opacities around the negative-extent cut 0.9999/255.

CPU tests: with px and power in fp64 the oracle's value is oracle.c's fp64 composite; the oracle's fp32 power is
oracle.c's fp32 power bit for bit; oracle.c's fp32 composite is an admissible execution; a numpy fp32 emulation of the
kernel -- per-warp culling included, expf perturbed within 2 ulp, the epilogue contracted at random -- stays within the
bound; and ten corruptions of that emulation are each caught.

The measured worst |kernel - S| / B per family and the undetermined counts are in DESIGN.md (3.1, numerics note).
"""
import math

import numpy as np
import pytest
import torch

import synthetic
from oracle import cpu_oracle, fwd_exact
from test_backward_exact import _fma as _fma32, _tile_pixels, records_of, scene_stack

K = fwd_exact.MASK_K
UND_SHARE = 2e-3          # most pixels with an undetermined decision a scene may have
CAUGHT = 10.0             # a corruption is caught when some output is this many bounds away (or leaves its set)
F32 = np.float32
AMIN = F32(1.0) / F32(255.0)


# ======================================================================================================================
# scenes
# ======================================================================================================================
def _flat_scene(W, H, u, v, z, sig1, sig2, theta, opac, colors, seed=0, jitter=0.0, bg=(0.1, 0.3, 0.2), ks=0.1):
    """A scene of flat Gaussians under the identity camera of synthetic.make_camera: Gaussian i projects to pixel
    (u_i, v_i) with a 2D covariance R(theta_i) diag(sig1_i^2, sig2_i^2) R(theta_i)^T (+ kernel_size)."""
    cam = synthetic.make_camera(W, H)
    f = 0.9 * W
    u, v, z = (np.asarray(a, np.float64) for a in (u, v, z))
    x = (u - (W - 1) / 2.0) * z / f
    y = (v - (H - 1) / 2.0) * z / f
    P = u.size
    s = np.stack([np.asarray(sig1) * z / f, np.asarray(sig2) * z / f, np.full(P, 1e-7)], 1)
    th = np.asarray(theta, np.float64)
    rot = np.stack([np.cos(th / 2), np.zeros(P), np.zeros(P), np.sin(th / 2)], 1)
    g = torch.Generator().manual_seed(seed + 900)
    scene = dict(cam)
    scene.update(image_width=int(W), image_height=int(H), kernel_size=float(ks), scale_modifier=1.0, prefiltered=False,
                 debug=False, means3D=torch.tensor(np.stack([x, y, z], 1), dtype=torch.float32),
                 scales=torch.tensor(s, dtype=torch.float32), rotations=torch.tensor(rot, dtype=torch.float32),
                 opacities=torch.tensor(np.asarray(opac, np.float64).reshape(P, 1), dtype=torch.float32),
                 colors_precomp=torch.tensor(np.asarray(colors, np.float64).reshape(P, 3), dtype=torch.float32),
                 sh_degree=0, bg=torch.tensor(bg, dtype=torch.float32))
    if jitter > 0:
        scene["subpixel_offset"] = ((torch.rand(H, W, 2, generator=g) - 0.5) * 2 * jitter).float().contiguous()
    else:
        scene["subpixel_offset"] = torch.zeros((H, W, 2), dtype=torch.float32)
    scene["dL_dpix"] = torch.zeros((3, H, W), dtype=torch.float32)
    return scene


def saturating_opacity(s):
    """Alpha a with (1 - a)^s > 1e-4 > (1 - a)^(s + 1): a stack of such splats saturates at list position s."""
    return 1.0 - 1e-4 ** (1.0 / (s + 0.5))


def scene_early_out(seed=311):
    """Four tiles in a row.  Block 0 of tile 0: two copies of a sharp opaque splat on every pixel (list positions 0..127),
    so its pixels saturate inside round 0 while the other blocks of the tile walk a faint 700-deep stack; tile 3 under
    twenty wide opaque splats saturates everywhere in round 0 (the block-wide vote)."""
    W, H = 64, 16
    g = np.random.default_rng(seed)
    us, vs, zs, s1, s2, th, op, col = [], [], [], [], [], [], [], []
    for c in range(2):                                       # sharp splats on block 0 of tile 0, front
        for y in range(8):
            for x in range(8):
                us.append(x); vs.append(y); zs.append(2.0 + 0.01 * c); s1.append(1.5); s2.append(1.5); th.append(0.0)
                op.append(0.999); col.append(g.uniform(0, 1, 3))
    for c in range(20):                                      # wide opaque splats over tile 3
        us.append(55.5); vs.append(7.5); zs.append(2.5 + 0.01 * c); s1.append(14.0); s2.append(12.0); th.append(0.3)
        op.append(0.999); col.append(g.uniform(0, 1, 3))
    for i in range(700):                                     # faint wide stack everywhere
        us.append(g.uniform(0, 64)); vs.append(g.uniform(0, 16)); zs.append(3.0 + 0.001 * i); s1.append(200.0)
        s2.append(150.0); th.append(g.uniform(0, 3)); op.append(0.006); col.append(g.uniform(0, 1, 3))
    return _flat_scene(W, H, us, vs, zs, s1, s2, th, op, col, seed=seed)


# ---- the culling rim ---------------------------------------------------------------------------------------------------
RIM_ROT = [0.0, 1e-3, math.pi / 8, math.pi / 4, 3 * math.pi / 8, math.pi / 2 - 1e-3]
# (long-axis sigma in pixels, ratio of the effective 2D eigenvalues): the last three straddle the cdet gate at 45 degrees
RIM_ANISO = [(4.0, 1.0), (7.0, 4.0), (12.0, 30.0), (40.0, 2000.0), (40.0, 8000.0), (40.0, 16000.0)]
RIM_Q0 = [2.0, 3.0, 4.0]
RIM_SIDES = ["left", "right", "top", "bottom", "tl", "tr", "bl", "br"]


def _block_samples(W, H, so, tx, ty, b):
    """fp32 sample positions (ux + so.x, uy + so.y) of the inside pixels of 8x8 block b of tile (tx, ty)."""
    x0, y0 = tx * 16 + 8 * (b % 2), ty * 16 + 8 * (b // 2)
    ys, xs = np.mgrid[y0:min(y0 + 8, H), x0:min(x0 + 8, W)]
    xs, ys = xs.ravel(), ys.ravel()
    return xs, ys, xs.astype(F32) + so[ys, xs, 0], ys.astype(F32) + so[ys, xs, 1]


def power32(x, y, A, B, C, px, py):
    """The kernel's fp32 power (render_fwd.cu:201-205)."""
    x, y, A, B, C = (F32(v) for v in (x, y, A, B, C))
    dx = x + (-np.asarray(px, F32))
    dy = y + (-np.asarray(py, F32))
    t1 = A * dx
    t3 = dy * (C * dy)
    un = dy * ((-B) * dx)
    return _fma32(_fma32(dx, t1, t3), F32(-0.5), un)


def rim_targets(W, H, so, seed, n_max=90):
    """Designed rim Gaussians: for a spread of warp blocks, a centre beyond an edge or a corner of the block at which
    q = d^T Sigma^-1 d reaches q0 exactly on the block's extreme sample, with the block on the far side of the tangent
    line.  Returns a list of dicts (block, centre, Sigma (effective 2D covariance), q0, kind, ...)."""
    g = np.random.default_rng(seed)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    blocks = [(tx, ty, b) for ty in range(gy) for tx in range(gx) for b in range(4)
              if tx * 16 + 8 * (b % 2) < W and ty * 16 + 8 * (b // 2) < H]
    g.shuffle(blocks)
    out = []
    for i, (tx, ty, b) in enumerate(blocks[:n_max]):
        side = RIM_SIDES[i % len(RIM_SIDES)]
        th = RIM_ROT[(i // len(RIM_SIDES)) % len(RIM_ROT)]
        sig, ratio = RIM_ANISO[(i // 3) % len(RIM_ANISO)]
        q0 = RIM_Q0[i % len(RIM_Q0)]
        l1 = sig * sig
        l2 = max(l1 / ratio, 0.1)
        c, s = math.cos(th), math.sin(th)
        R = np.array([[c, -s], [s, c]])
        Sig = R @ np.diag([l1, l2]) @ R.T
        xs, ys, px, py = _block_samples(W, H, so, tx, ty, b)
        if side in ("left", "right", "top", "bottom"):
            key = {"left": px, "right": -px, "top": py, "bottom": -py}[side]
            j = int(g.choice(np.flatnonzero(key == key.min())))       # without jitter: any sample of the edge
            n = {"left": (1, 0), "right": (-1, 0), "top": (0, 1), "bottom": (0, -1)}[side]
        else:
            sx = 1 if side[1] == "l" else -1
            sy = 1 if side[0] == "t" else -1
            j = int(np.argmin(sx * px.astype(np.float64) + sy * py.astype(np.float64)))
            phi = g.uniform(0.3, 1.27)
            n = (sx * math.cos(phi), sy * math.sin(phi))
        n = np.array(n, np.float64)
        lam = math.sqrt(q0 / float(n @ Sig @ n))
        d = lam * (Sig @ n)
        centre = np.array([float(px[j]), float(py[j])]) - d
        out.append(dict(tile=ty * gx + tx, tx=tx, ty=ty, block=b, side=side, theta=th, sig=sig, ratio=ratio, q0=q0,
                        Sigma=Sig, l1=l1, l2=l2, centre=centre, sample=(int(xs[j]), int(ys[j]))))
    return out


def rim_opacity(rec, W, H, so, t, rel):
    """Opacity o (fp32) at which the largest alpha of record rec over the target block is AMIN * (1 + rel), and the
    largest fp32 power there."""
    xs, ys, px, py = _block_samples(W, H, so, t["tx"], t["ty"], t["block"])
    pw = power32(rec[0], rec[1], rec[4], rec[5], rec[6], px, py)
    pmax = float(pw.max())
    return float(AMIN) * (1.0 + rel) / math.exp(pmax), pmax


RIM_REL = (4e-4, -4e-4)   # designed largest alpha over the target block: AMIN (1 + rel), above and (mirror) below


def rim_plan(W, H, so, seed):
    """The rim targets and, per target, which side of 1/255 it is designed on; every fifth target is a mirror case."""
    ts = rim_targets(W, H, so, seed)
    for i, t in enumerate(ts):
        t["rel"] = RIM_REL[1] if i % 5 == 4 else RIM_REL[0]
        t["color"] = 0.9 + 0.1 * ((i * 37) % 11) / 10.0
    return ts


def scene_rim(jitter, seed=401, W=150, H=120, n_back=3000):
    """GPU rim family: the designed rim Gaussians in front (depth order = target order), opacities solved on the
    preprocessed records (cpu_oracle's preprocess gives the kernel's bits, test_gpu_parity pins that), a few
    opacities at the negative-extent cut 0.9999/255, and an ordinary cloud behind."""
    so_t = ((torch.rand(H, W, 2, generator=torch.Generator().manual_seed(seed)) - 0.5) * 2 * jitter).float() \
        if jitter > 0 else torch.zeros((H, W, 2))
    so = so_t.numpy()
    ts = rim_plan(W, H, so, seed)
    g = np.random.default_rng(seed)
    n = len(ts)
    u = [t["centre"][0] for t in ts]; v = [t["centre"][1] for t in ts]
    z = [2.0 + 0.01 * i for i in range(n)]
    s1, s2, th = [], [], []
    for t in ts:
        # projected minor variance at least 1e-3: the low-pass filter's opacity compensation (det_0 > 1e-6) stays non-zero
        s1.append(math.sqrt(t["l1"] - 0.1)); s2.append(math.sqrt(max(t["l2"] - 0.1, 1e-3))); th.append(t["theta"])
    # negative-extent cut: splats centred inside a block with o*coef just below / at / above 0.9999/255 and at 1/255 (1 + 1e-5)
    cuts = [0.9999 / 255 * (1 - 1e-5), 0.9999 / 255 * (1 + 1e-5), float(AMIN) * (1 + 1e-5)] * 4
    for k, _ in enumerate(cuts):
        u.append(g.uniform(4, W - 4)); v.append(g.uniform(4, H - 4)); z.append(1.5 + 0.01 * k)
        s1.append(3.0); s2.append(2.0); th.append(g.uniform(0, 3))
    # ordinary cloud behind
    for _ in range(n_back):
        u.append(g.uniform(-10, W + 10)); v.append(g.uniform(-10, H + 10)); z.append(g.uniform(4.0, 8.0))
        s1.append(g.uniform(0.5, 4.0)); s2.append(g.uniform(0.5, 4.0)); th.append(g.uniform(0, 3))
    P = len(u)
    col = g.uniform(0, 1, (P, 3))
    col[:n] = np.array([t["color"] for t in ts])[:, None] * np.array([1.0, 0.97, 0.94])
    op = np.concatenate([np.ones(n + len(cuts)), g.uniform(0.05, 0.6, n_back)])
    sc = _flat_scene(W, H, u, v, z, s1, s2, th, op, col, seed=seed)
    sc["subpixel_offset"] = so_t.float().contiguous()
    st = cpu_oracle.forward(sc, stages=("preprocess",))
    coef = st["conic_opacity"][:, 3].astype(np.float64)            # o * coef with o = 1
    rec = records_of(st)
    for i, t in enumerate(ts):
        o, _ = rim_opacity(rec[i], W, H, so, t, t["rel"])
        op[i] = o / coef[i]
    for k, c in enumerate(cuts):
        op[n + k] = c / coef[n + k]
    # fp32 opacity: the product fl(o coef) lands within a few ulp of the designed value, far inside the 1e-3 band
    sc["opacities"] = torch.tensor(op.reshape(P, 1), dtype=torch.float32)
    return sc, ts, n, len(cuts)


# ======================================================================================================================
# GPU helpers
# ======================================================================================================================
def _run(scene, shard=None):
    """Forward through the C ABI.  Returns the kernel's outputs and the oracle's inputs."""
    from diff_gaussian_rasterization import _C
    from make_golden import call_args
    from test_blend_masks import masks_of
    d = synthetic.to_device(scene, torch.device("cuda:0"))
    W, H = d["image_width"], d["image_height"]
    P = d["means3D"].shape[0]
    M = d["shs"].shape[1] if "shs" in d else 0
    _C.set_geometry_cache(False)
    if shard is not None:
        _C.set_tile_row_shard(*shard)
    try:
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(*call_args(d))
        v = _C.debug_views(geom, binning, img, P, M, W, H, R)
        torch.cuda.synchronize()
        masks = masks_of(v, img, W, H)
        out = dict(color=color.cpu().numpy(), final_T=v["final_T"].cpu().numpy(),
                   n_contrib=v["n_contrib"].cpu().numpy().astype(np.int64), masks=masks, R=R)
        colors = v["rgb"] if M > 0 else d["colors_precomp"]
        ins = dict(records=v["records"].cpu().numpy(), colors=colors.cpu().numpy(),
                   point_list=v["point_list"].cpu().numpy(), ranges=v["ranges"].cpu().numpy(),
                   subpixel_offset=d["subpixel_offset"].cpu().numpy(), bg=d["bg"].cpu().numpy(), W=W, H=H)
    finally:
        _C.set_geometry_cache(True)
        if shard is not None:
            _C.set_tile_row_shard(0, 0)
    return out, ins


def _assert_within(name, out, res, und_share=UND_SHARE, masks=True):
    c = fwd_exact.check(res, out["color"], out["final_T"], out["n_contrib"], out["masks"] if masks else None)
    y0, y1 = fwd_exact.band_rows(res)
    npx = (y1 - y0) * res["W"]
    n_und = int((res["und"][y0:y1] > 0).sum())
    worst = ", ".join(f"{k} {v:.2e}" for k, v in c["ratio"].items())
    mk = f"; mask bits compared {c['mask_compared']}, unsure {c['mask_unsure']}" if masks else ""
    print(f"{name}: pixels {npx} blended pairs {res['blended_pairs']} undetermined pixels {n_und} "
          f"({n_und / max(npx, 1):.1e}) infinite {res['overflow_pixels']}; worst |kernel - S|/B: {worst}; "
          f"determined only: {max(c['ratio_det'].values()):.2e}{mk}")
    assert c["violations"].size == 0, (name, "pixels beyond their bound", c["violations"][:10].tolist())
    assert c["nc_outside"].size == 0, (name, "n_contrib not admissible (the nominal value where determined)",
                                       c["nc_outside"][:10].tolist())
    if masks:
        assert len(c["mask_differ"]) == 0, (name, "sure mask bits differ", c["mask_differ"][:10].tolist())
    if und_share is not None:
        assert n_und <= max(2, und_share * npx), (name, "undetermined pixels", n_und)
    return c


def _check_scene(name, scene, shard=None, und_share=UND_SHARE, masks=True):
    out, ins = _run(scene, shard)
    res = fwd_exact.bound(**ins, tile_rows=shard or (0, 0), n_contrib=out["n_contrib"])
    c = _assert_within(name, out, res, und_share=und_share, masks=masks)
    return out, ins, res, c


# ======================================================================================================================
# GPU tests
# ======================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small_320x240", "small_300x200_jitter", "posed_bg"])
def test_ordinary_scenes(name):
    from test_backward_exact import ordinary_scenes
    out, ins, res, c = _check_scene(name, ordinary_scenes()[name])
    assert res["blended_pairs"] > 100_000 and c["mask_compared"] > 10_000


@pytest.mark.gpu
def test_dense_beyond_mask_k():
    from test_blend_masks import DENSE, DENSE_OPACITY, _scene
    out, ins, res, c = _check_scene("dense", _scene(DENSE, DENSE_OPACITY))
    assert int(out["n_contrib"].max()) > K + 128, "scene does not reach the positions beyond MASK_K"


# list lengths at the forward's 128-instance rounds, its 32-wide warp batches / mask words, and MASK_K +- 1; every
# pixel's n_contrib equals the list length
STACKS = [1, 31, 32, 33, 64, 96, 127, 128, 129, 255, 256, 257, 383, 384, 385, K - 1, K, K + 1]


@pytest.mark.gpu
@pytest.mark.parametrize("n", STACKS)
def test_list_position_boundaries(n):
    out, ins, res, c = _check_scene(f"stack_{n}", scene_stack(n))
    nc = out["n_contrib"]
    assert int(nc.max()) == n and int(nc.min()) == n, (n, int(nc.min()), int(nc.max()))
    assert int(np.diff(ins["ranges"][0])[0]) == n


SATURATE = [127, 128, 129, 255, 256, 257]


@pytest.mark.gpu
@pytest.mark.parametrize("s", SATURATE)
def test_saturation_at_round_boundaries(s):
    """A stack of 400 splats that saturates (T (1 - alpha) < 1e-4) at list position s: n_contrib = s in the pixels."""
    out, ins, res, c = _check_scene(f"saturate_{s}", scene_stack(400, seed=321, opacity=saturating_opacity(s) / 1.01))
    nc = out["n_contrib"]
    assert (out["final_T"] < 2e-4).all() and int(nc.max()) < 400
    assert abs(int(np.median(nc)) - s) <= 1 and int((nc == s).sum()) > 0, (s, np.unique(nc))


@pytest.mark.gpu
def test_early_out_blocks():
    # identical stacked copies give whole groups of pixels the same T sequence, so one near-threshold stop test is
    # undetermined in several pixels at once: a wider cap than the ordinary scenes'
    out, ins, res, c = _check_scene("early_out", scene_early_out(), und_share=1e-2)
    nc, T = out["n_contrib"], out["final_T"]
    # the faint stack blends in every pixel, so n_contrib < 128 means the stop test ended the walk in round 0
    assert (nc[:8, :8] < 128).all(), "block 0 does not saturate in round 0"
    assert (nc[10:, :16] > 512).all(), "blocks 2 and 3 of tile 0 do not run many rounds"
    assert (nc[:, 48:] < 128).all(), "tile 3 does not saturate in round 0"
    assert (T[:8, :8] < 1e-2).all() and (T[:, 48:] < 1e-2).all()


@pytest.mark.gpu
def test_opaque_stacks_at_the_clamp():
    from test_adversarial_scenes import scene_opaque
    out, ins, res, c = _check_scene("opaque", scene_opaque())
    assert (ins["records"][:, 7] >= 0.99).sum() > 100
    W, H = ins["W"], ins["H"]
    lens = np.diff(ins["ranges"].astype(np.int64), axis=1).reshape((H + 15) // 16, (W + 15) // 16)
    lens = lens.repeat(16, 0).repeat(16, 1)[:H, :W]
    assert ((out["final_T"] < 1e-3) & (out["n_contrib"] < lens)).mean() > 0.3, "too few pixels saturate"


@pytest.mark.gpu
def test_faint_scene():
    from test_adversarial_scenes import scene_faint
    out, ins, res, c = _check_scene("faint", scene_faint(), und_share=None)
    assert res["blended_pairs"] == 0 and not np.any(out["n_contrib"])
    assert np.all(out["final_T"] == 1.0) and not np.any(res["B"])       # T = 1 exactly: bound 0, exact agreement


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", [(1, 1), (1, 37), (17, 33), (4095, 3)])
def test_image_shapes(W, H):
    from test_adversarial_scenes import scene_shape
    _check_scene(f"shape_{W}x{H}", scene_shape(W, H))


@pytest.mark.gpu
def test_tile_row_band():
    from test_blend_masks import SMALL, _scene
    out, ins, res, c = _check_scene("band_3_9", _scene(SMALL[0]), shard=(3, 9))
    assert res["blended_pairs"] > 10_000


@pytest.mark.gpu
def test_widest_strip():
    from test_adversarial_scenes import scene_widest_strip
    out, ins, res, c = _check_scene("widest_strip", scene_widest_strip())
    rg = ins["ranges"]
    assert rg.shape[0] == 65535 and int(rg[-1, 1] - rg[-1, 0]) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("ks", [0.0, 0.1])
def test_kernel_size(ks):
    from test_adversarial_scenes import scene_settings
    _check_scene(f"kernel_size_{ks}", scene_settings(ks, 1.0))


@pytest.mark.gpu
@pytest.mark.parametrize("ks", [0.0, 0.1])
def test_degenerate_splats(ks):
    from test_adversarial_scenes import scene_degenerate
    out, ins, res, c = _check_scene(f"degenerate_{ks}", scene_degenerate(ks))
    rec = ins["records"]
    if ks == 0.0:
        assert int((rec[:, 2] >= 1e29).sum()) > 100, "no splat reaches the cdet gate"


def rim_reach(ins, res, ts, jitter):
    """Where the designed rim pairs landed: per target, the largest oracle alpha over the block relative to 1/255, whether
    it is determined, where its sample lies on the warp box, and which side of the cdet gate the record is."""
    W, H = ins["W"], ins["H"]
    so = np.asarray(ins["subpixel_offset"], F32).reshape(H, W, 2)
    rows = []
    for i, t in enumerate(ts):
        rec = np.asarray(ins["records"][i], np.float64)
        xs, ys, px, py = _block_samples(W, H, so, t["tx"], t["ty"], t["block"])
        pw = power32(rec[0], rec[1], rec[4], rec[5], rec[6], px, py).astype(np.float64)
        a = np.minimum(0.99, rec[7] * np.exp(pw))
        j = int(np.argmax(a))
        rel = a[j] / float(AMIN) - 1.0
        corner = px[j] in (px.min(), px.max()) and py[j] in (py.min(), py.max())
        edge = px[j] in (px.min(), px.max()) or py[j] in (py.min(), py.max())
        cdet = rec[4] * rec[6] - rec[5] * rec[5]
        rows.append(dict(rel=rel, det=abs(rel) > 1e-5 and pw[j] <= 0, corner=corner, edge=edge,
                         gate_off=not cdet > 1e-3 * rec[4] * rec[6], box=rec[2], q=-2 * pw[j],
                         L=2 * math.log(255 * rec[7]), sample=(int(xs[j]), int(ys[j]))))
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize("jitter", [0.0, 0.3])
def test_culling_rim(jitter):
    sc, ts, n, n_cut = scene_rim(jitter)
    out, ins, res, c = _check_scene(f"rim_{jitter}", sc)
    rows = rim_reach(ins, res, ts, jitter)
    above = [r for r, t in zip(rows, ts) if t["rel"] > 0]
    assert all(1e-5 < r["rel"] < 1e-3 and r["det"] for r in above), "a rim pair left the band above 1/255"
    below = [r for r, t in zip(rows, ts) if t["rel"] < 0]
    assert below and all(-1e-3 < r["rel"] < -1e-5 for r in below)
    assert sum(r["edge"] for r in above) >= 30
    if jitter == 0.0:
        assert sum(r["corner"] for r in above) >= 15, "too few rim samples at a corner of the warp box"
    assert sum(r["gate_off"] for r in above) >= 3 and sum(not r["gate_off"] for r in above) >= 30, "cdet gate: one side"
    assert sum(r["box"] < 1e29 and r["box"] >= 6.0 for r in above) >= 10, "too few tight boxes"
    # every rim Gaussian is in its target tile's list (so the culling saw it there), some on tiles partly outside the image
    W, H = ins["W"], ins["H"]
    for i, t in enumerate(ts):
        r0, r1 = (int(v) for v in ins["ranges"][t["tile"]])
        assert i in ins["point_list"][r0:r1], ("rim Gaussian not binned to its target tile", i, t["tile"])
    partial = [t for t in ts if t["rel"] > 0 and (16 * t["tx"] + 16 > W or 16 * t["ty"] + 16 > H)]
    assert len(partial) >= 5, "too few rim targets on tiles partly outside the image"
    # negative-extent cut: records with o below 0.9999/255 carry negative extents, the others keep theirs
    cut = ins["records"][n:n + n_cut]
    assert (cut[:, 2] < 0).sum() >= 4 and (cut[:, 2] > 0).sum() >= 8


# ======================================================================================================================
# CPU tests
# ======================================================================================================================
def cpu_cases():
    from test_adversarial_scenes import scene_guard_band, scene_posed
    return {"small": synthetic.make_scene(2000, 64, 48, seed=5, subpixel_jitter=0.3, bg=(0.2, 0.5, 0.1)),
            "posed": scene_posed("precomp", P=3000, W=70, H=50),
            "guard_band": scene_guard_band(P=3000, W=70, H=50),
            "opaque": {**synthetic.make_scene(1500, 48, 32, seed=6, subpixel_jitter=0.3, bg=(0.3, 0.1, 0.6),
                                              scale_range=(0.02, 0.1)), "opacities": torch.full((1500, 1), 0.999)}}


@pytest.mark.parametrize("name", ["small", "posed", "guard_band", "opaque"])
def test_oracle_value_is_the_fp64_composite(name):
    """With px and power in fp64 (and the fp64 constants), S equals oracle.c's fp64 composite to 1e-12 of each channel's
    magnitude, and the nominal n_contrib is its n_contrib."""
    sc = cpu_cases()[name]
    st = cpu_oracle.forward(sc, np.float64)
    res = fwd_exact.bound(records_of(st), st["colors"], st["point_list"], st["ranges"], sc["subpixel_offset"], sc["bg"],
                          st["W"], st["H"], alpha_max=0.99, alpha_min=1.0 / 255.0, t_min=1e-4, debug_f64=True)
    assert res["blended_pairs"] > 1000
    want = np.concatenate([st["out_color"], st["final_T"][None]])
    for ch in range(4):
        scale = float(np.abs(want[ch]).max()) + 1e-300
        assert float(np.abs(res["S"][ch] - want[ch]).max()) <= 1e-12 * scale, (name, ch)
    assert np.array_equal(res["nc_nom"], st["n_contrib"])


def all_pairs(st):
    """Every (list position, pixel) pair of every tile of a CPU-oracle forward: Gaussian ids and pixel coordinates."""
    W, H = st["W"], st["H"]
    gx = (W + 15) // 16
    g, ux, uy = [], [], []
    for t in range(st["ranges"].shape[0]):
        r0, r1 = (int(v) for v in st["ranges"][t])
        if r1 == r0:
            continue
        tx, ty = t % gx, t // gx
        ys, xs = np.mgrid[ty * 16:min(ty * 16 + 16, H), tx * 16:min(tx * 16 + 16, W)]
        ids = st["point_list"][r0:r1].astype(np.int64)
        g.append(np.repeat(ids, xs.size)); ux.append(np.tile(xs.ravel(), ids.size)); uy.append(np.tile(ys.ravel(), ids.size))
    return np.concatenate(g), np.concatenate(ux), np.concatenate(uy)


@pytest.mark.parametrize("name", ["small", "posed", "guard_band", "opaque"])
def test_fp32_power_is_oracle_c_power(name):
    """The fp32 power the oracle walks with (fwd_bound.c, render_fwd.cu:201-205: fma(fma(dx, A dx, dy (C dy)), -0.5,
    dy ((-B) dx))) and oracle.c's fp32 pair_power (the reference's contraction, fma(fma(A dx, dx, (C dy) dy), -0.5,
    -(B dx) dy)), both computed by their own libraries from the records, the pixel and its sub-pixel offset: the same
    bits on every pair of every pixel."""
    sc = cpu_cases()[name]
    st = cpu_oracle.forward(sc)
    g, ux, uy = all_pairs(st)
    so = np.asarray(sc["subpixel_offset"], F32).reshape(st["H"], st["W"], 2)[uy, ux]
    theirs = cpu_oracle.pair_power(st["means2D"], st["conic_opacity"], g, ux, uy, so)
    ours = fwd_exact.pair_power(records_of(st), g, ux, uy, so)
    differ = np.flatnonzero(theirs.view(np.uint32) != ours.view(np.uint32))
    assert differ.size == 0, (name, differ.size, "pairs differ, first", differ[:5].tolist())
    # pairs at every scale of the exponent, the blending range (power in [-2 ln 255, 0]) well covered
    assert g.size > 100_000 and int(((ours <= 0) & (ours > -11.1)).sum()) > 10_000


@pytest.mark.parametrize("name", ["small", "posed", "guard_band", "opaque"])
def test_oracle_c_fp32_composite_is_admissible(name):
    """oracle.c's fp32 composite (glibc expf, within 1 ulp; the epilogue contracted) is one execution the bound admits:
    image and final_T within B, n_contrib in its set."""
    sc = cpu_cases()[name]
    st = cpu_oracle.forward(sc)
    res = fwd_exact.bound(records_of(st), st["colors"], st["point_list"], st["ranges"], sc["subpixel_offset"], sc["bg"],
                          st["W"], st["H"], n_contrib=st["n_contrib"])
    c = fwd_exact.check(res, st["out_color"], st["final_T"], st["n_contrib"])
    print(name, {k: f"{v:.3f}" for k, v in c["ratio"].items()}, "undetermined pixels", res["undetermined_pixels"])
    assert c["violations"].size == 0 and c["nc_outside"].size == 0
    assert res["overflow_pixels"] == 0


# ---- numpy fp32 emulation of render_fwd_packed_kernel<false, false> ----------------------------------------------------
def box_may_touch(g, box, shrink=1.0):
    x, y, hx, hy = (F32(v) for v in g[:4])
    hx, hy = F32(hx * F32(shrink)), F32(hy * F32(shrink))
    x0, x1, y0, y1 = box
    return ~((hx < 0) | (x + hx < x0) | (x - hx > x1) | (y + hy < y0) | (y - hy > y1))


def ellipse_may_touch(g, box, lower=0.0):
    """render_common.cuh:63-75 in fp32 as written in the source: each product and sum rounded on its own (nvcc's default
    contraction may fuse some of them) and numpy's float32 log for __logf.  Both differences are a few ulp, far below
    the test's own margins (1e-3 of the term magnitudes, 2e-3 on the bound), so the emulation culls the same pairs
    except within those ulps of its margins."""
    x, y, A, B, C, o = (F32(v) for v in (g[0], g[1], g[4], g[5], g[6], g[7]))
    x0, x1, y0, y1 = box
    u0, u1, v0, v1 = x - x1, x - x0, y - y1, y - y0
    inside = (u0 <= 0) & (u1 >= 0) & (v0 <= 0) & (v1 >= 0)
    if not (A > 0 and C > 0):
        return np.ones_like(inside)
    rA, rC = F32(1) / A, F32(1) / C

    def q_lo(u, v):
        a, c, m = A * u * u, C * v * v, F32(2) * B * u * v
        return (a + c + m) - F32(1e-3) * (a + c + np.abs(m))

    cl = lambda t, lo, hi: np.minimum(np.maximum(t, lo), hi)
    q = np.minimum(np.minimum(q_lo(u0, cl(-B * u0 * rC, v0, v1)), q_lo(u1, cl(-B * u1 * rC, v0, v1))),
                   np.minimum(q_lo(cl(-B * v0 * rA, u0, u1), v0), q_lo(cl(-B * v1 * rA, u0, u1), v1)))
    with np.errstate(divide="ignore", invalid="ignore"):
        L = F32(2) * np.log(F32(255) * o).astype(F32) + F32(2e-3) - F32(lower)
    return inside | ~(q > L)


def emulate(case, rng, mut=None):
    """The kernel's outputs, emulated in numpy fp32: out_color [3, H, W], final_T, n_contrib [H, W] and the blend masks
    [T, 4, 32].  expf is perturbed at random within +-2 ulp (expf(0) = 1 exactly), the epilogue contracted or not at
    random.  ``mut`` corrupts one step: "cull" = (tile, warp, position) culled although it blends, "le" (<= in the stop
    test), "T_on_stop", "zero_based", "no_subpixel", "no_bg", "prev_round" (the previous round's record at a round's
    first position), "tested_bit" (a mask bit for every pair the culling kept), "ellipse_low" (the ellipse bound lowered
    by 0.01), "box_shrink" (the box extents shrunk by 1 %)."""
    rec, col, pl, rg = case["records"], case["colors"], case["point_list"], case["ranges"]
    W, H = case["W"], case["H"]
    so = np.asarray(case["subpixel_offset"], F32).reshape(H, W, 2)
    bg = np.asarray(case["bg"], F32)
    kind = mut[0] if mut else None
    gx, gy = (W + 15) // 16, (H + 15) // 16
    out = np.zeros((3, H, W), F32)
    fT = np.ones((H, W), F32)
    ncon = np.zeros((H, W), np.int64)
    masks = np.zeros((gx * gy, 4, 32), np.uint32)
    rec32 = np.asarray(rec, F32)
    col32 = np.asarray(col, F32)
    for t in range(gx * gy):
        ux, uy = _tile_pixels(t % gx, t // gx)
        inside = (ux < W) & (uy < H)
        cx, cy = np.minimum(ux, W - 1), np.minimum(uy, H - 1)
        px, py = ux.astype(F32), uy.astype(F32)
        if kind != "no_subpixel":
            px = np.where(inside, px + so[cy, cx, 0], px)
            py = np.where(inside, py + so[cy, cx, 1], py)
        boxes = []
        for w in range(4):
            m = inside[64 * w:64 * w + 64]
            if m.any():
                boxes.append((px[64 * w:64 * w + 64][m].min(), px[64 * w:64 * w + 64][m].max(),
                              py[64 * w:64 * w + 64][m].min(), py[64 * w:64 * w + 64][m].max()))
            else:
                boxes.append((F32(3e38), F32(-3e38), F32(3e38), F32(-3e38)))
        r0, r1 = (int(v) for v in rg[t])
        live = inside.copy()
        T = np.ones(256, F32)
        C = np.zeros((3, 256), F32)
        last = np.zeros(256, np.int64)
        for p in range(r1 - r0):
            if not live.any():
                break
            src = p - 128 if (kind == "prev_round" and p >= 128 and p % 128 == 0) else p
            g = int(pl[r0 + src])
            G = rec32[g]
            rel = np.zeros(256, bool)
            for w in range(4):
                keep = bool(box_may_touch(G, boxes[w], 0.99 if kind == "box_shrink" else 1.0)) and \
                    bool(ellipse_may_touch(G, boxes[w], 0.01 if kind == "ellipse_low" else 0.0))
                if kind == "cull" and (t, w, p) == mut[1]:
                    keep = False
                rel[64 * w:64 * w + 64] = keep
            if not rel.any():
                continue
            pw = power32(G[0], G[1], G[4], G[5], G[6], px, py)
            with np.errstate(over="ignore", invalid="ignore"):
                e = np.exp(pw.astype(np.float64)).astype(F32)
                steps = rng.integers(-2, 3, 256)
                for s_ in (1, 2):
                    up = steps >= s_
                    dn = steps <= -s_
                    e = np.where(up, np.nextafter(e, F32(np.inf)), np.where(dn, np.nextafter(e, F32(0)), e))
                e = np.where(pw == 0, F32(1), e)
                oG = G[7] * e
                a = np.where(np.isnan(oG), F32(0.99), np.minimum(F32(0.99), oG))
                test_T = T * (F32(1) + (-a))
            blend = live & rel & ~(pw > 0) & ~(a < AMIN)
            stop = blend & ((test_T <= F32(1e-4)) if kind == "le" else (test_T < F32(1e-4)))
            live &= ~stop
            upd = blend & ~stop
            if kind == "T_on_stop":
                T = np.where(stop, test_T, T)
            for ch in range(3):
                C[ch] = np.where(upd, _fma32(T, a * col32[g, ch], C[ch]), C[ch])
            T = np.where(upd, test_T, T)
            last = np.where(upd, p if kind == "zero_based" else p + 1, last)
            if p < K:
                for w in range(4):
                    hit = (rel & live | rel & stop)[64 * w:64 * w + 64].any() if kind == "tested_bit" else \
                        upd[64 * w:64 * w + 64].any()
                    if hit:
                        masks[t, w, p // 32] |= np.uint32(1) << np.uint32(p % 32)
        contract = rng.integers(0, 2, 256).astype(bool)
        for ch in range(3):
            if kind == "no_bg":
                o_ = C[ch]
            else:
                o_ = np.where(contract, _fma32(T, bg[ch], C[ch]), C[ch] + T * bg[ch])
            out[ch, uy[inside], ux[inside]] = o_[inside]
        fT[uy[inside], ux[inside]] = T[inside]
        ncon[uy[inside], ux[inside]] = last[inside]
    return out, fT, ncon, masks


def _bin(centres, radius, W, H):
    """Tile lists in index (= depth) order for Gaussians with the given centres and pixel radii."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    lists = [[] for _ in range(gx * gy)]
    for i, ((x, y), r) in enumerate(zip(centres, radius)):
        tx0, tx1 = max(0, int((x - r) // 16)), min(gx - 1, int((x + r) // 16))
        ty0, ty1 = max(0, int((y - r) // 16)), min(gy - 1, int((y + r) // 16))
        for ty in range(ty0, ty1 + 1):
            for tx in range(tx0, tx1 + 1):
                lists[ty * gx + tx].append(i)
    pl = np.array([i for l in lists for i in l], np.int64)
    ends = np.cumsum([len(l) for l in lists])
    ranges = np.stack([ends - np.array([len(l) for l in lists]), ends], 1)
    return pl, ranges


def _extents(Sig, op):
    """preprocess_fwd.cu:238-249 in numpy fp32 (logf as numpy's)."""
    if op < F32(1.0 / 255.0) * F32(0.9999):
        return F32(-1), F32(-1)
    tau = F32(np.log(F32(255) * F32(op))) * F32(1.0001) + F32(1e-4)
    hx = F32(np.sqrt(F32(2) * tau * F32(Sig[0, 0]))) * F32(1.0001) + F32(0.05)
    hy = F32(np.sqrt(F32(2) * tau * F32(Sig[1, 1]))) * F32(1.0001) + F32(0.05)
    return hx, hy


def _record2d(centre, Sig, op):
    """fp32 record {x, y, hx, hy, A, B, C, o} of a 2D Gaussian (conic = fp32 inverse of the effective covariance)."""
    inv = np.linalg.inv(Sig)
    A, B, C = F32(inv[0, 0]), F32(inv[0, 1]), F32(inv[1, 1])
    hx, hy = _extents(Sig, op)
    cdet = float(A) * float(C) - float(B) * float(B)
    if op >= F32(1.0 / 255.0) * F32(0.9999) and not cdet > 1e-3 * float(A) * float(C):
        hx = hy = F32(1e30)
    return np.array([F32(centre[0]), F32(centre[1]), hx, hy, A, B, C, F32(op)], np.float64)


def rim_case(jitter, seed=501, W=70, H=56):
    """CPU rim family: the designed rim Gaussians as 2D records (opacity solved on the fp32 record), in front, over a few
    ordinary splats behind."""
    g = np.random.default_rng(seed)
    so = ((g.random((H, W, 2)) - 0.5) * 2 * jitter).astype(F32) if jitter > 0 else np.zeros((H, W, 2), F32)
    ts = rim_plan(W, H, so, seed)
    recs, radius, cols = [], [], []
    for t in ts:
        r = _record2d(t["centre"], t["Sigma"], F32(0.5))
        o, _ = rim_opacity(r, W, H, so, t, t["rel"])
        recs.append(_record2d(t["centre"], t["Sigma"], F32(o)))
        radius.append(3 * math.sqrt(t["l1"]) + 2)
        cols.append(t["color"] * np.array([1.0, 0.97, 0.94]))
    for _ in range(200):
        th, s1, s2 = g.uniform(0, 3), g.uniform(0.7, 4), g.uniform(0.7, 4)
        R = np.array([[math.cos(th), -math.sin(th)], [math.sin(th), math.cos(th)]])
        Sig = R @ np.diag([s1 * s1 + 0.1, s2 * s2 + 0.1]) @ R.T
        c = (g.uniform(-5, W + 5), g.uniform(-5, H + 5))
        recs.append(_record2d(c, Sig, F32(g.uniform(0.05, 0.9))))
        radius.append(3 * max(s1, s2) + 2)
        cols.append(g.uniform(0, 1, 3))
    pl, ranges = _bin([r[:2] for r in recs], radius, W, H)
    return dict(records=np.array(recs), colors=np.array(cols), point_list=pl, ranges=ranges, subpixel_offset=so,
                bg=np.array([0.2, 0.4, 0.1]), W=W, H=H, targets=ts)


def tie_case():
    """One tile; at pixel (5, 5) a splat of alpha 1 - 2^13 1e-4f then thirteen of alpha 0.5, all centred exactly on the
    sample (power 0, expf(0) = 1): test_T reaches 1e-4f exactly on the 14th splat, which blends (1e-4f < 1e-4f is
    false) and the 15th stops the pixel."""
    m = F32(1e-4) * F32(8192)
    Sig = np.eye(2) * 4.0
    recs = [_record2d((5.0, 5.0), Sig, F32(1) - m)] + [_record2d((5.0, 5.0), Sig, F32(0.5)) for _ in range(14)]
    n = len(recs)
    return dict(records=np.array(recs), colors=np.full((n, 3), 0.8), point_list=np.arange(n),
                ranges=np.array([[0, n]]), subpixel_offset=np.zeros((16, 16, 2), F32), bg=np.array([0.1, 0.2, 0.3]),
                W=16, H=16)


def scene_case(name):
    """Emulation cases from cpu_oracle's preprocess and binning (the kernel's records without the extents, which are
    recomputed here the way preprocess_fwd.cu does)."""
    sc = {"small": lambda: synthetic.make_scene(2500, 40, 36, seed=9, subpixel_jitter=0.3, bg=(0.2, 0.5, 0.1)),
          "opaque": lambda: cpu_cases()["opaque"]}[name]()
    st = cpu_oracle.forward(sc)
    rec = records_of(st)
    for i in range(st["P"]):
        A, B, C = rec[i, 4:7]
        if st["radii"][i] <= 0:
            continue
        Sig = np.linalg.inv(np.array([[A, B], [B, C]]))
        hx, hy = _extents(Sig, F32(rec[i, 7]))
        cdet = A * C - B * B
        if rec[i, 7] >= F32(1.0 / 255.0) * F32(0.9999) and not cdet > 1e-3 * A * C:
            hx = hy = F32(1e30)
        rec[i, 2:4] = (hx, hy)
    return dict(records=rec, colors=st["colors"], point_list=st["point_list"].astype(np.int64),
                ranges=st["ranges"].astype(np.int64), subpixel_offset=np.asarray(sc["subpixel_offset"], F32),
                bg=np.asarray(sc["bg"], np.float64), W=st["W"], H=st["H"])


def emu_case(name):
    if name == "rim_0.0":
        return rim_case(0.0)
    if name == "rim_0.3":
        return rim_case(0.3)
    if name == "tie":
        return tie_case()
    return scene_case(name)


def _bound(case, n_contrib=None):
    return fwd_exact.bound(case["records"], case["colors"], case["point_list"], case["ranges"], case["subpixel_offset"],
                           case["bg"], case["W"], case["H"], n_contrib=n_contrib)


def _judge(case, emu):
    """Worst |emulated - S| / B (inf where B = 0 and they differ), n_contrib not admissible, sure mask bits differing."""
    out, fT, nc, masks = emu
    res = _bound(case, nc)
    got = np.concatenate([out.astype(np.float64), fT[None].astype(np.float64)])
    d = np.abs(got - res["S"])
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0, 0.0, d / res["B"])
    c = fwd_exact.check(res, out, fT, nc, masks)
    return float(np.nan_to_num(r, nan=0.0).max()), c["nc_outside"].size, len(c["mask_differ"]), c


EMU_CASES = ["small", "opaque", "rim_0.0", "rim_0.3", "tie"]


@pytest.mark.parametrize("name", EMU_CASES)
def test_bound_holds_for_an_fp32_emulation(name):
    case = emu_case(name)
    res = _bound(case)
    assert res["overflow_pixels"] == 0 and res["blended_pairs"] > (100 if name != "tie" else 10)
    for seed in range(3):
        e, nbad, mbad, c = _judge(case, emulate(case, np.random.default_rng(seed)))
        print(f"{name} seed {seed}: worst |emulated - S| / B = {e:.3f}, sure mask bits {c['mask_compared']}")
        assert e <= 1.0 and nbad == 0 and mbad == 0, (name, seed, e, nbad, mbad)


def _rim_cull_target(case):
    """(tile, warp, position) of the first designed rim pair above 1/255: the pair blends at its target sample."""
    for i, t in enumerate(case["targets"]):
        if t["rel"] > 0:
            r0, r1 = case["ranges"][t["tile"]]
            pos = int(np.nonzero(case["point_list"][r0:r1] == i)[0][0])
            return (t["tile"], t["block"], pos)
    raise AssertionError("no rim target")


MUTATIONS = [("cull", "rim_0.0"), ("le", "tie"), ("T_on_stop", "opaque"), ("zero_based", "small"),
             ("no_subpixel", "small"), ("no_bg", "small"), ("prev_round", "small"), ("tested_bit", "small"),
             ("ellipse_low", "rim_0.0"), ("box_shrink", "rim_0.0")]


@pytest.mark.parametrize("kind,name", MUTATIONS)
def test_mutations_are_caught(kind, name):
    """Each corruption of the emulated kernel puts some output CAUGHT bounds away from S, n_contrib outside its set or a
    sure mask bit off."""
    case = emu_case(name)
    mut = (kind, _rim_cull_target(case)) if kind == "cull" else (kind,)
    e, nbad, mbad, c = _judge(case, emulate(case, np.random.default_rng(7), mut))
    print(f"{kind} on {name}: worst |mutated - S| / B = {e:.3g}, n_contrib off {nbad}, sure mask bits off {mbad}")
    assert e >= CAUGHT or nbad > 0 or mbad > 0, (kind, e, nbad, mbad)
    if kind in ("cull", "le", "T_on_stop", "no_subpixel", "no_bg", "ellipse_low", "box_shrink"):
        assert e >= CAUGHT, (kind, "a value corruption must show in the values", e)
    if kind == "zero_based":
        assert nbad > 0
    if kind == "tested_bit":
        assert mbad > 0


def test_rim_case_reaches_the_cull_edges():
    """The CPU rim family is tight where the two culling corruptions bite: rim pairs whose q lies within 2e-3 of
    2 ln(255 o), some of them on a box edge with extents of 6 px or more and the box enabled, and both sides of the
    cdet gate."""
    case = rim_case(0.0)
    ins = dict(records=case["records"], subpixel_offset=case["subpixel_offset"], W=case["W"], H=case["H"])
    rows = rim_reach(ins, None, case["targets"], 0.0)
    above = [r for r, t in zip(rows, case["targets"]) if t["rel"] > 0]
    assert all(0 <= r["L"] - r["q"] < 2e-3 for r in above), max(r["L"] - r["q"] for r in above)
    assert sum(r["edge"] and 6.0 <= r["box"] < 1e29 for r in above) >= 5
    assert sum(r["corner"] for r in above) >= 5
    assert sum(r["gate_off"] for r in above) >= 2 and sum(not r["gate_off"] for r in above) >= 10
