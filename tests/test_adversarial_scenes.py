"""Rasterizer parity on scenes outside what ``synthetic.make_scene`` generates: posed cameras (non-identity view
matrix, camera centre far from the origin, fx != fy, off-centre principal point), depths spanning 0.2 .. 1000 and
Gaussians a few ulps either side of the near plane, exact depth ties, centres in the frustum guard band, other
``kernel_size`` / ``scale_modifier`` settings, degenerate splats, opaque and faint composites, and odd image shapes.

Each scene is built in camera space and mapped to world space with a seeded rigid transform, so the visible set stays
under control; each family asserts that it reaches the edge it is there for.

References (GPU tests):
* the compiled reference (``oracle/_ref/libdgr_ref.so``, skipped when absent): integer artefacts (R, radii, the sorted
  instance list, tile ranges, n_contrib) bit-exact, projected state (depths, means2D, conic/opacity, SH colours) with
  the same bits, pixels within 1e-4, gradients under ``check_grad``'s noise-tied bar;
* the fp64 CPU oracle run on the CUDA forward's own artefacts (the fp32 oracle's state cast to float64, n_contrib and
  final_T taken from the kernel where an alpha threshold flipped): for each gradient tensor, over the entries above
  1e-3 of its largest magnitude, the element-wise relative error of the kernel to that fp64 gradient must be within
  max(4 x the reference's own error to the same answer, 1e-5), or within 1e-3 when the reference is absent.

Measured on an H100 SXM (80 GB, default power limit): the worst element-wise relative error to fp64 of either
implementation ranges from 1e-5 to 8e-2 (one entry of dL/dscales on the posed scene), and ours stayed within 4x of the
reference's in every tensor (largest ratio 2.7, dL/dmeans3D of the single-tile crowd); see ``MEASURED_REF_FP64``.
Degenerate splats are held to the fp64 bar only, not entry by entry to the reference (see test_degenerate_splats).

CPU tests (no GPU): the fp64 oracle's backward against finite differences on a small posed scene with guard-band
Gaussians and ``kernel_size`` 0, the oracle against golden vectors of the unmodified reference on posed / guard-band
scenes (``tests/golden/make_golden_posed.py``), and the C ABI's rejection of images past the tile / cell limits.
"""
import math
import os
from ctypes import byref, c_int

import numpy as np
import pytest
import torch

import synthetic
from oracle import cpu_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_DIR = os.path.join(HERE, "golden")
GRAD_NAMES = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales",
              "dL_drotations")
PIX_TOL = 1e-4
K = 1024                 # per-tile list positions the composites record blend masks for
FP64_BAR_ABSENT = 1e-3   # element-wise relative bar to fp64 when the compiled reference is not there to calibrate it

# Worst element-wise relative error of the compiled reference's gradients to the fp64 answer, over all gradient tensors
# of each scene (entries above 1e-3 of the tensor's maximum), measured on an H100 SXM 80 GB at its default power limit.
# Ours was within 4x of it in every tensor; the worst cases are single entries where fp32 cancellation hits both
# implementations alike (the same entries, the same error).  Without the reference, the bar is 4x this number but at
# least FP64_BAR_ABSENT.  Families not listed measured below 1e-4.
MEASURED_REF_FP64 = {
    "posed_precomp": 8.0e-2, "posed_sh3": 2.0e-4, "depth_span": 3.6e-4, "ties": 1.0e-4, "guard_band": 1.1e-3,
    "settings_0.0_0.6": 1.3e-4, "settings_0.3_1.7": 1.7e-4, "settings_0.0_1.7": 4.5e-2, "opaque": 3.9e-3,
    "shape_15x17": 2.7e-4, "shape_16x16": 1.5e-4, "shape_17x33": 2.3e-4, "shape_4095x3": 2.6e-2, "one_tile": 4.9e-4,
    "widest_strip": 3.2e-4,
    # needles, sub-pixel splats, unnormalised quaternions: the fp32 gradients of both implementations are far from fp64;
    # with kernel_size 0 nearly singular conics blend only through fp32 rounding, so fp64 describes another composite
    "degenerate_0.1": 4.9e-3, "degenerate_0.0": 1.8e2,
}


# ======================================================================================================================
# scene builders (seeded, CPU torch)
# ======================================================================================================================
def _quat_to_R(q):
    q = q / q.norm()
    r, x, y, z = [float(v) for v in q]
    return torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                         [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                         [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]], dtype=torch.float64)


def posed_camera(W, H, seed, z_axis_only=False):
    """A camera the way method.py builds one from a pose and OpenCV intrinsics: world -> camera x_c = R x_w + t,
    fx != fy, principal point off centre.  ``z_axis_only``: R rotates about the optical axis and t has no z part, so
    view-space z equals world z bit for bit (near-plane and equal-depth scenes)."""
    g = torch.Generator().manual_seed(int(seed) + 77)
    U = lambda: float(torch.rand((), generator=g))
    fx = 0.9 * W * (0.85 + 0.3 * U())
    fy = fx * (0.7 + 0.2 * U())
    cx = W * (0.5 + 0.16 * (U() - 0.5))
    cy = H * (0.5 + 0.16 * (U() - 0.5))
    if z_axis_only:
        a = 2 * math.pi * U()
        R = torch.tensor([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]],
                         dtype=torch.float64)
        t = torch.tensor([6 * U() - 3 + 5.0, 6 * U() - 3 - 4.0, 0.0], dtype=torch.float64)
    else:
        R = _quat_to_R(torch.randn(4, generator=g, dtype=torch.float64))
        t = torch.randn(3, generator=g, dtype=torch.float64) * 4.0 + torch.tensor([3.0, -5.0, 7.0], dtype=torch.float64)
    wv = torch.eye(4, dtype=torch.float64)
    wv[:3, :3], wv[:3, 3] = R, t
    view = wv.float().transpose(0, 1).contiguous()
    proj = synthetic.projection_from_opencv(W, H, fx, fy, cx, cy, 0.01, 100.0).transpose(0, 1)
    full = view.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0).contiguous()
    campos = view.inverse()[3, :3].contiguous()
    tanfovx = math.tan(2 * math.atan(W / (2 * fx)) * 0.5)     # focal2fov, then tan(fov / 2), as method.py does
    tanfovy = math.tan(2 * math.atan(H / (2 * fy)) * 0.5)
    return dict(viewmatrix=view, projmatrix=full, campos=campos, tanfovx=tanfovx, tanfovy=tanfovy,
                R=R, t=t, fx=fx, fy=fy, cx=cx, cy=cy)


def to_world(cam, xyz_cam):
    """Inverse of x_c = R x_w + t for camera-space points (float64), rounded to float32."""
    x = xyz_cam.double()
    return ((x - cam["t"]) @ cam["R"]).float().contiguous()


def view_space(scene):
    """View-space positions of the scene's (float32) world means, in float64."""
    V = scene["viewmatrix"].double()
    m = scene["means3D"].double()
    return m @ V[:3, :3] + V[3, :3]


def build_scene(cam, W, H, seed, xyz_cam, scales, rots, opac, sh_degree=None, cov3D_precomp=False, kernel_size=0.1,
                scale_modifier=1.0, bg=(0.1, 0.3, 0.2), subpixel_jitter=0.0, exact_world=None):
    g = torch.Generator().manual_seed(int(seed) + 500)
    P = xyz_cam.shape[0]
    scene = {k: cam[k] for k in ("viewmatrix", "projmatrix", "campos", "tanfovx", "tanfovy")}
    scene.update(image_width=int(W), image_height=int(H), kernel_size=float(kernel_size),
                 scale_modifier=float(scale_modifier), prefiltered=False, debug=False,
                 means3D=to_world(cam, xyz_cam) if exact_world is None else exact_world,
                 opacities=opac.float().reshape(P, 1).contiguous(), bg=torch.tensor(bg, dtype=torch.float32))
    if cov3D_precomp:
        q = rots.double() / rots.double().norm(dim=1, keepdim=True)
        r, x, y, z = q.unbind(1)
        Rm = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                          2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                          2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=1).view(P, 3, 3)
        Mm = Rm * (scale_modifier * scales.double())[:, None, :]
        S = Mm @ Mm.transpose(1, 2)
        scene["cov3D_precomp"] = torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]],
                                             dim=1).float().contiguous()
    else:
        scene["scales"] = scales.float().contiguous()
        scene["rotations"] = rots.float().contiguous()
    if sh_degree is None:
        scene["colors_precomp"] = torch.rand(P, 3, generator=g).float().contiguous()
        scene["sh_degree"] = 0
    else:
        sh = 0.3 * torch.randn(P, 16, 3, generator=g)
        sh[:, 0, :] = (torch.rand(P, 3, generator=g) - 0.5) / synthetic.C0
        scene["shs"] = sh.float().contiguous()
        scene["sh_degree"] = int(sh_degree)
    if subpixel_jitter > 0:
        scene["subpixel_offset"] = ((torch.rand(H, W, 2, generator=g) - 0.5) * 2 * subpixel_jitter).float().contiguous()
    else:
        scene["subpixel_offset"] = torch.zeros((H, W, 2), dtype=torch.float32)
    scene["dL_dpix"] = torch.randn(3, H, W, generator=g).float().contiguous()
    return scene


def _cloud(g, P, cam, z=None, spread=1.1, scale_range=(0.002, 0.03), opac_range=(0.02, 1.0)):
    U = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    if z is None:
        z = 2.0 + 4.0 * U(P)
    x = (2 * U(P) - 1) * z * cam["tanfovx"] * spread
    y = (2 * U(P) - 1) * z * cam["tanfovy"] * spread
    lo, hi = math.log(scale_range[0]), math.log(scale_range[1])
    s = torch.exp(lo + (hi - lo) * U(P))[:, None] * torch.exp(0.3 * torch.randn(P, 3, generator=g, dtype=torch.float64))
    rot = torch.randn(P, 4, generator=g, dtype=torch.float64)
    rot = rot / rot.norm(dim=1, keepdim=True)
    opac = opac_range[0] + (opac_range[1] - opac_range[0]) * U(P)
    return torch.stack([x, y, z], 1), s, rot, opac


def scene_posed(kind, seed=101, P=30_000, W=320, H=240):
    cam = posed_camera(W, H, seed)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, P, cam)
    return build_scene(cam, W, H, seed, xyz, s, rot, op, sh_degree=3 if kind == "sh3" else None,
                       cov3D_precomp=kind == "cov3d", subpixel_jitter=0.3 if kind == "precomp" else 0.0)


def scene_depth_span(seed=111, P=30_000, W=320, H=240):
    """Depths log-uniform in [0.2, 1000] with scales proportional to depth, plus Gaussians a few ulps either side of
    the near plane z = 0.2 (view-space z equals world z bit for bit under this camera)."""
    cam = posed_camera(W, H, seed, z_axis_only=True)
    g = torch.Generator().manual_seed(seed)
    z = torch.exp(math.log(0.2) + (math.log(1000.0) - math.log(0.2)) * torch.rand(P, generator=g, dtype=torch.float64))
    xyz, s, rot, op = _cloud(g, P, cam, z=z, scale_range=(0.001, 0.01))
    s = s * z[:, None]
    near = np.float32(0.2)
    zs = []
    for k in range(-6, 7):
        v = near
        for _ in range(abs(k)):
            v = np.nextafter(v, np.float32(1.0 if k > 0 else 0.0), dtype=np.float32)
        zs.append(v)
    n_near = 40 * len(zs)
    zn = torch.tensor(np.repeat(np.array(zs, np.float32), 40), dtype=torch.float64)
    xn, sn, rn, on = _cloud(g, n_near, cam, z=zn, scale_range=(0.0005, 0.003))
    xyz, s, rot, op = torch.cat([xyz, xn]), torch.cat([s, sn]), torch.cat([rot, rn]), torch.cat([op, on])
    world = to_world(cam, xyz)
    world[:, 2] = xyz[:, 2].float()                   # exact: view z = world z under a z-axis-only camera
    return build_scene(cam, W, H, seed, xyz, s, rot, op, exact_world=world)


def scene_ties(seed=121, W=320, H=240):
    """Exact duplicates (each Gaussian 2-8 times at interleaved indices) and a fronto-parallel plane of equal z."""
    cam = posed_camera(W, H, seed, z_axis_only=True)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, 4_000, cam, scale_range=(0.004, 0.04))
    reps = torch.randint(2, 9, (4_000,), generator=g)
    idx = torch.repeat_interleave(torch.arange(4_000), reps)
    idx = idx[torch.randperm(idx.numel(), generator=g)]           # copies spread over the index range
    zp = torch.full((6_000,), 3.0, dtype=torch.float64)
    xp, sp, rp, opp = _cloud(g, 6_000, cam, z=zp, scale_range=(0.004, 0.04))
    xyz = torch.cat([xyz[idx], xp]); s = torch.cat([s[idx], sp]); rot = torch.cat([rot[idx], rp])
    op = torch.cat([op[idx], opp])
    world = to_world(cam, xyz)
    world[:, 2] = xyz[:, 2].float()
    sc = build_scene(cam, W, H, seed, xyz, s, rot, op, exact_world=world)
    # duplicated Gaussians carry the same colour, so they are the same Gaussian
    base = sc["colors_precomp"].clone()
    sc["colors_precomp"][: idx.numel()] = base[idx]
    return sc


def scene_guard_band(seed=131, P=30_000, W=320, H=240):
    """15 % of the centres at |x/z| or |y/z| in (1.35, 3.5) tanfov, with splats large enough to reach the image."""
    cam = posed_camera(W, H, seed)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, P, cam)
    n = int(0.15 * P)
    U = lambda *sh: torch.rand(*sh, generator=g, dtype=torch.float64)
    z = 2.0 + 4.0 * U(n)
    ratio = 1.35 + 2.15 * U(n)
    sign = torch.where(U(n) < 0.5, -1.0, 1.0)
    axis_x = U(n) < 0.5
    tx, ty = cam["tanfovx"], cam["tanfovy"]
    x = torch.where(axis_x, sign * ratio * tx, (2 * U(n) - 1) * tx) * z
    y = torch.where(axis_x, (2 * U(n) - 1) * ty, sign * ratio * ty) * z
    xyz[:n] = torch.stack([x, y, z], 1)
    s[:n] = (z * (0.25 + 0.5 * U(n)))[:, None] * torch.exp(0.2 * torch.randn(n, 3, generator=g, dtype=torch.float64))
    op[:n] = 0.02 + 0.3 * U(n)
    return build_scene(cam, W, H, seed, xyz, s, rot, op)


def scene_settings(kernel_size, scale_modifier, seed=141, P=30_000, W=320, H=240):
    cam = posed_camera(W, H, seed)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, P, cam)
    return build_scene(cam, W, H, seed, xyz, s, rot, op, kernel_size=kernel_size, scale_modifier=scale_modifier)


def scene_degenerate(kernel_size, seed=151, P=30_000, W=320, H=240):
    """Needles (one or two scales 1e-5 of the third), sub-pixel splats whose 2D covariance is the low-pass filter's,
    and unnormalised quaternions scaled by 1e-3 and 1e3."""
    cam = posed_camera(W, H, seed)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, P, cam, scale_range=(0.005, 0.05))
    q = P // 5
    s[0 * q:1 * q, 0] *= 1e-5                                         # needles: one thin axis
    s[1 * q:2 * q, 1:] *= 1e-5                                        # needles: two thin axes
    s[2 * q:3 * q] = 1e-5 * xyz[2 * q:3 * q, 2:3] * torch.exp(torch.randn(q, 3, generator=g, dtype=torch.float64))
    rot[3 * q:3 * q + q // 2] *= 1e-3                                  # unnormalised quaternions
    rot[3 * q + q // 2:4 * q] *= 1e3
    s[3 * q + q // 2:4 * q] *= 1e-6                                    # the rotation matrix scales with |q|^2
    return build_scene(cam, W, H, seed, xyz, s, rot, op, kernel_size=kernel_size)


def scene_opaque(seed=161, P=20_000, W=320, H=240):
    """Opaque stacks: opacity 0.999, large splats: most pixels end with T < 1e-4, centres hit the 0.99 alpha clamp."""
    cam = posed_camera(W, H, seed)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, P, cam, scale_range=(0.02, 0.12), opac_range=(0.999, 0.999))
    return build_scene(cam, W, H, seed, xyz, s, rot, op)


def scene_faint(seed=171, P=20_000, W=320, H=240):
    """Every alpha below 1/255: the image is the background, nothing blends, every gradient is exactly zero."""
    cam = posed_camera(W, H, seed)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, P, cam, scale_range=(0.01, 0.1), opac_range=(0.0005, 0.0038))
    return build_scene(cam, W, H, seed, xyz, s, rot, op)


SHAPES = [(1, 1), (1, 37), (37, 1), (15, 17), (16, 16), (17, 33), (4095, 3)]


def scene_shape(W, H, seed=181):
    cam = posed_camera(W, H, seed + W * 7 + H)
    g = torch.Generator().manual_seed(seed + W * 7 + H)
    P = int(min(20_000, max(2_000, 4 * W * H)))
    xyz, s, rot, op = _cloud(g, P, cam, scale_range=(0.3, 4.0))       # 0.3 .. 4 pixels
    s = s * (xyz[:, 2] / cam["fx"])[:, None]
    return build_scene(cam, W, H, seed, xyz, s, rot, op, subpixel_jitter=0.4)


def scene_one_tile_crowd(seed=191, P=300_000):
    """One 16x16 image (a single tile and cell) under ~300k faint, wide Gaussians: lists far beyond K."""
    W = H = 16
    cam = posed_camera(W, H, seed)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, P, cam, spread=1.0, scale_range=(0.3, 1.0), opac_range=(0.0045, 0.008))
    return build_scene(cam, W, H, seed, xyz, s, rot, op)


def scene_widest_strip(seed=201, P=20_000):
    """The widest image the rasterizer accepts: 65535 tiles x 1 tile row."""
    W, H = 65535 * 16, 16
    cam = posed_camera(W, H, seed)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, P, cam, spread=1.05, scale_range=(1.0, 30.0))     # 1 .. 30 pixels
    s = s * (xyz[:, 2] / cam["fx"])[:, None]
    # some at the right end of the strip
    xyz[:200, 0] = xyz[:200, 2] * (W - cam["cx"] - 40 * torch.rand(200, generator=g, dtype=torch.float64)) / cam["fx"]
    return build_scene(cam, W, H, seed, xyz, s, rot, op)


# ======================================================================================================================
# comparisons
# ======================================================================================================================
def rel_errors_to(ref64, grads):
    """Largest element-wise relative error of `grads` to the fp64 gradients, per tensor, over the entries above 1e-3 of
    the tensor's largest magnitude (tensors that are zero in fp64 are compared exactly)."""
    out = {}
    for n in GRAD_NAMES:
        want = np.asarray(ref64[n], np.float64)
        if want.size == 0:
            continue
        got = np.asarray(grads[n], np.float64).reshape(want.shape)
        scale = float(np.abs(want).max())
        if scale == 0.0:
            out[n] = 0.0 if not np.any(got) else math.inf
            continue
        big = np.abs(want) > 1e-3 * scale
        out[n] = float((np.abs(got[big] - want[big]) / np.abs(want[big])).max())
    return out


def fp64_gradients(scene, st32, final_T, n_contrib):
    """The oracle's backward in float64 on the forward the kernel ran: the fp32 oracle's projected state cast to
    float64, with the kernel's n_contrib / final_T wherever an alpha threshold came out differently."""
    st = dict(st32)
    for k in ("depths", "means2D", "cov3D", "conic_opacity", "rgb", "out_color", "final_T", "colors"):
        st[k] = np.ascontiguousarray(st32[k], np.float64)
    st["dtype"] = np.dtype(np.float64)
    flip = st32["n_contrib"].astype(np.int64) != n_contrib.astype(np.int64)
    st["n_contrib"] = np.where(flip, n_contrib.astype(np.uint32), st32["n_contrib"]).astype(np.uint32)
    st["final_T"] = np.where(flip, final_T.astype(np.float64), st["final_T"])
    return cpu_oracle.backward(st, scene["dL_dpix"]), int(flip.sum())


def _np_grads(grads):
    return {n: g.detach().cpu().numpy() for n, g in grads.items()}


def run_and_compare(C, scene, name, ref_gradients=True):
    """Ours against the compiled reference (when present) and both against fp64.  Returns what the edge checks need.
    ``ref_gradients=False``: gradients are judged against fp64 only (the 4x-reference bar), not entry by entry against
    the reference's (see test_degenerate_splats)."""
    from test_gpu_parity import check_grad, run_ours
    from make_golden import backward_args, call_args
    from oracle import ref_cuda
    dev = torch.device("cuda:0")
    d = synthetic.to_device(scene, dev)
    C.set_geometry_cache(False)
    try:
        o = run_ours(C, d)
    finally:
        C.set_geometry_cache(True)
    v = o["views"]
    ours = _np_grads(o["grads"])
    vis = o["radii"] > 0

    have_ref = ref_cuda.available()
    ref_err = None
    if have_ref:
        R, color, radii, geom, binning, img = ref_cuda.rasterize_gaussians(*call_args(d))
        P = d["means3D"].shape[0]
        rv = ref_cuda.debug_views(geom, binning, img, P, d["image_width"], d["image_height"], R)
        bargs = backward_args(d, radii, geom, R, binning, img)
        rg = dict(zip(GRAD_NAMES, ref_cuda.rasterize_gaussians_backward(*bargs)))
        rg2 = dict(zip(GRAD_NAMES, ref_cuda.rasterize_gaussians_backward(*bargs)))
        torch.cuda.synchronize()
        assert o["R"] == R, (name, o["R"], R)
        assert torch.equal(o["radii"], radii), name
        assert torch.equal(v["ranges"], rv["ranges"]), name
        assert torch.equal(v["point_list"], rv["point_list"]), (name, "sorted instance list differs")
        assert torch.equal(v["n_contrib"], rv["n_contrib"]), name
        assert torch.equal(v["depths"][vis].view(torch.int32), rv["depths"][vis].view(torch.int32)), name
        assert torch.equal(v["records"][vis][:, 0:2].contiguous().view(torch.int32), rv["means2D"][vis].view(torch.int32))
        assert torch.equal(v["records"][vis][:, 4:8].contiguous().view(torch.int32),
                           rv["conic_opacity"][vis].view(torch.int32)), name
        if "shs" in scene:
            assert torch.equal(v["rgb"][vis].view(torch.int32), rv["rgb"][vis].view(torch.int32)), name
        assert float((o["color"] - color).abs().max()) <= PIX_TOL, name
        assert float((v["final_T"] - rv["final_T"]).abs().max()) <= PIX_TOL, name
        for n in GRAD_NAMES:
            if ref_gradients and rg[n].numel() and float(rg[n].abs().max()) > 0:
                check_grad(n, o["grads"][n].view_as(rg[n]), rg[n], rg2[n])
        ref_np = _np_grads(rg)

    # fp64: integer artefacts of the fp32 oracle equal the kernel's, then the fp64 backward on the kernel's forward
    st = cpu_oracle.forward(scene)
    assert st["num_rendered"] == o["R"], name
    assert np.array_equal(st["radii"], o["radii"].cpu().numpy()), name
    assert np.array_equal(st["point_list"].astype(np.int32), v["point_list"].cpu().numpy()), name
    assert np.array_equal(st["ranges"].astype(np.int32), v["ranges"].cpu().numpy()), name
    assert np.abs(st["out_color"] - o["color"].cpu().numpy()).max() <= PIX_TOL, name
    g64, flips = fp64_gradients(scene, st, v["final_T"].cpu().numpy(), v["n_contrib"].cpu().numpy())
    assert flips <= max(2, 1e-4 * v["n_contrib"].numel()), (name, flips)
    our_err = rel_errors_to(g64, ours)
    if have_ref:
        ref_err = rel_errors_to(g64, ref_np)
    for n, e in our_err.items():
        bar = max(4.0 * ref_err[n], 1e-5) if have_ref else max(FP64_BAR_ABSENT, 4.0 * MEASURED_REF_FP64.get(name, 0.0))
        print(f"fp64 {name} {n}: ours {e:.2e}" + (f" reference {ref_err[n]:.2e}" if have_ref else ""))
        assert e <= bar, (name, n, "element-wise relative error to fp64", e, "bar", bar)
    return dict(o=o, st=st, vis=vis.cpu().numpy(), ours=ours, g64=g64)


# ======================================================================================================================
# GPU tests
# ======================================================================================================================
@pytest.fixture(scope="module")
def C():
    from diff_gaussian_rasterization import _C
    return _C


def _tanfov_ratio(scene):
    vs = view_space(scene)
    return (vs[:, 0] / vs[:, 2]).abs().numpy() / scene["tanfovx"], (vs[:, 1] / vs[:, 2]).abs().numpy() / scene["tanfovy"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["precomp", "sh3", "cov3d"])
def test_posed_camera(C, kind):
    scene = scene_posed(kind)
    V = scene["viewmatrix"]
    assert float((V - torch.eye(4)).abs().max()) > 0.5 and float(V[3, :3].abs().max()) > 1.0
    assert float(scene["campos"].norm()) > 3.0 and abs(scene["tanfovx"] / scene["tanfovy"] - 320 / 240) > 0.05
    r = run_and_compare(C, scene, f"posed_{kind}")
    assert int(r["vis"].sum()) >= 10_000, "the posed camera does not see the cloud"


@pytest.mark.gpu
def test_mark_visible_under_a_posed_camera(C):
    from oracle import ref_cuda
    scene = scene_depth_span()
    dev = torch.device("cuda:0")
    d = synthetic.to_device(scene, dev)
    ours = C.mark_visible(d["means3D"], d["viewmatrix"], d["projmatrix"]).cpu().numpy()
    want = cpu_oracle.mark_visible(scene["means3D"], scene["viewmatrix"])
    z = scene["means3D"][:, 2].numpy()
    near = np.abs(z - np.float32(0.2)) < 1e-6
    assert near.sum() >= 400 and 0 < ours[near].sum() < near.sum(), "scene does not straddle the near plane"
    assert np.array_equal(ours, want)
    assert np.array_equal(ours, z > np.float32(0.2))                # view z == world z under this camera
    # a rotated, translated camera with points on both sides of the near plane
    posed = scene_posed("precomp")
    g = torch.Generator().manual_seed(5)
    xyz = torch.randn(20_000, 3, generator=g, dtype=torch.float64) * torch.tensor([2.0, 2.0, 0.5], dtype=torch.float64)
    posed["means3D"] = to_world(posed_camera(320, 240, 101), xyz + torch.tensor([0.0, 0.0, 0.2], dtype=torch.float64))
    dp = synthetic.to_device(posed, dev)
    ours_p = C.mark_visible(dp["means3D"], dp["viewmatrix"], dp["projmatrix"]).cpu().numpy()
    vz = view_space(posed)[:, 2].numpy()
    sure = np.abs(vz - 0.2) > 1e-5
    assert np.array_equal(ours_p[sure], (vz > 0.2)[sure]) and 0.3 < ours_p.mean() < 0.7
    assert np.array_equal(ours_p, cpu_oracle.mark_visible(posed["means3D"], posed["viewmatrix"]))
    if ref_cuda.available():
        assert np.array_equal(ours, ref_cuda.mark_visible(d["means3D"], d["viewmatrix"], d["projmatrix"]).cpu().numpy())
        assert np.array_equal(ours_p, ref_cuda.mark_visible(dp["means3D"], dp["viewmatrix"],
                                                            dp["projmatrix"]).cpu().numpy())


@pytest.mark.gpu
def test_depth_span_and_near_plane(C):
    scene = scene_depth_span()
    r = run_and_compare(C, scene, "depth_span")
    vis = r["vis"]
    top = np.unique(r["o"]["views"]["depths"].cpu().numpy()[vis].view(np.uint32) >> 24)
    assert top.size >= 5, f"depth keys use only top bytes {top}"
    z = scene["means3D"][:, 2].numpy()
    near = np.abs(z - np.float32(0.2)) < 1e-6
    assert vis[near & (z > np.float32(0.2))].sum() >= 100, "no Gaussian just beyond the near plane is rendered"
    assert not vis[near & (z <= np.float32(0.2))].any()


def _tied_pairs(o):
    v = o["views"]
    pl = v["point_list"].long()
    rg = v["ranges"].long()
    ne = rg[:, 1] > rg[:, 0]
    tile_of = torch.repeat_interleave(torch.arange(rg.shape[0], device=pl.device)[ne], (rg[ne, 1] - rg[ne, 0]))
    key = (tile_of << 32) | v["depths"].view(torch.int32).long()[pl]
    same = key[1:] == key[:-1]
    assert bool((pl[1:][same] > pl[:-1][same]).all()), "depth ties are not in Gaussian-index order"
    return int(same.sum())


@pytest.mark.gpu
def test_exact_depth_ties(C):
    scene = scene_ties()
    r = run_and_compare(C, scene, "ties")
    assert _tied_pairs(r["o"]) >= 5_000, "scene has too few tied (tile, depth) pairs"


@pytest.mark.gpu
def test_guard_band(C):
    scene = scene_guard_band()
    r = run_and_compare(C, scene, "guard_band")
    rx, ry = _tanfov_ratio(scene)
    band = (rx > 1.31) | (ry > 1.31)
    assert int((band & r["vis"]).sum()) >= 500, "too few guard-band Gaussians rendered"


@pytest.mark.gpu
@pytest.mark.parametrize("ks,mod", [(0.0, 0.6), (0.3, 1.7), (0.0, 1.7)])
def test_kernel_size_and_scale_modifier(C, ks, mod):
    scene = scene_settings(ks, mod)
    r = run_and_compare(C, scene, f"settings_{ks}_{mod}")
    assert int(r["vis"].sum()) >= 10_000


@pytest.mark.gpu
@pytest.mark.parametrize("ks", [0.0, 0.1])
def test_degenerate_splats(C, ks):
    """Forward bit-exact against the reference; gradients against fp64 under the 4x-reference bar.  Entry by entry
    against the reference's gradients is the wrong yardstick here: for needles and huge unnormalised quaternions both
    implementations' fp32 gradients are 1e-3 .. 1 of the tensor maximum away from the fp64 answer, in different
    entries and in both directions.  Measured (max |difference| / max |reference|): kernel_size 0.1, dL/dcov3D ours
    1.2e-3, reference 1.2e-3 from fp64, 3.4e-4 from each other; kernel_size 0, dL/dscales ours 2.8e-2, reference 2.1e-1,
    dL/drotations ours 2.6e-2, reference 1.0.  With kernel_size 0, needles with two thin axes blend only through fp32
    rounding of their nearly singular conic (in fp64 they do not blend at all), in both implementations alike."""
    scene = scene_degenerate(ks)
    r = run_and_compare(C, scene, f"degenerate_{ks}", ref_gradients=False)
    P = scene["means3D"].shape[0]
    q = P // 5
    vis = r["vis"]
    assert vis[:2 * q].sum() >= 1_000 and vis[2 * q:3 * q].sum() >= 1_000 and vis[3 * q:4 * q].sum() >= 1_000
    # sub-pixel splats: the 2D covariance is the low-pass filter's (or, without one, singular to fp32)
    conic_w = r["st"]["conic_opacity"][:, 3]
    if ks == 0.0:
        assert int((vis & (conic_w == 0)).sum()) >= 100, "no splat reaches the degenerate-determinant branch"
    assert int(np.count_nonzero(r["ours"]["dL_dopacity"][3 * q:4 * q])) >= 1_000, "unnormalised splats do not blend"


@pytest.mark.gpu
def test_opaque_stacks(C):
    scene = scene_opaque()
    r = run_and_compare(C, scene, "opaque")
    # terminated by the T < 1e-4 test: transmittance at the end below 1e-3 with list entries left unvisited
    v = r["o"]["views"]
    W, H = scene["image_width"], scene["image_height"]
    lens = (v["ranges"][:, 1] - v["ranges"][:, 0]).view((H + 15) // 16, (W + 15) // 16)
    lens = lens.repeat_interleave(16, 0).repeat_interleave(16, 1)[:H, :W]
    term = ((v["final_T"] < 1e-3) & (v["n_contrib"] < lens)).float().mean()
    assert float(term) >= 0.3, f"only {float(term):.2f} of the pixels terminate"
    assert int((r["vis"] & (r["st"]["conic_opacity"][:, 3] >= 0.99)).sum()) >= 100, "no Gaussian reaches the alpha clamp"


@pytest.mark.gpu
def test_faint_scene_is_background(C):
    scene = scene_faint()
    r = run_and_compare(C, scene, "faint")
    o = r["o"]
    assert int(r["vis"].sum()) >= 5_000
    W, H = scene["image_width"], scene["image_height"]
    assert torch.equal(o["color"].cpu(), scene["bg"][:, None, None].expand(3, H, W))
    assert int(o["views"]["n_contrib"].abs().max()) == 0
    for n, g in o["grads"].items():
        assert g.numel() == 0 or float(g.abs().max()) == 0.0, n


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", SHAPES, ids=lambda v: str(v))
def test_image_shapes(C, W, H):
    scene = scene_shape(W, H)
    r = run_and_compare(C, scene, f"shape_{W}x{H}")
    assert int(r["vis"].sum()) > 0 and r["o"]["R"] > 0


@pytest.mark.gpu
def test_one_tile_list_far_beyond_K(C):
    scene = scene_one_tile_crowd()
    r = run_and_compare(C, scene, "one_tile")
    assert int(r["o"]["views"]["n_contrib"].max()) > K, "scene does not exercise the positions beyond K"
    assert r["o"]["R"] >= 100_000


@pytest.mark.gpu
def test_widest_strip(C):
    scene = scene_widest_strip()
    r = run_and_compare(C, scene, "widest_strip")
    rg = r["o"]["views"]["ranges"]
    assert rg.shape[0] == 65535
    assert int(rg[-1, 1] - rg[-1, 0]) > 0, "nothing lands in the last tile of the strip"


# ======================================================================================================================
# method level: the reference's own _render_internal under a posed camera
# ======================================================================================================================
@pytest.mark.gpu
def test_render_internal_under_a_posed_camera():
    """method.py builds the view matrix, the camera centre (the SH view direction) and tanfov from the camera-to-world
    pose and the intrinsics.  One step through ``_render_internal`` on the drop-in, on the reference's compiled core
    behind the same names, and with ``wildgaussians_fused.enable`` (cached camera constants, the fused colour op's view
    direction), all under a rotated, translated camera with fx != fy and an off-centre principal point."""
    import types
    import wg_harness as wh
    from oracle import ref_cuda
    if not ref_cuda.available():
        pytest.skip("oracle/_ref/libdgr_ref.so not present")
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    import bench
    import diff_gaussian_rasterization as ours
    import wildgaussians_fused as wf
    ref_api = bench.make_reference_api(ref_cuda)
    dev = torch.device("cuda:0")
    W, H, seed = 400, 272, 65
    scene = scene_posed("sh3", seed=seed, P=60_000, W=W, H=H)
    cam = posed_camera(W, H, seed)
    c2w = torch.eye(4, dtype=torch.float64)
    c2w[:3, :3], c2w[:3, 3] = cam["R"].T, -cam["R"].T @ cam["t"]
    camera = types.SimpleNamespace(poses=c2w[:3].numpy().astype(np.float32), image_sizes=np.array([W, H], np.int32),
                                   intrinsics=np.array([cam["fx"], cam["fy"], cam["cx"], cam["cy"]], np.float32))
    model, cfg = wh.make_model(m, Config, scene, dev, seed=seed)
    g = torch.Generator().manual_seed(seed + 100)
    G1, G2 = torch.randn(3, H, W, generator=g).to(dev), torch.randn(3, H, W, generator=g).to(dev)

    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    ours._C.set_geometry_cache(True)
    a = wh.collect(model, wh.train_step(model, cfg, camera, G1, G2))
    wf.enable(model)
    try:
        f = wh.collect(model, wh.train_step(model, cfg, camera, G1, G2))
    finally:
        wf.disable(model)
    wh.use_backend(m, ref_api["GaussianRasterizer"], ref_api["GaussianRasterizationSettings"])
    try:
        b = wh.collect(model, wh.train_step(model, cfg, camera, G1, G2))
        b2 = wh.collect(model, wh.train_step(model, cfg, camera, G1, G2))
    finally:
        wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    torch.cuda.synchronize()

    assert int((a["radii"] > 0).sum()) >= 20_000, "the posed camera does not see the cloud"
    assert float(a["render"].abs().max()) > 0.05
    # drop-in against the reference backend
    assert torch.equal(a["radii"], b["radii"])
    for k in ("render", "raw_render", "accumulation"):
        assert float((a[k] - b[k]).abs().max()) <= 1e-4, k
    for k in a:
        if not (k.startswith("g_") or k == "viewspace_grad"):
            continue
        scale = float(b[k].abs().max()) + 1e-30
        err = float((a[k] - b[k]).abs().max()) / scale
        noise = float((b2[k] - b[k]).abs().max()) / scale
        assert err <= max(20.0 * noise, 2e-5), (k, err, noise)
    # fused path against the reference method (tolerances of test_method_py: bf16 MLP operands)
    assert torch.equal(f["radii"], b["radii"])
    assert float((f["raw_render"] - b["raw_render"]).abs().max()) < 2e-4
    assert float((f["render"] - b["render"]).abs().max()) < 1e-3
    for k in f:
        if not (k.startswith("g_") or k == "viewspace_grad"):
            continue
        x, y = f[k].double().flatten(), b[k].double().flatten()
        cos = float(x @ y) / (float(x.norm()) * float(y.norm()) + 1e-300)
        ratio = float(x.norm()) / (float(y.norm()) + 1e-300)
        assert cos >= 0.99 and abs(ratio - 1) < 0.03, (k, cos, ratio)
        if k in ("g_xyz", "g_scales", "g_rotations", "g_opacities", "viewspace_grad"):
            assert float((f[k] - b[k]).abs().max()) / (float(b[k].abs().max()) + 1e-30) < 2e-3, k


# ======================================================================================================================
# CPU: the oracle itself on the new geometry, and the C ABI's size limits
# ======================================================================================================================
def scene_fd(seed=211, P=60, W=48, H=32):
    """Small posed scene, kernel_size 0, a fifth of the centres in the guard band, every alpha below the 0.99 clamp
    (the reference's backward ignores the clamp, so only then is its gradient the true derivative)."""
    cam = posed_camera(W, H, seed)
    g = torch.Generator().manual_seed(seed)
    xyz, s, rot, op = _cloud(g, P, cam, scale_range=(0.08, 0.4), opac_range=(0.02, 0.88))
    n = P // 5
    ratio = 1.4 + 1.5 * torch.rand(n, generator=g, dtype=torch.float64)
    xyz[:n, 0] = ratio * cam["tanfovx"] * xyz[:n, 2] * torch.where(torch.arange(n) % 2 == 0, 1.0, -1.0)
    s[:n] = 0.5 * xyz[:n, 2:3] * (0.5 + torch.rand(n, 3, generator=g, dtype=torch.float64))
    return build_scene(cam, W, H, seed, xyz, s, rot, op, kernel_size=0.0, sh_degree=2)


def _loss64(scene):
    st = cpu_oracle.forward(scene, dtype=np.float64)
    return float((st["out_color"] * scene["dL_dpix"].numpy()).sum()), st


def test_oracle_backward_matches_finite_differences_posed_guard_band():
    """Scale, rotation, opacity and SH gradients are checked on guard-band Gaussians too.  Mean gradients are checked
    on Gaussians inside the band only: where the clamp is active the reference's dL/dt_z (backward.cu) treats the
    clamped t_x = 1.3 tanfov t_z as independent of t_z, so its mean gradient there is not the derivative of its
    forward (about 20 % off on this scene).  The oracle and the kernels restate that formula; the compiled-reference
    tests pin it."""
    scene = scene_fd()
    scene = {k: (v.double() if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in scene.items()}
    _, st = _loss64(scene)
    g = cpu_oracle.backward(st, scene["dL_dpix"])
    vis = np.nonzero(st["radii"] > 0)[0]
    rx, _ = _tanfov_ratio(scene)
    band = np.intersect1d(vis, np.nonzero(rx > 1.35)[0])
    assert band.size >= 5, "no guard-band Gaussian is rendered"
    assert float(np.max(st["conic_opacity"][vis, 3])) < 0.99
    rng = np.random.default_rng(1)
    for key, gname in (("means3D", "dL_dmeans3D"), ("opacities", "dL_dopacity"), ("scales", "dL_dscales"),
                       ("rotations", "dL_drotations"), ("shs", "dL_dsh")):
        x = scene[key]
        flat_g = g[gname].reshape(x.shape)
        errs = []
        for k in range(12):
            inner = np.setdiff1d(vis, band)
            i = int(rng.choice(band if (k % 2 == 0 and key != "means3D") else inner))   # half in the guard band
            j = tuple(int(rng.integers(0, s_)) for s_ in x.shape[1:])
            if key == "shs":
                j = (int(rng.integers(0, 9)), j[1])                 # active degree 2
            idx = (i,) + j
            eps = 1e-6 * max(1.0, abs(float(x[idx])))
            xp = x.clone(); xp[idx] += eps
            xm = x.clone(); xm[idx] -= eps
            fd = (_loss64({**scene, key: xp})[0] - _loss64({**scene, key: xm})[0]) / (2 * eps)
            an = float(flat_g[idx])
            errs.append(abs(fd - an) / max(1e-6, abs(fd), abs(an)))
        errs = np.sort(np.array(errs))
        assert errs[9] < 1e-4, (key, errs)


POSED_GOLDEN = ("posed_sh3_small", "guard_band_small", "posed_cov3d_ks0")


def golden_posed_scene(name):
    """Scenes of the posed golden vectors (tests/golden/make_golden_posed.py)."""
    if name == "posed_sh3_small":
        return scene_posed("sh3", seed=221, P=3_000, W=144, H=112)
    if name == "guard_band_small":
        return scene_guard_band(seed=222, P=2_000, W=128, H=96)
    if name == "posed_cov3d_ks0":
        return {**scene_posed("cov3d", seed=223, P=2_000, W=128, H=96), "kernel_size": 0.0}
    raise KeyError(name)


SCALARS = ("image_width", "image_height", "tanfovx", "tanfovy", "kernel_size", "scale_modifier", "sh_degree")


def load_posed_inputs(name, directory=GOLDEN_DIR):
    inp = dict(np.load(os.path.join(directory, name + ".inputs.npz")))
    scene = dict(prefiltered=False, debug=False)
    for k, v in inp.items():
        if k in SCALARS:
            scene[k] = int(v) if k in ("image_width", "image_height", "sh_degree") else float(v)
        else:
            scene[k] = torch.from_numpy(np.ascontiguousarray(v))
    return scene


def load_posed_case(name):
    """The committed inputs (tensors and scalars) and the reference's outputs on them."""
    return load_posed_inputs(name), dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))


@pytest.mark.parametrize("name", POSED_GOLDEN)
def test_oracle_against_posed_golden(name):
    from golden_util import bits, rel_err
    scene, gold = load_posed_case(name)
    V = scene["viewmatrix"]
    assert float((V - torch.eye(4)).abs().max()) > 0.5 and float(scene["campos"].norm()) > 3.0
    st = cpu_oracle.forward(scene)
    vis = gold["radii"] > 0
    assert st["num_rendered"] == int(gold["num_rendered"])
    assert np.array_equal(st["radii"], gold["radii"])
    assert np.array_equal(st["point_list"].astype(np.int32), gold["point_list"]), "sorted instance list differs"
    assert np.array_equal(st["ranges"].astype(np.int32), gold["ranges"])
    for k in ("depths", "means2D", "conic_opacity"):
        assert np.array_equal(bits(st[k][vis]), bits(gold[k][vis])), k
    if "shs" in scene:
        assert np.array_equal(bits(st["rgb"][vis]), bits(gold["rgb"][vis]))
    assert np.abs(st["out_color"] - gold["out_color"]).max() < PIX_TOL
    assert (st["n_contrib"].astype(np.int32) != gold["n_contrib"]).mean() <= 1e-4
    if name == "guard_band_small":
        rx, ry = _tanfov_ratio(scene)
        assert int((vis & ((rx > 1.31) | (ry > 1.31))).sum()) >= 20, "no guard-band Gaussian rendered"
    g = cpu_oracle.backward(st, scene["dL_dpix"])
    for n in GRAD_NAMES:
        ref = gold[n]
        if ref.size == 0 or not np.any(ref):
            continue
        got = g[n].reshape(ref.shape)
        assert rel_err(got, ref) < 1e-4, n
        big = np.abs(ref) > 1e-3 * np.abs(ref).max()
        assert float((np.abs(got[big] - ref[big]) / np.abs(ref[big])).max()) < 2e-3, (n, "element-wise")


def test_image_size_limits_are_rejected_through_the_c_abi():
    """One tile past the width limit and one binning cell past the 65536-cell limit are refused with a message before
    anything runs; the widest accepted strip (65535 x 1 tiles) and exactly 65536 cells pass the check."""
    import diff_gaussian_rasterization._C as C
    lib = C._lib
    R, N1 = c_int(0), c_int(0)

    def call(W, H):
        a = C.GsrForwardArgs()
        a.P, a.W, a.H = 0, W, H
        return lib.gsr_forward_geometry(byref(a), None, None, None, byref(R), byref(N1))

    assert call(65535 * 16, 16) == 0
    assert call(65535 * 16 + 1, 16) == -1 and b"image too large" in lib.gsr_last_error()
    assert call(16, 65535 * 16 + 1) == -1 and b"image too large" in lib.gsr_last_error()
    assert call(256 * 128, 256 * 128) == 0                          # 256 x 256 cells of 8 x 8 tiles
    assert call(256 * 128 + 1, 256 * 128) == -1 and b"image too large" in lib.gsr_last_error()
    assert call(256 * 128, 256 * 128 + 1) == -1 and b"image too large" in lib.gsr_last_error()
