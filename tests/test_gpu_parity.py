"""GPU parity tests (run on an H100 with ``-m gpu``): the CUDA path, called through the C ABI
(``diff_gaussian_rasterization._C`` is a ctypes shim over ``include/gsrast.h``) and through the drop-in Python
API, against (a) the committed golden vectors of the reference, (b) the compiled reference itself when
``oracle/_ref/libdgr_ref.so`` travelled with the snapshot, (c) the CPU oracle; plus size-independent
properties at BASELINE.json's full sizes.

Bars: tile / sort indices bit-exact; pixels and final_T the reference's bits where the reference's own outputs are
there (golden vectors, the compiled reference), within 1e-4 of the CPU oracle (glibc expf); gradients within 1e-3 of
the largest gradient magnitude (the reference's own float-atomic run-to-run noise is ~1e-6).
"""
import numpy as np
import pytest
import torch

import synthetic
from golden_util import GRAD_NAMES, GRAD_TOL, PIX_TOL, bits, load_case, rel_err
from make_golden import CASES, backward_args, call_args

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    from diff_gaussian_rasterization import _C
    return _C


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def run_ours(C, d):
    R, color, radii, geom, binning, img = C.rasterize_gaussians(*call_args(d))
    P = d["means3D"].shape[0]
    M = d["shs"].shape[1] if "shs" in d else 0
    v = C.debug_views(geom, binning, img, P, M, d["image_width"], d["image_height"], R) if P else {}
    grads = C.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))
    torch.cuda.synchronize()
    return dict(R=R, color=color, radii=radii, views=v, grads=dict(zip(GRAD_NAMES, grads)), bufs=(geom, binning, img))


# ------------------------------------------------------------------------------------------------------
# (a) golden vectors of the reference
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_against_reference_golden(C, dev, name):
    scene, gold = load_case(name)
    o = run_ours(C, synthetic.to_device(scene, dev))
    v = o["views"]
    vis = gold["radii"] > 0
    # integer artefacts: bit-exact
    assert o["R"] == int(gold["num_rendered"])
    assert np.array_equal(o["radii"].cpu().numpy(), gold["radii"])
    assert np.array_equal(v["tiles_touched"].cpu().numpy()[vis], gold["tiles_touched"][vis])
    assert np.array_equal(v["point_list"].cpu().numpy(), gold["point_list"]), "sorted instance list differs"
    assert np.array_equal(v["ranges"].cpu().numpy(), gold["ranges"])
    assert np.array_equal(v["n_contrib"].cpu().numpy(), gold["n_contrib"])
    # projected state: same bits (numerics notes N1/N2)
    rec = v["records"].cpu().numpy()
    assert np.array_equal(bits(v["depths"].cpu().numpy()[vis]), bits(gold["depths"][vis]))
    assert np.array_equal(bits(np.ascontiguousarray(rec[vis][:, 0:2])), bits(gold["means2D"][vis]))
    assert np.array_equal(bits(np.ascontiguousarray(rec[vis][:, 4:8])), bits(gold["conic_opacity"][vis]))
    if "shs" in scene:
        assert np.array_equal(bits(v["rgb"].cpu().numpy()[vis]), bits(gold["rgb"][vis]))
    # pixels and final_T: the reference's bits (render_fwd.cu numerics contract; tests/test_forward_exact.py bounds them)
    assert np.array_equal(bits(o["color"].cpu().numpy()), bits(gold["out_color"]))
    assert np.array_equal(bits(v["final_T"].cpu().numpy()), bits(gold["final_T"]))
    # gradients: 1e-3 of the tensor's largest magnitude
    for n in GRAD_NAMES:
        if gold[n].size:
            assert rel_err(o["grads"][n].cpu().numpy().reshape(gold[n].shape), gold[n]) < GRAD_TOL, n


# ------------------------------------------------------------------------------------------------------
# (b) the compiled reference, same process, same tensors
# ------------------------------------------------------------------------------------------------------
REF_SCENES = [
    dict(P=200_000, W=800, H=800, sh_degree=3, seed=21),
    dict(P=300_000, W=1000, H=700, sh_degree=None, seed=22),
    dict(P=50_000, W=333, H=211, sh_degree=2, seed=23, subpixel_jitter=0.5, bg=(1.0, 0.5, 0.25)),
    dict(P=20_000, W=640, H=360, sh_degree=None, seed=24, scale_range=(0.05, 0.5)),       # huge splats
    dict(P=100_000, W=512, H=512, sh_degree=None, seed=25, normalize_rot=False),
    dict(P=60_000, W=400, H=300, sh_degree=None, seed=26, cov3D_precomp=True),
    # more than 256 binning cells (8x8 tiles each): the coarse-item sort needs two radix passes
    dict(P=150_000, W=4096, H=2304, sh_degree=None, seed=27),
    # medium-to-large splats: binning units whose output exceeds the staging buffer (multi-walk scatter)
    dict(P=100_000, W=1280, H=720, sh_degree=None, seed=28, scale_range=(0.01, 0.15)),
    # SH tensors with 4 coefficients (128-bit row accesses) and 9 coefficients (rows not 16-byte multiples: scalar path)
    dict(P=30_000, W=320, H=240, sh_degree=1, max_sh_degree=1, seed=29),
    dict(P=30_000, W=320, H=240, sh_degree=2, max_sh_degree=2, seed=30),
    dict(P=30_000, W=320, H=240, sh_degree=1, max_sh_degree=3, seed=31),
]


def check_grad(name, ours, ref, ref_again, exact=None):
    """Gradient bar tied to the reference's own noise: the reference accumulates with float atomics, so two runs of
    it on the same inputs differ (`ref_noise`).  Ours must be within max(20 x that noise, 1e-5) of the tensor's largest
    magnitude -- two orders tighter than BASELINE.json's 1e-3 -- and every entry above 1e-3 of the maximum must
    also agree RELATIVELY within 2e-3 + the noise (small-gradient Gaussians are not hidden behind the largest one).

    The run-to-run noise understates the reference's error where its atomics are biased: in the |.| channel of
    dL/dmeans2D each pixel's term is added on its own to a sum that grows to 1e4-1e5, and terms below half an ulp of
    it are lost, so the reference sits up to ~4e-5 of the maximum below the fp64 value while two of its runs agree to
    ~2e-6 (measured at P=100k, 1280x720).  ``exact(name)`` (fp64 gradients of the same forward) then decides: ours
    must be within the same bar of fp64 and closer to it than the reference."""
    ours, ref, ref_again = ours.double(), ref.double(), ref_again.double()
    scale = float(ref.abs().max()) + 1e-30
    ours_err = float((ours - ref).abs().max()) / scale
    ref_noise = float((ref_again - ref).abs().max()) / scale
    bar = max(20.0 * ref_noise, 1e-5)
    if ours_err > bar and exact is not None:
        want = torch.as_tensor(np.asarray(exact(name), np.float64), device=ours.device).reshape(ours.shape)
        ours64 = float((ours - want).abs().max()) / scale
        ref64 = float((ref - want).abs().max()) / scale
        assert ours64 <= bar and ours64 < ref64, (name, "to fp64: ours", ours64, "reference", ref64, "bar", bar)
    else:
        assert ours_err <= bar, (name, ours_err, ref_noise)
    assert ours_err < GRAD_TOL, (name, ours_err)
    big = ref.abs() > 1e-3 * scale
    if bool(big.any()):
        noise_abs = (ref_again - ref).abs()
        rel = ((ours - ref).abs()[big] - 20.0 * noise_abs[big]).clamp_min(0) / ref.abs()[big]
        assert float(rel.max()) < 2e-3, (name, "per-element relative", float(rel.max()))
    return ours_err, ref_noise


@pytest.mark.parametrize("kw", REF_SCENES, ids=lambda k: f"P{k['P']}_{k['W']}x{k['H']}_s{k['seed']}")
def test_against_compiled_reference(C, dev, kw):
    from oracle import ref_cuda
    if not ref_cuda.available():
        pytest.skip("oracle/_ref/libdgr_ref.so not present")
    scene = synthetic.make_scene(**kw)
    d = synthetic.to_device(scene, dev)
    o = run_ours(C, d)
    R, color, radii, geom, binning, img = ref_cuda.rasterize_gaussians(*call_args(d))
    P = d["means3D"].shape[0]
    rv = ref_cuda.debug_views(geom, binning, img, P, d["image_width"], d["image_height"], R)
    rg = dict(zip(GRAD_NAMES, ref_cuda.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))))
    rg2 = dict(zip(GRAD_NAMES, ref_cuda.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))))
    torch.cuda.synchronize()
    v = o["views"]
    assert o["R"] == R
    assert torch.equal(o["radii"], radii)
    assert torch.equal(v["point_list"], rv["point_list"])
    assert torch.equal(v["ranges"], rv["ranges"])
    assert torch.equal(v["n_contrib"], rv["n_contrib"])
    vis = radii > 0
    assert torch.equal(v["depths"][vis].view(torch.int32), rv["depths"][vis].view(torch.int32))
    assert torch.equal(v["records"][vis][:, 0:2].contiguous().view(torch.int32), rv["means2D"][vis].view(torch.int32))
    assert torch.equal(v["records"][vis][:, 4:8].contiguous().view(torch.int32),
                       rv["conic_opacity"][vis].view(torch.int32))
    assert torch.equal(o["color"].view(torch.int32), color.view(torch.int32)), "pixels differ from the reference's bits"
    assert torch.equal(v["final_T"].view(torch.int32), rv["final_T"].view(torch.int32))
    g64 = {}

    def exact(n):         # fp64 gradients on the kernel's forward, computed only if a bar needs them
        if not g64:
            from test_adversarial_scenes import fp64_gradients
            from oracle import cpu_oracle
            st = cpu_oracle.forward(scene)
            g, flips = fp64_gradients(scene, st, v["final_T"].cpu().numpy(), v["n_contrib"].cpu().numpy())
            assert flips <= max(2, 1e-4 * v["n_contrib"].numel()), flips
            g64.update(g)
        return g64[n]

    for n in GRAD_NAMES:
        if rg[n].numel() == 0:
            continue
        check_grad(n, o["grads"][n].view_as(rg[n]), rg[n], rg2[n], exact)


# ------------------------------------------------------------------------------------------------------
# (c) the CPU oracle
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(P=20_000, W=320, H=240, sh_degree=3, seed=31),
                                dict(P=30_000, W=300, H=200, sh_degree=None, seed=32, subpixel_jitter=0.3)])
def test_against_cpu_oracle(C, dev, kw):
    from oracle import cpu_oracle
    scene = synthetic.make_scene(**kw)
    o = run_ours(C, synthetic.to_device(scene, dev))
    st = cpu_oracle.forward(scene)
    g = cpu_oracle.backward(st, scene["dL_dpix"])
    assert o["R"] == st["num_rendered"]
    assert np.array_equal(o["radii"].cpu().numpy(), st["radii"])
    assert np.array_equal(o["views"]["point_list"].cpu().numpy(), st["point_list"].astype(np.int32))
    assert np.array_equal(o["views"]["ranges"].cpu().numpy(), st["ranges"].astype(np.int32))
    assert np.abs(o["color"].cpu().numpy() - st["out_color"]).max() < PIX_TOL
    ne = (o["views"]["n_contrib"].cpu().numpy() != st["n_contrib"].astype(np.int32)).mean()
    assert ne <= 1e-4      # CUDA expf vs glibc expf can flip an alpha threshold
    for n in GRAD_NAMES:
        ref = g[n]
        if ref.size:
            assert rel_err(o["grads"][n].cpu().numpy().reshape(ref.shape), ref) < GRAD_TOL, n


# ------------------------------------------------------------------------------------------------------
# drop-in Python API (what wildgaussians/method.py:1529-1631 does)
# ------------------------------------------------------------------------------------------------------
def _settings(d, debug=False):
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    return GaussianRasterizationSettings(
        image_height=d["image_height"], image_width=d["image_width"], tanfovx=d["tanfovx"], tanfovy=d["tanfovy"],
        kernel_size=d["kernel_size"], subpixel_offset=d["subpixel_offset"], bg=d["bg"], scale_modifier=1.0,
        viewmatrix=d["viewmatrix"], projmatrix=d["projmatrix"], sh_degree=d["sh_degree"], campos=d["campos"],
        prefiltered=False, debug=debug, return_accumulation=True)


def test_autograd_two_passes_like_method_py(C, dev):
    """Two rasterizer calls on the same geometry (raw + toned colours), one backward: the shared
    `screenspace_points` gradient accumulates both passes (method.py:1495,1573-1611,1470-1477)."""
    from diff_gaussian_rasterization import GaussianRasterizer
    scene = synthetic.make_scene(P=30_000, W=320, H=208, sh_degree=None, seed=41)
    d = synthetic.to_device(scene, dev)
    leaves = {k: d[k].clone().requires_grad_(True) for k in ("means3D", "opacities", "scales", "rotations")}
    col_a = d["colors_precomp"].clone().requires_grad_(True)
    col_b = (1.0 - d["colors_precomp"]).clone().requires_grad_(True)
    means2D = torch.zeros_like(leaves["means3D"], requires_grad=True) + 0
    means2D.retain_grad()
    rast = GaussianRasterizer(_settings(d))
    kw = dict(means3D=leaves["means3D"], means2D=means2D, opacities=leaves["opacities"], scales=leaves["scales"],
              rotations=leaves["rotations"], shs=None, cov3D_precomp=None)
    C.set_geometry_cache(True)
    C.clear_geometry_cache()
    hits0 = C.geometry_cache_hits()
    img_a, radii, acc = rast(colors_precomp=col_a, **kw)
    img_b, radii_b, acc_b = rast(colors_precomp=col_b, **kw)
    # the second pass reused the projection / depth order / tile lists of the first (SURVEY 8f-1)
    assert C.geometry_cache_hits() == hits0 + 1
    assert img_a.shape == (3, 208, 320) and radii.dtype == torch.int32 and acc.shape == (208, 320)
    assert torch.equal(radii, radii_b) and torch.equal(acc, acc_b)
    (img_a * d["dL_dpix"]).sum().backward(retain_graph=True)
    g_a = {k: v.grad.clone() for k, v in leaves.items()}
    m2d_a = means2D.grad.clone()
    (img_b * d["dL_dpix"]).sum().backward()
    torch.cuda.synchronize()
    # reference values from the raw C-level call
    o_a = run_ours(C, d)
    d_b = dict(d); d_b["colors_precomp"] = (1.0 - d["colors_precomp"]).contiguous()
    o_b = run_ours(C, d_b)
    assert torch.equal(img_a.detach(), o_a["color"]) and torch.equal(img_b.detach(), o_b["color"])
    fT = o_a["views"]["final_T"]
    assert torch.allclose(acc, 1.0 - fT)
    for k, n in (("means3D", "dL_dmeans3D"), ("scales", "dL_dscales"), ("rotations", "dL_drotations"),
                 ("opacities", "dL_dopacity")):
        ref_a = o_a["grads"][n].view_as(g_a[k])
        assert rel_err(g_a[k].cpu().numpy(), ref_a.cpu().numpy()) < GRAD_TOL
        both = ref_a + o_b["grads"][n].view_as(ref_a)
        assert rel_err(leaves[k].grad.cpu().numpy(), both.cpu().numpy()) < GRAD_TOL
    assert rel_err(m2d_a.cpu().numpy(), o_a["grads"]["dL_dmeans2D"].cpu().numpy()) < GRAD_TOL
    assert rel_err(col_a.grad.cpu().numpy(), o_a["grads"]["dL_dcolors"].cpu().numpy()) < GRAD_TOL
    assert (means2D.grad[:, 2] >= 0).all()          # abs-gradient channel


def test_geometry_cache_is_invalidated_by_in_place_updates(C, dev):
    """The reuse keys on tensor identity + version: an optimizer-style in-place update, another tensor object, other
    settings or a disabled cache all force a full forward; a hit gives bit-identical outputs."""
    scene = synthetic.make_scene(P=20_000, W=256, H=160, sh_degree=None, seed=43)
    d = synthetic.to_device(scene, dev)
    C.set_geometry_cache(True)
    C.clear_geometry_cache()
    args = list(call_args(d))
    h0 = C.geometry_cache_hits()
    R1, c1, radii1, g1, b1, i1 = C.rasterize_gaussians(*args)
    R2, c2, radii2, g2, b2, i2 = C.rasterize_gaussians(*args)
    assert C.geometry_cache_hits() == h0 + 1
    assert R1 == R2 and torch.equal(c1, c2) and torch.equal(radii1, radii2)
    assert g2.data_ptr() == g1.data_ptr() and b2.data_ptr() == b1.data_ptr() and i2.data_ptr() != i1.data_ptr()
    v1 = C.debug_views(g1, b1, i1, d["means3D"].shape[0], 0, 256, 160, R1)
    v2 = C.debug_views(g2, b2, i2, d["means3D"].shape[0], 0, 256, 160, R2)
    for k in ("final_T", "n_contrib", "ranges", "point_list"):
        assert torch.equal(v1[k], v2[k]), k
    # in-place update of a geometry input -> version bump -> miss, and the new result reflects the update
    d["means3D"].mul_(1.001)
    R3, c3, *_ = C.rasterize_gaussians(*args)
    assert C.geometry_cache_hits() == h0 + 1
    assert not torch.equal(c3, c1)
    # a different colour tensor alone is a hit; a different opacity tensor object is a miss
    args_c = list(args); args_c[2] = (1.0 - d["colors_precomp"]).contiguous()
    C.rasterize_gaussians(*args_c)
    assert C.geometry_cache_hits() == h0 + 2
    args_o = list(args); args_o[3] = d["opacities"].clone()
    C.rasterize_gaussians(*args_o)
    assert C.geometry_cache_hits() == h0 + 2
    C.set_geometry_cache(False)
    C.rasterize_gaussians(*args_o)
    C.rasterize_gaussians(*args_o)
    assert C.geometry_cache_hits() == h0 + 2
    C.set_geometry_cache(True)


def test_sh_path_and_debug_flag(C, dev):
    from diff_gaussian_rasterization import GaussianRasterizer
    scene = synthetic.make_scene(P=5_000, W=160, H=96, sh_degree=2, seed=42)
    d = synthetic.to_device(scene, dev)
    shs = d["shs"].clone().requires_grad_(True)
    means2D = torch.zeros_like(d["means3D"], requires_grad=True)
    img, radii, acc = GaussianRasterizer(_settings(d, debug=True))(
        means3D=d["means3D"], means2D=means2D, opacities=d["opacities"], shs=shs, scales=d["scales"],
        rotations=d["rotations"])
    (img * d["dL_dpix"]).sum().backward()
    o = run_ours(C, d)
    assert torch.equal(img.detach(), o["color"])
    assert rel_err(shs.grad.cpu().numpy(), o["grads"]["dL_dsh"].cpu().numpy()) < GRAD_TOL
    # coefficients above the active degree (2) get no gradient
    assert float(shs.grad[:, 9:].abs().max()) == 0.0


def test_mark_visible(C, dev):
    from diff_gaussian_rasterization import GaussianRasterizer
    scene = synthetic.make_scene(P=10_000, W=64, H=64, sh_degree=None, seed=43)
    d = synthetic.to_device(scene, dev)
    vis = GaussianRasterizer(_settings(d)).markVisible(d["means3D"])
    assert vis.dtype == torch.bool
    assert torch.equal(vis.cpu(), scene["means3D"][:, 2] > 0.2)


# ------------------------------------------------------------------------------------------------------
# edge cases
# ------------------------------------------------------------------------------------------------------
def test_empty_cloud(C, dev):
    scene = synthetic.make_scene(P=10, W=70, H=50, sh_degree=None, seed=44, bg=(0.1, 0.2, 0.3))
    for k in ("means3D", "opacities", "scales", "rotations", "colors_precomp"):
        scene[k] = scene[k][:0]
    d = synthetic.to_device(scene, dev)
    R, color, radii, geom, binning, img = C.rasterize_gaussians(*call_args(d))
    assert R == 0 and radii.numel() == 0 and color.shape == (3, 50, 70)
    assert float(color.abs().max()) == 0.0       # the reference skips everything for P == 0 (rasterize_points.cu:83)
    grads = C.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))
    assert all(g.shape[0] == 0 for g in grads)


def test_everything_culled_renders_background(C, dev):
    scene = synthetic.make_scene(P=1000, W=70, H=50, sh_degree=None, seed=45, bg=(0.1, 0.2, 0.3))
    scene["means3D"][:, 2] = -scene["means3D"][:, 2].abs() - 1
    d = synthetic.to_device(scene, dev)
    o = run_ours(C, d)
    assert o["R"] == 0 and int(o["radii"].abs().max()) == 0
    assert torch.allclose(o["color"], d["bg"][:, None, None].expand(3, 50, 70))
    assert all(float(g.abs().max()) == 0 for g in o["grads"].values() if g.numel())


def test_tile_row_shards_compose(C, dev):
    """The multi-GPU partition: bands rendered separately reproduce the full image bit for bit and their
    per-Gaussian gradients sum to the full gradients."""
    scene = synthetic.make_scene(P=40_000, W=300, H=212, sh_degree=None, seed=46)
    d = synthetic.to_device(scene, dev)
    full = run_ours(C, d)
    rows = (212 + 15) // 16
    parts = []
    try:
        for y0, y1 in ((0, 5), (5, 9), (9, rows)):
            C.set_tile_row_shard(y0, y1)
            parts.append(((y0, y1), run_ours(C, d)))
    finally:
        C.set_tile_row_shard(0, 0)
    assert sum(p["R"] for _, p in parts) == full["R"]
    img = torch.zeros_like(full["color"])
    for (y0, y1), p in parts:
        assert torch.equal(p["radii"], full["radii"])
        img[:, 16 * y0:16 * y1] = p["color"][:, 16 * y0:16 * y1]
    assert torch.equal(img, full["color"])
    for n in GRAD_NAMES:
        tot = sum(p["grads"][n] for _, p in parts)
        if tot.numel():
            assert rel_err(tot.cpu().numpy(), full["grads"][n].cpu().numpy()) < GRAD_TOL, n


def test_prefiltered_violation_raises(C, dev):
    scene = synthetic.make_scene(P=2000, W=64, H=64, sh_degree=None, seed=47)
    d = synthetic.to_device(scene, dev)
    args = list(call_args(d)); args[19] = True
    with pytest.raises(RuntimeError, match="filtered although prefiltered"):
        C.rasterize_gaussians(*args)


# ------------------------------------------------------------------------------------------------------
# size-independent properties at BASELINE.json's full sizes
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", ["C2", "C3", "C5"])
def test_full_size_properties(C, dev, cfg):
    kw = dict(synthetic.CONFIGS[cfg]); kw["seed"] = 0
    scene = synthetic.make_scene(**kw)
    d = synthetic.to_device(scene, dev)
    o = run_ours(C, d)
    v, R = o["views"], o["R"]
    W, H = d["image_width"], d["image_height"]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    tiles = v["tiles_touched"].long()
    vis = o["radii"] > 0
    # R is the sum of the tile counts of the rendered Gaussians
    assert int(tiles[vis].sum()) == R
    # the tile ranges partition [0, R) in tile order
    rg = v["ranges"].long()
    ne = rg[:, 1] > rg[:, 0]
    assert int((rg[ne, 1] - rg[ne, 0]).sum()) == R
    starts, ends = rg[ne, 0], rg[ne, 1]
    assert int(starts[0]) == 0 and int(ends[-1]) == R and torch.equal(starts[1:], ends[:-1])
    # inside every tile the list is ordered by depth, ties by Gaussian index (stable sort, note N4)
    pl = v["point_list"].long()
    depth_bits = v["depths"].view(torch.int32).long()[pl]
    tile_of = torch.repeat_interleave(torch.arange(T, device=dev)[ne], (ends - starts))
    key = (tile_of << 32) | depth_bits
    assert bool((key[1:] >= key[:-1]).all()), "instance list is not (tile, depth) sorted"
    same = key[1:] == key[:-1]
    assert bool((pl[1:][same] > pl[:-1][same]).all()), "depth ties are not in Gaussian-index order"
    # histogram of Gaussian ids in the list == tiles_touched
    assert torch.equal(torch.bincount(pl, minlength=tiles.numel()), tiles * vis)
    # n_contrib never exceeds the tile's list length; transmittance in [0, 1]
    lens = (rg[:, 1] - rg[:, 0]).view((H + 15) // 16, (W + 15) // 16)
    per_pix = lens.repeat_interleave(16, 0).repeat_interleave(16, 1)[:H, :W]
    assert bool((v["n_contrib"].long() <= per_pix).all())
    assert float(v["final_T"].min()) >= 0.0 and float(v["final_T"].max()) <= 1.0
    # the forward is deterministic: a second run gives the same bits
    o2 = run_ours(C, d)
    assert torch.equal(o2["color"], o["color"]) and torch.equal(o2["views"]["point_list"], v["point_list"])
    # the backward is linear in the upstream gradient
    d2 = dict(d); d2["dL_dpix"] = 2.0 * d["dL_dpix"]
    R2, color2, radii2, geom, binning, img = C.rasterize_gaussians(*call_args(d2))
    g2 = dict(zip(GRAD_NAMES, C.rasterize_gaussians_backward(*backward_args(d2, radii2, geom, R2, binning, img))))
    for n in ("dL_dmeans3D", "dL_dopacity", "dL_dscales", "dL_dcolors"):
        if g2[n].numel():
            assert rel_err(g2[n].cpu().numpy(), 2.0 * o["grads"][n].cpu().numpy()) < GRAD_TOL, n
    # invisible Gaussians get exactly zero gradient
    for n in ("dL_dmeans3D", "dL_dscales", "dL_drotations", "dL_dopacity"):
        if o["grads"][n].numel():
            assert float(o["grads"][n][~vis].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------------
# the BENCHMARKED configurations, value-checked against the compiled reference (same process, same tensors)
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", ["C2", "C3", "C5"])
def test_benchmarked_config_against_compiled_reference(C, dev, cfg):
    """BASELINE.json configs 2 (500k, 800x800, SH degree 3 in-kernel), 3 (3M, 1080p, colours precomputed -- the
    bench.py workload) and 5 on one GPU (6M, 4096x2160): R, radii, the sorted instance list, the tile ranges and
    n_contrib bit-exact; pixels and final_T the reference's bits; all gradient tensors within the noise-tied bar of
    check_grad."""
    from oracle import ref_cuda
    if not ref_cuda.available():
        pytest.skip("oracle/_ref/libdgr_ref.so not present")
    kw = dict(synthetic.CONFIGS[cfg]); kw["seed"] = 0
    scene = synthetic.make_scene(**kw)
    d = synthetic.to_device(scene, dev)
    C.set_geometry_cache(False)
    o = run_ours(C, d)
    R, color, radii, geom, binning, img = ref_cuda.rasterize_gaussians(*call_args(d))
    P = d["means3D"].shape[0]
    rv = ref_cuda.debug_views(geom, binning, img, P, d["image_width"], d["image_height"], R)
    v = o["views"]
    assert o["R"] == R
    assert torch.equal(o["radii"], radii)
    assert torch.equal(v["ranges"], rv["ranges"])
    assert torch.equal(v["point_list"], rv["point_list"]), "sorted instance list differs"
    assert torch.equal(v["n_contrib"], rv["n_contrib"])
    assert torch.equal(o["color"].view(torch.int32), color.view(torch.int32)), \
        float((o["color"] - color).abs().max())
    assert torch.equal(v["final_T"].view(torch.int32), rv["final_T"].view(torch.int32))
    bargs = backward_args(d, radii, geom, R, binning, img)
    rg = dict(zip(GRAD_NAMES, ref_cuda.rasterize_gaussians_backward(*bargs)))
    rg2 = dict(zip(GRAD_NAMES, ref_cuda.rasterize_gaussians_backward(*bargs)))
    torch.cuda.synchronize()
    for n in GRAD_NAMES:
        if rg[n].numel() == 0 or (n == "dL_dcov3D"):     # dL_dcov3D is an intermediate with scales/rotations given
            continue
        check_grad(n, o["grads"][n].view_as(rg[n]), rg[n], rg2[n])
    C.set_geometry_cache(True)


def test_gsr_forward_through_the_allocation_callback(C, dev):
    """gsr_forward() -- the single call INTEGRATION.md tells a maintainer to bind, with the C allocation callback
    standing in for the reference's three resize lambdas (rasterize_points.cu:27-33,78-80) -- gives the same image,
    radii and instance list as the staged entry points the Python shim uses."""
    import ctypes
    from ctypes import CFUNCTYPE, byref, c_int, c_size_t, c_void_p
    scene = synthetic.make_scene(P=50_000, W=400, H=304, sh_degree=2, seed=51)
    d = synthetic.to_device(scene, dev)
    o = run_ours(C, d)
    P, W, H, M = 50_000, 400, 304, d["shs"].shape[1]
    a = C.GsrForwardArgs()
    a.P, a.D, a.M, a.W, a.H = P, d["sh_degree"], M, W, H
    out_color = torch.zeros((3, H, W), device=dev)
    radii = torch.zeros((P,), dtype=torch.int32, device=dev)
    for name, key in (("background", "bg"), ("means3D", "means3D"), ("shs", "shs"), ("opacities", "opacities"),
                      ("scales", "scales"), ("rotations", "rotations"), ("viewmatrix", "viewmatrix"),
                      ("projmatrix", "projmatrix"), ("campos", "campos"), ("subpixel_offset", "subpixel_offset")):
        setattr(a, name, d[key].contiguous().data_ptr())
    a.scale_modifier, a.tan_fovx, a.tan_fovy, a.kernel_size = 1.0, d["tanfovx"], d["tanfovy"], d["kernel_size"]
    a.out_color, a.radii = out_color.data_ptr(), radii.data_ptr()
    bufs, calls = {}, []

    @CFUNCTYPE(c_void_p, c_void_p, c_int, c_size_t)
    def alloc(_ctx, which, nbytes):
        calls.append((which, nbytes))
        bufs[which] = torch.empty((int(nbytes) + 256,), dtype=torch.uint8, device=dev)
        p = bufs[which].data_ptr()
        return (p + 255) // 256 * 256

    lib = C._lib
    lib.gsr_forward.argtypes = [ctypes.POINTER(C.GsrForwardArgs), CFUNCTYPE(c_void_p, c_void_p, c_int, c_size_t), c_void_p,
                                c_void_p, ctypes.POINTER(c_int)]
    lib.gsr_forward.restype = c_int
    R = c_int(0)
    rc = lib.gsr_forward(byref(a), alloc, None, torch.cuda.current_stream(dev).cuda_stream, byref(R))
    torch.cuda.synchronize()
    assert rc == 0, lib.gsr_last_error()
    assert sorted(w for w, _ in calls) == [0, 1, 2, 3]          # GEOM, BINNING, IMG, SCRATCH each asked once
    assert R.value == o["R"]
    assert torch.equal(out_color, o["color"]) and torch.equal(radii, o["radii"])
    pl = c_void_p()
    binning_ptr = (bufs[1].data_ptr() + 255) // 256 * 256
    assert lib.gsr_binning_views(binning_ptr, R.value, byref(pl)) == 0
    off = pl.value - bufs[1].data_ptr()
    mine = bufs[1][off:off + 4 * R.value].view(torch.int32)
    assert torch.equal(mine, o["views"]["point_list"])
    # NULL callback is rejected with a message
    assert lib.gsr_forward(byref(a), CFUNCTYPE(c_void_p, c_void_p, c_int, c_size_t)(0), None, None, byref(R)) == -1


def test_geometry_cache_hits_with_a_non_contiguous_view_matrix(C, dev):
    """wildgaussians/method.py:1516 passes `torch.tensor(...).transpose(0, 1).to(device)` -- a NON-contiguous view matrix
    whose contiguous copy is a new tensor on every call.  The reuse is keyed on the caller's own tensor objects, so
    the second composite of a step still hits; the caller's radii tensor is its own copy."""
    scene = synthetic.make_scene(P=20_000, W=256, H=160, sh_degree=None, seed=44)
    d = synthetic.to_device(scene, dev)
    d["viewmatrix"] = d["viewmatrix"].t().contiguous().t()      # same values, transposed strides
    d["projmatrix"] = d["projmatrix"].t().contiguous().t()
    assert not d["viewmatrix"].is_contiguous()
    C.set_geometry_cache(True)
    C.clear_geometry_cache()
    args = list(call_args(d))
    h0 = C.geometry_cache_hits()
    R1, c1, radii1, g1, b1, i1 = C.rasterize_gaussians(*args)
    radii1.zero_()                                              # a caller scribbling over its radii ...
    R2, c2, radii2, g2, b2, i2 = C.rasterize_gaussians(*args)
    assert C.geometry_cache_hits() == h0 + 1
    assert torch.equal(c1, c2) and int(radii2.max()) > 0        # ... does not corrupt the cached state
    ref = run_ours(C, d)                                        # (its backward drops the cache entry)
    assert torch.equal(ref["color"], c1) and torch.equal(ref["radii"], radii2)
    R3, *_ = C.rasterize_gaussians(*args)
    assert C.geometry_cache_hits() == h0 + 2                    # (run_ours' forward hit too) the entry was released when its backward started


def test_render_counts_too_small_for_the_scene_render_nothing(C, dev):
    """gsr_forward_render takes the instance and coarse-item counts from its caller.  Counts smaller than the scene's
    bin nothing (empty tile ranges, no write beyond the buffers sized for them) and leave the background; a following
    call with the right counts on the same geometry is bit-identical to the ordinary forward."""
    from ctypes import byref, c_size_t
    scene = synthetic.make_scene(P=60_000, W=480, H=320, sh_degree=None, seed=52, bg=(0.2, 0.1, 0.3))
    d = synthetic.to_device(scene, dev)
    C.set_geometry_cache(False)
    want = run_ours(C, d)
    P, W, H = d["means3D"].shape[0], d["image_width"], d["image_height"]
    out_color, radii = torch.empty((3, H, W), device=dev), torch.empty((P,), dtype=torch.int32, device=dev)
    a = C.forward_args(background=d["bg"], means3D=d["means3D"], colors=d["colors_precomp"], opacities=d["opacities"],
                       scales=d["scales"], rotations=d["rotations"], viewmatrix=d["viewmatrix"],
                       projmatrix=d["projmatrix"], campos=d["campos"], tan_fovx=d["tanfovx"], tan_fovy=d["tanfovy"],
                       kernel_size=d["kernel_size"], subpixel_offset=d["subpixel_offset"], H=H, W=W, radii=radii,
                       out_color=out_color)
    stream = torch.cuda.current_stream(dev).cuda_stream
    geom, img, binning, scratch, R, N1 = C._forward_geometry(a, dev, stream)
    assert R == want["R"] and R > 1 and N1 > 1
    for r, n1 in ((1, 1), (0, 0)):
        bb, sb = c_size_t(0), c_size_t(0)
        C._check(C._lib.gsr_binning_sizes(P, W, H, r, n1, byref(bb), byref(sb)), "gsr_binning_sizes")
        small_bin = torch.empty((bb.value,), dtype=torch.uint8, device=dev)
        small_scratch = torch.empty((sb.value,), dtype=torch.uint8, device=dev)
        out_color.fill_(float("nan"))
        C._check(C._lib.gsr_forward_render(byref(a), geom.data_ptr(), img.data_ptr(), small_bin.data_ptr(),
                                           small_scratch.data_ptr(), r, n1, stream), "gsr_forward_render")
        ranges = C.debug_views(geom, small_bin, img, P, 0, W, H, 0)["ranges"]
        torch.cuda.synchronize()
        assert torch.equal(ranges[:, 0], ranges[:, 1]), (r, n1)
        assert torch.equal(out_color, d["bg"].view(3, 1, 1).expand(3, H, W)), (r, n1)
    C._check(C._lib.gsr_forward_render(byref(a), geom.data_ptr(), img.data_ptr(), binning.data_ptr(), scratch.data_ptr(),
                                       R, N1, stream), "gsr_forward_render")
    v = C.debug_views(geom, binning, img, P, 0, W, H, R)
    torch.cuda.synchronize()
    assert torch.equal(out_color, want["color"]) and torch.equal(radii, want["radii"])
    for k in ("point_list", "ranges", "n_contrib", "final_T"):
        assert torch.equal(v[k], want["views"][k]), k
    C.set_geometry_cache(True)


def test_defer_composite_inputs_waits_before_the_composite(C, dev):
    """Host-buffer pipelines: the forward may be started when only the geometry inputs are on the device; the composite
    stage waits for the event that marks the arrival of colours / background / sub-pixel offsets."""
    import diff_gaussian_rasterization as dgr
    scene = synthetic.make_scene(P=30_000, W=320, H=208, sh_degree=None, seed=53, bg=(0.2, 0.1, 0.3), subpixel_jitter=0.4)
    d = synthetic.to_device(scene, dev)
    ref = run_ours(C, d)
    C.set_geometry_cache(False)
    side = torch.cuda.Stream(dev)
    host = {k: scene[k].contiguous().pin_memory() for k in ("colors_precomp", "bg", "subpixel_offset")}
    late = {k: torch.zeros_like(d[k]) for k in host}            # wrong values until the side stream has delivered
    ev = torch.cuda.Event()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                           # ~0.1 s: the copies land long after the forward was issued
        for k in host:
            late[k].copy_(host[k], non_blocking=True)
        ev.record(side)
    d2 = dict(d); d2.update(late)
    dgr.defer_composite_inputs(ev)
    R, color, radii, geom, binning, img = C.rasterize_gaussians(*call_args(d2))
    torch.cuda.synchronize()
    assert torch.equal(color, ref["color"]) and R == ref["R"]
    assert C._render_wait["event"] is None                       # one-shot
    C.set_geometry_cache(True)
