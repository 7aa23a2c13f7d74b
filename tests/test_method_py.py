"""The reference's own ``wildgaussians/method.py``, UNMODIFIED, running on the drop-in package (SURVEY.md 4.5,
BASELINE.json north star: "so wildgaussians/method.py drops onto it unchanged").

``GaussianModel._render_internal`` (method.py:1479-1632; appearance on, uncertainty off) is executed once on this repo's
``diff_gaussian_rasterization`` and once on the reference's compiled CUDA rasterizer behind the same two names; images,
radii, accumulation and every parameter gradient of a train-step-like loss must agree.  It is also the real call
pattern of the geometry reuse (SURVEY 8f-1): two rasterizer calls per step on the same geometry tensors, the view
matrix a non-contiguous transposed tensor (method.py:1516) -> exactly one cache hit per step.
"""
import os
import sys

import pytest
import torch

import synthetic
import wg_harness as wh

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ref_api():
    from oracle import ref_cuda
    if not ref_cuda.available():
        pytest.skip("oracle/_ref/libdgr_ref.so not present")
    sys.path.insert(0, ROOT)
    import bench
    return bench.make_reference_api(ref_cuda)


@pytest.mark.parametrize("kw", [dict(P=150_000, W=640, H=400, seed=61), dict(P=40_000, W=333, H=211, seed=62)],
                         ids=lambda k: f"P{k['P']}_{k['W']}x{k['H']}")
def test_render_internal_on_the_drop_in_equals_reference_backend(kw, ref_api):
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    import diff_gaussian_rasterization as ours
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    scene = synthetic.make_scene(sh_degree=3, **kw)
    model, cfg = wh.make_model(m, Config, scene, dev, seed=kw["seed"])
    cam = wh.make_camera(scene)
    g = torch.Generator().manual_seed(kw["seed"] + 100)
    G1 = torch.randn(3, kw["H"], kw["W"], generator=g).to(dev)
    G2 = torch.randn(3, kw["H"], kw["W"], generator=g).to(dev)

    # ---- ours: the names method.py imported at :26 ARE this package's
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    _C.set_geometry_cache(True)
    _C.clear_geometry_cache()
    h0 = _C.geometry_cache_hits()
    a = wh.collect(model, wh.train_step(model, cfg, cam, G1, G2))
    assert _C.geometry_cache_hits() == h0 + 1, "the second composite of the step did not reuse the first one's geometry"
    a2 = wh.collect(model, wh.train_step(model, cfg, cam, G1, G2))      # next step: fresh tensors -> miss, then hit
    assert _C.geometry_cache_hits() == h0 + 2
    assert torch.equal(a["render"], a2["render"]) and torch.equal(a["raw_render"], a2["raw_render"])

    # ---- the reference's compiled CUDA core behind the same two names
    wh.use_backend(m, ref_api["GaussianRasterizer"], ref_api["GaussianRasterizationSettings"])
    b = wh.collect(model, wh.train_step(model, cfg, cam, G1, G2))
    b2 = wh.collect(model, wh.train_step(model, cfg, cam, G1, G2))      # the reference's own atomic-order noise
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    torch.cuda.synchronize()

    assert torch.equal(a["radii"], b["radii"])
    assert float((a["render"] - b["render"]).abs().max()) <= 1e-4
    assert float((a["raw_render"] - b["raw_render"]).abs().max()) <= 1e-4
    assert float((a["accumulation"] - b["accumulation"]).abs().max()) <= 1e-4
    assert float(a["render"].abs().max()) > 0.05 and float((a["render"] - a["raw_render"]).abs().max()) > 1e-3
    for k in a:
        if not (k.startswith("g_") or k == "viewspace_grad"):
            continue
        scale = float(b[k].abs().max()) + 1e-30
        err = float((a[k] - b[k]).abs().max()) / scale
        noise = float((b2[k] - b[k]).abs().max()) / scale
        assert err <= max(20.0 * noise, 2e-5), (k, err, noise)
        assert err < 1e-3, (k, err)


def test_fused_render_internal_matches_the_reference_method():
    """wildgaussians_fused.enable(model): same output dictionary as the unmodified ``_render_internal`` -- images within
    1e-3 (the MLP runs with bf16 operands, its output is scaled by 0.01), rasterizer-side gradients within 1e-3, gradients
    that pass through the MLP in direction and size (cosine >= 0.99; see tests/test_appearance.py for why not entry-wise)."""
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    import diff_gaussian_rasterization as ours
    import wildgaussians_fused as wf
    dev = torch.device("cuda:0")
    kw = dict(P=120_000, W=640, H=400, seed=63)
    scene = synthetic.make_scene(sh_degree=3, **kw)
    model, cfg = wh.make_model(m, Config, scene, dev, seed=63)
    cam = wh.make_camera(scene)
    g = torch.Generator().manual_seed(163)
    G1, G2 = torch.randn(3, 400, 640, generator=g).to(dev), torch.randn(3, 400, 640, generator=g).to(dev)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    ours._C.set_geometry_cache(True)
    a = wh.collect(model, wh.train_step(model, cfg, cam, G1, G2))
    wf.enable(model)
    h0 = ours._C.geometry_cache_hits()
    b = wh.collect(model, wh.train_step(model, cfg, cam, G1, G2))
    assert ours._C.geometry_cache_hits() == h0 + 1
    wf.disable(model)
    c = wh.collect(model, wh.train_step(model, cfg, cam, G1, G2))
    torch.cuda.synchronize()
    assert torch.equal(a["render"], c["render"])                       # disable() restores the original method
    assert torch.equal(a["radii"], b["radii"])
    # the raw colours agree to fp32 rounding (different summation order of the 16 SH terms); a pixel sums hundreds of them
    assert float((a["raw_render"] - b["raw_render"]).abs().max()) < 2e-4
    assert float((a["render"] - b["render"]).abs().max()) < 1e-3
    for k in a:
        if not (k.startswith("g_") or k == "viewspace_grad"):
            continue
        x, y = b[k].double().flatten(), a[k].double().flatten()
        cos = float(x @ y) / (float(x.norm()) * float(y.norm()) + 1e-300)
        ratio = float(x.norm()) / (float(y.norm()) + 1e-300)
        assert cos >= 0.99 and abs(ratio - 1) < 0.03, (k, cos, ratio)
        if k in ("g_xyz", "g_scales", "g_rotations", "g_opacities", "viewspace_grad"):
            # the colours feeding the rasterizer differ by ~1e-5, the geometry gradients follow
            assert float((b[k] - a[k]).abs().max()) / (float(a[k].abs().max()) + 1e-30) < 2e-3, k


def test_densification_stats_kernel_matches_the_reference_statements():
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    import wildgaussians_fused as wf
    dev = torch.device("cuda:0")
    P = 50_001
    scene = synthetic.make_scene(P=P, W=64, H=48, sh_degree=3, seed=64)
    g = torch.Generator().manual_seed(7)
    radii = (torch.randint(0, 40, (P,), generator=g) * (torch.rand(P, generator=g) > 0.3)).to(torch.int32).to(dev)
    vsp = torch.zeros(P, 3, device=dev, requires_grad=True)
    vsp.grad = torch.randn(P, 3, generator=g).to(dev)
    models = []
    for _ in range(2):
        model, cfg = wh.make_model(m, Config, scene, dev, seed=64)
        gg = torch.Generator().manual_seed(8)
        for name in ("max_radii2D", "xyz_grad", "denom", "xyz_gradient_accum_abs", "xyz_gradient_accum_abs_max"):
            getattr(model, name).copy_(torch.rand(getattr(model, name).shape, generator=gg).to(dev) * 5)
        models.append(model)
    ref, fused = models
    vis = radii > 0                                                    # method.py:1997-1998
    ref.max_radii2D[vis] = torch.max(ref.max_radii2D[vis], radii[vis])
    ref.add_densification_stats(vsp, vis)
    wf.densification_stats(fused, vsp, radii)
    torch.cuda.synchronize()
    for name in ("max_radii2D", "xyz_grad", "denom", "xyz_gradient_accum_abs", "xyz_gradient_accum_abs_max"):
        assert torch.allclose(getattr(ref, name), getattr(fused, name), rtol=1e-6, atol=1e-6), name
