"""Inference render on one display composite (``fused_render``, ``wildgaussians_fused.enable_method(method, render=True)``).

CPU: the C entry point's argument checks, the dispatch predicate for every fall-back condition, and the hook's binding.
GPU: colour and accumulation bit for bit those of ``WildGaussians.render`` under ``enable_method(method)``, depth within
1e-6 of the largest visible distance, the shipped method within 1e-3 (colour) and 1e-4 (accumulation), the display epilogue
against the ordinary composite on colours the test supplies, edge cases, fresh result arrays, the host synchronisations
and copies of a profiled call, and both reference evaluation protocols.
"""
from __future__ import annotations

import ctypes
import sys
import types

import numpy as np
import pytest
import torch


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_display_entry_point_validates_its_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib
    E = -1
    assert lib.gsr_forward_display(None, None, None, None, None, None, 0, 0, None) == E
    assert b"NULL" in lib.gsr_last_error()
    a, d = _C.GsrForwardArgs(), _C.GsrDisplayArgs()
    a.P, a.W, a.H = -1, 16, 16
    assert lib.gsr_forward_display(ctypes.byref(a), ctypes.byref(d), None, None, None, None, 0, 0, None) == E
    assert b"bad sizes" in lib.gsr_last_error()
    a.P = 10
    assert lib.gsr_forward_display(ctypes.byref(a), ctypes.byref(d), None, None, None, None, 0, 0, None) == E
    assert b"NULL" in lib.gsr_last_error()                                  # every pointer NULL
    for f in ("means3D", "opacities", "viewmatrix", "projmatrix", "background", "subpixel_offset", "radii",
              "colors_precomp", "scales", "rotations", "campos"):
        setattr(a, f, 256)                                                  # never dereferenced: every call fails first
    assert lib.gsr_forward_display(ctypes.byref(a), ctypes.byref(d), None, None, None, None, 0, 0, None) == E
    assert b"NULL" in lib.gsr_last_error()                                  # no display image
    d.out_color = 256
    a.tile_y0, a.tile_y1 = 0, 1
    assert lib.gsr_forward_display(ctypes.byref(a), ctypes.byref(d), None, None, None, None, 0, 0, None) == E
    assert b"tile-row shard" in lib.gsr_last_error()
    a.tile_y0, a.tile_y1 = 0, 0
    a.peer_images, a.n_peer_images = 256, 1
    assert lib.gsr_forward_display(ctypes.byref(a), ctypes.byref(d), None, None, None, None, 0, 0, None) == E
    assert b"peer images" in lib.gsr_last_error()
    a.peer_images, a.n_peer_images = None, 0
    assert lib.gsr_forward_display(ctypes.byref(a), ctypes.byref(d), None, None, None, None, -1, 0, None) == E
    assert b"bad counts" in lib.gsr_last_error()
    assert lib.gsr_forward_display(ctypes.byref(a), ctypes.byref(d), None, None, None, None, 0, 0, None) == E
    assert b"out_accum" in lib.gsr_last_error()
    d.out_accum, d.depth = 256, 1
    assert lib.gsr_forward_display(ctypes.byref(a), ctypes.byref(d), None, None, None, None, 0, 0, None) == E
    assert b"out_depth" in lib.gsr_last_error()
    d.out_depth = 256
    assert lib.gsr_forward_display(ctypes.byref(a), ctypes.byref(d), None, None, None, None, 0, 0, None) == E
    assert b"depth_scratch" in lib.gsr_last_error()
    d.depth_scratch = 256
    assert lib.gsr_forward_display(ctypes.byref(a), ctypes.byref(d), None, None, None, None, 5, 5, None) == E
    assert b"buffer is NULL" in lib.gsr_last_error()
    a.P = 0                                                                 # no Gaussians: nothing to do
    assert lib.gsr_forward_display(ctypes.byref(a), ctypes.byref(d), None, None, None, None, 0, 0, None) == 0


def camera_model_to_int(name):          # looked up in the model class's module, as in wildgaussians/method.py
    return {"pinhole": 0}.get(name, 1)


class _FakeModel(types.SimpleNamespace):
    pass


def _fake_method(cuda=True, appearance=True, debug=False, model_sh=False, P=10, dtype=torch.float32):
    t = lambda *s: types.SimpleNamespace(is_cuda=cuda, dtype=dtype, shape=s)
    mlp = torch.nn.Sequential(torch.nn.Linear(59, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128), torch.nn.ReLU(),
                              torch.nn.Linear(128, 6))
    cfg = types.SimpleNamespace(appearance_enabled=appearance, appearance_separate_tuned_color=True,
                                appearance_model_sh=model_sh, sh_degree=3, appearance_embedding_dim=32, debug=debug)
    model = _FakeModel(config=cfg, xyz=t(P, 3), features_dc=t(P, 3), features_rest=t(P, 45), embeddings=t(P, 24),
                       scales=t(P, 3), opacities=t(P, 1), rotations=t(P, 4), filter_3D=t(P, 1),
                       appearance_embeddings=t(4, 32), appearance_mlp=types.SimpleNamespace(mlp=mlp))
    return types.SimpleNamespace(model=model, config=cfg)


def _fake_camera(model_id=0):
    cam = types.SimpleNamespace(camera_models=model_id)
    cam.item = lambda: cam
    return cam


def test_supported_falls_back_for_each_condition(monkeypatch):
    import fused_render as fr
    from diff_gaussian_rasterization import _C
    # the fake's MLP parameters live on the CPU: report every tensor as CUDA to isolate each condition
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    ok, cam = _fake_method(), _fake_camera()
    emb32 = np.zeros(32, np.float32)
    assert fr.supported(ok, cam)
    assert fr.supported(ok, cam, {"embedding": emb32, "outputs": ("color", "depth")})
    assert fr.supported(_fake_method(appearance=False), cam)                                   # SH colours
    assert fr.supported(_fake_method(appearance=False), cam, {"embedding": emb32.astype(np.float64)})   # ignored
    assert not fr.supported(_fake_method(model_sh=True), cam)                                  # configuration
    assert not fr.supported(_fake_method(debug=True), cam)
    assert not fr.supported(_fake_method(appearance=False, debug=True), cam)
    assert not fr.supported(ok, _fake_camera(model_id=1))                                      # not pinhole
    assert not fr.supported(ok, cam, {"embedding": emb32.astype(np.float64)})                  # not float32
    assert not fr.supported(ok, cam, {"embedding": np.zeros(16, np.float32)})
    assert not fr.supported(ok, cam, {"embedding": torch.zeros(32)})                           # not numpy
    assert not fr.supported(_fake_method(P=0), cam)
    assert not fr.supported(_fake_method(dtype=torch.float64), cam)
    _C.set_tile_row_shard(0, 1)
    try:
        assert not fr.supported(ok, cam)                                                       # tile-row shard
    finally:
        _C.set_tile_row_shard(0, 0)
    assert fr.supported(ok, cam)
    monkeypatch.undo()
    assert not fr.supported(_fake_method(cuda=False), cam)                                     # CPU tensors
    assert not fr.supported(_fake_method(cuda=False, appearance=False), cam)


class _Method:
    def __init__(self):
        self.model = _FakeModel(optimizer=None)
        self.config = types.SimpleNamespace()

    def render(self, camera, options=None):
        return "class render"


def test_enable_method_binds_render_only_when_asked():
    import wildgaussians_fused as wf
    method = _Method()
    wf.enable_method(method)
    assert "render" not in method.__dict__ and method.render(None) == "class render"
    assert "optimize_embedding" in method.__dict__
    wf.enable_method(method, render=True)
    assert method.render.__func__ is wf.render and method.render.__self__ is method
    wf.disable_method(method)
    assert "render" not in method.__dict__ and "optimize_embedding" not in method.__dict__
    assert method.render(None) == "class render"


# ---------------------------------------------------------------------------------------------------------------- GPU
MODELS = [dict(P=150_000, W=640, H=400, seed=3), dict(P=40_000, W=333, H=211, seed=5)]
MODEL_IDS = ["P150k_640x400", "P40k_333x211"]


def _method_module():
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    import diff_gaussian_rasterization as ours
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    return m, Config


def _camera(m, method, i=0, pose=None):
    from wildgaussians.types import new_cameras
    c = method.train_cameras[i]
    poses = c.poses if pose is None else pose
    return new_cameras(poses=poses[None].astype(np.float32), intrinsics=c.intrinsics[None].astype(np.float32),
                       camera_models=np.array([m.camera_model_to_int("pinhole")], np.int32),
                       distortion_parameters=np.zeros((1, 0), np.float32), image_sizes=c.image_sizes[None])


def _make(kw, appearance):
    import synthetic
    import wg_train
    m, Config = _method_module()
    dev = torch.device("cuda:0")
    scene = synthetic.make_scene(kw["P"], kw["W"], kw["H"], sh_degree=3, seed=kw["seed"])
    method = wg_train.make_method(m, Config, scene, dev, appearance=appearance, seed=kw["seed"])
    return m, method


def _fresh():
    import wildgaussians_fused as wf
    return wf


def _today(method, cam, options):
    """``WildGaussians.render`` under ``enable_method(method)`` (the fused caller without the fused render)."""
    wf = _fresh()
    wf.enable_method(method)
    try:
        assert "render" not in method.__dict__
        return type(method).render(method, cam, options)
    finally:
        wf.disable_method(method)


def _max_visible_distance(method, cam):
    wf = _fresh()
    model = method.model
    m = sys.modules[type(model).__module__]
    cc = wf._camera_constants(m, cam.item(), model.xyz.device)
    with torch.no_grad():
        out = wf.render_internal(model, cam.item(), method.config, kernel_size=method.config.kernel_size,
                                 embedding=model.get_embedding(None), return_raw=False)
        dist = torch.norm(model.xyz - cc["cam_center"][None], dim=-1)
        return float(dist[out["radii"] > 0].max())


def _same_layout(ours, ref):
    assert sorted(ours) == sorted(ref)
    for k in ref:
        assert ours[k].shape == ref[k].shape and ours[k].dtype == ref[k].dtype, k
    assert ours["color"].flags["C_CONTIGUOUS"]


@pytest.mark.gpu
@pytest.mark.parametrize("appearance", [True, False], ids=["appearance", "sh"])
@pytest.mark.parametrize("kw", MODELS, ids=MODEL_IDS)
def test_bitwise_against_the_fused_caller(kw, appearance):
    import fused_render as fr
    m, method = _make(kw, appearance)
    cam = _camera(m, method)
    embeddings = [None, np.linspace(-0.5, 0.5, 32).astype(np.float32)]
    if appearance:
        embeddings.append(method.model.appearance_embeddings[1].detach().cpu().numpy())
    bar = 1e-6 * _max_visible_distance(method, cam)
    for emb in embeddings:
        for outputs in (("color",), ("color", "depth")):
            options = {"embedding": emb, "outputs": outputs}
            assert fr.supported(method, cam, options)
            ref = _today(method, cam, options)
            ours = fr.render(method, cam, options)
            _same_layout(ours, ref)
            assert np.array_equal(ours["color"], ref["color"]), (emb is None, outputs)
            assert np.array_equal(ours["accumulation"], ref["accumulation"])
            if "depth" in outputs:
                err = float(np.abs(ours["depth"].astype(np.float64) - ref["depth"]).max())
                print(f"depth: max |diff| {err:.3e} (bar {bar:.3e}), bitwise {np.array_equal(ours['depth'], ref['depth'])}")
                assert err <= bar, (err, bar)


@pytest.mark.gpu
@pytest.mark.parametrize("appearance", [True, False], ids=["appearance", "sh"])
@pytest.mark.parametrize("kw", MODELS, ids=MODEL_IDS)
def test_against_the_shipped_method(kw, appearance):
    import fused_render as fr
    m, method = _make(kw, appearance)
    cam = _camera(m, method)
    for emb in (None, np.linspace(-0.5, 0.5, 32).astype(np.float32)):
        options = {"embedding": emb, "outputs": ("color", "depth")}
        ref = m.WildGaussians.render(method, cam, options)
        ours = fr.render(method, cam, options)
        _same_layout(ours, ref)
        # the colour bars of the fused caller, which this path matches bit for bit (test above).  Without appearance its
        # SH colours differ from the shipped statements by up to 9.2e-4 on the 150 k scene, above test_method_py.py's 2e-4
        # raw-colour bar on its own scene
        assert float(np.abs(ours["color"] - ref["color"]).max()) <= 1e-3
        assert float(np.abs(ours["accumulation"] - ref["accumulation"]).max()) <= 1e-4


def _scene(P, W, H, seed):
    import synthetic
    return synthetic.to_device(synthetic.make_scene(P, W, H, sh_degree=None, seed=seed), torch.device("cuda:0"))


def _display(d, colors, **kw):
    import fused_render as fr
    return fr.display_composite(d["bg"], d["means3D"], colors, d["opacities"], d["scales"], d["rotations"], d["viewmatrix"],
                                d["projmatrix"], d["campos"], d["tanfovx"], d["tanfovy"], d["kernel_size"],
                                d["subpixel_offset"], d["image_height"], d["image_width"], **kw)


def _ordinary(d, colors):
    from diff_gaussian_rasterization import _C
    e = torch.Tensor([])
    R, img, radii, geom, binning, ibuf = _C.rasterize_gaussians(
        d["bg"], d["means3D"], colors, d["opacities"], d["scales"], d["rotations"], 1.0, e, d["viewmatrix"],
        d["projmatrix"], d["tanfovx"], d["tanfovy"], d["kernel_size"], d["subpixel_offset"], d["image_height"],
        d["image_width"], e, 0, d["campos"], False, False)
    P, H, W = int(d["means3D"].shape[0]), d["image_height"], d["image_width"]
    return img, _C.debug_views(geom, binning, ibuf, P, 0, W, H, R)["final_T"], radii


@pytest.mark.gpu
@pytest.mark.parametrize("P,W,H,seed", [(40_000, 333, 211, 11), (150_000, 640, 400, 12)])
def test_display_epilogue_against_the_ordinary_composite(P, W, H, seed):
    """Colours with NaN, values above 1 and negative values: clamp(0, 1).nan_to_num_(0) of the ordinary composite, HWC."""
    from diff_gaussian_rasterization import _C
    _C.clear_geometry_cache()
    d = _scene(P, W, H, seed)
    g = torch.Generator().manual_seed(seed)
    colors = (torch.randn(P, 3, generator=g) * 1.5 + 0.5).to(d["means3D"].device)
    colors[torch.randperm(P, generator=g)[: P // 50].to(colors.device), 1] = float("nan")
    values = (torch.rand(P, generator=g) * 7 - 1).to(colors.device)
    HW = H * W
    img, final_T, _ = _ordinary(d, colors)
    want = img.clamp(0, 1).nan_to_num_(0).permute(1, 2, 0).reshape(-1)
    assert bool(img.isnan().any()) and bool((img > 1).any()) and bool((img < 0).any())
    for kw in (dict(), dict(depth=True, depth_values=values), dict(depth=True)):
        out = _display(d, colors, **kw)
        assert torch.equal(out[:3 * HW], want)
        assert torch.equal(out[3 * HW:4 * HW], (1 - final_T).reshape(-1))
        if kw.get("depth_values") is not None:          # a fourth channel with the colours' recurrence: bit for bit
            _C.clear_geometry_cache()
            dimg = _ordinary(d, values[:, None].repeat(1, 3).contiguous())[0]
            assert torch.equal(out[4 * HW:], dimg[0].reshape(-1))
        elif kw:                                         # camera distances against torch.norm's
            dist = torch.norm(d["means3D"] - d["campos"][None], dim=-1)
            _C.clear_geometry_cache()
            dimg, _, radii = _ordinary(d, dist[:, None].repeat(1, 3).contiguous())
            err = float((out[4 * HW:] - dimg[0].reshape(-1)).abs().max())
            assert err <= 1e-6 * float(dist[radii > 0].max()), err


@pytest.mark.gpu
def test_render_clamps_and_an_empty_view_is_zero():
    import fused_render as fr
    m, method = _make(MODELS[1], False)
    with torch.no_grad():                                # bright SH colours: some pixels exceed 1 before the clamp
        method.model.features_dc.fill_(1.0)
        method.model.features_rest.fill_(1.0)
    cam = _camera(m, method)
    wf = _fresh()
    with torch.no_grad():
        raw = wf.render_internal(method.model, cam.item(), method.config, kernel_size=method.config.kernel_size,
                                 embedding=method.model.get_embedding(None), return_raw=False)["render"]
    over = (raw > 1).permute(1, 2, 0).cpu().numpy()
    assert over.any()
    ours = fr.render(method, cam)
    assert np.all(ours["color"][over] == 1.0)
    assert np.array_equal(ours["color"], _today(method, cam, None)["color"])
    # a camera far behind the scene and turned away from it sees no Gaussian
    away = np.concatenate([np.diag([-1.0, 1.0, -1.0]).astype(np.float32), np.array([[0.0], [0.0], [-1000.0]], np.float32)],
                          axis=1)
    cam2 = _camera(m, method, pose=away)
    options = {"outputs": ("color", "depth")}
    ours, ref = fr.render(method, cam2, options), m.WildGaussians.render(method, cam2, options)
    _same_layout(ours, ref)
    for k in ref:
        assert not ours[k].any() and np.array_equal(ours[k], ref[k]), k


@pytest.mark.gpu
def test_embedding_edge_cases():
    import fused_render as fr
    m, method = _make(MODELS[1], True)
    cam = _camera(m, method)
    bad = {"embedding": np.zeros(32, np.float64)}
    assert not fr.supported(method, cam, bad)
    with pytest.raises(Exception) as want:
        m.WildGaussians.render(method, cam, bad)
    with pytest.raises(type(want.value)) as got:
        fr.render(method, cam, bad)
    assert str(got.value) == str(want.value)
    # a model without appearance ignores the embedding
    m, plain = _make(MODELS[1], False)
    cam = _camera(m, plain)
    a = fr.render(plain, cam)
    for emb in (np.ones(32, np.float32), np.ones(32, np.float64)):
        assert fr.supported(plain, cam, {"embedding": emb})
        b = fr.render(plain, cam, {"embedding": emb})
        assert all(np.array_equal(a[k], b[k]) for k in a)


@pytest.mark.gpu
def test_results_are_fresh_and_repeatable():
    import fused_render as fr
    m, method = _make(MODELS[1], True)
    cam0, cam1 = _camera(m, method, 0), _camera(m, method, 1)
    options = {"outputs": ("color", "depth")}
    a = fr.render(method, cam0, options)
    keep = {k: v.copy() for k, v in a.items()}
    b = fr.render(method, cam1, options)
    assert not np.array_equal(a["color"], b["color"])
    assert all(np.array_equal(a[k], keep[k]) for k in a)         # the second call did not write into the first result
    c = fr.render(method, cam0, options)
    assert all(a[k].tobytes() == c[k].tobytes() for k in a)


# Synchronising runtime calls.  cudaDeviceSynchronize is left out: the call makes none, and the profiler itself makes
# one when it stops.
SYNC_CALLS = ("cudaStreamSynchronize", "cudaEventSynchronize", "cudaMemcpy")


@pytest.mark.gpu
@pytest.mark.parametrize("appearance", [True, False], ids=["appearance", "sh"])
def test_profiled_call_synchronises_twice_without_pageable_copies(appearance):
    import fused_render as fr
    from torch.profiler import ProfilerActivity, profile
    m, method = _make(MODELS[1], appearance)
    cam = _camera(m, method)
    options = {"embedding": np.linspace(-0.5, 0.5, 32).astype(np.float32), "outputs": ("color", "depth")}
    fr.render(method, cam, options)                             # the camera's constants are computed once
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        out = fr.render(method, cam, options)
    names = [e.name for e in prof.events()]
    syncs = [n for n in names if n in SYNC_CALLS]
    copies = [n for n in names if n.startswith("Memcpy")]
    print(f"synchronising calls {syncs}; copies {copies}; .item() {names.count('aten::item')}")
    assert len(syncs) <= 2, syncs
    assert not any("DtoH" in n and "Pageable" in n for n in copies), copies
    assert names.count("aten::item") == 0 and names.count("aten::nonzero") == 0
    assert sum(1 for n in copies if "DtoH" in n) <= 1, copies
    assert out["color"].base is not None


@pytest.mark.gpu
def test_reference_protocols_give_the_same_metrics():
    import wildgaussians_fused as wf
    m, method = _make(MODELS[1], True)
    import wildgaussians.evaluation as ev
    from wildgaussians.datasets.phototourism import NerfWEvaluationProtocol

    class ZeroLPIPS(torch.nn.Module):
        def forward(self, a, b):
            return a.new_zeros((a.shape[0], 1, 1, 1))

    saved = dict(ev._LPIPS_CACHE)
    ev._LPIPS_CACHE.clear()
    ev._LPIPS_CACHE["alex"] = ZeroLPIPS()
    try:
        gt = np.clip(method.train_images[2].permute(1, 2, 0).numpy(), 0, 1)
        ds = {"cameras": _camera(m, method, 2), "images": [gt], "masks": None, "metadata": {"color_space": "srgb"}}
        results = []
        recorded = {}
        for fused in (True, False):
            wf.enable_method(method, render=fused)
            try:
                if fused:
                    opt = method.optimize_embedding
                    method.optimize_embedding = lambda d, embedding=None: recorded.setdefault("pred", opt(d, embedding=embedding))
                else:                                   # the same embedding: the loop's atomics may change its last bits
                    method.optimize_embedding = lambda d, embedding=None: recorded["pred"]
                assert ("render" in method.__dict__) == fused
                row = []
                for proto in (ev.DefaultEvaluationProtocol(), NerfWEvaluationProtocol()):
                    pred = proto.render(method, ds)
                    row.append((pred["color"], proto.evaluate(pred, ds)))
                results.append(row)
            finally:
                wf.disable_method(method)
        for (ca, ma), (cb, mb) in zip(*results):
            assert np.array_equal(ca, cb)
            assert ma == mb, (ma, mb)
    finally:
        ev._LPIPS_CACHE.clear()
        ev._LPIPS_CACHE.update(saved)
