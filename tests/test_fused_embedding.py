"""Test-time appearance optimisation on one geometry pass (``fused_embedding``, ``wildgaussians_fused.optimize_embedding``).

CPU: the reduction the embedding-only kernel implements (d(embedding) = W1[:, 27:59]^T . sum dZ1) against autograd, the
C entry points' argument checks, and the dispatch predicate.  GPU: the colour-only composite backward against the full
backward, the embedding-only colour-op backward against ``fused_colors`` and the oracles, and whole
``optimize_embedding`` calls against the reference method (wildgaussians/method.py:1755-1830) on the same model.
"""
from __future__ import annotations

import ctypes
import sys
import types

import numpy as np
import pytest
import torch

from oracle import color_torch as ct


def embedding_grad_oracle(dc, rest, gemb, aemb, W1, b1, W2, b2, W3, b3, means, campos, deg, dL_dtoned):
    """d(image embedding) as W1[:, 27:59]^T . sum_rows dZ1, dZ1 from the bf16-emulated colour op (color_torch): the
    embedding enters only through the layer-1 bias, so sum_rows dZ1 is the gradient of b1."""
    b1 = b1.detach().clone().requires_grad_(True)
    _, toned = ct.colors(dc, rest, gemb, aemb.detach(), W1, b1, W2, b2, W3, b3, means, campos, deg, emulate_bf16=True)
    (sum_dz1,) = torch.autograd.grad(toned, b1, dL_dtoned)
    return W1[:, 27:].T @ sum_dz1


def _random_colour_inputs(P, dev, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    R = lambda *s, scale=1.0: (torch.randn(*s, generator=g, dtype=torch.float64) * scale).to(device=dev, dtype=dtype)
    ins = [R(P, 3), R(P, 45, scale=0.3), R(P, 24, scale=0.5), R(32, scale=0.5), R(P, 3, scale=2.0)]
    torch.manual_seed(seed)
    mlp = torch.nn.Sequential(torch.nn.Linear(59, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128), torch.nn.ReLU(),
                              torch.nn.Linear(128, 6)).to(device=dev, dtype=dtype)
    with torch.no_grad():
        mlp[4].bias[3:] = 80.0
    campos = torch.tensor([0.1, -0.2, 0.3], device=dev, dtype=dtype)
    return ins, mlp, campos, R(P, 3)


def _cos_ratio(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float(a @ b) / (float(a.norm()) * float(b.norm()) + 1e-300), float(a.norm()) / (float(b.norm()) + 1e-300)


def test_oracle_embedding_grad_is_the_autograd_gradient():
    for P, deg in ((1, 3), (37, 3), (300, 1)):
        ins, mlp, campos, dL = _random_colour_inputs(P, "cpu", 11 + P)
        aemb = ins[3].clone().requires_grad_(True)
        _, toned = ct.colors(ins[0], ins[1], ins[2], aemb, mlp[0].weight, mlp[0].bias, mlp[2].weight, mlp[2].bias,
                             mlp[4].weight, mlp[4].bias, ins[4], campos, deg, emulate_bf16=True)
        (want,) = torch.autograd.grad(toned, aemb, dL)
        got = embedding_grad_oracle(ins[0], ins[1], ins[2], ins[3], mlp[0].weight, mlp[0].bias, mlp[2].weight, mlp[2].bias,
                                    mlp[4].weight, mlp[4].bias, ins[4], campos, deg, dL)
        assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max()) + 1e-12, (P, got, want)


def test_entry_points_exported_and_reject_bad_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib
    for name in ("gsr_backward_colors", "gsr_appearance_embedding_backward"):
        assert hasattr(lib, name)
    GSR_E_INVALID = -1
    assert lib.gsr_backward_colors(None, None) == GSR_E_INVALID
    a = _C.GsrBackwardArgs()
    a.P, a.W, a.H, a.R = -1, 16, 16, 0
    assert lib.gsr_backward_colors(ctypes.byref(a), None) == GSR_E_INVALID
    a.P, a.W, a.H, a.R = 10, 0, 16, 0
    assert lib.gsr_backward_colors(ctypes.byref(a), None) == GSR_E_INVALID
    a.P, a.W, a.H, a.R = 10, 16, 16, -1
    assert lib.gsr_backward_colors(ctypes.byref(a), None) == GSR_E_INVALID
    a.R = 5                                                   # every buffer NULL
    assert lib.gsr_backward_colors(ctypes.byref(a), None) == GSR_E_INVALID
    assert b"NULL" in lib.gsr_last_error()

    assert lib.gsr_appearance_embedding_backward(None, None) == GSR_E_INVALID
    b = _C.GsrAppearanceArgs()
    b.P, b.sh_degree = 5, 4
    assert lib.gsr_appearance_embedding_backward(ctypes.byref(b), None) == GSR_E_INVALID
    b.P, b.sh_degree = -1, 3
    assert lib.gsr_appearance_embedding_backward(ctypes.byref(b), None) == GSR_E_INVALID
    b.P = 5                                                   # grad_pack NULL
    assert lib.gsr_appearance_embedding_backward(ctypes.byref(b), None) == GSR_E_INVALID
    b.grad_pack = 256                                         # inputs NULL (checked before any CUDA call)
    assert lib.gsr_appearance_embedding_backward(ctypes.byref(b), None) == GSR_E_INVALID
    for f in ("features_dc", "features_rest", "embeddings", "means3D", "campos", "packed_weights", "dL_dcolors_toned"):
        setattr(b, f, 4096)
    b.features_rest = 4100                                    # misaligned
    assert lib.gsr_appearance_embedding_backward(ctypes.byref(b), None) == GSR_E_INVALID
    assert b"aligned" in lib.gsr_last_error()


# ---- dispatch predicate (no device needed: the CUDA-ness is read from attributes) -------------------------------------
def camera_model_to_int(name):          # looked up in the model class's module, as in wildgaussians/method.py
    return {"pinhole": 0, "opencv": 1}[name]


class _FakeModel(types.SimpleNamespace):
    pass


def _fake_method(cuda=True, optim="dssim+l1-scaled", appearance=True, hidden=128):
    t = lambda *s: types.SimpleNamespace(is_cuda=cuda, dtype=torch.float32, shape=s)
    mlp = torch.nn.Sequential(torch.nn.Linear(59, hidden), torch.nn.ReLU(), torch.nn.Linear(hidden, 128), torch.nn.ReLU(),
                              torch.nn.Linear(128, 6))
    cfg = types.SimpleNamespace(appearance_enabled=appearance, appearance_separate_tuned_color=True, appearance_model_sh=False,
                                sh_degree=3, appearance_embedding_dim=32, debug=False, appearance_optim_type=optim)
    model = _FakeModel(config=cfg, xyz=t(10, 3), features_dc=t(10, 3), features_rest=t(10, 45), embeddings=t(10, 24),
                       scales=t(10, 3), opacities=t(10, 1), rotations=t(10, 4), filter_3D=t(10, 1),
                       appearance_embeddings=t(4, 32), appearance_mlp=types.SimpleNamespace(mlp=mlp))
    return types.SimpleNamespace(model=model, config=cfg)


def _fake_dataset(model_id=0):
    cam = types.SimpleNamespace(camera_models=model_id)
    cam.item = lambda: cam
    return {"cameras": cam, "images": [None], "masks": None}


def test_dispatch_predicate_falls_back(monkeypatch):
    import fused_embedding as fe
    # MLP parameters of the fake live on the CPU: report every tensor as CUDA to isolate each condition
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    ok = _fake_method()
    assert fe.supported(ok, _fake_dataset())                         # the default configuration is accelerated
    assert fe.supported(_fake_method(optim="mse"), _fake_dataset())
    assert fe.supported(_fake_method(optim="dssim+l1"), _fake_dataset())
    assert not fe.supported(ok, _fake_dataset(model_id=1))          # not a pinhole camera
    assert not fe.supported(_fake_method(optim="l1"), _fake_dataset())
    assert not fe.supported(_fake_method(optim="dssim+l1-weird"), _fake_dataset())
    assert not fe.supported(_fake_method(appearance=False), _fake_dataset())
    assert not fe.supported(_fake_method(hidden=64), _fake_dataset())
    assert not fe.supported(ok, _fake_dataset(), embedding=np.zeros(32, dtype=np.float64))
    assert fe.supported(ok, _fake_dataset(), embedding=np.zeros(32, dtype=np.float32))
    monkeypatch.undo()
    assert not fe.supported(_fake_method(cuda=False), _fake_dataset())   # CPU tensors


# ======================================================================================================================
# GPU
# ======================================================================================================================
def _scene_buffers(P, W, H, seed, dev):
    import synthetic
    from diff_gaussian_rasterization import _C
    from make_golden import call_args
    d = synthetic.to_device(synthetic.make_scene(P, W, H, sh_degree=None, seed=seed), dev)
    R, img, radii, geom, binning, ibuf = _C.rasterize_gaussians(*call_args(d))
    return d, R, img, radii, geom, binning, ibuf


def color_backward(d, R, geom, binning, ibuf, dL_dpix):
    from diff_gaussian_rasterization import _C
    P = int(d["means3D"].shape[0])
    H, W = int(d["image_height"]), int(d["image_width"])
    out = torch.full((P, 3), float("nan"), device=dL_dpix.device)    # the call writes every row
    a = _C.GsrBackwardArgs()
    a.P, a.M, a.R, a.W, a.H = P, 0, int(R), W, H
    a.subpixel_offset = d["subpixel_offset"].data_ptr()
    a.geom_buffer, a.binning_buffer, a.img_buffer = geom.data_ptr(), binning.data_ptr(), ibuf.data_ptr()
    a.dL_dpix, a.dL_dcolor = dL_dpix.data_ptr(), out.data_ptr()
    _C._check(_C._lib.gsr_backward_colors(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "gsr_backward_colors")
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("P,W,H,seed", [(150_000, 640, 400, 3), (40_000, 333, 211, 5), (3_000_000, 1920, 1080, 7)])
def test_color_backward_matches_the_full_backward(P, W, H, seed):
    """dL/dcolour of the colour-only walk (forward-order T alpha) against the full backward's colour gradient (T
    reconstructed back to front by division), on the same geometry and dL/dpix, within 20x the full backward's own
    run-to-run spread or 1e-6 of the largest entry; rows of Gaussians with radii == 0 are exactly zero; the recolour
    pass's image buffer gives the same result."""
    from diff_gaussian_rasterization import _C
    from make_golden import backward_args, call_args
    dev = torch.device("cuda:0")
    _C.set_geometry_cache(True)
    d, R, img, radii, geom, binning, ibuf = _scene_buffers(P, W, H, seed, dev)
    # a second forward on the same tensors re-composites on the cached geometry (gsr_forward_recolor's image buffer)
    R2, img2, _, geom2, binning2, ibuf2 = _C.rasterize_gaussians(*call_args(d))
    assert geom2 is geom and ibuf2 is not ibuf and torch.equal(img2, img)
    ours = color_backward(d, R, geom, binning, ibuf, d["dL_dpix"])
    ours2 = color_backward(d, R, geom, binning, ibuf, d["dL_dpix"])
    ours_rc = color_backward(d, R, geom, binning, ibuf2, d["dL_dpix"])
    full = [_C.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, ibuf))[1] for _ in range(2)]
    torch.cuda.synchronize()
    noise = float((full[0] - full[1]).abs().max())
    scale = float(full[0].abs().max())
    err = float((ours - full[0]).abs().max())
    bar = max(20 * noise, 1e-6 * scale)
    print(f"P={P} {W}x{H}: max|dcolor|={scale:.3e} err={err:.3e} full-backward spread={noise:.3e} "
          f"own spread={float((ours - ours2).abs().max()):.3e} bar={bar:.3e}")
    assert not torch.isnan(ours).any()
    assert torch.count_nonzero(ours[radii == 0]) == 0
    assert err <= bar, (err, bar)
    assert float((ours_rc - ours).abs().max()) <= bar


def embedding_backward(ins, mlp, campos, dL, deg=3):
    """d(image embedding) [32] through gsr_appearance_embedding_backward + gsr_appearance_unpack_grads."""
    from diff_gaussian_rasterization import _C
    lib = _C._lib
    dev = dL.device
    P = int(ins[0].shape[0])
    s = torch.cuda.current_stream().cuda_stream
    w = [t.detach().contiguous() for i in (0, 2, 4) for t in (mlp[i].weight, mlp[i].bias)]
    blob = torch.empty((lib.gsr_appearance_packed_weight_bytes(),), dtype=torch.uint8, device=dev)
    aemb = ins[3].detach().contiguous()
    _C._check(lib.gsr_appearance_pack_weights(*[t.data_ptr() for t in w], aemb.data_ptr(), blob.data_ptr(), s), "pack")
    pack = torch.full((lib.gsr_appearance_grad_pack_bytes() // 4,), float("nan"), device=dev)
    a = _C.GsrAppearanceArgs()
    a.P, a.sh_degree = P, deg
    x = [t.detach().contiguous() for t in (ins[0], ins[1], ins[2], ins[4], dL)]
    if P > 0:
        a.features_dc, a.features_rest, a.embeddings, a.means3D = (t.data_ptr() for t in x[:4])
        a.campos, a.packed_weights, a.dL_dcolors_toned = campos.data_ptr(), blob.data_ptr(), x[4].data_ptr()
    a.grad_pack = pack.data_ptr()
    _C._check(lib.gsr_appearance_embedding_backward(ctypes.byref(a), s), "gsr_appearance_embedding_backward")
    outs = [torch.empty(sh, device=dev) for sh in ((128, 59), (128,), (128, 128), (128,), (6, 128), (6,), (32,))]
    _C._check(lib.gsr_appearance_unpack_grads(pack.data_ptr(), w[0].data_ptr(), aemb.data_ptr(), *[t.data_ptr() for t in outs],
                                              s), "unpack")
    return outs[-1]


@pytest.mark.gpu
@pytest.mark.parametrize("P", [0, 1000, 100_003, 3_000_000])
def test_embedding_backward_against_fused_colors_and_oracles(P):
    import fused_colors as fc
    dev = torch.device("cuda:0")
    ins, mlp, campos, dL = _random_colour_inputs(P, dev, 21 + P % 97)
    ours = [embedding_backward(ins, mlp, campos, dL) for _ in range(2)]
    if P == 0:
        torch.cuda.synchronize()
        assert torch.count_nonzero(ours[0]) == 0
        return
    full = []
    for _ in range(2):
        aemb = ins[3].clone().requires_grad_(True)
        _, toned = fc.fused_colors(ins[0], ins[1], ins[2], aemb, mlp, ins[4], campos, 3, want_raw=False)
        (g,) = torch.autograd.grad(toned, aemb, dL)
        full.append(g)
    bf16 = embedding_grad_oracle(ins[0], ins[1], ins[2], ins[3], mlp[0].weight, mlp[0].bias, mlp[2].weight, mlp[2].bias,
                                 mlp[4].weight, mlp[4].bias, ins[4], campos, 3, dL).detach()
    aemb = ins[3].clone().requires_grad_(True)
    _, toned = ct.colors(ins[0], ins[1], ins[2], aemb, mlp[0].weight, mlp[0].bias, mlp[2].weight, mlp[2].bias, mlp[4].weight,
                         mlp[4].bias, ins[4], campos, 3)
    (fp32,) = torch.autograd.grad(toned, aemb, dL)
    torch.cuda.synchronize()
    scale = float(full[0].abs().max())
    noise = max(float((full[0] - full[1]).abs().max()), float((ours[0] - ours[1]).abs().max()))
    err = float((ours[0] - full[0]).abs().max())
    bar = max(20 * noise, 1e-6 * scale)
    cb, rb = _cos_ratio(ours[0], bf16)
    c32, r32 = _cos_ratio(ours[0], fp32)
    print(f"P={P}: max|d emb|={scale:.3e} err vs fused_colors={err:.3e} spread={noise:.3e} bar={bar:.3e}; "
          f"bf16 oracle cos={cb:.6f} ratio={rb:.5f}; fp32 cos={c32:.5f} ratio={r32:.4f}")
    assert err <= bar, (err, bar)
    assert cb >= 0.999 and abs(rb - 1) < 0.01
    assert c32 >= 0.99 and abs(r32 - 1) < 0.03


# ---- whole optimize_embedding calls against the reference method --------------------------------------------------------
def _setup(scene_kw, seed=63, uncertainty=False):
    import synthetic
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    import diff_gaussian_rasterization as ours
    dev = torch.device("cuda:0")
    scene = synthetic.make_scene(sh_degree=3, seed=seed, **scene_kw)
    model, cfg = wh.make_model(m, Config, scene, dev, seed=seed)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    cam = wh.make_camera(scene)
    cam.camera_models = m.camera_model_to_int("pinhole")
    cam.item = lambda: cam
    if uncertainty:           # random backbone weights; eval(): no dropout, so every get_loss call gives the same map
        import wg_uncertainty
        model.uncertainty_model = wg_uncertainty.make_uncertainty_model(m, Config, "dino", dev, seed=seed)[0].eval()
    # the target: the render at a DIFFERENT training embedding than the start (zeros)
    import wildgaussians_fused as wf
    with torch.no_grad():
        gt = wf.render_internal(model, cam, cfg, kernel_size=cfg.kernel_size, embedding=model.appearance_embeddings[1],
                                return_raw=False)["render"]
    gt_np = gt.clamp(0, 1).permute(1, 2, 0).cpu().numpy().astype(np.float32)
    return m, model, cfg, cam, gt_np


def _dataset(cam, gt_np, mask=None):
    return {"cameras": cam, "images": [gt_np], "masks": None if mask is None else [mask]}


def _snapshot(model):
    return {n: p.detach().clone() for n, p in model.named_parameters()}


def _ref_call(m, model, cfg, ds, embedding=None):
    import wildgaussians_fused as wf
    ns = types.SimpleNamespace(model=model, config=cfg)
    # the fused caller and the same SSIM kernel as the fused loop: the comparison isolates the loop itself
    wf.enable(model, optimizer=False, ssim=True)
    try:
        out = m.WildGaussians.optimize_embedding(ns, ds, embedding=embedding)
    finally:
        wf.disable(model)
    for p in model.parameters():
        p.grad = None
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("setup", ["dssim+l1-scaled+mask", "mse", "dssim+l1-nomask"])
def test_optimize_embedding_matches_the_reference_method(setup):
    import fused_embedding as fe
    kw = dict(P=40_000, W=333, H=211)
    m, model, cfg, cam, gt_np = _setup(kw, uncertainty=setup.startswith("dssim+l1-scaled"))
    cfg.appearance_optim_type = {"dssim+l1-scaled+mask": "dssim+l1-scaled", "mse": "mse", "dssim+l1-nomask": "dssim+l1"}[setup]
    mask = None
    if setup != "dssim+l1-nomask":
        mask = np.ones((211, 333), dtype=np.float32)
        mask[50:120, 100:220] = 0.0
    ds = _dataset(cam, gt_np, mask)
    params = _snapshot(model)
    refs = [_ref_call(m, model, cfg, ds) for _ in range(2)]
    model.train()
    start = np.zeros(32, dtype=np.float32)
    ns = types.SimpleNamespace(model=model, config=cfg)
    assert fe.supported(ns, ds, start)
    ours = fe.optimize_embedding(ns, ds, embedding=start)
    torch.cuda.synchronize()
    # state after the call
    assert not model.training
    assert all(torch.equal(p, params[n]) for n, p in model.named_parameters())
    assert all(p.grad is None for p in model.parameters())
    assert np.array_equal(start, np.zeros(32, dtype=np.float32))
    # structure
    assert set(ours) == set(refs[0]) and set(ours["metrics"]) == set(refs[0]["metrics"])
    for k in ours["metrics"]:
        assert len(ours["metrics"][k]) == len(refs[0]["metrics"][k]) == cfg.appearance_embedding_optim_iters
        assert all(type(v) is float for v in ours["metrics"][k])
    assert ours["embedding"].shape == refs[0]["embedding"].shape and ours["embedding"].dtype == np.float32
    psnr = np.array(ours["metrics"]["psnr"])
    ref_psnr = np.array(refs[0]["metrics"]["psnr"])
    # with random backbone weights the uncertainty map (loss_mult > 1) can be all zero: then no gradient reaches the
    # embedding and the reference does not move either
    if ref_psnr[-1] > ref_psnr[0] + 1.0:
        assert psnr[-1] > psnr[0] + 1.0
    else:
        assert np.array_equal(ours["embedding"], refs[0]["embedding"]) and psnr[-1] == psnr[0]
    # agreement with the reference, bars from the reference's own run-to-run spread
    curves = {k: [np.array(r["metrics"][k]) for r in refs] + [np.array(ours["metrics"][k])] for k in ("loss", "psnr")}
    emb = [r["embedding"] for r in refs] + [ours["embedding"]]
    lspread = float(np.abs(curves["loss"][0] - curves["loss"][1]).max() / np.abs(curves["loss"][0]).max())
    lerr = float(np.abs(curves["loss"][2] - curves["loss"][0]).max() / np.abs(curves["loss"][0]).max())
    pspread = abs(curves["psnr"][0][-1] - curves["psnr"][1][-1])
    perr = abs(curves["psnr"][2][-1] - curves["psnr"][0][-1])
    espread = float(np.abs(emb[0] - emb[1]).max())
    eerr = float(np.abs(emb[2] - emb[0]).max())
    enorm = float(np.abs(emb[0]).max())
    print(f"{setup}: psnr {psnr[0]:.2f} -> {psnr[-1]:.3f} (reference {curves['psnr'][0][-1]:.3f}); loss rel err {lerr:.2e} "
          f"(spread {lspread:.2e}); final psnr err {perr:.2e} (spread {pspread:.2e}); embedding err {eerr:.2e} "
          f"(spread {espread:.2e}, max {enorm:.2e})")
    assert lerr <= max(20 * lspread, 1e-3)
    assert perr <= max(20 * pspread, 0.02)
    assert eerr <= max(20 * espread, 1e-2 * enorm)


@pytest.mark.gpu
def test_first_iteration_image_and_gradient_match_the_reference_statements():
    """Iteration 0: the image equals the fused _render_internal's bit for bit; dL/d(embedding) of one iteration matches the
    reference statements of method.py:1786-1808 run once with autograd, on the fused colours (bars of the colour-op
    test) and on the unmodified fp32 path."""
    import fused_embedding as fe
    import wildgaussians_fused as wf
    m, model, cfg, cam, gt_np = _setup(dict(P=150_000, W=640, H=400))
    mask = np.ones((400, 640), dtype=np.float32)
    mask[:100] = 0.0
    ds = _dataset(cam, gt_np, mask)
    cfg.appearance_optim_type = "dssim+l1"
    ns = types.SimpleNamespace(model=model, config=cfg)
    start = (np.random.default_rng(0).normal(size=32) * 0.2).astype(np.float32)
    loop = fe.EmbeddingLoop(ns, ds, start)
    image = loop.render().clone()
    x = image.clone().requires_grad_(True)
    with torch.enable_grad():
        loss, _ = loop.loss(x)
        loss.backward()
    ours = loop.embedding_grad(x.grad).clone()

    def reference_grad(fused):
        emb = torch.nn.Parameter(torch.from_numpy(start).cuda().requires_grad_(True))
        if fused:
            wf.enable(model, optimizer=False)
        try:
            with torch.enable_grad():
                img = model._render_internal(cam, config=cfg, embedding=emb, kernel_size=cfg.kernel_size)["render"]
                y = m.scale_grads(img, loop.mask)
                l1 = torch.nn.functional.l1_loss(y, loop.gt)
                loss = (1.0 - cfg.lambda_dssim) * l1 + cfg.lambda_dssim * (1.0 - m.ssim(y, loop.gt, size_average=True))
                loss.backward()
        finally:
            wf.disable(model)
        for p in model.parameters():
            p.grad = None
        return img.detach(), emb.grad.detach()

    img_f, g_f = reference_grad(True)
    img_f2, g_f2 = reference_grad(True)
    _, g_32 = reference_grad(False)
    torch.cuda.synchronize()
    assert torch.equal(image, img_f), float((image - img_f).abs().max())
    scale = float(g_f.abs().max())
    noise = float((g_f - g_f2).abs().max())
    err = float((ours - g_f).abs().max())
    c, r = _cos_ratio(ours, g_f)
    c32, r32 = _cos_ratio(ours, g_32)
    print(f"iteration-0 gradient: err vs fused statements {err:.3e} (spread {noise:.3e}, max {scale:.3e}) cos {c:.6f} "
          f"ratio {r:.5f}; vs fp32 cos {c32:.5f} ratio {r32:.4f}")
    assert c >= 0.999 and abs(r - 1) < 0.01
    assert c32 >= 0.99 and abs(r32 - 1) < 0.03


@pytest.mark.gpu
def test_iterations_do_not_synchronise_and_leave_the_model_alone():
    import fused_embedding as fe
    m, model, cfg, cam, gt_np = _setup(dict(P=40_000, W=333, H=211))
    ds = _dataset(cam, gt_np, np.ones((211, 333), dtype=np.float32))
    params = _snapshot(model)
    loop = fe.EmbeddingLoop(types.SimpleNamespace(model=model, config=cfg), ds, None)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(4):
            loop.step(i)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(torch.equal(p, params[n]) for n, p in model.named_parameters())
    # with an optimizer on the model, its gradients are left as the reference leaves them (zeroed)
    model.optimizer = torch.optim.Adam(model.parameters(), lr=1e-3)
    try:
        for p in model.parameters():
            p.grad = torch.ones_like(p)
        fe.optimize_embedding(types.SimpleNamespace(model=model, config=cfg), ds)
        assert all(p.grad is None for p in model.parameters())
    finally:
        model.optimizer = None


@pytest.mark.gpu
def test_unsupported_configurations_run_the_reference_method():
    import fused_embedding as fe
    import wildgaussians_fused as wf
    m, model, cfg, cam, gt_np = _setup(dict(P=20_000, W=160, H=112))
    ds = _dataset(cam, gt_np)
    cfg.appearance_optim_type = "l1"
    ns = types.SimpleNamespace(model=model, config=cfg)
    assert not fe.supported(ns, ds)
    with pytest.raises(ValueError, match="Unknown appearance optimization type l1"):
        fe.optimize_embedding(ns, ds)
    with pytest.raises(ValueError, match="Unknown appearance optimization type l1"):
        m.WildGaussians.optimize_embedding(ns, ds)
    # enable_method routes the instance's method; disable_method restores the class's
    cfg.appearance_optim_type = "mse"
    cfg.appearance_embedding_optim_iters = 3
    method = m.WildGaussians.__new__(m.WildGaussians)
    method.model, method.config = model, cfg
    wf.enable_method(method, optimizer=False)
    assert "optimize_embedding" in method.__dict__ and "_render_internal" in model.__dict__
    out = method.optimize_embedding(ds)
    assert len(out["metrics"]["psnr"]) == 3
    wf.disable_method(method)
    assert "optimize_embedding" not in method.__dict__ and "_render_internal" not in model.__dict__
