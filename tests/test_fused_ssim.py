"""Fused SSIM of the photometric loss (csrc/ssim.cu, fused_ssim.py, wildgaussians_fused.enable(ssim=True)).

CPU: the float64 oracle against the reference's own goldens, the C entry points' argument checks, the Python wrapper's
refusals and the hook's fall-back.  GPU: map, mean and dL/dimg1 against the oracle (goldens, 1080p, 4K), ranks and
reductions, determinism, no host synchronisation, and the loss block of method.py:1948-1966 through the unmodified
reference against its own ``ssim``.
"""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import ssim_oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["ssim_textured", "ssim_small", "ssim_batched", "ssim_flat"]
TEXTURED = [c for c in CASES if c != "ssim_flat"]


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: torch.from_numpy(np.asarray(z[k])) for k in z.files}


# ---------------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_goldens(name):
    c = load(name)
    smap, mean, grad = ssim_oracle.ssim_and_grad(c["img1"], c["img2"], c["dL_dmap"])
    assert smap.shape == c["map"].shape and grad.shape == c["img1"].shape
    assert float((smap - c["map"]).abs().max()) <= 1e-12
    assert abs(float(mean) - float(c["mean"])) <= 1e-12
    assert float((grad - c["grad"]).abs().max()) <= 1e-12


def test_c_entry_points_reject_bad_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib
    p = ctypes.c_void_p(256)                     # never dereferenced: every call below fails its checks first
    assert lib.gsr_ssim_forward(0, 8, 8, p, p, p, None, None) == -1
    assert b"bad sizes" in lib.gsr_last_error()
    assert lib.gsr_ssim_forward(1, 8, -3, p, p, p, None, None) == -1
    assert lib.gsr_ssim_forward(1, 8, 8, p, None, p, None, None) == -1
    assert b"NULL" in lib.gsr_last_error()
    assert lib.gsr_ssim_backward(1, 0, 8, p, p, p, p, p, None) == -1
    assert b"bad sizes" in lib.gsr_last_error()
    assert lib.gsr_ssim_backward(1, 8, 8, p, p, None, p, p, None) == -1
    assert b"NULL" in lib.gsr_last_error()
    assert lib.gsr_ssim_backward(1, 8, 8, p, p, p, p, None, None) == -1
    assert b"NULL" in lib.gsr_last_error()


def test_wrapper_refuses_cpu_tensors():
    import fused_ssim
    a, b = torch.rand(3, 16, 16), torch.rand(3, 16, 16)
    assert not fused_ssim.supported(a, b)
    with pytest.raises(RuntimeError, match="CUDA"):
        fused_ssim.ssim(a, b)


def fake_method_module(name="_fake_wg_method"):
    """A module with a module-level ``ssim`` and a model class defined in it, like wildgaussians.method."""
    m = types.ModuleType(name)
    calls = []

    def ssim(img1, img2, window_size=11, size_average=True):
        calls.append(img1.device.type)
        return ssim_oracle.ssim(img1, img2, window_size, size_average, dtype=img1.dtype)

    class Model(torch.nn.Module):
        pass

    Model.__module__ = name
    m.ssim, m.Model, m.calls = ssim, Model, calls
    sys.modules[name] = m
    return m


def test_hook_falls_back_to_the_original_and_disable_restores_it():
    import wildgaussians_fused as wf
    m = fake_method_module()
    try:
        original = m.ssim
        model = m.Model()
        wf.enable(model, optimizer=False)
        assert m.ssim is original                     # default: the loss is untouched
        wf.enable(model, optimizer=False, ssim=True)
        assert m.ssim is not original
        wf.enable(model, optimizer=False, ssim=True)  # idempotent
        assert m.ssim.__wrapped__ is original
        a, b = torch.rand(3, 12, 14), torch.rand(3, 12, 14)
        out = m.ssim(a, b, size_average=False)        # CPU tensors: the original runs
        assert m.calls == ["cpu"] and out.shape == (12, 14)
        wf.disable(model)
        assert m.ssim is original
    finally:
        sys.modules.pop(m.__name__, None)


# ---------------------------------------------------------------------------------------------------------------- GPU

def fused_map_mean_grad(img1, img2, dL_dmap):
    import fused_ssim
    x = img1.detach().clone().requires_grad_(True)
    smap = fused_ssim.ssim(x, img2, size_average=False)
    (smap * dL_dmap).sum().backward()
    mean = fused_ssim.ssim(img1, img2, size_average=True)
    return smap.detach(), mean.detach(), x.grad


def errors(got, want):
    gmap, gmean, ggrad = got
    wmap, wmean, wgrad = want
    return (float((gmap.double() - wmap.to(gmap.device)).abs().max()), abs(float(gmean) - float(wmean)),
            float((ggrad.double() - wgrad.to(ggrad.device)).abs().max()) / float(wgrad.abs().max()))


@pytest.mark.gpu
@pytest.mark.parametrize("name", TEXTURED)
def test_fused_against_reference_goldens(name):
    c = load(name)
    dev = torch.device("cuda:0")
    got = fused_map_mean_grad(c["img1"].to(dev), c["img2"].to(dev), c["dL_dmap"].to(dev))
    emap, emean, egrad = errors(got, (c["map"], c["mean"], c["grad"]))
    assert emap <= 2e-5 and emean <= 1e-6 and egrad <= 2e-5, (name, emap, emean, egrad)


@pytest.mark.gpu
def test_fused_near_flat_within_twice_the_fp32_statements():
    """On a near-flat image E[x^2] - mu^2 cancels; the bar is the reference's statements evaluated in fp32."""
    c = load("ssim_flat")
    dev = torch.device("cuda:0")
    want = (c["map"], c["mean"], c["grad"])
    got = fused_map_mean_grad(c["img1"].to(dev), c["img2"].to(dev), c["dL_dmap"].to(dev))
    f32 = ssim_oracle.ssim_and_grad(c["img1"], c["img2"], c["dL_dmap"], dtype=torch.float32)   # CPU: no TF32
    ours, theirs = errors(got, want), errors(f32, want)
    for what, e_ours, e_ref in zip(("map", "mean", "grad"), ours, theirs):
        assert e_ours <= 2 * e_ref + 1e-9, (what, e_ours, e_ref)


def textured_pair(H, W, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    gt = torch.rand(3, H, W, generator=g, device=dev)
    blur = torch.nn.functional.avg_pool2d(gt[None], 5, 1, 2)[0]
    img = (blur + 0.05 * torch.randn(3, H, W, generator=g, device=dev)).clamp(0, 1)
    return img, gt, torch.randn(H, W, generator=g, device=dev)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(1080, 1920), (2160, 4096)])
def test_fused_against_oracle_at_image_sizes(H, W):
    dev = torch.device("cuda:0")
    img, gt, G = textured_pair(H, W, 7, dev)
    got = fused_map_mean_grad(img, gt, G)
    torch.backends.cudnn.allow_tf32, was = False, torch.backends.cudnn.allow_tf32
    try:
        want = ssim_oracle.ssim_and_grad(img, gt, G)     # fp64 on the GPU
    finally:
        torch.backends.cudnn.allow_tf32 = was
    emap, emean, egrad = errors(got, want)
    assert emap <= 2e-5 and emean <= 1e-6 and egrad <= 2e-5, (H, W, emap, emean, egrad)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 7, 5), (3, 1, 1), (3, 17, 33), (2, 3, 40, 70), (1, 3, 31, 64)])
def test_ranks_reductions_and_odd_sizes(shape):
    import fused_ssim
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(3)
    a, b = torch.rand(shape, generator=g, device=dev), torch.rand(shape, generator=g, device=dev)
    map_shape = shape[:-3] + shape[-2:]
    G = torch.randn(map_shape, generator=g, device=dev)
    smap, mean, grad = fused_map_mean_grad(a, b, G)
    assert smap.shape == map_shape and mean.shape == () and grad.shape == shape
    want = ssim_oracle.ssim_and_grad(a.cpu(), b.cpu(), G.cpu())
    emap, emean, egrad = errors((smap, mean, grad), want)
    assert emap <= 2e-5 and emean <= 1e-6 and egrad <= 2e-5, (shape, emap, emean, egrad)
    with torch.no_grad():                                # no gradient wanted: no factors, same map
        assert torch.equal(fused_ssim.ssim(a, b, size_average=False), smap)


@pytest.mark.gpu
def test_two_runs_are_bitwise_identical():
    dev = torch.device("cuda:0")
    img, gt, G = textured_pair(540, 960, 11, dev)
    r1 = fused_map_mean_grad(img, gt, G)
    r2 = fused_map_mean_grad(img, gt, G)
    assert all(torch.equal(x, y) for x, y in zip(r1, r2))


@pytest.mark.gpu
def test_forward_backward_do_not_synchronise():
    import fused_ssim
    dev = torch.device("cuda:0")
    img, gt, G = textured_pair(200, 300, 13, dev)
    x = img.clone().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for size_average in (False, True):
            s = fused_ssim.ssim(x, gt, size_average=size_average)
            ((1.0 - s) * 1.0).mean().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert x.grad is not None


@pytest.mark.gpu
def test_wrapper_refuses_unsupported_input():
    import fused_ssim
    dev = torch.device("cuda:0")
    a, b = torch.rand(3, 16, 16, device=dev), torch.rand(3, 16, 16, device=dev)
    for args, kw in [((a.double(), b.double()), {}), ((a, b), {"window_size": 7}), ((a[:2], b[:2]), {}),
                     ((a, b[:, :8]), {}), ((a, b.clone().requires_grad_(True)), {}), ((a, b.cpu()), {})]:
        assert not fused_ssim.supported(*args, **kw)
        with pytest.raises(RuntimeError):
            fused_ssim.ssim(*args, **kw)


@pytest.mark.gpu
def test_hook_falls_back_for_unsupported_input_on_the_gpu():
    import fused_ssim
    import wildgaussians_fused as wf
    m = fake_method_module("_fake_wg_method_gpu")
    try:
        original = m.ssim
        model = m.Model()
        wf.enable(model, optimizer=False, ssim=True)
        dev = torch.device("cuda:0")
        a, b = torch.rand(3, 20, 24, device=dev), torch.rand(3, 20, 24, device=dev)
        fused = m.ssim(a, b, size_average=False)
        assert m.calls == [] and torch.equal(fused, fused_ssim.ssim(a, b, size_average=False))
        m.ssim(a.double(), b.double())                              # fp64
        m.ssim(a, b.clone().requires_grad_(True))                   # a gradient for img2
        m.ssim(a.cpu(), b.cpu())                                    # CPU tensors
        assert m.calls == ["cuda", "cuda", "cpu"]
        wf.disable(model)
        assert m.ssim is original
    finally:
        sys.modules.pop(m.__name__, None)


def loss_block(m, image, gt_image, lambda_dssim=0.2, retain_graph=False):
    """The statements of method.py:1948-1966 with loss_mult = 1 and no uncertainty model (``ssim`` looked up in `m`)."""
    Ll1 = torch.nn.functional.l1_loss(image, gt_image, reduction="none")
    ssim_value = m.ssim(image, gt_image, size_average=False)
    loss = (1.0 - lambda_dssim) * (Ll1 * 1.0).mean() + lambda_dssim * ((1.0 - ssim_value) * 1.0).mean() + 0
    loss.backward(retain_graph=retain_graph)
    return loss


@pytest.mark.gpu
def test_loss_block_through_the_unmodified_method_py():
    """`enable(model, ssim=True)`: the loss statements of method.py:1948-1966 on `_render_internal`'s image give every
    parameter gradient within 1e-4 of its tensor's maximum of the run with the reference's own ``ssim`` (TF32 off).

    One render, three backward passes through it: the reference's ``ssim``, the hooked one, and the float64 oracle.  A
    gradient that is nearly cancelled (its maximum far below the terms it sums) amplifies the fp32 rounding of dL/dimage
    in both implementations; such a tensor passes when the fused result is at most twice as far from the float64 run as
    the reference's own (the bar of the near-flat image)."""
    import synthetic
    import wg_harness as wh
    import wildgaussians_fused as wf
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    import diff_gaussian_rasterization as ours
    dev = torch.device("cuda:0")
    kw = dict(P=30_000, W=320, H=200, seed=31)
    scene = synthetic.make_scene(sh_degree=3, **kw)
    cam = wh.make_camera(scene)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    gt = torch.rand(3, kw["H"], kw["W"], generator=torch.Generator().manual_seed(4)).to(dev)
    model, cfg = wh.make_model(m, Config, scene, dev, seed=kw["seed"])
    original = m.ssim
    f64 = types.SimpleNamespace(ssim=lambda a, b, size_average=True: ssim_oracle.ssim(a, b, size_average=size_average).float())
    was = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    grads = {}
    try:
        wf.enable(model, optimizer=False)
        out = model._render_internal(cam, cfg, kernel_size=cfg.kernel_size, embedding=model.appearance_embeddings[0])
        for arm in ("reference", "fused", "float64"):
            for p in model.parameters():
                p.grad = None
            if arm == "fused":
                wf.enable(model, optimizer=False, ssim=True)
                assert m.ssim is not original
            loss_block(f64 if arm == "float64" else m, out["render"], gt, retain_graph=True)
            grads[arm] = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
            wf.disable(model)
            assert m.ssim is original
    finally:
        torch.backends.cudnn.allow_tf32 = was
        m.ssim = original
    ref, fused, exact = grads["reference"], grads["fused"], grads["float64"]
    assert ref.keys() == fused.keys() and len(ref) >= 6
    for n, g0 in ref.items():
        d = float((fused[n] - g0).abs().max())
        if d <= 1e-4 * float(g0.abs().max()):
            continue
        e_fused, e_ref = float((fused[n] - exact[n]).abs().max()), float((g0 - exact[n]).abs().max())
        assert e_fused <= 2 * e_ref, (n, d, float(g0.abs().max()), e_fused, e_ref)
