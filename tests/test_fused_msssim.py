"""Fused msssim / ssim_down of the uncertainty loss (csrc/msssim.cu, fused_ssim.py, wildgaussians_fused.enable(msssim=True)).

CPU: the float64 oracle against the reference's own goldens, the C entry points' argument checks, the wrappers'
refusals and the hook's fall-back.  GPU: both maps against the oracle (goldens, 1080p, 4K, edge shapes) within twice
the error of the reference's fp32 statements, determinism, no host synchronisation, launch counts, and
``UncertaintyModel._compute_losses`` of the unmodified ``method.py`` hooked against unhooked.
"""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import msssim_oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["msssim_resize", "msssim_noresize", "msssim_upsample", "msssim_batched", "msssim_flat"]


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    c = {k: torch.from_numpy(np.asarray(z[k])) for k in z.files}
    c["max_size"] = None if int(c["max_size"]) < 0 else int(c["max_size"])
    c["min_size"], c["stride"] = int(c["min_size"]), int(c["stride"])
    return c


def both(fn_ms, fn_sd, c, x, y):
    """(msssim, ssim_down) of one golden case's parameters, on the golden's output grid."""
    s = c["stride"]
    ms = fn_ms(x, y, max_size=c["max_size"], min_size=c["min_size"])
    sd = fn_sd(x, y, max_size=c["max_size"])
    return ms[:, ::s, ::s], sd[:, ::s, ::s]


# ---------------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_goldens(name):
    c = load(name)
    ms, sd = both(msssim_oracle.msssim, msssim_oracle.ssim_down, c, c["img1"], c["img2"])
    assert ms.shape == c["msssim"].shape and sd.shape == c["ssim_down"].shape
    assert float((ms - c["msssim"]).abs().max()) <= 1e-12
    assert float((sd - c["ssim_down"]).abs().max()) <= 1e-12


def test_c_entry_points_reject_bad_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib
    p = ctypes.c_void_p(256)                     # never dereferenced: every call below fails its checks first
    assert lib.gsr_msssim_scratch_bytes(1, 0, 8, 4) == 0
    assert lib.gsr_msssim_scratch_bytes(1, 400, 711, 80) > 0
    assert lib.gsr_msssim_forward(0, 8, 8, 8, 8, 4, p, p, p, p, None) == -1
    assert b"bad sizes" in lib.gsr_last_error()
    assert lib.gsr_msssim_forward(1, 8, -1, 8, 8, 4, p, p, p, p, None) == -1
    assert b"bad sizes" in lib.gsr_last_error()
    assert lib.gsr_msssim_forward(1, 8, 8, 0, 8, 4, p, p, p, p, None) == -1
    assert b"bad sizes" in lib.gsr_last_error()
    assert lib.gsr_msssim_forward(1, 8, 8, 8, 8, 0, p, p, p, p, None) == -1
    assert b"min_size" in lib.gsr_last_error()
    assert lib.gsr_msssim_forward(70000, 8, 8, 8, 8, 4, p, p, p, p, None) == -1
    assert b"too large" in lib.gsr_last_error()
    for i in range(4):
        args = [p, p, p, p]
        args[i] = None
        assert lib.gsr_msssim_forward(1, 8, 8, 8, 8, 4, *args, None) == -1
        assert b"NULL" in lib.gsr_last_error()
    assert lib.gsr_ssim_down_scratch_bytes(1, 4, 0) == 0
    assert lib.gsr_ssim_down_forward(1, 8, 8, 8, -2, p, p, p, p, None) == -1
    assert b"bad sizes" in lib.gsr_last_error()
    assert lib.gsr_ssim_down_forward(70000, 8, 8, 4, 4, p, p, p, p, None) == -1
    assert b"too large" in lib.gsr_last_error()
    assert lib.gsr_ssim_down_forward(1, 8, 8, 4, 4, p, p, p, None, None) == -1     # a resize needs scratch
    assert b"NULL" in lib.gsr_last_error()
    assert lib.gsr_ssim_down_forward(1, 8, 8, 4, 4, p, None, p, p, None) == -1
    assert b"NULL" in lib.gsr_last_error()


def test_wrappers_refuse_cpu_tensors():
    import fused_ssim
    a, b = torch.rand(1, 3, 16, 16), torch.rand(1, 3, 16, 16)
    assert not fused_ssim.supported_msssim(a, b) and not fused_ssim.supported_ssim_down(a, b)
    with pytest.raises(RuntimeError, match="CUDA"):
        fused_ssim.msssim(a, b)
    with pytest.raises(RuntimeError, match="CUDA"):
        fused_ssim.ssim_down(a, b, max_size=8)


def fake_method_module(name="_fake_wg_method_ms"):
    """A module with module-level ``msssim`` / ``ssim_down`` and a model class defined in it, like wildgaussians.method."""
    m = types.ModuleType(name)
    calls = []

    def msssim(x, y, max_size=None, min_size=200):
        calls.append(("msssim", x.device.type))
        return msssim_oracle.msssim(x, y, max_size, min_size, dtype=x.dtype)

    def ssim_down(x, y, max_size=None):
        calls.append(("ssim_down", x.device.type))
        return msssim_oracle.ssim_down(x, y, max_size, dtype=x.dtype)

    def ssim(img1, img2, window_size=11, size_average=True):
        return None

    class Model(torch.nn.Module):
        pass

    Model.__module__ = name
    m.msssim, m.ssim_down, m.ssim, m.Model, m.calls = msssim, ssim_down, ssim, Model, calls
    sys.modules[name] = m
    return m


def test_hook_falls_back_to_the_original_and_disable_restores_both():
    import wildgaussians_fused as wf
    m = fake_method_module()
    try:
        ms0, sd0, ssim0 = m.msssim, m.ssim_down, m.ssim
        model = m.Model()
        wf.enable(model, optimizer=False)
        wf.enable(model, optimizer=False, ssim=True)
        assert m.msssim is ms0 and m.ssim_down is sd0                 # default: untouched, also with ssim=True
        wf.disable(model)
        wf.enable(model, optimizer=False, msssim=True)
        assert m.msssim is not ms0 and m.ssim_down is not sd0 and m.ssim is ssim0
        hooked = (m.msssim, m.ssim_down)
        wf.enable(model, optimizer=False, msssim=True)                # idempotent
        assert (m.msssim, m.ssim_down) == hooked and m.msssim.__wrapped__ is ms0 and m.ssim_down.__wrapped__ is sd0
        a, b = torch.rand(1, 3, 30, 40), torch.rand(1, 3, 30, 40)
        assert m.msssim(a, b, max_size=20, min_size=8).shape == (1, 30, 40)   # CPU tensors: the originals run
        assert m.ssim_down(a, b, max_size=20).shape == (1, 30, 40)
        assert m.calls == [("msssim", "cpu"), ("ssim_down", "cpu")]
        wf.disable(model)
        assert m.msssim is ms0 and m.ssim_down is sd0 and m.ssim is ssim0
    finally:
        sys.modules.pop(m.__name__, None)


# ---------------------------------------------------------------------------------------------------------------- GPU

def no_tf32():
    class _Ctx:
        def __enter__(self):
            self.was = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = False

        def __exit__(self, *exc):
            torch.backends.cudnn.allow_tf32 = self.was
    return _Ctx()


def max_err(a, b):
    return float((a.double() - b.to(device=a.device, dtype=torch.float64)).abs().max())


def check_against_oracle(x, y, max_size, min_size, what=""):
    """Both fused maps vs the float64 oracle: max error <= 2x the fp32 statements' + 1e-9, mean error <= 1e-6."""
    import fused_ssim
    got = (fused_ssim.msssim(x, y, max_size=max_size, min_size=min_size), fused_ssim.ssim_down(x, y, max_size=max_size))
    with no_tf32():
        want = (msssim_oracle.msssim(x, y, max_size, min_size), msssim_oracle.ssim_down(x, y, max_size))
        f32 = (msssim_oracle.msssim(x, y, max_size, min_size, dtype=torch.float32),
               msssim_oracle.ssim_down(x, y, max_size, dtype=torch.float32))
    for name, g, w, r in zip(("msssim", "ssim_down"), got, want, f32):
        assert g.shape == w.shape and g.dtype == torch.float32, (what, name, g.shape, w.shape)
        e_ours, e_ref = max_err(g, w), max_err(r, w)
        assert e_ours <= 2 * e_ref + 1e-9, (what, name, e_ours, e_ref)
        assert abs(float(g.double().mean()) - float(w.mean())) <= 1e-6, (what, name)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_fused_against_reference_goldens(name):
    import fused_ssim
    c = load(name)
    dev = torch.device("cuda:0")
    x, y = c["img1"].to(dev), c["img2"].to(dev)
    got = both(fused_ssim.msssim, fused_ssim.ssim_down, c, x, y)
    with no_tf32():
        f32 = both(lambda *a, **k: msssim_oracle.msssim(*a, **k, dtype=torch.float32),
                   lambda *a, **k: msssim_oracle.ssim_down(*a, **k, dtype=torch.float32), c, x, y)
    for what, g, r in zip(("msssim", "ssim_down"), got, f32):
        want = c[what]
        e_ours, e_ref = max_err(g, want), max_err(r, want)
        assert e_ours <= 2 * e_ref + 1e-9, (name, what, e_ours, e_ref)
        m_ours, m_ref = (abs(float(t.double().mean()) - float(want.mean())) for t in (g, r))
        # on the near-flat pair E[x^2] - mu^2 cancels, and sigma = sqrt(.) amplifies that near 0: there the bar for the
        # mean is also twice the fp32 statements' error, as for the photometric SSIM's near-flat golden
        assert m_ours <= (2 * m_ref + 1e-9 if name == "msssim_flat" else 1e-6), (name, what, m_ours, m_ref)


def textured_pair(B, H, W, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    gt = torch.rand(B, 3, H // 8 + 1, W // 8 + 1, generator=g, device=dev)
    gt = torch.nn.functional.interpolate(gt, size=(H, W), mode="bilinear", align_corners=False)
    pred = (gt + 0.05 * torch.randn(B, 3, H, W, generator=g, device=dev)).clamp(0, 1)
    return pred, gt


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(1080, 1920), (2160, 4096)])
def test_fused_against_oracle_at_image_sizes(H, W):
    dev = torch.device("cuda:0")
    pred, gt = textured_pair(1, H, W, 7, dev)
    check_against_oracle(gt, pred, 400, 80, (H, W))


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,max_size,min_size", [
    (1, 7, 9, None, 3),          # smaller than the window
    (1, 9, 40, 20, 4),           # H below 11, area upsample in ssim_down
    (1, 50, 64, None, 50),       # at min_size: no coarse level
    (1, 51, 70, None, 50),       # min_size + 1: one coarse level
    (2, 45, 77, 30, 8),          # batched, resized
    (1, 60, 90, None, 200),      # max_size None, the default min_size
])
def test_edge_shapes(B, H, W, max_size, min_size):
    dev = torch.device("cuda:0")
    pred, gt = textured_pair(B, H, W, 3, dev)
    ms, sd = check_against_oracle(gt, pred, max_size, min_size, (B, H, W, max_size, min_size))
    assert ms.shape == (B, H, W) and sd.shape == (B, H, W)


@pytest.mark.gpu
def test_two_runs_are_bitwise_identical():
    import fused_ssim
    dev = torch.device("cuda:0")
    pred, gt = textured_pair(1, 540, 960, 11, dev)
    r1 = (fused_ssim.msssim(gt, pred, 400, 80), fused_ssim.ssim_down(gt, pred, 400))
    r2 = (fused_ssim.msssim(gt, pred, 400, 80), fused_ssim.ssim_down(gt, pred, 400))
    assert all(torch.equal(a, b) for a, b in zip(r1, r2))


@pytest.mark.gpu
def test_no_host_synchronisation():
    import fused_ssim
    dev = torch.device("cuda:0")
    pred, gt = textured_pair(1, 200, 300, 13, dev)
    fused_ssim.msssim(gt, pred, 150, 40)                 # warm: caching allocator pools exist
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for max_size in (None, 150, 400):
            fused_ssim.msssim(gt, pred, max_size=max_size, min_size=40)
            fused_ssim.ssim_down(gt, pred, max_size=max_size)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_launch_counts():
    import fused_ssim
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    pred, gt = textured_pair(1, 1080, 1920, 5, dev)

    def launches(fn):
        n0 = _C.launch_count()
        fn()
        return _C.launch_count() - n0

    assert launches(lambda: fused_ssim.msssim(gt, pred, max_size=400, min_size=80)) == 10   # 400x711 + 3 coarse levels
    assert launches(lambda: fused_ssim.ssim_down(gt, pred, max_size=400)) == 3
    assert launches(lambda: fused_ssim.ssim_down(gt, pred)) == 1
    assert launches(lambda: fused_ssim.msssim(gt[..., :300, :400], pred[..., :300, :400], min_size=80)) == 6   # 2 coarse


@pytest.mark.gpu
def test_wrappers_refuse_unsupported_input():
    import fused_ssim
    dev = torch.device("cuda:0")
    a, b = torch.rand(1, 3, 16, 16, device=dev), torch.rand(1, 3, 16, 16, device=dev)
    for args, kw in [((a.double(), b.double()), {}), ((a[0], b[0]), {}), ((a[:, :2], b[:, :2]), {}),
                     ((a, b[..., :8]), {}), ((a.clone().requires_grad_(True), b), {}),
                     ((a, b.clone().requires_grad_(True)), {}), ((a, b.cpu()), {}), ((a, b), {"max_size": 0})]:
        assert not fused_ssim.supported_msssim(*args, **kw) and not fused_ssim.supported_ssim_down(*args, **kw)
        with pytest.raises(RuntimeError):
            fused_ssim.msssim(*args, **kw)
        with pytest.raises(RuntimeError):
            fused_ssim.ssim_down(*args, **kw)
    assert not fused_ssim.supported_msssim(a, b, min_size=0)
    assert not fused_ssim.supported_msssim(a, b, min_size=2.5)


@pytest.mark.gpu
def test_hook_falls_back_for_unsupported_input_on_the_gpu():
    import fused_ssim
    import wildgaussians_fused as wf
    m = fake_method_module("_fake_wg_method_ms_gpu")
    try:
        model = m.Model()
        wf.enable(model, optimizer=False, msssim=True)
        dev = torch.device("cuda:0")
        a, b = torch.rand(1, 3, 20, 24, device=dev), torch.rand(1, 3, 20, 24, device=dev)
        assert torch.equal(m.msssim(a, b, max_size=16, min_size=4), fused_ssim.msssim(a, b, 16, 4))
        assert torch.equal(m.ssim_down(a, b, max_size=16), fused_ssim.ssim_down(a, b, 16))
        assert m.calls == []
        m.msssim(a.double(), b.double(), min_size=4)
        m.ssim_down(a, b.clone().requires_grad_(True), max_size=16)
        assert m.calls == [("msssim", "cuda"), ("ssim_down", "cuda")]
        wf.disable(model)
    finally:
        sys.modules.pop(m.__name__, None)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["l2reg", "dino+mssim", "dino"])
def test_compute_losses_through_the_unmodified_method_py(mode):
    """`enable(model, msssim=True)`: ``UncertaintyModel._compute_losses`` (method.py:363-433) with a random-weight
    backbone, hooked against the reference's own functions (TF32 off), and a third arm with the float64 oracle."""
    import wg_harness as wh
    import wg_uncertainty as wu
    import wildgaussians_fused as wf
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    dev = torch.device("cuda:0")
    pred, gt = textured_pair(1, 420, 616, 17, dev)
    model, _ = wu.make_uncertainty_model(m, Config, mode, dev, seed=3)
    originals = (m.msssim, m.ssim_down)
    f64 = (lambda x, y, max_size=None, min_size=200: msssim_oracle.msssim(x, y, max_size, min_size).float(),
           lambda x, y, max_size=None: msssim_oracle.ssim_down(x, y, max_size).float())
    res = {}
    fake = type("Probe", (), {"__module__": m.__name__})()      # enable() finds the method module through the type
    try:
        with no_tf32():
            for arm in ("reference", "fused", "float64"):
                if arm == "fused":
                    wf.enable(fake, optimizer=False, msssim=True)
                    assert m.msssim is not originals[0] and m.ssim_down is not originals[1]
                elif arm == "float64":
                    m.msssim, m.ssim_down = f64
                res[arm] = wu.compute_losses(model, gt[0], pred[0], seed=5)
                wf.disable(fake)
                m.msssim, m.ssim_down = originals
    finally:
        m.msssim, m.ssim_down = originals
    (l0, met0, lm0, g0), (l1, met1, lm1, g1), (_, _, _, g2) = res["reference"], res["fused"], res["float64"]
    assert abs(float(l1) - float(l0)) <= 1e-5
    for k in ("loss", "msssim", "ssim_discounted"):
        assert abs(met1[k] - met0[k]) <= 1e-5, (k, met1[k], met0[k])
    assert float((lm1 - lm0).abs().max()) <= 1e-5
    assert g0.keys() == g1.keys() and len(g0) >= 2
    for n, r in g0.items():
        d = float((g1[n] - r).abs().max())
        if d <= 1e-4 * float(r.abs().max()):
            continue
        e_fused, e_ref = float((g1[n] - g2[n]).abs().max()), float((r - g2[n]).abs().max())
        assert e_fused <= 2 * e_ref, (n, d, float(r.abs().max()), e_fused, e_ref)
