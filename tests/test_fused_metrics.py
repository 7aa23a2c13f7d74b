"""Fused evaluation metrics (csrc/metrics.cu, fused_metrics.py, wildgaussians_fused.enable_metrics).

CPU: the float64 oracle against the reference's own goldens, the C entry point's argument checks, and the hook's
rebinding and fall-back.  GPU: the fused ``compute_metrics`` against the goldens, the oracle and the live reference
(``oracle/_ref/py``) at evaluation sizes; LPIPS through seeded random-weight networks; edge cases; determinism, launches
and synchronisations; and the hook through the reference's unmodified evaluation protocols.
"""
import ctypes
import glob
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import metrics_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = sorted(os.path.basename(p)[len("metrics_"):-len(".npz")] for p in glob.glob(os.path.join(GOLDEN, "metrics_*.npz")))
KEYS = ("psnr", "ssim", "mae", "mse")


def load(name):
    z = np.load(os.path.join(GOLDEN, f"metrics_{name}.npz"))
    c = {k: z[k] for k in z.files}
    if int(c["half"]):
        c["pred"], c["gt"] = c["pred"][:, c["pred"].shape[1] // 2:], c["gt"][:, c["gt"].shape[1] // 2:]
    return c


def f32_ulps(x, ref):
    """|x - ref| in units of the float32 spacing at ref."""
    ref = np.asarray(ref, dtype=np.float32)
    return np.abs(np.asarray(x, dtype=np.float64) - ref.astype(np.float64)) / np.spacing(np.abs(ref)).astype(np.float64)


# ---------------------------------------------------------------------------------------------------------------- CPU

def test_golden_cases_cover_the_issue_matrix():
    assert {"nerfw_half_u8", "batch_f32", "rgba_pred", "out_of_range", "constant_u8", "tiny_11x11"} <= set(CASES)
    assert not load("nerfw_half_u8")["gt"].flags.c_contiguous


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_goldens(name):
    c = load(name)
    o = mo.metrics(c["pred"], c["gt"])
    assert o["ssim"].shape == c["ssim"].shape
    assert np.abs(o["ssim"] - c["ssim"]).max() <= 1e-12
    # the reference's float32 np.mean is within a few ulp of the exact mean
    for k in ("mse", "mae"):
        assert f32_ulps(c[k], o[k].astype(np.float32)).max() <= 4, (k, c[k], o[k])


def test_taps_are_the_oracles_gaussian():
    import fused_metrics as fm
    assert np.abs(fm.dmpix_taps() - mo.gaussian_taps()).max() <= 1e-17
    assert fm._C1 == mo.C1 and fm._C2 == mo.C2


def test_metrics_entry_point_validates_its_arguments():
    import diff_gaussian_rasterization._C as C
    lib = C._lib
    assert lib.gsr_metrics_scratch_bytes(1, 10, 64, 3) == 0
    assert lib.gsr_metrics_scratch_bytes(1, 64, 10, 3) == 0
    assert lib.gsr_metrics_scratch_bytes(0, 64, 64, 3) == 0
    assert lib.gsr_metrics_scratch_bytes(70000, 64, 64, 1) == 0
    assert lib.gsr_metrics_scratch_bytes(2, 11, 11, 3) == 2 * 3 * 3 * 8       # one CTA per (image, channel)
    assert lib.gsr_metrics_scratch_bytes(1, 1080, 960, 3) == 30 * 67 * 3 * 3 * 8
    assert lib.gsr_metrics_forward(None, None) == -1 and b"args is NULL" in lib.gsr_last_error()
    a = C.GsrMetricsArgs(B=1, H=10, W=64, C=3)
    assert lib.gsr_metrics_forward(ctypes.byref(a), None) == -1 and b"bad metric sizes" in lib.gsr_last_error()
    a = C.GsrMetricsArgs(B=1, H=64, W=64, C=3)
    assert lib.gsr_metrics_forward(ctypes.byref(a), None) == -1 and b"NULL" in lib.gsr_last_error()
    a.a = a.b = a.sums = a.scratch = 256
    a.lpips_a = 256
    assert lib.gsr_metrics_forward(ctypes.byref(a), None) == -1 and b"lpips_a and lpips_b" in lib.gsr_last_error()
    a.lpips_a = None
    a.taps[3] = float("nan")
    assert lib.gsr_metrics_forward(ctypes.byref(a), None) == -1 and b"taps[3]" in lib.gsr_last_error()


def _fake_evaluation():
    """A module holding a stand-in ``compute_metrics`` by name, and a second module that imported it."""
    calls = []

    def compute_metrics(pred, gt, *, reduce=True, run_lpips_vgg=False):
        calls.append((pred.shape, reduce, run_lpips_vgg))
        return {"psnr": float(np.sum(pred)), "reduce": reduce}

    ev = types.ModuleType("fake_wg_evaluation")
    ev.compute_metrics = compute_metrics
    user = types.ModuleType("fake_wg_train")
    user.compute_metrics = compute_metrics
    other = types.ModuleType("fake_wg_other")
    other.compute_metrics = lambda *a, **k: None
    return ev, user, other, calls


def test_enable_metrics_rebinds_by_identity_and_falls_back(monkeypatch):
    import wildgaussians_fused as wf
    ev, user, other, calls = _fake_evaluation()
    original, unrelated = ev.compute_metrics, other.compute_metrics
    for m in (ev, user, other):
        monkeypatch.setitem(sys.modules, m.__name__, m)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)        # as on a CPU-only machine
    wf.enable_metrics(ev)
    hook = ev.compute_metrics
    assert hook is not original and hook.__wrapped__ is original
    assert user.compute_metrics is hook and other.compute_metrics is unrelated
    wf.enable_metrics(ev)                                                # enabling twice does not wrap twice
    assert ev.compute_metrics is hook
    x = np.full((1, 16, 16, 3), 0.5, np.float32)
    assert hook(x, x, reduce=False, run_lpips_vgg=True) == original(x, x, reduce=False, run_lpips_vgg=True)
    assert calls[0] == calls[1] == ((1, 16, 16, 3), False, True)
    small = np.zeros((8, 8, 3), np.uint8)
    assert hook(small, small) == original(small, small)
    wf.disable_metrics(ev)
    assert ev.compute_metrics is original and user.compute_metrics is original and other.compute_metrics is unrelated
    wf.disable_metrics(ev)
    assert ev.compute_metrics is original


def test_supported_matrix(monkeypatch):
    import fused_metrics as fm
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    u8 = np.zeros((20, 30, 3), np.uint8)
    assert fm.supported(u8, u8)
    assert fm.supported(np.zeros((2, 20, 30, 4), np.float16), np.zeros((2, 20, 30, 3), np.float64))   # RGBA pred
    assert fm.supported(u8[:, 15:], u8[:, 15:])                                                       # not contiguous
    assert "smaller" in fm.why_unsupported(u8[:10], u8[:10])
    assert "smaller" in fm.why_unsupported(u8[:, :10], u8[:, :10])
    assert "dtype" in fm.why_unsupported(u8.astype(np.int16), u8)
    assert "shapes" in fm.why_unsupported(u8[:, :, :2], u8)
    assert "shapes" in fm.why_unsupported(u8[None], u8)
    assert "shapes" in fm.why_unsupported(u8[0], u8[0])
    assert "numpy" in fm.why_unsupported(torch.zeros(20, 30, 3), u8)
    assert "images" in fm.why_unsupported(np.zeros((0, 20, 30, 3), np.uint8), np.zeros((0, 20, 30, 3), np.uint8))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    assert "CUDA" in fm.why_unsupported(u8, u8)


# ---------------------------------------------------------------------------------------------------------------- GPU

class ZeroLPIPS(torch.nn.Module):
    def forward(self, a, b):
        return a.new_zeros((a.shape[0], 1, 1, 1))


@pytest.fixture
def ev():
    """The reference's evaluation module (oracle/_ref/py) with a zero LPIPS network in its cache."""
    ref = os.path.join(ROOT, "oracle", "_ref", "py")
    assert os.path.exists(os.path.join(ref, "wildgaussians", "evaluation.py")), "build() copies the reference package"
    if ref not in sys.path:
        sys.path.insert(0, ref)
    import wildgaussians.evaluation as m
    saved = dict(m._LPIPS_CACHE)
    m._LPIPS_CACHE.clear()
    m._LPIPS_CACHE["alex"] = ZeroLPIPS()
    yield m
    m._LPIPS_CACHE.clear()
    m._LPIPS_CACHE.update(saved)


def fused(pred, gt, ev, **kw):
    import fused_metrics as fm
    assert fm.supported(pred, gt)
    return fm.compute_metrics(pred, gt, evaluation=ev, **kw)


def same_types(a, b):
    assert list(a) == list(b)
    for k in a:
        assert type(a[k]) is type(b[k]), (k, type(a[k]), type(b[k]))
        assert np.shape(a[k]) == np.shape(b[k]) and getattr(a[k], "dtype", None) == getattr(b[k], "dtype", None), k


def check_against(out, ref, pred, gt):
    """The thresholds of the fused path: SSIM within 1e-10 of the reference; MSE and MAE within 1 ulp of the exact
    mean and no further from the reference than the reference is from the exact mean (+1 ulp); PSNR from the MSE."""
    exact = mo.metrics(pred, gt)
    assert np.all(np.abs(np.asarray(out["ssim"]) - np.asarray(ref["ssim"])) <= 1e-10)
    assert np.all(np.abs(np.asarray(out["ssim"]) - exact["ssim"]) <= 1e-10)
    for k in ("mse", "mae"):
        e32 = exact[k].astype(np.float32)
        assert f32_ulps(out[k], e32).max() <= 1, (k, out[k], exact[k])
        spread = np.abs(np.asarray(ref[k], np.float64) - exact[k]) + np.spacing(np.abs(e32)).astype(np.float64)
        assert np.all(np.abs(np.asarray(out[k], np.float64) - np.asarray(ref[k], np.float64)) <= spread), k
    assert np.array_equal(np.asarray(out["psnr"]), np.asarray(-10 * np.log10(out["mse"])))


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_fused_matches_goldens(name, ev):
    c = load(name)
    out = fused(c["pred"], c["gt"], ev, reduce=False)
    ref = ev.compute_metrics(c["pred"], c["gt"], reduce=False)
    same_types(out, ref)
    for k in KEYS:
        assert np.shape(out[k]) == c[k].shape
    check_against(out, ref, c["pred"], c["gt"])
    exact = mo.metrics(c["pred"], c["gt"])
    for k in ("mse", "mae"):                                  # the float32 rounding of the exact mean, on every golden
        assert np.array_equal(np.asarray(out[k]), exact[k].astype(np.float32)), (k, out[k], exact[k])
    assert np.all(np.abs(np.asarray(out["ssim"]) - c["ssim"]) <= 1e-10)


def _photo(rng, shape):
    """A textured uint8 photograph-like image and a noisy rendering of it."""
    H, W = shape[-3], shape[-2]
    y, x = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    base = 0.5 + 0.25 * np.sin(x / 17.0)[..., None] * np.cos(y[..., None] / 23.0 + np.arange(shape[-1]))
    gt = np.clip(base * 255 + rng.normal(0, 6, shape), 0, 255).astype(np.uint8)
    pred = np.clip(gt + rng.normal(0, 10, shape), 0, 255).astype(np.uint8)
    return pred, gt


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["nerfw_half_u8", "full_f32", "batch_f32"])
@pytest.mark.parametrize("reduce", [False, True])
def test_fused_matches_live_reference(kind, reduce, ev):
    rng = np.random.default_rng(11)
    if kind == "nerfw_half_u8":
        pred, gt = _photo(rng, (1080, 1920, 3))
        pred, gt = pred[:, 960:], gt[:, 960:]                 # NerfWEvaluationProtocol.evaluate's right half
    elif kind == "full_f32":
        pred, gt = (x[None].astype(np.float32) / 255 for x in _photo(rng, (1080, 1920, 3)))
    else:
        pred, gt = (x.astype(np.float32) / 255 for x in _photo(rng, (2, 3, 67, 93, 3)))
    out = fused(pred, gt, ev, reduce=reduce)
    ref = ev.compute_metrics(pred, gt, reduce=reduce)
    same_types(out, ref)
    if not reduce:
        check_against(out, ref, pred, gt)
    else:
        exact = mo.metrics(pred, gt)
        assert abs(out["ssim"] - ref["ssim"]) <= 1e-10
        for k in ("mse", "mae"):
            e32 = np.float32(np.mean(exact[k].astype(np.float32)))
            assert abs(out[k] - ref[k]) <= abs(ref[k] - float(exact[k].mean())) + 2 * float(np.spacing(e32)), k
        assert out["lpips"] == ref["lpips"] == 0.0


@pytest.mark.gpu
def test_lpips_through_seeded_random_networks(ev):
    """alex and vgg with seeded random weights in _LPIPS_CACHE: the fused path feeds the same values in the same layout,
    so LPIPS agrees to 1e-6 (bitwise equality is reported)."""
    from wildgaussians._metrics_lpips import LPIPS
    torch.manual_seed(0)
    ev._LPIPS_CACHE["alex"] = LPIPS(pretrained=False, net="alex", pnet_rand=True, verbose=False)
    ev._LPIPS_CACHE["vgg"] = LPIPS(pretrained=False, net="vgg", pnet_rand=True, verbose=False)
    rng = np.random.default_rng(3)
    pred, gt = _photo(rng, (2, 180, 240, 3))
    ref = ev.compute_metrics(pred, gt, reduce=False, run_lpips_vgg=True)
    out = fused(pred, gt, ev, reduce=False, run_lpips_vgg=True)
    same_types(out, ref)
    for k in ("lpips", "lpips_vgg"):
        assert np.abs(out[k] - ref[k]).max() <= 1e-6, (k, out[k], ref[k])
        print(f"{k}: bitwise equal {np.array_equal(out[k], ref[k])}, max diff {np.abs(out[k] - ref[k]).max():.3e}")
    red = fused(pred, gt, ev, reduce=True, run_lpips_vgg=True)
    assert abs(red["lpips_vgg"] - float(ref["lpips_vgg"].mean())) <= 1e-6


@pytest.mark.gpu
def test_edge_cases_equal_the_reference(ev):
    import fused_metrics as fm
    from diff_gaussian_rasterization import _C
    rng = np.random.default_rng(5)
    pred, gt = (x.astype(np.float32) / 255 for x in _photo(rng, (1, 64, 80, 3)))
    # a NaN pixel: NaN wherever the reference gives NaN
    p = pred.copy()
    p[0, 30, 40, 1] = np.nan
    out, ref = fused(p, gt, ev, reduce=False), ev.compute_metrics(p, gt, reduce=False)
    for k in KEYS:
        assert np.array_equal(np.isnan(out[k]), np.isnan(ref[k])), k
    assert np.isnan(out["mse"]).all() and np.isnan(out["ssim"]).all()
    # a difference confined to the last 10 rows and columns, outside the SSIM's valid map
    p = gt.copy()
    p[0, -10:, :, 0] += 0.25
    p[0, :, -10:, 2] -= 0.125
    out, ref = fused(p, gt, ev, reduce=False), ev.compute_metrics(p, gt, reduce=False)
    assert out["mse"][0] > 0 and out["mae"][0] > 0
    check_against(out, ref, p, gt)
    # RGBA pred, float64 and float16 inputs
    rgba = np.concatenate([pred, rng.random((1, 64, 80, 1), dtype=np.float32)], -1)
    for p, g in ((rgba, gt), (pred.astype(np.float64), gt.astype(np.float64)), (pred.astype(np.float16), gt.astype(np.float16))):
        out, ref = fused(p, g, ev, reduce=False), ev.compute_metrics(p, g, reduce=False)
        same_types(out, ref)
        check_against(out, ref, p, g)
    # H or W < 11: the reference runs, the fused entry point is not called
    before = _C._lib.gsr_launch_count()
    for shape in ((10, 40, 3), (40, 10, 3)):
        p, g = _photo(rng, shape)
        assert not fm.supported(p, g)
        out, ref = fm.compute_metrics(p, g, reduce=False, evaluation=ev), ev.compute_metrics(p, g, reduce=False)
        same_types(out, ref)
        for k in KEYS:
            assert np.array_equal(out[k], ref[k], equal_nan=True)
    assert _C._lib.gsr_launch_count() == before


# Synchronising runtime calls.  cudaDeviceSynchronize is left out: the call makes none, and the profiler itself makes
# one when it stops.
SYNC_CALLS = ("cudaStreamSynchronize", "cudaEventSynchronize", "cudaMemcpy")


@pytest.mark.gpu
def test_deterministic_two_launches_one_synchronisation(ev):
    import fused_metrics as fm
    from diff_gaussian_rasterization import _C
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(9)
    pred, gt = _photo(rng, (1080, 1920, 3))
    pred, gt = pred[:, 960:], gt[:, 960:]
    first = fused(pred, gt, ev, reduce=False)
    second = fused(pred, gt, ev, reduce=False)
    for k in first:
        assert np.asarray(first[k]).tobytes() == np.asarray(second[k]).tobytes(), k
    torch.cuda.synchronize()
    before = _C._lib.gsr_launch_count()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fused(pred, gt, ev, reduce=True)
    assert _C._lib.gsr_launch_count() - before == fm.LAUNCHES
    names = [e.name for e in prof.events()]
    syncs = [n for n in names if n in SYNC_CALLS]
    copies = [n for n in names if n.startswith("Memcpy")]
    print(f"synchronising calls {syncs}; copy calls {names.count('cudaMemcpyAsync')}; copies recorded on the device {copies}")
    assert syncs == ["cudaStreamSynchronize"], syncs
    # Copies are counted at the runtime API: the profiler can drop the device records of copies that run at the very
    # start of its window (after other profiled tests it kept the two read-backs and lost both uploads).  Four calls:
    # one upload per image, the sums and the LPIPS values back.
    assert names.count("cudaMemcpyAsync") == 4, names
    assert not any("Pageable" in n for n in copies), copies
    staging = fm._buffers[torch.device("cuda", torch.cuda.current_device())].t
    assert all(staging[k].is_pinned() for k in ("host0", "host1", "host_sums", "host_lpips"))


def _dataset(gt):
    return {"images": [gt], "metadata": {"color_space": "srgb"}}


@pytest.mark.gpu
def test_hook_through_the_reference_protocols(ev):
    import fused_metrics as fm
    import wildgaussians_fused as wf
    from diff_gaussian_rasterization import _C
    from wildgaussians.datasets.phototourism import NerfWEvaluationProtocol
    rng = np.random.default_rng(13)
    pred, gt = (x.astype(np.float32) / 255 for x in _photo(rng, (240, 320, 3)))
    pred_rgba = np.concatenate([pred, np.ones_like(pred[..., :1])], -1)
    original = ev.compute_metrics
    unhooked = [ev.DefaultEvaluationProtocol().evaluate({"color": pred_rgba}, _dataset(gt)),
                NerfWEvaluationProtocol().evaluate({"color": pred}, _dataset(gt))]
    before_enable = NerfWEvaluationProtocol()
    wf.enable_metrics(ev)
    try:
        launches = _C._lib.gsr_launch_count()
        hooked = [ev.DefaultEvaluationProtocol().evaluate({"color": pred_rgba}, _dataset(gt)),
                  NerfWEvaluationProtocol().evaluate({"color": pred}, _dataset(gt))]
        assert _C._lib.gsr_launch_count() - launches == 2 * fm.LAUNCHES
        assert before_enable._compute_metrics is original            # captured before enable_metrics: unchanged
    finally:
        wf.disable_metrics(ev)
    assert ev.compute_metrics is original
    for u, h in zip(unhooked, hooked):
        same_types(h, u)
        assert abs(h["ssim"] - u["ssim"]) <= 1e-10
        for k in ("mse", "mae", "psnr"):
            assert abs(h[k] - u[k]) <= 4 * np.spacing(np.float32(abs(u[k]))), (k, h[k], u[k])
