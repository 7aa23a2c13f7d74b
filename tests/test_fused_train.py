"""The fused training iteration (``fused_train``, ``csrc/train_loss.cu``): the loss op against a float64 oracle, the
byte staging of training images, the whole ``train_iteration`` against the reference's own, and its host
synchronisations."""
import ctypes
import os
import random
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "wild-gaussians_b200"), ROOT, os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)


# ---------------------------------------------------------------------------------------------------------------- CPU

class _FakeModel(types.SimpleNamespace):
    pass


def _fake_method(cuda=True, appearance=True, sh_degree=3, uncertainty="disabled", max_size=None, debug=False, masks=False,
                 image_dtype=torch.float32):
    t = lambda *s: types.SimpleNamespace(is_cuda=cuda, dtype=torch.float32, shape=s)
    cfg = types.SimpleNamespace(appearance_enabled=appearance, appearance_separate_tuned_color=True, appearance_model_sh=False,
                                sh_degree=sh_degree, appearance_embedding_dim=32, debug=debug, uncertainty_mode=uncertainty,
                                uncertainty_dino_max_size=max_size)
    um = None if uncertainty == "disabled" else types.SimpleNamespace(config=cfg)
    model = _FakeModel(config=cfg, xyz=t(10, 3), features_rest=t(10, 45), embeddings=t(10, 24) if appearance else None,
                       appearance_mlp=object() if appearance else None, uncertainty_model=um)
    images = [torch.zeros(3, 4, 5, dtype=image_dtype) for _ in range(2)]
    return types.SimpleNamespace(model=model, config=cfg, train_images=images,
                                 train_masks=[torch.ones(1, 4, 5) for _ in range(2)] if masks else None)


def test_supported_matrix():
    import fused_train as ft
    assert ft.supported(_fake_method())                                   # appearance on (the preset)
    assert ft.supported(_fake_method(appearance=False))                   # appearance off, SH degree 3
    assert ft.supported(_fake_method(uncertainty="dino"))
    assert ft.supported(_fake_method(masks=True))
    assert ft.supported(_fake_method(appearance=False, uncertainty="dino", masks=True))
    assert not ft.supported(_fake_method(appearance=False, sh_degree=0))
    assert not ft.supported(_fake_method(uncertainty="l2reg"))
    assert not ft.supported(_fake_method(uncertainty="dino+mssim"))
    assert not ft.supported(_fake_method(uncertainty="dino", max_size=224))
    assert not ft.supported(_fake_method(debug=True))
    assert not ft.supported(_fake_method(cuda=False))
    assert not ft.supported(_fake_method(image_dtype=torch.float64))
    bad = _fake_method(masks=True)
    bad.train_masks = bad.train_masks[:1]
    assert not ft.supported(bad)


class _CountingList(list):
    """A list that counts the passes over it."""

    def __init__(self, *a):
        super().__init__(*a)
        self.passes = 0

    def __iter__(self):
        self.passes += 1
        return super().__iter__()


class _Method:                                  # hashable and weak-referenceable, as WildGaussians is
    def __init__(self, **kw):
        self.__dict__.update(kw)


def test_images_are_checked_once_per_list_not_per_step():
    import fused_train as ft
    fake = _fake_method(masks=True)
    n = 1700                                                            # a phototourism scene's image count
    images = _CountingList([torch.zeros(3, 4, 5) for _ in range(n)])
    masks = _CountingList([torch.ones(1, 4, 5) for _ in range(n)])
    method = _Method(model=fake.model, config=fake.config, train_images=images, train_masks=masks)
    assert ft.supported(method)
    passes = (images.passes, masks.passes)
    assert passes[0] >= 1 and passes[1] >= 1
    for _ in range(5):                                                  # later steps: no pass over the dataset
        assert ft.supported(method)
    assert (images.passes, masks.passes) == passes
    images.append(torch.zeros(3, 4, 6))                                 # a list that changed is checked again
    assert not ft.supported(method)
    assert images.passes > passes[0]
    method.train_images = _CountingList(list(images)[:n])
    assert ft.supported(method)


def test_every_byte_value_round_trips_bit_for_bit():
    import fused_train as ft
    k = np.arange(256, dtype=np.float32) / np.float32(255)
    u8 = ft.as_bytes(k)
    assert u8 is not None and np.array_equal(u8, np.arange(256))
    assert np.array_equal((u8.astype(np.float32) / np.float32(255)).view(np.uint32), k.view(np.uint32))
    # the reference's own conversion (method.py:50) gives the same bits
    assert np.array_equal((np.arange(256, dtype=np.uint8).astype(np.float32) / 255.0).view(np.uint32), k.view(np.uint32))
    for off in (np.float32(0.5) / np.float32(255), np.float32(-0.0), np.float32(1.5), np.float32(np.nan)):
        x = k.copy()
        x[17] = off if not np.isnan(off) else off
        assert ft.as_bytes(x) is None, off


def test_an_image_with_one_non_byte_value_is_staged_as_fp32():
    import fused_train as ft
    img = np.rint(np.random.default_rng(0).random((6, 7, 3)) * 255).astype(np.uint8).astype(np.float32) / np.float32(255)
    e = ft._Entry(torch.from_numpy(np.moveaxis(img, -1, 0)), torch.ones(1, 6, 7))
    assert e.img_u8 is not None and e.img_f32 is None and e.mask_u8 is not None and e.mask_binary
    assert np.array_equal(e.img_u8, np.rint(img * 255).astype(np.uint8))
    img[3, 2, 1] = np.float32(0.3)
    frac = torch.full((1, 6, 7), np.float32(128) / np.float32(255))
    e = ft._Entry(torch.from_numpy(np.moveaxis(img, -1, 0)), frac)
    assert e.img_u8 is None and e.img_f32 is not None and e.mask_u8 is not None and not e.mask_binary
    e = ft._Entry(torch.from_numpy(np.moveaxis(img, -1, 0)), torch.full((1, 6, 7), 0.3))
    assert e.mask_u8 is None and e.mask_f32 is not None


def test_c_entry_points_reject_bad_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib

    def args(**kw):
        a = _C.GsrTrainLossArgs()
        a.H, a.W, a.c_l1, a.c_ssim = 8, 8, 0.8, 0.2
        for n in ("toned", "raw", "gt", "ssim_map", "ssim_partials", "loss", "metrics", "scratch", "dL_dloss", "dL_dmap",
                  "d_toned", "d_raw", "raw_scaled"):
            setattr(a, n, 0x1000)
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    fwd = lambda a: lib.gsr_train_loss_forward(ctypes.byref(a), None)
    bwd = lambda a: lib.gsr_train_loss_backward(ctypes.byref(a), None)
    for name in ("toned", "raw", "gt", "ssim_map", "loss", "metrics", "scratch"):
        assert fwd(args(**{name: None})) == -1, name
        assert "NULL" in lib.gsr_last_error().decode()
    for name in ("ssim_partials", "dL_dloss", "dL_dmap", "d_toned", "d_raw"):
        assert bwd(args(**{name: None})) == -1, name
    assert fwd(args(mask=0x2000, raw_scaled=None)) == -1
    assert bwd(args(grad_scale=0x2000, raw_scaled=None)) == -1
    for kw in (dict(H=0), dict(W=-3), dict(H=70000, W=70000), dict(c_l1=float("nan")), dict(c_ssim=float("inf"))):
        assert fwd(args(**kw)) == -1, kw
        assert bwd(args(**kw)) == -1, kw
    assert lib.gsr_train_loss_forward(None, None) == -1
    assert lib.gsr_train_loss_scratch_bytes() >= 1024 * 9 * 8
    assert lib.gsr_unpack_u8(8, 8, None, None, 0x1000, 0x1000, None) == -1
    assert lib.gsr_unpack_u8(0, 8, 0x1000, None, 0x1000, None, None) == -1
    assert lib.gsr_unpack_u8(8, 8, 0x1000, None, None, None, None) == -1
    assert lib.gsr_unpack_u8(8, 8, None, 0x1000, None, None, None) == -1


# ---------------------------------------------------------------------------------------------------------------- GPU

class no_tf32:
    def __enter__(self):
        self.was = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.was


def _inputs(H, W, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    smooth = lambda: torch.nn.functional.interpolate(torch.rand(1, 3, H // 6 + 2, W // 6 + 2, generator=g, device=dev),
                                                     size=(H, W), mode="bilinear")[0]
    gt = smooth()
    toned = (gt + 0.08 * torch.randn(3, H, W, generator=g, device=dev)).clamp(0, 1)
    raw = (0.9 * gt + 0.05 + 0.05 * torch.randn(3, H, W, generator=g, device=dev)).clamp(0, 1)
    toned[:, : H // 5, : W // 5] = gt[:, : H // 5, : W // 5]            # exact ties: sign(0) = 0
    u = torch.rand(1, H, W, generator=g, device=dev)
    binary = (u > 0.3).float()
    return toned, raw, gt, binary, u


def _weight(kind, u, binary):
    if kind is None:
        return None
    if kind == "binary":
        return binary
    if kind == "ramped":                                   # method.py:1939-1940
        return 1 + 0.37 * (binary - 1)
    if kind == "centred":                                  # method.py:1942
        return binary.sub(binary.mean() - 1).clamp(0, 2)
    raise ValueError(kind)


# (mask, weight, scale_grad)
BRANCHES = {
    "plain": (None, None, False),
    "mask": ("binary", None, False),
    "fractional_mask": ("fractional", None, False),
    "w_binary": (None, "binary", False),
    "w_ramped": (None, "ramped", False),
    "w_centred": (None, "centred", False),
    "scale_grad_ramped": (None, "ramped", True),
    "mask_scale_grad_centred": ("binary", "centred", True),
    "fractional_mask_w_ramped": ("fractional", "ramped", False),
}
SIZES = {"odd": (37, 53), "S1": (400, 640), "C3": (1080, 1920)}
CASES = [("odd", b) for b in BRANCHES] + [(s, b) for s in ("S1", "C3") for b in ("plain", "mask_scale_grad_centred",
                                                                                 "w_ramped")]


def _case(size, branch, dev, seed=3):
    H, W = SIZES[size]
    toned, raw, gt, binary, u = _inputs(H, W, seed, dev)
    mk, wk, sg = BRANCHES[branch]
    mask = None if mk is None else (binary if mk == "binary" else torch.round(u * 255) / 255)
    w = _weight(wk, u, binary)
    return toned, raw, gt, mask, (None if sg else w), (w if sg else None)


def _fused(toned, raw, gt, mask, weight, grad_scale, lam=0.2):
    import fused_train as ft
    T, R = toned.clone().requires_grad_(True), raw.clone().requires_grad_(True)
    loss, met = ft.train_loss(T, R, gt, lam, mask=mask, weight=weight, grad_scale=grad_scale)
    loss.backward()
    return loss.detach(), met, T.grad, R.grad


def _bar_check(name, got, ref32, want, inherited=0.0):
    """|got - want| <= 2 |ref32 - want| + one fp32 ulp of the scale (the project's bar) + `inherited`."""
    got, ref32, want = (torch.as_tensor(x, dtype=torch.float64).cpu() for x in (got, ref32, want))
    e = float((got - want).abs().max())
    r = float((ref32 - want).abs().max())
    ulp = float(np.spacing(np.float32(float(want.abs().max()))))
    assert e <= 2 * r + ulp + inherited, f"{name}: error {e:.3e}, reference fp32 error {r:.3e}, ulp {ulp:.3e}, " \
                                         f"inherited {inherited:.3e}"
    return e, r


def _inherited_ssim_error(raw, gt, mask, weight, grad_scale, lam):
    """The loss's SSIM term is computed on the map of the existing fused SSIM op (tests/test_fused_ssim.py holds the
    map to its own bars).  That map's error against float64 enters the loss as lam * mean((1 - S) w): this is it."""
    import fused_ssim
    from oracle import ssim_oracle
    from oracle import train_loss_oracle as tlo
    r = raw
    for s in (mask, grad_scale):
        if s is not None:
            r = tlo.scale_grads(r, s)                                   # the fp32 values the op feeds the SSIM
    w = 1.0 if weight is None else weight[0].double()
    s32 = fused_ssim.ssim(r, gt, size_average=False).double()
    s64 = ssim_oracle.ssim(r, gt, size_average=False)
    return lam * abs(float(((1 - s32) * w).mean() - ((1 - s64) * w).mean()))


@pytest.mark.gpu
@pytest.mark.parametrize("size,branch", CASES)
def test_loss_op_against_float64(size, branch):
    import fused_train as ft
    from oracle import train_loss_oracle as tlo
    dev = torch.device("cuda:0")
    toned, raw, gt, mask, weight, grad_scale = _case(size, branch, dev)
    loss, met, dT, dR = _fused(toned, raw, gt, mask, weight, grad_scale)
    with no_tf32():
        r_loss, r_met, r_dT, r_dR = tlo.loss_and_grads(toned, raw, gt, 0.2, mask, weight, grad_scale, dtype=torch.float32)
    w_loss, w_met, w_dT, w_dR = tlo.loss_and_grads(toned, raw, gt, 0.2, mask, weight, grad_scale)
    _bar_check("loss", loss, r_loss, w_loss, _inherited_ssim_error(raw, gt, mask, weight, grad_scale, 0.2))
    _bar_check("dL/dtoned", dT, r_dT, w_dT)
    _bar_check("dL/draw", dR, r_dR, w_dR)
    values = met.tolist()
    for i, k in enumerate(ft.METRICS):
        if k in w_met:
            _bar_check(k, values[i], r_met[k], w_met[k])
        else:
            assert values[i] == 0.0, k


@pytest.mark.gpu
def test_loss_op_is_bitwise_reproducible_and_launch_count_is_pinned():
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    args = _case("S1", "mask_scale_grad_centred", dev)
    runs = []
    for _ in range(2):
        torch.cuda.synchronize()
        n0 = _C._lib.gsr_launch_count()
        import fused_train as ft
        T, R = args[0].clone().requires_grad_(True), args[1].clone().requires_grad_(True)
        loss, met = ft.train_loss(T, R, args[2], 0.2, mask=args[3], weight=args[4], grad_scale=args[5])
        n1 = _C._lib.gsr_launch_count()
        loss.backward()
        n2 = _C._lib.gsr_launch_count()
        assert (n1 - n0, n2 - n1) == (3, 2)
        runs.append([loss.detach(), met, T.grad, R.grad])
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.gpu
def test_unpack_matches_the_reference_conversion():
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    H, W = 37, 53
    img = np.random.default_rng(1).integers(0, 256, (H, W, 3), dtype=np.uint8)
    img[0, :3, 0] = [0, 255, 128]
    mask = np.random.default_rng(2).integers(0, 256, (H, W), dtype=np.uint8)
    out, mout = torch.empty(3, H, W, device=dev), torch.empty(H, W, device=dev)
    di, dm = torch.from_numpy(img).to(dev), torch.from_numpy(mask).to(dev)
    _C._check(_C._lib.gsr_unpack_u8(H, W, di.data_ptr(), dm.data_ptr(), out.data_ptr(), mout.data_ptr(),
                                    torch.cuda.current_stream().cuda_stream), "gsr_unpack_u8")
    want = np.moveaxis(img.astype(np.float32) / 255.0, -1, 0)                # method.py:50, 1717
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32))
    assert np.array_equal(mout.cpu().numpy().view(np.uint32), (mask.astype(np.float32) / 255.0).view(np.uint32))


# ---- whole step -------------------------------------------------------------------------------------------------------

# Small intervals around iteration 1000 (the SH-degree increase is hard-wired there): densification from 995 every 5,
# an opacity reset at 1008 (then 3 protected iterations), the uncertainty warm-up from 1000 over 6 iterations.
SCHEDULE = dict(iterations=1100, densify_from_iter=995, densify_until_iter=1030, densification_interval=5,
                opacity_reset_interval=1008, uncertainty_protected_iters=3, uncertainty_warmup_start=1000,
                uncertainty_warmup_iters=6)
FIRST, LAST = 990, 1012


def _method(variant, dev):
    import synthetic
    import wg_harness as wh
    import wg_train
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    scene = synthetic.make_scene(20_000, 224, 168, sh_degree=3, seed=4)
    scene = synthetic.to_device(scene, dev)
    kw = dict(SCHEDULE)
    if variant == "uncertainty_masks":
        return m, wg_train.make_method(m, Config, scene, dev, uncertainty=True, masks=True, active_sh_degree=2, **kw)
    if variant == "masks":
        return m, wg_train.make_method(m, Config, scene, dev, masks=True, active_sh_degree=2, **kw)
    if variant == "no_appearance_scale_grad":
        # centring needs a tensor loss_mult (the reference fails before the warm-up start): the warm-up starts earlier
        kw.update(uncertainty_warmup_start=990, uncertainty_warmup_iters=15)
        return m, wg_train.make_method(m, Config, scene, dev, uncertainty=True, appearance=False, active_sh_degree=2,
                                       uncertainty_scale_grad=True, uncertainty_center_mult=True, **kw)
    return m, wg_train.make_method(m, Config, scene, dev, active_sh_degree=2, **kw)


def _run(variant, fused, steps, dev, on_step=None):
    import diff_gaussian_rasterization as ours
    import wg_harness as wh
    import wildgaussians_fused as wf
    m, method = _method(variant, dev)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    wf.enable_method(method, train=fused, ssim=True, msssim=True, dino=True, uncertainty=True)
    assert ("train_iteration" in method.__dict__) == fused
    method.start = {(g["name"], i): p.detach().clone() for g in method.model.optimizer.param_groups
                    for i, p in enumerate(g["params"])}
    random.seed(123)
    torch.manual_seed(7)
    out = []
    try:
        with no_tf32():
            for step in steps:
                metrics = method.train_iteration(step)
                out.append((list(method._viewpoint_stack), metrics, len(method.model.xyz)))
                if on_step is not None:
                    on_step(step, method)
    finally:
        wf.disable_method(method)
    return method, out


VARIANTS = ["plain", "uncertainty_masks", "no_appearance_scale_grad"]


DENSIFICATION_BUFFERS = ("xyz_grad", "denom", "max_radii2D", "xyz_gradient_accum_abs", "xyz_gradient_accum_abs_max")


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_one_step_matches_the_reference_step(variant):
    """One step from identical states: metrics, the densification statistics, Adam moments and parameters."""
    dev = torch.device("cuda:0")
    res = {}
    for fused in (False, True):
        method, out = _run(variant, fused, [FIRST + 10], dev)        # iteration 1001: warm-up ramp, statistics
        model, opt = method.model, method.model.optimizer
        state = {}
        for grp in opt.param_groups:
            for pi, p in enumerate(grp["params"]):
                st = opt.state.get(p, {})
                state[(grp["name"], pi)] = (p.detach().clone(), st.get("exp_avg"), st.get("exp_avg_sq"), float(grp["lr"]))
        bufs = {n: getattr(model, n).detach().clone() for n in DENSIFICATION_BUFFERS if getattr(model, n, None) is not None}
        res[fused] = (out, state, bufs, method.start)
    (o0, s0, b0, start), (o1, s1, b1, _) = res[False], res[True]
    assert o0[0][0] == o1[0][0]                                       # the same camera was drawn
    assert list(o0[0][1]) == list(o1[0][1])                           # same keys, same order
    for k, v in o0[0][1].items():
        w = o1[0][1][k]
        assert isinstance(w, (int, float)) and type(w) is type(v), k
        assert abs(w - v) <= 2e-5 * max(1.0, abs(v)), (k, v, w)
    # densification statistics (wildgaussians_fused.densification_stats against method.py:1997-1998): the radii of
    # both arms come from the same render, so the maxima and the visibility counts agree exactly; the gradient norms
    # carry the last-bit differences of the loss gradient
    assert set(b0) == set(b1)
    for n, a in b0.items():
        b = b1[n]
        assert float(a.abs().max()) > 0, n                            # the step did write them
        if n in ("denom", "max_radii2D"):
            assert torch.equal(a, b), n
        else:
            assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max()), n
    for key, (p0, m0, v0, lr) in s0.items():
        p1, m1, v1, _ = s1[key]
        for name, a, b in (("exp_avg", m0, m1), ("exp_avg_sq", v0, v1)):
            if a is None:
                assert b is None, (key, name)
                continue
            scale = float(a.abs().max()) + 1e-30
            assert float((a - b).abs().max()) <= 2e-3 * scale, (key, name)
        # The first Adam step from zero moments moves each element by lr * g / (|g| + eps), i.e. by about lr: a bar
        # tied to max|p| could not fail for small-lr groups.  So the bar is per element and in units of the group's
        # lr; only elements whose gradient is ~0 (where a last-bit difference can flip its sign) may exceed it.
        d = (p0 - p1).abs()
        allowed = 1e-3 * lr + 4 * torch.finfo(torch.float32).eps * start[key].abs()
        off = d > allowed
        if m0 is not None and bool(off.any()):
            assert float(off.float().mean()) <= 1e-3, (key, int(off.sum()))
            assert float(m0[off].abs().max()) <= 1e-3 * float(m0.abs().max()), key
        else:
            assert not bool(off.any()), key
        moved = (p0 - start[key]).abs().max()
        if m0 is not None and float(m0.abs().max()) > 0:
            assert float(moved) > 0.5 * lr, (key, float(moved), lr)   # the step did move the group


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_short_run_crosses_the_schedule_like_the_reference(variant):
    """23 steps (iterations 991-1013) over the SH increase (1000), the warm-up, three densifications (1000, 1005, 1010),
    an opacity reset (1008) and its protected iterations.  Every metric, the uncertainty ones included, is compared.
    Gaussian counts after each densification may differ slightly: the densification thresholds compare accumulated
    gradient norms, and last-bit differences of the gradients (reordered sums) flip Gaussians that sit at a threshold;
    the bar is 1 % of the count, and the metrics' bar 2 % for the same reason."""
    dev = torch.device("cuda:0")
    steps = list(range(FIRST, LAST + 1))
    _, ref = _run(variant, False, steps, dev)
    method, got = _run(variant, True, steps, dev)
    assert int(method.model.active_sh_degree) == 3
    for step, (r, g) in zip(steps, zip(ref, got)):
        assert r[0] == g[0], step                                     # the same cameras in the same order
        assert list(r[1]) == list(g[1]), step
        for k, v in r[1].items():
            assert np.isfinite(g[1][k]), (step, k)
            assert abs(g[1][k] - v) <= 2e-2 * max(1.0, abs(v)), (step, k, v, g[1][k])
        assert abs(r[2] - g[2]) <= 0.01 * r[2], (step, r[2], g[2])


# Synchronising runtime calls a step can make.  cudaDeviceSynchronize is left out: neither arm calls it, and the
# profiler itself calls it once when it stops.
SYNC_CALLS = ("cudaStreamSynchronize", "cudaEventSynchronize", "cudaMemcpy")


def _syncs_seen_per_count_readback(dev):
    """How many synchronising runtime calls the profiler records for one rasterizer count read-back (the library links
    the CUDA runtime statically; whether its calls are traced depends on the profiler build)."""
    import synthetic
    from torch.profiler import ProfilerActivity, profile
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    d = synthetic.to_device(synthetic.make_scene(2000, 96, 64, sh_degree=None, seed=3), dev)
    settings = GaussianRasterizationSettings(
        image_height=d["image_height"], image_width=d["image_width"], tanfovx=d["tanfovx"], tanfovy=d["tanfovy"],
        kernel_size=d["kernel_size"], subpixel_offset=d["subpixel_offset"], bg=d["bg"], scale_modifier=1.0,
        viewmatrix=d["viewmatrix"], projmatrix=d["projmatrix"], sh_degree=0, campos=d["campos"], prefiltered=False,
        debug=False, return_accumulation=True)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        GaussianRasterizer(settings)(means3D=d["means3D"], means2D=torch.zeros_like(d["means3D"]), opacities=d["opacities"],
                                     colors_precomp=d["colors_precomp"], scales=d["scales"], rotations=d["rotations"])
    return sum(e.name in SYNC_CALLS for e in prof.events())


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["masks", "uncertainty_masks"])
def test_an_ordinary_step_synchronises_once(variant):
    """torch.profiler over one ordinary fused step: one synchronisation besides the rasterizer's instance-count
    read-back (counted by wrapping the library), and, without the uncertainty model, no pageable host-to-device copy
    (with it, a feature-cache hit copies the cached features from pageable memory, as the fused uncertainty loss does).
    The shipped arm's counts are printed beside it."""
    from torch.profiler import ProfilerActivity, profile
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    per_readback = _syncs_seen_per_count_readback(dev)
    results = {}
    for fused in (False, True):
        import diff_gaussian_rasterization as ours
        import wg_harness as wh
        import wildgaussians_fused as wf
        m, method = _method(variant, dev)
        wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
        wf.enable_method(method, train=fused, ssim=True, msssim=True, dino=True, uncertainty=True)
        random.seed(5)
        try:
            for step in range(1040, 1048):                            # warm-up: every image staged, every cache filled
                method.train_iteration(step)
            torch.cuda.synchronize()
            counted = _CountingLib(_C._lib)
            _C._lib = counted
            try:
                with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    method.train_iteration(1050)                     # no densification, reset or SH change
            finally:
                _C._lib = counted.lib
        finally:
            wf.disable_method(method)
        names = [e.name for e in prof.events()]
        syncs = [n for n in names if n in SYNC_CALLS]
        pageable = [n for n in names if "Pageable" in n and "HtoD" in n]
        results[fused] = (len(syncs), counted.readbacks, pageable, syncs)
    n, readbacks, pageable, syncs = results[True]
    print(f"{variant}: shipped arm {results[False][0]} synchronising calls, {results[False][1]} count read-backs, "
          f"{len(results[False][2])} pageable copies; fused arm {n} ({syncs}), {readbacks} count read-backs, "
          f"{len(pageable)} pageable copies; {per_readback} profiler events per read-back")
    assert n == per_readback * readbacks + 1, syncs
    if variant == "masks":
        assert not pageable, pageable


class _CountingLib:
    """Delegates to the library and counts the calls that read the rasterizer's instance counts back."""

    def __init__(self, lib):
        self.lib = lib
        self.readbacks = 0

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if name in ("gsr_forward_geometry", "gsr_forward_status"):
            def counted(*a, **k):
                self.readbacks += 1
                return fn(*a, **k)
            return counted
        return fn
