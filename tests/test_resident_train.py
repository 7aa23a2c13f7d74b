"""Device-resident training data for the fused training iteration: the byte check and pack kernel
(``gsr_pack_u8_exact``) against ``fused_train.as_bytes``, the store's budget, training bit for bit equal to the staged
path, the device feature cache and its undo, and the copies and synchronisations of a resident step."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "wild-gaussians_b200"), ROOT, os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)


# ---------------------------------------------------------------------------------------------------------------- CPU

def kernel_predicate(x):
    """pack_u8_exact_kernel (csrc/train_loss.cu) per element, in numpy: (bytes, exact, binary)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    with np.errstate(invalid="ignore"):
        t = np.fmin(np.fmax(np.rint(x * np.float32(255)), np.float32(0)), np.float32(255))    # fmaxf: NaN -> 0
    u = t.astype(np.uint8)
    exact = (u.astype(np.float32) / np.float32(255)).view(np.uint32) == x.view(np.uint32)
    return u, exact, (x == 0) | (x == 1)


def _ties():
    """fp32 values x with x * 255f exactly k + 0.5: the rounding ties of rint."""
    out = []
    for k in range(255):
        c = np.float32((k + 0.5) / 255)
        for d in range(-4, 5):
            x = c
            for _ in range(abs(d)):
                x = np.nextafter(x, np.float32(np.sign(d)), dtype=np.float32)
            if x * np.float32(255) == np.float32(k + 0.5):
                out.append(x)
    return np.array(out, dtype=np.float32)


def crafted():
    """The k / 255 grid, its +-1-ulp neighbours, the rounding ties and the special values."""
    k = np.arange(256, dtype=np.float32) / np.float32(255)
    up = np.nextafter(k, np.float32(2), dtype=np.float32)
    down = np.nextafter(k, np.float32(-1), dtype=np.float32)
    special = np.array([-0.0, np.nan, np.inf, -np.inf, -1e-8, np.nextafter(np.float32(1), np.float32(2))],
                       dtype=np.float32)
    return np.concatenate([k, up, down, _ties(), special])


def test_the_kernel_predicate_is_that_of_as_bytes():
    import fused_train as ft
    x = crafted()
    ties = _ties()
    assert len(ties) >= 200                                   # the search found ties for most k
    u, exact, _ = kernel_predicate(x)
    for i, v in enumerate(x):
        want = ft.as_bytes(np.array([v], dtype=np.float32))
        assert (want is not None) == bool(exact[i]), (i, float(v))
        if want is not None:
            assert want[0] == u[i], (i, float(v))
    assert exact[:256].all() and not exact[256:768].any()    # the grid passes, its neighbours fail
    assert not exact[-6:].any()                               # -0.0, NaN, +-inf, -1e-8, 1 + 1 ulp
    # a whole image: as_bytes accepts it exactly when every element passes, and then gives the same bytes
    grid = np.arange(256 * 3, dtype=np.float32).reshape(16, 16, 3) % 256 / np.float32(255)
    assert np.array_equal(ft.as_bytes(grid), kernel_predicate(grid)[0])
    grid[3, 4, 1] = np.float32(-0.0)
    assert ft.as_bytes(grid) is None and not kernel_predicate(grid)[1].all()


def test_budget_picks_cameras_first_fit_in_index_order():
    import fused_train as ft
    sizes = [100, 400, 100, 100]
    assert ft.plan(sizes, 0) == [False] * 4
    assert ft.plan(sizes, 700) == [True] * 4                  # exact fit
    assert ft.plan(sizes, 699) == [True, True, True, False]   # one byte short
    assert ft.plan(sizes, 500) == [True, True, False, False]
    assert ft.plan(sizes, 300) == [True, False, True, True]   # the larger camera is skipped, later ones still fit
    assert ft.plan([], 10) == []
    # mixed entries: byte-exact images as uint8 (3 B per pixel), the rest fp32 (12 B), masks 1 or 4 B per pixel
    H, W = 10, 20
    rb = ft.resident_bytes
    assert (rb(H, W, True, False, True), rb(H, W, False, False, True)) == (600, 2400)
    assert (rb(H, W, True, True, True), rb(H, W, True, True, False), rb(H, W, False, True, False)) == (800, 1400, 3200)
    mixed = [rb(H, W, True, True, True), rb(H, W, False, True, True), rb(H, W, True, True, False), rb(H, W, True, True, True)]
    assert ft.plan(mixed, 800 + 2600) == [True, True, False, False]
    assert ft.plan(mixed, 800 + 2600 + 800) == [True, True, False, True]
    assert ft.plan(mixed, sum(mixed)) == [True] * 4
    assert ft.plan(mixed, sum(mixed) - 1) == [True, True, True, False]


def test_pack_entry_point_rejects_bad_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib

    def call(n=1, **kw):
        arr = (_C.GsrPackItem * max(n, 1))()
        for a in arr:
            a.src, a.dst, a.flags = 0x1000, 0x2000, 0x3000
            a.stride_c, a.stride_y, a.stride_x = 1, 30, 3
            a.H, a.W, a.C = 4, 10, 3
            for k, v in kw.items():
                setattr(a, k, v)
        return lib.gsr_pack_u8_exact(arr, n, None)

    assert lib.gsr_pack_u8_exact(None, 1, None) == -1
    for n in (0, -1, _C.PACK_MAX_ITEMS + 1):
        assert call(n) == -1, n
    for kw in (dict(H=0), dict(W=-2), dict(H=70000, W=70000), dict(C=2), dict(C=0), dict(src=None), dict(dst=None),
               dict(flags=None)):
        assert call(**kw) == -1, kw
        assert lib.gsr_last_error().decode()


def test_enable_method_marks_and_disable_method_unmarks():
    import types
    import fused_train as ft
    import fused_uncertainty as fu
    import wildgaussians_fused as wf

    class M:                                                   # hashable and weak-referenceable, as WildGaussians is
        pass

    um = types.SimpleNamespace(_images_cache={("train", 0): torch.zeros(2)})
    model = types.SimpleNamespace(uncertainty_model=um, optimizer=None)
    method = M()
    method.model = model
    wf.enable_method(method, train=True, resident=True, resident_bytes=1234, feature_cache_bytes=99)
    assert method.__dict__[ft.RESIDENT_MARK] == 1234 and um.__dict__[fu.RESIDENT_MARK] == [99]
    wf.disable_method(method)
    assert ft.RESIDENT_MARK not in method.__dict__ and fu.RESIDENT_MARK not in um.__dict__
    wf.enable_method(method, train=True)                       # without the option nothing is marked
    assert ft.RESIDENT_MARK not in method.__dict__ and fu.RESIDENT_MARK not in um.__dict__
    wf.disable_method(method)


# ---------------------------------------------------------------------------------------------------------------- GPU

def _gpu_pack(values, C):
    """Every value of `values` as its own 1x1 item (C channels of it) through gsr_pack_u8_exact: (bytes, flags)."""
    import fused_train as ft
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    x = torch.from_numpy(np.repeat(values[:, None], C, axis=1).copy()).to(dev)        # [n, C]
    dst = torch.empty((len(values), C), dtype=torch.uint8, device=dev)
    flags = torch.zeros((len(values),), dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream(dev)
    for a in range(0, len(values), _C.PACK_MAX_ITEMS):
        ft._pack_items([(x[i], (1, C, C), C, 1, 1, dst[i], flags[i]) for i in range(a, min(a + _C.PACK_MAX_ITEMS, len(values)))],
                       stream)
    return dst.cpu().numpy(), flags.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 3])
def test_pack_kernel_matches_as_bytes_on_crafted_values(C):
    import fused_train as ft
    from diff_gaussian_rasterization import _C
    x = crafted()
    got, flags = _gpu_pack(x, C)
    for i, v in enumerate(x):
        want = ft.as_bytes(np.full((1, 1, C), v, dtype=np.float32))
        assert (want is not None) == (not flags[i] & _C.PACK_NOT_EXACT), (i, float(v), flags[i])
        if want is not None:
            assert np.array_equal(got[i], want.reshape(-1)), (i, float(v))
        binary = bool(np.all((np.float32(v) == 0) | (np.float32(v) == 1)))
        assert binary == (not flags[i] & _C.PACK_NOT_BINARY), (i, float(v))


def _reference_image(H, W, rng, exact=True):
    """A [3,H,W] fp32 view of an HWC array, as method.py:1716-1723 stores training images."""
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8).astype(np.float32) / np.float32(255)
    if not exact:
        img[H // 2, W // 3, 1] = np.float32(0.123456789)
    return torch.from_numpy(np.moveaxis(img, -1, 0))


def _mask(kind, H, W, rng):
    if kind == "none":
        return None
    m = (rng.random((H, W)) > 0.3).astype(np.float32)
    if kind == "fractional":
        m = rng.integers(0, 256, (H, W)).astype(np.float32) / np.float32(255)
    if kind == "one_over":
        m[H // 2, W // 2] = np.nextafter(np.float32(1), np.float32(2))
    return torch.from_numpy(m[None])


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(1, 1), (37, 53), (401, 599), (1080, 1920)])
@pytest.mark.parametrize("mask_kind", ["none", "binary", "fractional", "one_over"])
def test_pack_kernel_matches_as_bytes_on_images(H, W, mask_kind):
    import fused_train as ft
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(H * 7 + W)
    for exact in (True, False):
        img = _reference_image(H, W, rng, exact)
        d = img.to(dev)
        assert d.stride() == img.stride()                                    # the HWC memory order travels
        u8, ok, _ = ft.pack_u8_exact(d)
        want = ft.as_bytes(img.permute(1, 2, 0).numpy())
        assert ok == (want is not None)
        if want is not None:
            assert np.array_equal(u8.cpu().numpy(), want)
        u8c, okc, _ = ft.pack_u8_exact(d.contiguous())                       # the same from a CHW tensor
        assert okc == ok and torch.equal(u8c, u8)
    m = _mask(mask_kind, H, W, rng)
    if m is not None:
        u8, ok, binary = ft.pack_u8_exact(m.to(dev))
        mv = m.reshape(H, W).numpy()
        want = ft.as_bytes(mv)
        assert ok == (want is not None)
        if want is not None:
            assert np.array_equal(u8.cpu().numpy(), want)
        assert binary == bool(np.all((mv == 0) | (mv == 1)))


# ---- training: staged against resident, each pair in a fresh process under torch.use_deterministic_algorithms ----

_SCRIPT = r"""
import hashlib, json, os, random, sys
ROOT = sys.argv[1]
for p in (ROOT, os.path.join(ROOT, "wild-gaussians_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np
import torch
torch.use_deterministic_algorithms(True)
import test_resident_train as trt
print("RESULT " + json.dumps(trt._pair(*sys.argv[2:])))
"""


def _digest(t):
    import hashlib
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def _method(variant, dev, size=None):
    import synthetic
    import test_fused_train as tft
    import wg_harness as wh
    import wg_train
    import diff_gaussian_rasterization as ours
    if size is None:
        m, method = tft._method(variant, dev)
    else:
        m, Config = wh.import_method()
        if m is None:
            pytest.skip("reference python package not present (oracle/_ref/py)")
        scene = synthetic.to_device(synthetic.make_scene(20_000, size[1], size[0], sh_degree=3, seed=4), dev)
        method = wg_train.make_method(m, Config, scene, dev, uncertainty=True, masks=True, active_sh_degree=2,
                                      **tft.SCHEDULE)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    return method


def _sizes(method):
    """The resident bytes of each camera, from the host check."""
    import fused_train as ft
    out = []
    for i, img in enumerate(method.train_images):
        H, W = int(img.shape[1]), int(img.shape[2])
        m = None if method.train_masks is None else method.train_masks[i].reshape(H, W).numpy()
        out.append(ft.resident_bytes(H, W, ft.as_bytes(img.permute(1, 2, 0).numpy()) is not None, m is not None,
                                     m is not None and ft.as_bytes(m) is not None))
    return out


FLAGS = dict(train=True, ssim=True, msssim=True, dino=True, uncertainty=True)
STEPS = list(range(991, 1011))     # 20 steps: the SH increase (1000), densifications (1000, 1005, 1010), a reset (1008)


def _state(method, out):
    model, opt = method.model, method.model.optimizer
    for grp in opt.param_groups:
        for pi, p in enumerate(grp["params"]):
            out[f"{grp['name']}.{pi}"] = _digest(p)
            for k, v in opt.state.get(p, {}).items():
                out[f"{grp['name']}.{pi}.{k}"] = _digest(v) if isinstance(v, torch.Tensor) else repr(v)
    for n, b in model.named_buffers() if hasattr(model, "named_buffers") else ():
        out["buf." + n] = _digest(b)
    import test_fused_train as tft
    for n in tft.DENSIFICATION_BUFFERS:
        if getattr(model, n, None) is not None:
            out["dens." + n] = _digest(getattr(model, n))
    um = getattr(model, "uncertainty_model", None)
    if um is not None:
        for n, b in um.named_buffers():
            out["unc." + n] = _digest(b)
        for n, p in um.named_parameters():
            out["uncp." + n] = _digest(p)


def _train_arm(variant, resident, budget):
    import random
    import fused_train as ft
    import test_fused_train as tft
    import wildgaussians_fused as wf
    dev = torch.device("cuda:0")
    method = _method(variant, dev)
    kw = dict(FLAGS)
    info = {}
    if resident:
        sizes = _sizes(method)
        nbytes = {"none": None, "zero": 0, "half": sum(sizes[: len(sizes) // 2])}[budget]
        info["expect"] = [i for i, t in enumerate(ft.plan(sizes, nbytes)) if t] if nbytes is not None else \
            list(range(len(sizes)))
        kw.update(resident=True, resident_bytes=nbytes)
    wf.enable_method(method, **kw)
    random.seed(123)
    torch.manual_seed(7)
    out = {}
    try:
        with tft.no_tf32():
            for i, step in enumerate(STEPS):
                metrics = method.train_iteration(step)
                out[f"step{i}"] = repr((list(method._viewpoint_stack), sorted(metrics.items()), len(method.model.xyz)))
        if resident:
            store = ft._stores[method]
            info["resident"] = sorted(store.entries)
            info["staged"] = store.staged
            info["stager"] = sorted(ft._stagers[method].entries) if method in ft._stagers else []
            del store
        _state(method, out)
    finally:
        wf.disable_method(method)
    um = method.model.uncertainty_model
    if um is not None:
        for k, v in um._images_cache.items():
            out[f"cache.{k}"] = (_digest(v), v.is_cuda)
    return out, info


def _cache_arm(resident, budget_entries):
    """One warm step on the staged path, an emptied feature cache, then one epoch (four ordinary steps) on the arm; the
    class's ``_compute_losses`` and ``fused_uncertainty_modes`` against the cache; memory before and after."""
    import random
    import fused_train as ft
    import fused_uncertainty_modes as fum
    import test_fused_train as tft
    import wildgaussians_fused as wf
    dev = torch.device("cuda:0")
    method = _method("uncertainty_masks", dev, size=(480, 640))
    um = method.model.uncertainty_model
    random.seed(5)
    torch.manual_seed(3)
    out, info = {}, {}
    with tft.no_tf32():
        wf.enable_method(method, **FLAGS)
        method.train_iteration(1039)
        wf.disable_method(method)
        um._images_cache.clear()
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated(dev)
        kw = dict(FLAGS)
        if resident:
            kw.update(resident=True, feature_cache_bytes=budget_entries)
        wf.enable_method(method, **kw)
        for i, step in enumerate(range(1040, 1044)):
            metrics = method.train_iteration(step)
            out[f"step{i}"] = repr(sorted(metrics.items()))
        torch.cuda.synchronize()
        info["during"] = torch.cuda.memory_allocated(dev) - before
        info["cache"] = [(int(v.nbytes), bool(v.is_cuda)) for v in um._images_cache.values()]
        if resident:
            store = ft._stores[method]
            info["store_bytes"] = sum(e.img.nbytes + (0 if e.mask is None else e.mask.nbytes) for e in store.entries.values())
            del store                                            # disable_method frees what the store alone holds
        # the class's own method and the modes path, through the same cache keys
        for cid in range(len(method.train_images)):
            gt = method.train_images[cid].to(dev).contiguous()[None]
            pred = (gt * 0.9 + 0.05).contiguous()
            loss, met, mult = fum.compute_losses(um, gt, pred, _cache_entry=("train", cid))
            out[f"modes{cid}"] = (_digest(loss), sorted(met.items()), _digest(mult))
            loss, met, mult = type(um)._compute_losses(um, gt, pred, _cache_entry=("train", cid))
            out[f"class{cid}"] = (_digest(loss), sorted((k, float(v)) for k, v in met.items()), _digest(mult))
        del gt, pred, loss, met, mult
        wf.disable_method(method)
    torch.cuda.synchronize()
    info["after"] = torch.cuda.memory_allocated(dev) - before
    for k, v in um._images_cache.items():
        out[f"cache.{k}"] = (_digest(v), v.is_cuda)
    _state(method, out)
    return out, info


def _pair(what, variant, budget):
    if what == "train":
        staged, _ = _train_arm(variant, False, budget)
        resident, info = _train_arm(variant, True, budget)
    else:
        staged, sinfo = _cache_arm(False, None)
        sizes = [n for n, _ in sinfo["cache"]]
        budget_entries = sum(sizes[: len(sizes) // 2])
        resident, info = _cache_arm(True, budget_entries)
        import fused_train as ft
        info["expect_device"] = ft.plan(sizes, budget_entries)
    return {"staged": staged, "resident": resident, "info": info}


def _run_pair(*args):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-c", _SCRIPT, ROOT, *args], capture_output=True, text=True, env=env,
                       timeout=1800)
    if "reference python package not present" in r.stdout + r.stderr:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    line = [x for x in r.stdout.splitlines() if x.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


def _assert_same(a, b):
    assert a.keys() == b.keys(), sorted(set(a) ^ set(b))
    diff = [k for k in a if a[k] != b[k]]
    assert not diff, diff[:10]


@pytest.mark.gpu
@pytest.mark.parametrize("variant,budget", [("uncertainty_masks", "none"), ("plain", "none"),
                                            ("no_appearance_scale_grad", "none"), ("uncertainty_masks", "zero"),
                                            ("uncertainty_masks", "half")])
def test_resident_training_is_bitwise_the_staged_training(variant, budget):
    """20 steps from identical seeds, staged against resident: every metric, parameter, Adam moment, model and
    uncertainty buffer, and (after ``disable_method``) every feature-cache entry, bit for bit.  Image 1 is not
    byte-exact and mask 2 is fractional (tests/wg_train.py); the uncertainty runs miss the feature cache in the first
    epoch and hit it afterwards."""
    res = _run_pair("train", variant, budget)
    info = res["info"]
    assert info["resident"] == info["expect"], info
    assert info["staged"] == [i for i in range(4) if i not in info["expect"]]
    assert info["stager"] == info["staged"]            # the host check ran on the staged cameras only
    if budget == "half":
        assert info["resident"] == [0, 1]
    _assert_same(res["staged"], res["resident"])
    assert all(not v[1] for k, v in res["resident"].items() if k.startswith("cache."))


@pytest.mark.gpu
def test_device_feature_cache_and_its_undo():
    """After one epoch the entries within the budget are device tensors and the rest host tensors; the class's
    ``_compute_losses`` and ``fused_uncertainty_modes`` return what they return on the staged arm; after
    ``disable_method`` every entry is a host tensor equal to the staged arm's and the device memory is back."""
    res = _run_pair("cache", "uncertainty_masks", "none")
    info = res["info"]
    assert [d for _, d in info["cache"]] == info["expect_device"], info
    assert any(info["expect_device"]) and not all(info["expect_device"])
    held = info["store_bytes"] + sum(n for n, d in info["cache"] if d)
    assert held > 4 << 20 and info["during"] >= held, info
    assert abs(info["after"]) <= 1 << 20, info
    _assert_same(res["staged"], res["resident"])
    assert all(not v[1] for k, v in res["resident"].items() if k.startswith("cache."))


@pytest.mark.gpu
def test_a_resident_step_copies_nothing_to_the_device_and_synchronises_twice():
    """torch.profiler over three ordinary steps after two warm epochs, everything resident: no host-to-device copy, and
    per step the rasterizer's count read-back and the metric read-back only."""
    import random
    import test_fused_train as tft
    import wildgaussians_fused as wf
    from torch.profiler import ProfilerActivity, profile
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    per_readback = tft._syncs_seen_per_count_readback(dev)
    method = _method("uncertainty_masks", dev)
    wf.enable_method(method, resident=True, **FLAGS)
    random.seed(5)
    try:
        for step in range(1040, 1048):
            method.train_iteration(step)
        torch.cuda.synchronize()
        counted = tft._CountingLib(_C._lib)
        _C._lib = counted
        try:
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for step in (1050, 1051, 1052):
                    method.train_iteration(step)
        finally:
            _C._lib = counted.lib
    finally:
        wf.disable_method(method)
    names = [e.name for e in prof.events()]
    h2d = [n for n in names if "HtoD" in n]
    syncs = [n for n in names if n in tft.SYNC_CALLS]
    print(f"resident: {len(syncs)} synchronising calls over 3 steps ({syncs}), {counted.readbacks} count read-backs, "
          f"{per_readback} profiler events per read-back, host-to-device copies {h2d}")
    assert not h2d, h2d
    assert counted.readbacks == 3
    assert len(syncs) == 3 * (per_readback + 1), syncs
