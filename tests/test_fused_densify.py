"""Fused densification (``fused_densify``, ``csrc/densify.cu``): ``densify_and_prune`` and ``reset_opacity`` against the
reference's own methods from identical states, the GPU quantile against ``torch.quantile``, a model above torch's
2^24-element quantile limit, training runs with ``enable_method(..., densify=True)`` and the host synchronisations."""
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

def test_c_entry_points_reject_bad_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib
    assert lib.gsr_densify_scratch_bytes(-1) == 0 and lib.gsr_densify_scratch_bytes(_C.DENSIFY_MAX_P + 1) == 0
    assert lib.gsr_densify_scratch_bytes(1000) >= 4 * 8 * 1000

    def args(**kw):
        a = _C.GsrDensifyArgs()
        a.P = 10
        for n in ("xyz_grad", "denom", "xyz", "scales", "rotations", "opacities", "scratch", "counts"):
            setattr(a, n, 0x1000)
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    for name in ("xyz_grad", "denom", "xyz", "scales", "rotations", "opacities", "scratch", "counts"):
        assert lib.gsr_densify_plan(ctypes.byref(args(**{name: None})), None) == -1, name
        assert "NULL" in lib.gsr_last_error().decode()
    for P in (0, -1, _C.DENSIFY_MAX_P + 1):
        assert lib.gsr_densify_plan(ctypes.byref(args(P=P)), None) == -1, P
    assert lib.gsr_densify_plan(ctypes.byref(args(scratch=0x1004)), None) == -1
    assert lib.gsr_densify_plan(None, None) == -1
    seg = _C.GsrDensifySegment(0x1000, 0x2000, 3, _C.DENSIFY_XYZ)
    for bad in (dict(width=0), dict(width=4), dict(kind=7), dict(src=None), dict(dst=None)):
        s = _C.GsrDensifySegment(0x1000, 0x2000, 3, _C.DENSIFY_XYZ)
        for k, v in bad.items():
            setattr(s, k, v)
        assert lib.gsr_densify_apply(ctypes.byref(args()), ctypes.byref(s), 1, None) == -1, bad
    assert lib.gsr_densify_apply(ctypes.byref(args()), ctypes.byref(seg), _C.DENSIFY_MAX_SEGMENTS + 1, None) == -1
    assert lib.gsr_reset_opacity(-1, None, None, None, None, None) == -1
    assert lib.gsr_reset_opacity(0, None, None, None, None, None) == 0
    assert lib.gsr_reset_opacity(5, 0x1000, None, 0x1000, 0x1000, None) == -1


def test_enable_binds_and_disable_restores():
    import wildgaussians_fused as wf

    class Model(torch.nn.Module):
        def densify_and_prune(self, *a, **k):
            return "class"

        def reset_opacity(self):
            return "class"

    model = Model()
    wf.enable(model, optimizer=False)
    assert "densify_and_prune" not in model.__dict__ and "reset_opacity" not in model.__dict__   # opt-in
    wf.enable(model, optimizer=False, densify=True)
    assert model.densify_and_prune.__func__ is wf.densify_and_prune and model.reset_opacity.__func__ is wf.reset_opacity
    wf.disable(model)
    assert model.densify_and_prune() == "class" and model.reset_opacity() == "class"


def test_unsupported_models_are_refused_on_the_cpu():
    import fused_densify as fd
    cfg = types.SimpleNamespace(debug=False, use_gof_abs_gradient=False, percent_dense=0.01)
    xyz = torch.nn.Parameter(torch.zeros(4, 3))
    model = types.SimpleNamespace(config=cfg, xyz=xyz, _dynamically_sized_props=["xyz"],
                                  optimizer=torch.optim.Adam([{"params": [xyz], "name": "xyz"}]))
    assert not fd.supported(model)                                   # CPU tensors
    model.optimizer = torch.optim.SGD([{"params": [xyz], "name": "xyz"}], lr=1.0)
    assert not fd.supported(model)                                   # not Adam


# ---------------------------------------------------------------------------------------------------------------- GPU

def _reference():
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    return m, Config


def _make(appearance, use_abs, dev, *, P=3000, seed=0, **overrides):
    """A WildGaussians (optimizer set up) on a small synthetic scene, with a few very large and a few transparent
    Gaussians so that the size and opacity prunes both fire."""
    import synthetic
    import wg_harness as wh  # noqa: F401
    import wg_train
    m, Config = _reference()
    scene = synthetic.to_device(synthetic.make_scene(P, 96, 64, sh_degree=3, seed=seed), dev)
    method = wg_train.make_method(m, Config, scene, dev, appearance=appearance, use_gof_abs_gradient=use_abs, seed=seed,
                                  **overrides)
    model = method.model
    g = torch.Generator(device=dev).manual_seed(seed + 1)
    with torch.no_grad():
        big = torch.rand(P, generator=g, device=dev) < 0.02
        model.scales[big] = float(np.log(0.3))
        faint = torch.rand(P, generator=g, device=dev) < 0.03
        model.opacities[faint] = float(torch.special.logit(torch.tensor(0.002)))
        model.filter_3D.copy_(torch.rand(P, 1, generator=g, device=dev) * 0.004)
    return m, method


def _set_stats(model, kind, max_grad, dev, seed=3):
    """Densification statistics that select a few % of the Gaussians (kind "normal"), drive Q to 0 ("q_zero": almost
    every denom 0), or select nothing ("none")."""
    P = int(model.xyz.shape[0])
    g = torch.Generator(device=dev).manual_seed(seed)
    denom = torch.randint(0, 6, (P, 1), generator=g, device=dev).float()
    if kind == "q_zero":
        denom = torch.where(torch.rand(P, 1, generator=g, device=dev) < 0.97, 0.0, denom + 1)
    lg = lambda s: torch.exp(torch.randn(P, 1, generator=g, device=dev) * s) * max_grad
    grad = lg(0.8) * 0.45
    if kind == "q_zero":
        grad = torch.where(denom > 0, max_grad * 3, 0.0)
    if kind == "none":
        grad = grad * 0
    with torch.no_grad():
        model.denom.copy_(denom)
        model.xyz_grad.copy_(grad * denom)
        model.xyz_grad[:7] = torch.where(denom[:7] == 0, 1e-3, model.xyz_grad[:7])      # x / 0 = inf
        if model.xyz_gradient_accum_abs is not None:
            model.xyz_gradient_accum_abs.copy_(lg(1.0) * 0.3 * denom)
            model.xyz_gradient_accum_abs[::97] = torch.round(model.xyz_gradient_accum_abs[::97] * 1e4) / 1e4   # ties
            model.xyz_gradient_accum_abs_max.copy_(model.xyz_gradient_accum_abs * 0.5)
        model.max_radii2D.copy_(torch.randint(0, 30, (P,), generator=g, device=dev).float())


def _set_moments(model, dev, which):
    """Adam state for some dynamically sized groups (`which`: "all", "some", "none"); `step` 3."""
    opt = model.optimizer
    g = torch.Generator(device=dev).manual_seed(11)
    for i, grp in enumerate(opt.param_groups):
        if grp["name"] not in model._dynamically_sized_props:
            continue
        if which == "none" or (which == "some" and i % 2):
            continue
        p = grp["params"][0]
        opt.state[p] = {"step": torch.tensor(3.0), "exp_avg": torch.randn(p.shape, generator=g, device=dev),
                        "exp_avg_sq": torch.rand(p.shape, generator=g, device=dev)}


def _snapshot(model):
    opt = model.optimizer
    out = {}
    for name in model._dynamically_sized_props:
        t = getattr(model, name, None)
        out[name] = None if t is None else t.detach().clone()
    for grp in opt.param_groups:
        if grp["name"] not in model._dynamically_sized_props:
            continue
        p = grp["params"][0]
        assert p is getattr(model, grp["name"]), grp["name"]
        assert p.grad is None and p.requires_grad and isinstance(p, torch.nn.Parameter), grp["name"]
        st = opt.state.get(p, None)
        out["state:" + grp["name"]] = None if st is None else (float(st["step"]), st["exp_avg"].clone(), st["exp_avg_sq"].clone())
    return out


def _assert_same_state(ref, got, n_children):
    assert set(ref) == set(got)
    for k, a in ref.items():
        b = got[k]
        if a is None:
            assert b is None, k
            continue
        if k.startswith("state:"):
            assert b is not None and a[0] == b[0], k                                    # step kept
            for x, y in zip(a[1:], b[1:]):
                assert torch.equal(x.view(torch.int32), y.view(torch.int32)), k
            continue
        assert a.shape == b.shape, (k, a.shape, b.shape)
        if k == "xyz" and n_children:
            # the split children's positions: the reference multiplies with a cuBLAS bmm, the kernel in fp32 FMAs
            head = a.shape[0] - n_children
            assert torch.equal(a[:head].view(torch.int32), b[:head].view(torch.int32)), k
            bar = 4 * torch.finfo(torch.float32).eps * float(a[head:].abs().max())
            assert float((a[head:] - b[head:]).abs().max()) <= bar, k
        else:
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (k, int((a != b).sum()))


def _run_pair(appearance, use_abs, kind, size_pruning, moments, optimizer, dev, capsys):
    import fused_densify as fd
    import fused_adam
    max_grad, min_opacity, extent = 0.0002, 0.005, 1.5
    res = {}
    for fused in (False, True):
        m, method = _make(appearance, use_abs, dev)
        model = method.model
        _set_stats(model, kind, max_grad, dev)
        _set_moments(model, dev, moments)
        if optimizer == "fused_adam":
            fused_adam.adopt(model.optimizer)
        capsys.readouterr()
        torch.manual_seed(1234)
        if fused:
            assert fd.supported(model)
            n_children = 2 * fd.plan(model, max_grad, min_opacity, extent, size_pruning)[0]["kept_splits"]
            out = fd.densify_and_prune(model, max_grad, min_opacity, extent, size_pruning)
        else:
            out = type(model).densify_and_prune(model, max_grad, min_opacity, extent, size_pruning)
        torch.cuda.synchronize()
        printed = capsys.readouterr().out
        res[fused] = (out, printed, torch.cuda.get_rng_state(), _snapshot(model))
    (o0, p0, r0, s0), (o1, p1, r1, s1) = res[False], res[True]
    assert o1 == o0 and all(type(x) is int for x in o1), (o0, o1)
    assert p1 == p0, (p0, p1)
    assert torch.equal(r0, r1)                                                          # the generator ended alike
    _assert_same_state(s0, s1, n_children)                             # the split copies are the last rows
    return o0


PARITY = [
    # appearance, use_gof_abs_gradient, statistics, enable_size_pruning, moments, optimizer
    (True, True, "normal", True, "all", "adam"),
    (True, True, "normal", False, "some", "fused_adam"),
    (False, True, "normal", True, "none", "adam"),
    (False, False, "normal", True, "some", "adam"),
    (True, False, "normal", False, "all", "fused_adam"),
    (True, True, "q_zero", True, "all", "adam"),
    (False, False, "none", False, "all", "adam"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("appearance,use_abs,kind,size_pruning,moments,optimizer", PARITY)
def test_densify_and_prune_matches_the_reference(appearance, use_abs, kind, size_pruning, moments, optimizer, capsys):
    dev = torch.device("cuda:0")
    out = _run_pair(appearance, use_abs, kind, size_pruning, moments, optimizer, dev, capsys)
    if kind == "none":
        assert out[:2] == (0, 0), out
    else:
        assert out[0] > 0 and out[1] > 0 and out[2] > 0, out
    if kind == "q_zero":
        assert out[0] + out[1] > 1000, out                             # Q = 0: every zero-gradient Gaussian qualifies


# ---- quantile -----------------------------------------------------------------------------------------------------------

def _plan_q(ga, n_ge, dev, max_grad=1.0):
    """Q of the plan for accum_abs = ga (denom 1) with `n_ge` rows at |grad| >= max_grad; and torch's value."""
    import fused_densify as fd
    P = int(ga.numel())
    grad = torch.zeros(P, 1, device=dev)
    grad[:n_ge] = 2 * max_grad
    cfg = types.SimpleNamespace(use_gof_abs_gradient=True, percent_dense=0.01)
    model = types.SimpleNamespace(
        config=cfg, xyz=torch.zeros(P, 3, device=dev), scales=torch.zeros(P, 3, device=dev),
        rotations=torch.zeros(P, 4, device=dev), opacities=torch.zeros(P, 1, device=dev), xyz_grad=grad,
        denom=torch.ones(P, 1, device=dev), xyz_gradient_accum_abs=ga.reshape(P, 1).contiguous())
    counts, _, _ = fd.plan(model, max_grad, 0.005, 1.0, False)
    ratio = (torch.norm(grad, dim=-1) >= max_grad).float().mean()
    assert counts["n_ge"] == n_ge
    return counts["Q"], ratio


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3, 1000, (1 << 20) + 7, 1 << 24])
def test_quantile_equals_torch_bitwise(P):
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(P % 1000)
    inputs = {
        "spread": torch.rand(P, generator=g, device=dev) * torch.exp(torch.randn(P, generator=g, device=dev) * 3),
        "ties": torch.round(torch.rand(P, generator=g, device=dev) * 7) / 7,
        "all_equal": torch.full((P,), 0.37, device=dev),
        "zeros": torch.where(torch.rand(P, generator=g, device=dev) < 0.6, 0.0, torch.rand(P, generator=g, device=dev)),
    }
    ks = sorted({0, P, P // 3, (P * 2) // 7, max(P - 1, 0), min(1, P)})      # q = 1 - k / P: 1, 0 and in between
    for name, ga in inputs.items():
        for k in ks:
            q, ratio = _plan_q(ga, k, dev)
            want = torch.quantile(ga, 1 - ratio)
            assert np.float32(q).view(np.int32) == want.cpu().numpy().astype(np.float32).view(np.int32), (name, k, q, float(want))


@pytest.mark.gpu
def test_torch_quantile_refuses_above_2_pow_24():
    dev = torch.device("cuda:0")
    with pytest.raises(RuntimeError, match="too large"):
        torch.quantile(torch.zeros((1 << 24) + 1, device=dev), 0.5)


# ---- beyond 2^24 --------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_densify_beyond_torch_quantile_limit():
    """A lean model (appearance off, SH degree 0 storage) of 2^24 + 2^20 Gaussians densifies to completion; Q equals a
    torch.sort plus torch.quantile's fp32 rank formula, and the output rows are the reference's statements' selection."""
    import fused_densify as fd
    dev = torch.device("cuda:0")
    if torch.cuda.mem_get_info(dev)[0] < 30 * 2**30:
        pytest.skip("needs about 30 GB of free device memory (the device is shared)")
    m, Config = _reference()
    P = (1 << 24) + (1 << 20)
    cfg = Config(source_path="", model_path="", uncertainty_mode="disabled", appearance_enabled=False, sh_degree=0)
    model = m.GaussianModel(cfg, training_setup=False).to(dev)
    model._resize_parameters(P)
    g = torch.Generator(device=dev).manual_seed(5)
    max_grad, min_opacity, extent = 0.0002, 0.005, 1.5
    with torch.no_grad():
        model.xyz.copy_(torch.randn(P, 3, generator=g, device=dev))
        model.features_dc.copy_(torch.rand(P, 3, generator=g, device=dev))
        model.scales.copy_(torch.log(0.015 * torch.exp(0.3 * torch.randn(P, 3, generator=g, device=dev))))
        model.rotations.copy_(torch.randn(P, 4, generator=g, device=dev))
        model.opacities.copy_(torch.randn(P, 1, generator=g, device=dev) * 3)
        denom = torch.randint(0, 5, (P, 1), generator=g, device=dev).float()
        model.denom.copy_(denom)
        model.xyz_grad.copy_(torch.exp(torch.randn(P, 1, generator=g, device=dev) * 0.8) * max_grad * 0.45 * denom)
        model.xyz_gradient_accum_abs.copy_(torch.exp(torch.randn(P, 1, generator=g, device=dev)) * max_grad * 0.3 * denom)
    model.spatial_lr_scale.fill_(1.0)
    model._setup_optimizers()
    assert fd.supported(model)

    # the reference's statements, element by element, and the quantile by sort + torch.quantile's fp32 rank formula
    with torch.no_grad():
        grads = model.xyz_grad / model.denom
        grads[grads.isnan()] = 0.0
        ga = model.xyz_gradient_accum_abs / model.denom
        ga[ga.isnan()] = 0.0
        n_ge = int((torch.norm(grads, dim=-1) >= max_grad).sum())
        ratio = np.float32(n_ge) * (np.float32(1) / np.float32(P))
        rank = np.float32(np.float32(1) - ratio) * np.float32(P - 1)
        below = min(int(rank), P - 1)
        above = min(int(np.ceil(rank)), P - 1)
        w = np.float32(rank - np.float32(below))
        srt = torch.sort(ga.reshape(-1)).values
        Q = torch.lerp(srt[below:below + 1], srt[above:above + 1], torch.tensor([w], device=dev))
        del srt
        sel = (torch.norm(grads, dim=-1) >= max_grad) | (torch.norm(ga, dim=-1) >= Q)
        smax = torch.exp(model.scales).max(dim=1).values
        clone = sel & (smax <= 0.01 * extent)
        split = ((grads.squeeze() >= max_grad) | (ga.squeeze() >= Q)) & (smax > 0.01 * extent)
        faint = (torch.sigmoid(model.opacities) < min_opacity).squeeze()
        child_big = torch.exp(torch.log(torch.exp(model.scales) / 1.6)).max(dim=1).values > 0.1 * extent
        keep = ~faint & ~(smax > 0.1 * extent)
        keep_child = ~faint & ~child_big
        op = model.opacities.detach()
        want_op = torch.cat([op[~split & keep], op[clone & keep], op[split & keep_child], op[split & keep_child]])
        want = (int(clone.sum()), int(split.sum()))
        del grads, ga, sel, smax, child_big, faint
    counts, _, _ = fd.plan(model, max_grad, min_opacity, extent, True)
    assert np.float32(counts["Q"]).view(np.int32) == Q.cpu().numpy().view(np.int32)[0]
    out = fd.densify_and_prune(model, max_grad, min_opacity, extent, True)
    assert out[:2] == want, (out, want)
    assert torch.equal(model.opacities.detach().view(torch.int32), want_op.view(torch.int32))
    assert int(model.xyz.shape[0]) == int(want_op.shape[0]) and int(model.denom.shape[0]) == int(want_op.shape[0])


# ---- reset_opacity ------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("appearance", [True, False])
def test_reset_opacity_matches_the_reference(appearance):
    """Within 1 ulp of the reference: the kernel evaluates exp / sqrt / log with the same IEEE operations and libdevice
    functions torch's kernels call, in the same order, but is built by a different CUDA toolkit than the torch
    binary, whose libdevice may round a transcendental differently in the last place."""
    import fused_densify as fd
    dev = torch.device("cuda:0")
    res = []
    for fused in (False, True):
        _, method = _make(appearance, True, dev)
        model = method.model
        _set_moments(model, dev, "all")
        old = model.opacities
        (fd.reset_opacity if fused else type(model).reset_opacity)(model)
        st = model.optimizer.state[model.opacities]
        assert model.opacities is not old and old not in model.optimizer.state
        assert float(st["step"]) == 3.0 and not st["exp_avg"].any() and not st["exp_avg_sq"].any()
        res.append(model.opacities.detach().clone())
    a, b = (x.view(torch.int32).long() for x in res)
    assert int((a - b).abs().max()) <= 1, int((a - b).abs().max())


# ---- through training ---------------------------------------------------------------------------------------------------

# the short schedule of tests/test_fused_train.py: densification from 995 every 5 iterations, an opacity reset at 1008
SCHEDULE = dict(iterations=1100, densify_from_iter=995, densify_until_iter=1030, densification_interval=5,
                opacity_reset_interval=1008, uncertainty_protected_iters=3, uncertainty_warmup_start=1000,
                uncertainty_warmup_iters=6)
FIRST, LAST = 990, 1012


class no_tf32:
    def __enter__(self):
        self.was = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.was


def _train(dev, steps, **enable_kw):
    import synthetic
    import diff_gaussian_rasterization as ours
    import wg_harness as wh
    import wg_train
    import wildgaussians_fused as wf
    m, Config = _reference()
    scene = synthetic.to_device(synthetic.make_scene(20_000, 224, 168, sh_degree=3, seed=4), dev)
    method = wg_train.make_method(m, Config, scene, dev, active_sh_degree=2, **SCHEDULE)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    wf.enable_method(method, ssim=True, **enable_kw)
    random.seed(123)
    torch.manual_seed(7)
    out = []
    try:
        with no_tf32():
            for step in steps:
                metrics = method.train_iteration(step)
                out.append((metrics, len(method.model.xyz)))
    finally:
        wf.disable_method(method)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("train", [True, False])
def test_short_run_with_fused_densification(train):
    """23 steps over three densifications and an opacity reset: Gaussian counts within 1 % and metrics within 2 % of
    the reference run (test_fused_train.py's bars: last-bit gradient differences of the fused render and loss flip
    Gaussians that sit at a threshold)."""
    dev = torch.device("cuda:0")
    steps = list(range(FIRST, LAST + 1))
    ref = _train(dev, steps, train=train)
    got = _train(dev, steps, train=train, densify=True)
    assert ref[-1][1] != ref[0][1]                                    # the run did densify
    for step, (r, g) in zip(steps, zip(ref, got)):
        for k, v in r[0].items():
            assert np.isfinite(g[0][k]), (step, k)
            assert abs(g[0][k] - v) <= 2e-2 * max(1.0, abs(v)), (step, k, v, g[0][k])
        assert abs(r[1] - g[1]) <= 0.01 * r[1], (step, r[1], g[1])


@pytest.mark.gpu
def test_one_densifying_step_gives_exactly_the_reference_counts():
    """From identical states through the same render path, a densifying step's Gaussian count is exactly equal."""
    dev = torch.device("cuda:0")
    steps = list(range(FIRST, 1001))                                   # densifies at 1000 (and 995 is the start)
    ref = _train(dev, steps)
    got = _train(dev, steps, densify=True)
    assert [r[1] for r in ref] == [g[1] for g in got]
    assert ref[-1][1] != ref[0][1]


# ---- synchronisations ---------------------------------------------------------------------------------------------------

SYNC_CALLS = ("cudaStreamSynchronize", "cudaEventSynchronize", "cudaMemcpy")


@pytest.mark.gpu
def test_one_fused_densification_synchronises_once():
    import fused_densify as fd
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda:0")
    counts = {}
    for fused in (False, True):
        _, method = _make(True, True, dev)
        model = method.model
        _set_stats(model, "normal", 0.0002, dev)
        _set_moments(model, dev, "all")
        fd.plan(model, 0.0002, 0.005, 1.5, False)                        # warm-up: pinned buffer, modules loaded
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            if fused:
                fd.densify_and_prune(model, 0.0002, 0.005, 1.5, True)
            else:
                type(model).densify_and_prune(model, 0.0002, 0.005, 1.5, True)
        counts[fused] = [e.name for e in prof.events() if e.name in SYNC_CALLS]
    print(f"synchronising calls per densify_and_prune: reference {len(counts[False])}, fused {len(counts[True])}")
    assert len(counts[True]) == 1, counts[True]


@pytest.mark.gpu
def test_unsupported_model_runs_the_reference(capsys):
    """A model refused by `supported` (config.debug) runs the class's own method: the same result, bit for bit."""
    import fused_densify as fd
    dev = torch.device("cuda:0")
    res = []
    for fused in (False, True):
        _, method = _make(False, True, dev, debug=True)
        model = method.model
        _set_stats(model, "normal", 0.0002, dev)
        assert not fd.supported(model)
        torch.manual_seed(9)
        out = (fd.densify_and_prune if fused else type(model).densify_and_prune)(model, 0.0002, 0.005, 1.5, True)
        res.append((out, model.xyz.detach().clone()))
    assert res[0][0] == res[1][0] and torch.equal(res[0][1], res[1][1])
