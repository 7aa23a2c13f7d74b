"""SH colours of models without appearance (``fused_colors.fused_sh_colors``, ``csrc/sh_colors.cu``) and the fused caller
for such models (``wildgaussians_fused.enable`` on the NeRF On-the-go configuration: ``appearance_enabled = False``,
``sh_degree = 3``).

CPU: the C entry points' argument checks and the dispatch predicate.  GPU: the colour op against a float64 restatement
of method.py's statements (:1555-1565) with the reference's own fp32 statements as the yardstick; ``_render_internal``
as shipped against ``enable(model)`` on the same model; a short training loop (loss of ``train_iteration``, Adam)
in both arms from the same start; ``optimize_embedding`` still refusing an appearance-off model.
"""
from __future__ import annotations

import ctypes
import types

import pytest
import torch

from oracle import color_torch as ct

GSR_E_INVALID = -1


# ---- the reference's statements (method.py:1555-1565), any dtype -------------------------------------------------------
def restated_colors(features_dc, features_rest, means3D, campos, deg):
    P = features_dc.shape[0]
    features = torch.cat((features_dc, features_rest), dim=-1).clamp_max(1.0)
    dirs = torch.nn.functional.normalize(means3D - campos.repeat(P, 1), dim=1)
    shs = features.view(-1, 16, 3).transpose(1, 2).contiguous()
    return torch.clamp_min(ct.eval_sh(deg, shs, dirs) + 0.5, 0.0)


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def test_entry_points_reject_bad_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib
    null6 = [None] * 6
    assert lib.gsr_sh_colors_forward(-1, 3, *null6) == GSR_E_INVALID
    assert b"sh_degree" in lib.gsr_last_error()
    assert lib.gsr_sh_colors_forward(5, 4, *null6) == GSR_E_INVALID
    assert lib.gsr_sh_colors_forward(5, -1, *null6) == GSR_E_INVALID
    assert lib.gsr_sh_colors_forward(5, 3, *null6) == GSR_E_INVALID
    assert b"NULL" in lib.gsr_last_error()
    assert lib.gsr_sh_colors_forward(0, 3, *null6) == 0                  # P = 0 is valid and launches nothing
    ptrs = [4096] * 6
    ptrs[1] = 4100                                                       # features_rest misaligned
    assert lib.gsr_sh_colors_forward(5, 3, *ptrs) == GSR_E_INVALID
    assert b"aligned" in lib.gsr_last_error()

    null9 = [None] * 9
    assert lib.gsr_sh_colors_backward(-1, 3, *null9) == GSR_E_INVALID
    assert lib.gsr_sh_colors_backward(5, 4, *null9) == GSR_E_INVALID
    assert lib.gsr_sh_colors_backward(5, 3, *null9) == GSR_E_INVALID
    assert b"NULL" in lib.gsr_last_error()
    assert lib.gsr_sh_colors_backward(0, 0, *null9) == 0
    ptrs = [4096] * 9
    ptrs[4] = None                                                       # dL_dcolors is optional ...
    ptrs[6] = 4104                                                       # ... but dL_dfeatures_rest must be aligned
    assert lib.gsr_sh_colors_backward(5, 3, *ptrs) == GSR_E_INVALID
    assert b"aligned" in lib.gsr_last_error()
    for i in (0, 1, 2, 3, 5, 6, 7):                                      # each required pointer
        ptrs = [4096] * 9
        ptrs[i] = None
        assert lib.gsr_sh_colors_backward(5, 3, *ptrs) == GSR_E_INVALID, i


def test_colour_op_refuses_cpu_tensors():
    import fused_colors as fc
    P = 4
    with pytest.raises(RuntimeError, match="CUDA"):
        fc.fused_sh_colors(torch.zeros(P, 3), torch.zeros(P, 45), torch.zeros(P, 3), torch.zeros(3), 3)


def test_restatement_is_the_raw_part_of_the_pinned_colour_oracle():
    """``restated_colors`` is the raw-colour part of ``oracle/color_torch.colors`` (pinned to the reference's own outputs
    by tests/golden/colors_*.npz), in float64 and with every edge of ``_inputs``."""
    (dc, rest, means), campos, _ = _inputs(500, "cpu", seed=3)
    dc, rest, means, campos = (x.double() for x in (dc, rest, means, campos))
    torch.manual_seed(0)
    W = [torch.randn(128, 59), torch.randn(128), torch.randn(128, 128), torch.randn(128), torch.randn(6, 128), torch.randn(6)]
    for deg in range(4):
        raw, _ = ct.colors(dc, rest, torch.zeros(500, 24).double(), torch.zeros(32).double(), *(w.double() for w in W),
                           means, campos, deg)
        assert torch.equal(restated_colors(dc, rest, means, campos, deg), raw)


class _FakeModel(types.SimpleNamespace):
    def _render_internal(self, *args, **kwargs):            # the class method the fused caller falls through to
        return "as shipped"


def _fake_model(appearance=False, storage_degree=3, cuda=True):
    t = lambda *s: types.SimpleNamespace(is_cuda=cuda, dtype=torch.float32, shape=s)
    cfg = types.SimpleNamespace(appearance_enabled=appearance, appearance_separate_tuned_color=True, appearance_model_sh=False,
                                sh_degree=storage_degree, appearance_embedding_dim=32, debug=False)
    mlp = types.SimpleNamespace(mlp=None) if appearance else None
    return _FakeModel(config=cfg, xyz=t(10, 3), features_dc=t(10, 3),
                      features_rest=t(10, 45) if storage_degree == 3 else None,
                      embeddings=t(10, 24) if appearance else None, appearance_mlp=mlp)


def test_dispatch_predicate():
    import wildgaussians_fused as wf
    run = types.SimpleNamespace(debug=False)
    off = _fake_model()
    assert wf._supported_sh(off, run) and not wf._supported(off, run)           # appearance off, degree 3: fused
    on = _fake_model(appearance=True)
    assert wf._supported(on, run) and not wf._supported_sh(on, run)             # appearance on: as before
    assert not wf._supported_sh(_fake_model(storage_degree=0), run)             # storage degree 0: falls through
    assert not wf._supported_sh(off, types.SimpleNamespace(debug=True))          # debug
    assert not wf._supported_sh(_fake_model(cuda=False), run)                    # CPU tensors
    for model, cfg in ((_fake_model(storage_degree=0), run), (off, types.SimpleNamespace(debug=True)),
                       (_fake_model(cuda=False), run), (on, run)):              # (appearance on without an embedding)
        assert wf.render_internal(model, None, cfg, kernel_size=0.1, embedding=None) == "as shipped"


def test_embedding_optimisation_stays_unsupported_without_appearance():
    import fused_embedding as fe
    model = _fake_model()
    cfg = types.SimpleNamespace(**vars(model.config), appearance_optim_type="dssim+l1-scaled")
    cam = types.SimpleNamespace(camera_models=0)
    cam.item = lambda: cam
    assert not fe.supported(types.SimpleNamespace(model=model, config=cfg), {"cameras": cam, "images": [None], "masks": None})


# ---- GPU: the colour op --------------------------------------------------------------------------------------------------
CAMPOS = (0.1, -0.2, 0.3)


def _inputs(P, dev, seed):
    """Raw parameters reaching every edge: coefficients above 1 (clamped, gradient masked), colours clamped at 0
    (strongly negative DC rows), a Gaussian exactly at campos (row 0), and non-contiguous features_rest / means3D."""
    g = torch.Generator().manual_seed(seed)
    dc = torch.randn(P, 3, generator=g) * 0.6
    dc[torch.rand(P, generator=g) < 0.1] -= 3.0
    rest = (torch.randn(45, P, generator=g) * 0.5).t()                   # non-contiguous view [P, 45]
    means = (torch.randn(P, 4, generator=g) * 2.0)[:, :3]                # non-contiguous view [P, 3]
    campos = torch.tensor(CAMPOS)
    if P > 0:
        means[0] = campos
    assert P < 2 or not (rest.is_contiguous() or means.is_contiguous())
    return [x.to(dev) for x in (dc, rest, means)], campos.to(dev), torch.randn(P, 3, generator=g).to(dev)


def _run(fn, leaves, campos, dL, deg, dtype):
    L = [x.detach().to(dtype).requires_grad_(True) for x in leaves]
    colors = fn(L[0], L[1], L[2], campos.to(dtype), deg)
    colors.backward(dL.to(dtype))
    return colors.detach(), [x.grad for x in L]


@pytest.mark.gpu
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("P", [0, 1, 77, 100_037, 3_000_000])
def test_colour_op_against_fp64(P, deg):
    import fused_colors as fc
    dev = torch.device("cuda:0")
    leaves, campos, dL = _inputs(P, dev, seed=1000 + P + deg)
    ours, g_ours = _run(fc.fused_sh_colors, leaves, campos, dL, deg, torch.float32)
    ref, g_ref = _run(restated_colors, leaves, campos, dL, deg, torch.float32)
    want, g_want = _run(restated_colors, leaves, campos, dL, deg, torch.float64)
    torch.cuda.synchronize()
    assert ours.shape == (P, 3) and all(g is not None for g in g_ours)
    assert g_ours[1].shape == (P, 45)
    nk = (deg + 1) ** 2
    if P == 0:
        return
    # edges reached
    if P >= 77:
        assert bool((want == 0).any()) and bool((want > 0).any())
        assert bool((leaves[0] > 1).any()) and (deg == 0 or bool((leaves[1][:, : 3 * (nk - 1)] > 1).any()))

    floor = 2.0 ** -23                                                   # one ulp of a colour near 1
    err = float((ours.double() - want).abs().max())
    err_ref = float((ref.double() - want).abs().max())
    assert err <= 1e-5 and err <= 2 * err_ref + floor, (err, err_ref)
    # the gradient of the Gaussian at campos is 1e12 x the direction gradient (F.normalize's eps): compared on its own
    rest_rows = slice(1, None)
    # at degree 0 the statements do not use the direction: autograd leaves means3D.grad None there (zero)
    g_ref, g_want = ([torch.zeros_like(x) if gr is None else gr for x, gr in zip(leaves, gs)] for gs in (g_ref, g_want))
    for name, a, r, w in zip(("features_dc", "features_rest", "means3D"), g_ours, g_ref, g_want):
        for rows in (rest_rows, slice(0, 1)) if name == "means3D" else (slice(None),):
            a_, r_, w_ = a[rows].double(), r[rows].double(), w[rows]
            if w_.numel() == 0:
                continue
            scale = float(w_.abs().max()) + 1e-300
            e = float((a_ - w_).abs().max()) / scale
            e_ref = float((r_ - w_).abs().max()) / scale
            assert torch.isfinite(a_).all(), name
            assert e <= 2 * e_ref + 1e-7, (name, rows, e, e_ref)
    # exactly zero above the active degree (a zero tensor, not None, at degree 0)
    assert int(torch.count_nonzero(g_ours[1][:, 3 * (nk - 1):])) == 0
    if deg > 0 and P >= 77:
        assert int(torch.count_nonzero(g_ours[1][:, : 3 * (nk - 1)])) > 0
    # the raw output of the fused appearance op on the same inputs: same arithmetic
    torch.manual_seed(deg)
    mlp = torch.nn.Sequential(torch.nn.Linear(59, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128), torch.nn.ReLU(),
                              torch.nn.Linear(128, 6)).to(dev)
    with torch.no_grad():
        raw, _ = fc.fused_colors(leaves[0], leaves[1], torch.zeros(P, 24, device=dev), torch.zeros(32, device=dev), mlp,
                                 leaves[2], campos, deg)
    assert float((raw - ours).abs().max()) <= 1e-6


@pytest.mark.gpu
def test_missing_upstream_gradient_counts_as_zero():
    import fused_colors as fc
    dev = torch.device("cuda:0")
    (dc, rest, means), campos, _ = _inputs(1000, dev, seed=5)
    ctx = types.SimpleNamespace(saved_tensors=(dc.contiguous(), rest.contiguous(), means.contiguous(), campos), deg=3)
    d = fc._FusedSHColors.backward(ctx, None)
    assert [tuple(t.shape) for t in d[:3]] == [(1000, 3), (1000, 45), (1000, 3)] and d[3] is None and d[4] is None
    assert all(int(torch.count_nonzero(t)) == 0 for t in d[:3])


# ---- GPU: the fused caller on an appearance-off model --------------------------------------------------------------------
UNIT_QUATERNIONS = torch.tensor([[s * (i == j) for j in range(4)] for i in range(4) for s in (1.0, -1.0)] +
                                [[0.5 * a, 0.5 * b, 0.5 * c, 0.5 * d] for a in (1, -1) for b in (1, -1) for c in (1, -1)
                                 for d in (1, -1)])       # the 24 rotations of norm exactly 1 in fp32 (and 0.5 x 16 signs)


def make_model_off(m, Config, scene, device, seed=0, deg=3, filter_3d=0.002, exact_activations=False):
    """A ``GaussianModel`` with the NeRF On-the-go values (appearance off, SH degree 3, kernel_size 0.1; uncertainty off)
    holding the synthetic cloud of `scene` (synthetic.make_scene with sh_degree=3), parameters as in
    ``wg_harness.make_model``.

    ``exact_activations``: no 3D filter and rotations drawn from the 24 quaternions whose norm is exactly 1, so that
    ``get_gaussians`` and ``fused_activations`` give the same bits (their normalisation and filter arithmetic otherwise
    differ in the last bit).  A comparison of the colour paths then sees no alpha of the composite cross its 1/255
    cut-off between the two arms: such a flip moves a pixel by up to 1/255 and the gradients of the Gaussians behind it."""
    cfg = Config(source_path="", model_path="", uncertainty_mode="disabled", appearance_enabled=False, sh_degree=3,
                 kernel_size=0.1)
    torch.manual_seed(seed)
    model = m.GaussianModel(cfg, training_setup=False).to(device)
    P = scene["means3D"].shape[0]
    model._resize_parameters(P)
    shs = scene["shs"]
    with torch.no_grad():
        model.xyz.copy_(scene["means3D"])
        model.features_dc.copy_(shs[:, 0, :])
        model.features_rest.copy_(shs[:, 1:, :].reshape(P, -1))
        model.scales.copy_(torch.log(scene["scales"]))
        model.rotations.copy_(scene["rotations"])
        model.opacities.copy_(torch.special.logit(scene["opacities"].clamp(1e-4, 1 - 1e-4)))
        model.filter_3D.fill_(0.0 if exact_activations else filter_3d)
        if exact_activations:
            pick = torch.randint(0, len(UNIT_QUATERNIONS), (P,), generator=torch.Generator().manual_seed(seed + 11))
            model.rotations.copy_(UNIT_QUATERNIONS[pick])
        model.active_sh_degree.fill_(deg)
    assert model.appearance_mlp is None and model.embeddings is None and model.get_embedding(0) is None
    model.train()
    return model, cfg


PARAMS = ("xyz", "features_dc", "features_rest", "scales", "rotations", "opacities")


def _method():
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    import diff_gaussian_rasterization as ours
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    return m, Config


def _step(model, cfg, cam, G, return_raw, render_depth, grad):
    for p in model.parameters():
        p.grad = None
    with torch.set_grad_enabled(grad):
        out = model._render_internal(cam, cfg, kernel_size=cfg.kernel_size, embedding=model.get_embedding(0),
                                     return_raw=return_raw, render_depth=render_depth)
        if grad:
            loss = (out["render"] * G[0]).sum()
            if render_depth:
                loss = loss + (out["depth"] * G[1][0]).sum() * 1e-2
            loss.backward()
    res = {"keys": sorted(out), "same": return_raw and out["render"] is out["raw_render"], "radii": out["radii"].clone(),
           "render": out["render"].detach().clone(), "accumulation": out["accumulation"].detach().clone()}
    if render_depth:
        res["depth"] = out["depth"].detach().clone()
    if grad:
        res["viewspace_grad"] = out["viewspace_points"].grad.detach().clone()
        for n in PARAMS:
            g = getattr(model, n).grad
            assert g is not None, n
            res["g_" + n] = g.detach().clone()
    return res


CASES = [dict(deg=3, return_raw=True, render_depth=False, grad=True), dict(deg=0, return_raw=True, render_depth=False, grad=True),
         dict(deg=3, return_raw=False, render_depth=False, grad=True), dict(deg=3, return_raw=True, render_depth=True, grad=True),
         dict(deg=1, return_raw=False, render_depth=False, grad=False)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: "deg{deg}_raw{return_raw:d}_depth{render_depth:d}_grad{grad:d}".format(**c))
def test_fused_render_internal_matches_the_shipped_method(case):
    import synthetic
    import wg_harness as wh
    import wildgaussians_fused as wf
    m, Config = _method()
    dev = torch.device("cuda:0")
    kw = dict(P=150_000, W=640, H=400, seed=71)
    scene = synthetic.make_scene(sh_degree=3, **kw)
    model, cfg = make_model_off(m, Config, scene, dev, seed=71, deg=case["deg"], exact_activations=True)
    cam = wh.make_camera(scene)
    import fused_colors as fc
    with torch.no_grad():
        want = model.get_gaussians()
        got = fc.fused_activations(model.scales, model.opacities, model.rotations, model.filter_3D)
    for k, x in zip(("scales", "opacities", "rotations"), got):
        assert torch.equal(x, want[k]), k                                 # the geometry of both arms is the same
    gen = torch.Generator().manual_seed(171)
    G = (torch.randn(3, kw["H"], kw["W"], generator=gen).to(dev), torch.randn(3, kw["H"], kw["W"], generator=gen).to(dev))
    args = (model, cfg, cam, G, case["return_raw"], case["render_depth"], case["grad"])
    a = _step(*args)
    a2 = _step(*args)                                                    # the shipped path's own run-to-run spread
    wf.enable(model, optimizer=False)
    b = _step(*args)
    wf.disable(model)
    c = _step(*args)
    torch.cuda.synchronize()

    assert b["keys"] == a["keys"] and b["same"] == a["same"] == case["return_raw"]
    assert torch.equal(c["render"], a["render"]) and torch.equal(c["radii"], a["radii"])     # disable() restores the method
    assert torch.equal(a["radii"], b["radii"])
    assert float(a["render"].abs().max()) > 0.05
    for k in ("render", "accumulation") + (("depth",) if case["render_depth"] else ()):
        assert float((a[k] - b[k]).abs().max()) <= 2e-4 * (float(a[k].abs().max()) if k == "depth" else 1.0), k
    if not case["grad"]:
        return
    for k in a:
        if not (k.startswith("g_") or k == "viewspace_grad"):
            continue
        scale = float(a[k].abs().max()) + 1e-30
        err = float((a[k] - b[k]).abs().max()) / scale
        noise = float((a2[k] - a[k]).abs().max()) / scale
        assert err <= max(20.0 * noise, 2e-5), (k, err, noise)
        assert err < 1e-3, (k, err)
    if case["deg"] == 0:
        assert int(torch.count_nonzero(b["g_features_rest"])) == 0


def _optimizer(model):
    lrs = dict(xyz=1.6e-4, features_dc=2.5e-3, features_rest=2.5e-3 / 20, opacities=0.05, scales=5e-3, rotations=1e-3)
    return torch.optim.Adam([{"params": [getattr(model, n)], "lr": lr, "name": n} for n, lr in lrs.items()], lr=1.0, eps=1e-15)


@pytest.mark.gpu
def test_short_training_loop_matches_the_shipped_method():
    """5 steps of render -> train_iteration's loss (L1 on `render`, 0.2 DSSIM on `raw_render`, method.py:1948-1966 with
    loss_mult 1) -> backward -> optimizer.step(), as shipped (torch Adam) and with ``enable(model, ssim=True)`` (FusedAdam,
    fused SSIM) from the same start."""
    import synthetic
    import wg_harness as wh
    import wildgaussians_fused as wf
    m, Config = _method()
    dev = torch.device("cuda:0")
    kw = dict(P=100_000, W=480, H=320, seed=72)
    scene = synthetic.make_scene(sh_degree=3, **kw)
    cam = wh.make_camera(scene)
    gt = torch.rand(3, kw["H"], kw["W"], generator=torch.Generator().manual_seed(9)).to(dev)

    def arm(fused):
        model, cfg = make_model_off(m, Config, scene, dev, seed=72, exact_activations=True)
        model.optimizer = _optimizer(model)
        start = {n: getattr(model, n).detach().clone() for n in PARAMS}
        if fused:
            wf.enable(model, ssim=True)
            assert type(model.optimizer).__name__ == "FusedAdam"
        try:
            for _ in range(5):
                model.optimizer.zero_grad(set_to_none=True)
                out = model._render_internal(cam, config=cfg, embedding=model.get_embedding(0), kernel_size=cfg.kernel_size)
                image_toned, image = out["render"], out["raw_render"]
                Ll1 = torch.nn.functional.l1_loss(image_toned, gt, reduction="none")
                ssim_value = m.ssim(image, gt, size_average=False)
                loss = (1.0 - cfg.lambda_dssim) * Ll1.mean() + cfg.lambda_dssim * (1.0 - ssim_value).mean()
                loss.backward()
                for n in PARAMS:
                    assert getattr(model, n).grad is not None, n
                model.optimizer.step()
        finally:
            wf.disable(model)
        torch.cuda.synchronize()
        st = model.optimizer.state
        return ({n: getattr(model, n).detach().clone() for n in PARAMS}, start,
                {n: st[getattr(model, n)]["exp_avg"].clone() for n in PARAMS})

    a, a0, ma = arm(False)
    a2, _, ma2 = arm(False)
    b, _, mb = arm(True)
    # After the first step the arms' parameters differ in the last bits, so an alpha of the composite may cross its
    # 1/255 cut-off in one arm only and move the gradients of the few Gaussians behind that pixel: the bars are on
    # whole tensors (norms, means), not entries.
    for n in PARAMS:
        # first moments (the averaged gradients): relative L2 distance
        norm = float(ma[n].norm())
        err, noise = float((mb[n] - ma[n]).norm()) / norm, float((ma2[n] - ma[n]).norm()) / norm
        assert norm > 0 and err <= max(20 * noise, 1e-3), (n, err, noise)
        # parameters: Adam normalises each entry's step, so an entry whose gradient is ~0 may step either way in
        # either arm; the mean deviation against the mean step is what the loop must preserve
        step = float((a[n] - a0[n]).abs().mean())
        dev_ = float((b[n] - a[n]).abs().mean()) / step
        noise = float((a2[n] - a[n]).abs().mean()) / step
        assert step > 0 and dev_ <= max(20 * noise, 1e-2), (n, dev_, noise)


@pytest.mark.gpu
def test_enable_method_keeps_refusing_embedding_optimisation():
    import synthetic
    import wildgaussians_fused as wf
    m, Config = _method()
    dev = torch.device("cuda:0")
    scene = synthetic.make_scene(P=2000, W=64, H=48, sh_degree=3, seed=73)
    model, cfg = make_model_off(m, Config, scene, dev, seed=73)
    method = types.SimpleNamespace(model=model, config=cfg)
    wf.enable_method(method)
    cam = types.SimpleNamespace(camera_models=0)
    cam.item = lambda: cam
    with pytest.raises(NotImplementedError, match="appearance_enabled=False"):
        method.optimize_embedding({"cameras": cam, "images": [None], "masks": None})
    wf.disable_method(method)
