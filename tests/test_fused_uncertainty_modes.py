"""Fused uncertainty loss for the other modes, evaluation-mode calls and a capped head input (the ``gsr_uncertainty_mode_*``
entry points of csrc/uncertainty.cu, fused_uncertainty_modes.py, wildgaussians_fused.enable(uncertainty_modes=True)).

CPU: the float64 oracle against the reference's own goldens, the C entry points' argument checks, the dispatch
predicate (and that the ``dino`` path's predicates still refuse what they refused), the hook's install / restore and
fall-back.  GPU: every mode in training and evaluation mode against the reference's ``_compute_losses`` and the float64
oracle, with and without a cap; the ``loss_mult > 1`` map; determinism and launch count; backbone calls and host
synchronisations on a cache hit and in ``get_loss(gt, gt)``; ``optimize_embedding``; a short training loop.
"""
import ctypes
import os
import types
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_fused_uncertainty as tfu
from oracle import uncertainty_modes_oracle as uo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["uncertainty_modes_small_odd", "uncertainty_modes_resize", "uncertainty_modes_tall_down", "uncertainty_modes_cap"]
MODES = ("l2reg", "l1reg", "dino", "dino+mssim")
LAUNCHES = {"l2reg": 4 + 4, "l1reg": 4 + 4, "dino": 6 + 3, "dino+mssim": 6 + 3}     # forward + backward kernels


# ---------------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_goldens(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    t = {k: torch.from_numpy(np.asarray(z[k])) for k in z.files if z[k].dtype.kind != "U"}
    gt, pred = t["gt"].double() / 255, t["pred"].double() / 255
    ssim, msssim, msssim_down = (t[k].double() / float(z["stat_scale"]) for k in ("ssim", "msssim", "msssim_down"))
    H, W = gt.shape[2:]
    cap = int(z["cap"])
    s = int(z["stride"])
    rel = lambda a, b: float((a.double() - b.double()).abs().max()) / max(float(b.double().abs().max()), 1e-300)
    for run in z["runs"]:
        mode = {"l2reg": "l2reg", "l1reg": "l1reg", "dino": "dino", "dino_mssim": "dino+mssim"}[run.rsplit("_", 2)[0]]
        training = run.endswith("_train_")
        got = uo.compute_mode(t["feat"], t.get("feat_gt_down"), t.get("feat_pred_down"), t["mask"], t["conv_w"],
                              t["conv_b"], t["bn_w"], t["bn_b"], t["running_mean_in"], t["running_var_in"], gt, pred, ssim,
                              msssim, msssim_down, mode=mode, training=training,
                              head_hw=uo.head_size(H, W, None if cap < 0 else cap), clip_min=float(z["clip_min"]),
                              reg_weight=float(z["reg_weight"]), eps=float(z["eps"]), momentum=float(z["momentum"]))
        assert abs(got["loss"] - float(t[run + "loss"])) <= 1e-12, run
        assert np.allclose(got["metrics"], t[run + "metrics"].numpy(), rtol=1e-12, atol=1e-12), run
        assert rel(got["loss_mult"][..., ::s, ::s], t[run + "loss_mult"]) <= 1e-12, run
        for k in ("conv_w", "conv_b", "bn_w", "bn_b"):
            assert rel(got["grads"][k], t[run + "d_" + k]) <= 1e-10, (run, k)
        assert rel(got["running_mean"], t[run + "running_mean"]) <= 1e-12, run
        assert rel(got["running_var"], t[run + "running_var"]) <= 1e-12, run
        if not training:
            assert torch.equal(t[run + "running_mean"], t["running_mean_in"]), run


def test_goldens_cover_every_mode_in_both_batchnorm_modes():
    runs = set()
    for name in CASES:
        runs |= {str(r) for r in np.load(os.path.join(GOLDEN, name + ".npz"))["runs"]}
    assert runs == {f"{m}_{b}_" for m in ("l2reg", "l1reg", "dino_mssim") for b in ("train", "eval")} | {"dino_eval_"}


def _args(**kw):
    from diff_gaussian_rasterization import _C
    a = _C.GsrUncertaintyModeArgs()
    for k, v in dict(mode=3, training=1, C=384, th=3, tw=4, Hp=42, Wp=56, pad_top=1, pad_left=2, uh=40, uw=50, H=80, W=100,
                     nh=40, nw=50, ch=3, cw=4, nHp=42, nWp=56, npad_top=1, npad_left=2, clip_min=0.1, reg_weight=0.5,
                     bn_eps=1e-5, bn_momentum=0.1).items():
        setattr(a, k, v)
    for name, _ in _C.GsrUncertaintyModeArgs._fields_:
        if getattr(a, name) in (None, 0) and name not in ("pad_top", "pad_left", "npad_top", "npad_left"):
            setattr(a, name, 256)                  # never dereferenced: every call below fails its checks first
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_c_entry_points_reject_bad_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib

    def rejected(expect, backward=False, **kw):
        fn = lib.gsr_uncertainty_mode_backward if backward else lib.gsr_uncertainty_mode_forward
        assert fn(ctypes.byref(_args(**kw)), None) == -1, kw
        assert expect in lib.gsr_last_error(), (kw, lib.gsr_last_error())

    assert lib.gsr_uncertainty_mode_forward(None, None) == -1 and b"NULL" in lib.gsr_last_error()
    assert lib.gsr_uncertainty_mode_backward(None, None) == -1 and b"NULL" in lib.gsr_last_error()
    assert lib.gsr_uncertainty_mode_scratch_bytes(None) == 0
    assert lib.gsr_uncertainty_mode_scratch_bytes(ctypes.byref(_args(C=0))) == 0
    assert lib.gsr_uncertainty_mode_scratch_bytes(ctypes.byref(_args(mode=4))) == 0
    dino = lib.gsr_uncertainty_mode_scratch_bytes(ctypes.byref(_args()))
    l2 = lib.gsr_uncertainty_mode_scratch_bytes(ctypes.byref(_args(mode=0, nh=0, nw=0, ch=0, cw=0)))
    assert dino > 0 and l2 > 0                 # l2reg / l1reg read no 350-px size
    for mode in (-1, 4):
        rejected(b"bad mode", mode=mode)
        rejected(b"bad mode", backward=True, mode=mode)
    rejected(b"training", training=2)
    for C in (0, -1, 2049):
        rejected(b"channel count", C=C)
    for k in ("th", "tw", "Hp", "uh", "uw", "H", "W", "nw", "cw", "nHp"):
        rejected(b"positive", **{k: 0})
    rejected(b"more than one token", th=1, tw=1)
    rejected(b"token grid is larger", th=5, Hp=4, uh=4, pad_top=0)
    rejected(b"crop does not fit", uh=42)                       # 1 + 42 > 42
    rejected(b"crop does not fit", pad_left=-1)
    rejected(b"crop does not fit", nw=55)
    rejected(b"clip_min", clip_min=0.0)
    for k in ("feat", "feat_gt_down", "mask", "conv_b", "bn_b", "gt", "msssim", "msssim_down", "loss_mult", "metrics",
              "scratch"):
        rejected(b"NULL", **{k: None})
    rejected(b"NULL", training=0, running_var=None)             # evaluation mode reads the running statistics
    for k in ("dL_dloss", "d_conv_w", "d_bn_b"):
        rejected(b"gradient pointer is NULL", backward=True, **{k: None})


def _model_stub(**cfg):
    base = dict(uncertainty_mode="dino", uncertainty_dino_max_size=None)
    base.update(cfg)
    bn = torch.nn.SyncBatchNorm(8)
    return types.SimpleNamespace(config=types.SimpleNamespace(**base), training=True, bn=bn,
                                 conv_seg=torch.nn.Conv2d(8, 1, 1), backbone=types.SimpleNamespace(embed_dim=8),
                                 patch_size=14)


def _eval(stub):
    stub.training = False
    stub.bn.eval()
    return stub


def test_supported_matrix(monkeypatch):
    import fused_uncertainty_modes as fm
    x = torch.rand(1, 3, 28, 42)
    why = lambda model, a=x, b=x: fm._unsupported(model, a, b)
    for mode in MODES:                                           # get as far as the device check
        assert "CUDA" in why(_model_stub(uncertainty_mode=mode))
        assert "CUDA" in why(_eval(_model_stub(uncertainty_mode=mode)))
        assert "CUDA" in why(_model_stub(uncertainty_mode=mode, uncertainty_dino_max_size=504))
    assert "uncertainty_mode" in why(_model_stub(uncertainty_mode="disabled"))
    assert "uncertainty_mode" in why(_model_stub(uncertainty_mode="l3reg"))
    stub = _model_stub()
    stub.bn.eval()
    assert "same" in why(stub)
    stub = _model_stub()
    stub.training = False
    assert "same" in why(stub)
    assert "[1, 3, H, W]" in why(_model_stub(), x.expand(2, 3, 28, 42), x.expand(2, 3, 28, 42))
    assert "fp32" in why(_model_stub(), x.double(), x.double())
    assert not fm.supported(_model_stub(), x, x)
    # the dino modes under a cap whose 350-px grid differs from the image's: 1080 x 1920 at 504 gives a 294 x 504 head
    # input, whose 350-px map is 210 x 350 against 196 x 350
    assert fm.head_size(_model_stub(uncertainty_dino_max_size=504), 1080, 1920) == (294, 504)
    assert fm._down_size(294, 504, 350) == (210, 350) and fm._down_size(1080, 1920, 350) == (196, 350)
    monkeypatch.setattr(fm.fu, "_unsupported_inputs", lambda *a: None)
    big = torch.empty(1, 3, 1080, 1920)
    for mode in ("dino", "dino+mssim"):
        assert "350-px grid" in why(_model_stub(uncertainty_mode=mode, uncertainty_dino_max_size=504), big, big)
        assert why(_model_stub(uncertainty_mode=mode, uncertainty_dino_max_size=896), big, big) is None
    for mode in ("l2reg", "l1reg"):
        assert why(_model_stub(uncertainty_mode=mode, uncertainty_dino_max_size=504), big, big) is None
    tiny = torch.empty(1, 3, 10, 12)
    assert "more than one token" in why(_model_stub(uncertainty_mode="l2reg"), tiny, tiny)
    assert why(_eval(_model_stub(uncertainty_mode="l2reg")), tiny, tiny) is None
    monkeypatch.setattr(torch.distributed, "is_available", lambda: True)
    monkeypatch.setattr(torch.distributed, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.distributed, "get_world_size", lambda group=None: 2)
    assert "across processes" in why(_model_stub(uncertainty_mode="l2reg"), big, big)
    assert why(_eval(_model_stub(uncertainty_mode="l2reg")), big, big) is None    # evaluation mode does not synchronise


def test_dino_path_predicates_still_refuse_the_new_cases():
    import fused_train as ft
    import fused_uncertainty as fu
    import test_fused_train as tft
    import wildgaussians_fused as wf
    x = torch.rand(1, 3, 28, 42)
    for mode in ("l2reg", "l1reg", "dino+mssim"):
        assert "mode" in fu._unsupported(_model_stub(uncertainty_mode=mode), x, x)
    assert "max_size" in fu._unsupported(_model_stub(uncertainty_dino_max_size=504), x, x)
    assert "training" in fu._unsupported(_eval(_model_stub()), x, x)
    for kw in (dict(uncertainty="l2reg"), dict(uncertainty="l1reg"), dict(uncertainty="dino+mssim"),
               dict(uncertainty="dino", max_size=224), dict(uncertainty="l2reg", max_size=504)):
        method = tft._fake_method(**kw)
        method.model.uncertainty_model.__dict__[wf._MODES_MARK] = True       # a marked model changes nothing here
        assert not ft.supported(method), kw


def test_enable_installs_marks_and_restores_and_cpu_falls_back():
    import wg_uncertainty as wu
    import wildgaussians_fused as wf
    m, Config = tfu.import_method()
    model, _ = wu.make_uncertainty_model(m, Config, "l2reg", "cpu", seed=1)
    probe = tfu.probe_for(m, model)
    gt = torch.rand(3, 56, 70, generator=torch.Generator().manual_seed(1))
    pred = (gt + 0.1).clamp(0, 1)
    want = wu.compute_losses(model, gt, pred, seed=4)
    wf.enable(probe, optimizer=False, uncertainty=True)
    hooked = model.__dict__["_compute_losses"]
    assert wf._MODES_MARK not in model.__dict__                   # without the flag: exactly as before
    wf.enable(probe, optimizer=False, uncertainty=True, uncertainty_modes=True)
    assert model.__dict__["_compute_losses"] is hooked and model.__dict__[wf._MODES_MARK] is True
    assert model._compute_losses.__func__ is wf.uncertainty_compute_losses
    wf.enable(probe, optimizer=False, uncertainty_modes=True)     # idempotent
    assert model.__dict__["_compute_losses"] is hooked
    got = wu.compute_losses(model, gt, pred, seed=4)              # CPU input: the reference runs
    assert torch.equal(got[0], want[0]) and got[1] == want[1] and torch.equal(got[2], want[2])
    model.eval()
    want_eval = wu.compute_losses(model, gt, pred, seed=4)
    wf.disable(probe)
    assert "_compute_losses" not in model.__dict__ and wf._MODES_MARK not in model.__dict__
    assert model._compute_losses.__func__ is type(model)._compute_losses
    got_eval = wu.compute_losses(model, gt, pred, seed=4)
    assert torch.equal(got_eval[0], want_eval[0]) and got_eval[1] == want_eval[1]
    # the flag alone installs the hook; enable_method passes it through
    method = types.SimpleNamespace(model=probe)
    wf.enable_method(method, uncertainty_modes=True)
    assert model.__dict__[wf._MODES_MARK] is True and "_compute_losses" in model.__dict__
    wf.disable_method(method)
    assert wf._MODES_MARK not in model.__dict__ and "_compute_losses" not in model.__dict__


# ---------------------------------------------------------------------------------------------------------------- GPU

def make_model(dev, mode, training, cap=None, seed=3):
    m, model = tfu.make_model(dev, seed=seed)
    model.config.uncertainty_mode = mode
    model.config.uncertainty_dino_max_size = cap
    g = torch.Generator(device=dev).manual_seed(seed + 60)
    with torch.no_grad():                                            # running statistics the evaluation mode can see
        model.bn.running_mean.copy_(0.2 * torch.randn(model.bn.running_mean.shape, generator=g, device=dev))
        model.bn.running_var.copy_(0.5 + torch.rand(model.bn.running_var.shape, generator=g, device=dev))
    model.train(training)
    return m, model


def oracle_arm(model, m, gt, pred, seed=5):
    import fused_uncertainty as fu
    cfg = model.config
    mode, training = cfg.uncertainty_mode, model.training
    with torch.no_grad():
        head_in = model._scale_input(gt, cfg.uncertainty_dino_max_size)
        feat = fu._features(model, fu._normalised_padded(model, head_in)[0], None)
        fgd = fpd = msssim_down = None
        if mode.startswith("dino"):
            gd, pd = m.dino_downsample(gt, max_size=350), m.dino_downsample(pred, max_size=350)
            fgd = fu._features(model, fu._normalised_padded(model, gd)[0], None)
            fpd = fu._features(model, fu._normalised_padded(model, pd)[0], None)
            msssim_down = m.msssim(gd, pd, min_size=80) if mode == "dino+mssim" else None
        torch.manual_seed(seed)
        mask = F.dropout2d(torch.ones(1, feat.shape[1], 1, 1, device=gt.device), p=cfg.uncertainty_dropout,
                           training=True).reshape(-1)
        ssim = m.ssim_down(gt, pred, max_size=400)
        msssim = m.msssim(gt, pred, max_size=400, min_size=80)
    bn, conv = model.bn, model.conv_seg
    return uo.compute_mode(feat, fgd, fpd, mask, conv.weight, conv.bias, bn.weight, bn.bias, bn.running_mean,
                           bn.running_var, gt, pred, ssim, msssim, msssim_down, mode=mode, training=training,
                           head_hw=tuple(head_in.shape[2:]), clip_min=cfg.uncertainty_clip_min,
                           reg_weight=cfg.uncertainty_regularizer_weight, eps=bn.eps, momentum=bn.momentum)


def compare(H, W, mode, training, cap=None):
    import fused_uncertainty_modes as fm
    dev = torch.device("cuda:0")
    m, model = make_model(dev, mode, training, cap)
    gt, pred = tfu.images(H, W, 9, dev)
    assert fm.supported(model, gt, pred)
    snap = tfu.snapshot(model)
    with tfu.no_tf32():
        ref = tfu.run(model, model._compute_losses, gt, pred)
        tfu.restore(model, snap)
        fused = tfu.run(model, lambda *a, **k: fm.compute_losses(model, *a, **k), gt, pred)
        tfu.restore(model, snap)
        want = oracle_arm(model, m, gt, pred)
    what = f"{mode} {'train' if training else 'eval'} {H}x{W} cap {cap}"
    assert set(fused["metrics"]) == set(ref["metrics"]) and all(type(v) is float for v in fused["metrics"].values())
    assert fused["loss"].dim() == 0 and fused["loss_mult"].shape == (1, 1, H, W)
    tfu.check_against_oracle(ref, fused, want, what)
    if not training:
        assert fused["nbt"] == int(snap["bn.num_batches_tracked"])
        assert torch.equal(fused["running_mean"], snap["bn.running_mean"])
    # the map train_iteration and optimize_embedding use differs only where float64 puts the value within the bar of 1
    w = want["loss_mult"].double().cpu()
    e_ref = float((ref["loss_mult"].double().cpu() - w).abs().max())
    bar = 2 * e_ref + 2.0 ** -23 * float(w.abs().max())
    differ = (fused["loss_mult"].cpu() > 1) != (ref["loss_mult"].cpu() > 1)
    assert bool(((w - 1).abs()[differ] <= bar).all()), (what, int(differ.sum()))
    print(f"{what}: loss_mult > 1 on {float((w > 1).double().mean()):.3f} of the pixels, {int(differ.sum())} differ")


@pytest.mark.gpu
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("H,W", [(1080, 1920), (101, 157), (200, 301)])
def test_modes_against_reference_and_float64(H, W, mode, training):
    compare(H, W, mode, training)


@pytest.mark.gpu
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("mode,cap", [("l2reg", 504), ("dino", 896), ("dino+mssim", 896)])
def test_capped_head_input_against_reference_and_float64(mode, cap, training):
    compare(1080, 1920, mode, training, cap)


@pytest.mark.gpu
def test_two_runs_are_bitwise_identical_and_launch_count_is_pinned():
    import fused_uncertainty_modes as fm
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    for mode, training, cap in (("l2reg", True, None), ("l1reg", False, 504), ("dino", False, None),
                                ("dino+mssim", True, None)):
        m, model = make_model(dev, mode, training, cap)
        fused_fn = lambda *a, **k: fm.compute_losses(model, *a, **k)
        for H, W in ((1080, 1920), (200, 301)):
            gt, pred = tfu.images(H, W, 11, dev)
            snap = tfu.snapshot(model)
            n0 = _C.launch_count()
            a = tfu.run(model, fused_fn, gt, pred)
            assert _C.launch_count() - n0 == LAUNCHES[mode], mode   # statistics and backbone unhooked: PyTorch
            tfu.restore(model, snap)
            b = tfu.run(model, fused_fn, gt, pred)
            tfu.same(a, b)
            assert torch.equal(a["running_mean"], b["running_mean"]) and torch.equal(a["running_var"], b["running_var"])
            tfu.restore(model, snap)


def _syncs(fn):
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return out, [str(w.message) for w in rec if "called a synchronizing" in str(w.message)]


@pytest.mark.gpu
def test_l2reg_cache_hit_calls_no_backbone_and_synchronises_once():
    import wildgaussians_fused as wf
    dev = torch.device("cuda:0")
    m, model = make_model(dev, "l2reg", True)
    probe = tfu.probe_for(m, model)
    gt, pred = tfu.images(1080, 1920, 12, dev)
    wf.enable(probe, optimizer=False, msssim=True, dino=True, uncertainty=True, uncertainty_modes=True)
    try:
        calls = tfu.counting_backbone(model)
        model.get_loss(gt[0], pred[0], _cache_entry=("train", 0))         # miss: fills the cache
        assert len(calls) == 1 and calls[0][2:] == (1092, 1932)
        torch.cuda.synchronize()
        calls.clear()
        (loss, metrics, _), syncs = _syncs(lambda: model.get_loss(gt[0], pred[0], _cache_entry=("train", 0)))
        print("backbone calls on a hit:", calls, "synchronisations:", len(syncs), syncs)
        assert calls == [] and len(syncs) == 1, syncs
        assert np.isfinite(metrics["uncertainty_loss"])
        loss.backward()
    finally:
        wf.disable(probe)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["dino", "dino+mssim", "l2reg"])
def test_eval_get_loss_of_gt_against_itself_calls_the_backbone_once_per_resolution(mode):
    import fused_uncertainty_modes as fm
    import wildgaussians_fused as wf
    dev = torch.device("cuda:0")
    m, model = make_model(dev, mode, False)
    probe = tfu.probe_for(m, model)
    gt, _ = tfu.images(1080, 1920, 13, dev)
    snap = tfu.snapshot(model)
    img = gt[0]
    with torch.enable_grad():
        ref_loss, ref_metrics, ref_lm = model.get_loss(img, img)
    wf.enable(probe, optimizer=False, uncertainty=True, uncertainty_modes=True)
    try:
        calls = tfu.counting_backbone(model)
        rng = torch.cuda.get_rng_state()
        assert fm.supported(model, gt, gt)
        with torch.enable_grad():
            loss, metrics, lm = model.get_loss(img, img)
        assert torch.equal(torch.cuda.get_rng_state(), rng)
        assert len(calls) == (2 if mode.startswith("dino") else 1), calls
        assert calls[0][2:] == (1092, 1932)
        assert loss.requires_grad and ref_loss.requires_grad
        loss.backward()
        assert set(metrics) == set(ref_metrics) and lm.shape == ref_lm.shape
        assert all(torch.equal(v, snap[k]) for k, v in tfu.snapshot(model).items())
        assert abs(metrics["uncertainty_loss"] - ref_metrics["uncertainty_loss"]) <= 1e-4 * abs(ref_metrics["uncertainty_loss"]) + 1e-5
    finally:
        wf.disable(probe)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["l2reg", "dino"])
def test_optimize_embedding_uses_the_reference_uncertainty_map(mode, monkeypatch):
    import fused_embedding as fe
    import fused_uncertainty_modes as fm
    import test_fused_embedding as tfe
    import wildgaussians_fused as wf
    m, model, cfg, cam, gt_np = tfe._setup(dict(P=40_000, W=333, H=211), uncertainty=True)
    cfg.appearance_optim_type = "dssim+l1-scaled"
    um = model.uncertainty_model
    um.config.uncertainty_mode = mode
    g = torch.Generator(device=um.device).manual_seed(5)
    with torch.no_grad():                      # a head whose map has pixels on both sides of 1
        um.conv_seg.weight.normal_(0, 0.05, generator=g)
        um.conv_seg.bias.fill_(-0.3 if mode == "l2reg" else -0.6)
    maps = []

    def recording(self, *a, **k):
        out = type(self).get_loss(self, *a, **k)
        maps.append(out[2].detach().clone())
        return out

    um.get_loss = types.MethodType(recording, um)
    ds = tfe._dataset(cam, gt_np)
    tfe._ref_call(m, model, cfg, ds)                                   # the reference method, unhooked head
    model.train()
    taken = []
    real = fm.compute_losses
    monkeypatch.setattr(fm, "compute_losses", lambda *a, **k: taken.append(1) or real(*a, **k))
    wf.enable(model, optimizer=False, ssim=True, uncertainty=True, uncertainty_modes=True)
    try:
        ns = types.SimpleNamespace(model=model, config=cfg)
        fe.optimize_embedding(ns, ds, embedding=np.zeros(32, dtype=np.float32))
    finally:
        wf.disable(model)
    assert len(maps) == 2 and taken == [1]
    ref, fused = maps
    tol = 1e-5 * float(ref.abs().max())
    differ = (ref > 1) != (fused > 1)
    print(f"{mode}: loss_mult > 1 on {float((ref > 1).float().mean()):.3f}, {int(differ.sum())} pixels differ")
    assert bool(((ref - 1).abs()[differ] <= tol).all())
    assert float((fused - ref).abs().max()) <= tol


@pytest.mark.gpu
def test_short_l2reg_training_loop_matches_the_shipped_path():
    import wildgaussians_fused as wf
    dev = torch.device("cuda:0")
    res = {}
    for arm in ("shipped", "fused"):
        m, model = make_model(dev, "l2reg", True)
        probe = tfu.probe_for(m, model)
        method = types.SimpleNamespace(model=probe)
        if arm == "fused":
            wf.enable_method(method, ssim=True, msssim=True, uncertainty=True, uncertainty_modes=True)
        opt = torch.optim.Adam(model.parameters(), lr=model.config.uncertainty_lr)
        views = [tfu.images(540, 960, 20 + i, dev) for i in range(2)]
        torch.manual_seed(1)
        try:
            with tfu.no_tf32():
                for step in range(4):
                    gt, pred = views[step % 2]
                    opt.zero_grad()
                    loss, _, _ = model.get_loss(gt[0], pred[0], _cache_entry=("train", step % 2))
                    loss.backward()
                    opt.step()
        finally:
            wf.disable_method(method)
        res[arm] = {n: p.detach().clone() for n, p in model.named_parameters() if n in tfu.HEAD}
        res[arm + "_start"] = tfu.snapshot(make_model(dev, "l2reg", True)[1])
    for n in tfu.HEAD:
        moved = float((res["shipped"][n] - res["shipped_start"][n]).abs().max())
        d = float((res["fused"][n] - res["shipped"][n]).abs().max())
        print(f"{n}: moved {moved:.3e}, fused - shipped {d:.3e}")
        assert d <= 1e-3 * moved + 1e-7, (n, d, moved)
