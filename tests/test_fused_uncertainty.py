"""Fused head and ``dino``-mode loss of the uncertainty model (csrc/uncertainty.cu, fused_uncertainty.py,
wildgaussians_fused.enable(uncertainty=True)).

CPU: the float64 oracle against the reference's own goldens, the C entry points' argument checks, the dispatch
predicate's refusals, the hook's install / restore and fall-back, and the equivalence of the [1, C, 1, 1] dropout draw
with the reference's.  GPU: ``compute_losses`` against the reference's ``_compute_losses`` and the float64 oracle at
1080p, an odd size, a size below 350 px and 4K; the feature cache; determinism; launch count; host synchronisations;
a short training loop.
"""
import ctypes
import os
import types
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import uncertainty_oracle as uo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["uncertainty_small_odd", "uncertainty_resize", "uncertainty_tall_down"]
LAUNCHES = 6 + 3                                   # forward + backward kernels per call


def import_method():
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    return m, Config


def probe_for(m, um):
    """What ``enable`` needs of a GaussianModel: its module (for the msssim hooks) and ``uncertainty_model``."""
    probe = type("Probe", (), {"__module__": m.__name__})()
    probe.uncertainty_model = um
    return probe


# ---------------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_goldens(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    t = {k: torch.from_numpy(np.asarray(z[k])) for k in z.files}
    gt, pred = t["gt"].double() / 255, t["pred"].double() / 255
    ssim, msssim = (t[k].double() / float(z["stat_scale"]) for k in ("ssim", "msssim"))
    got = uo.compute(t["feat"], t["feat_gt_down"], t["feat_pred_down"], t["mask"], t["conv_w"], t["conv_b"], t["bn_w"],
                     t["bn_b"], t["running_mean_in"], t["running_var_in"], gt, pred, ssim, msssim,
                     clip_min=float(z["clip_min"]), reg_weight=float(z["reg_weight"]), eps=float(z["eps"]),
                     momentum=float(z["momentum"]))
    s = int(z["stride"])
    rel = lambda a, b: float((a.double() - b.double()).abs().max()) / max(float(b.double().abs().max()), 1e-300)
    assert abs(got["loss"] - float(t["loss"])) <= 1e-12
    assert np.allclose(got["metrics"], t["metrics"].numpy(), rtol=1e-12, atol=1e-12)
    assert rel(got["loss_mult"][..., ::s, ::s], t["loss_mult"]) <= 1e-12
    for k in ("conv_w", "conv_b", "bn_w", "bn_b"):
        assert rel(got["grads"][k], t["d_" + k]) <= 1e-10, k
    assert rel(got["running_mean"], t["running_mean"]) <= 1e-12 and rel(got["running_var"], t["running_var"]) <= 1e-12


def _args(**kw):
    from diff_gaussian_rasterization import _C
    a = _C.GsrUncertaintyArgs()
    for k, v in dict(C=384, th=3, tw=4, Hp=42, Wp=56, pad_top=1, pad_left=2, H=40, W=50, nh=40, nw=50, ch=3, cw=4, nHp=42,
                     nWp=56, npad_top=1, npad_left=2, clip_min=0.1, reg_weight=0.5, bn_eps=1e-5, bn_momentum=0.1).items():
        setattr(a, k, v)
    for name, _ in _C.GsrUncertaintyArgs._fields_:
        if getattr(a, name) in (None, 0) and name not in ("pad_top", "pad_left", "npad_top", "npad_left"):
            setattr(a, name, 256)                  # never dereferenced: every call below fails its checks first
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_c_entry_points_reject_bad_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib

    def rejected(expect, backward=False, **kw):
        fn = lib.gsr_uncertainty_backward if backward else lib.gsr_uncertainty_forward
        assert fn(ctypes.byref(_args(**kw)), None) == -1, kw
        assert expect in lib.gsr_last_error(), (kw, lib.gsr_last_error())

    assert lib.gsr_uncertainty_forward(None, None) == -1 and b"NULL" in lib.gsr_last_error()
    assert lib.gsr_uncertainty_scratch_bytes(None) == 0
    assert lib.gsr_uncertainty_scratch_bytes(ctypes.byref(_args(C=0))) == 0
    assert lib.gsr_uncertainty_scratch_bytes(ctypes.byref(_args())) > 0
    for C in (0, -1, 2049):
        rejected(b"channel count", C=C)
        rejected(b"channel count", backward=True, C=C)
    for k in ("th", "tw", "Hp", "H", "nw", "cw", "nHp"):
        rejected(b"positive", **{k: 0})
    rejected(b"more than one token", th=1, tw=1)
    rejected(b"token grid is larger", th=5, Hp=4, H=4, pad_top=0)
    rejected(b"crop does not fit", H=42)                        # 1 + 42 > 42
    rejected(b"crop does not fit", pad_left=-1)
    rejected(b"crop does not fit", nw=55)
    rejected(b"clip_min", clip_min=0.0)
    for k in ("feat", "feat_gt_down", "mask", "conv_b", "bn_b", "gt", "msssim", "loss_mult", "metrics", "scratch"):
        rejected(b"NULL", **{k: None})
    for k in ("dL_dloss", "d_conv_w", "d_bn_b"):
        rejected(b"gradient pointer is NULL", backward=True, **{k: None})


def _model_stub(**cfg):
    """Enough of an UncertaintyModel for the predicate's checks."""
    base = dict(uncertainty_mode="dino", uncertainty_dino_max_size=None)
    base.update(cfg)
    bn = torch.nn.SyncBatchNorm(8)
    return types.SimpleNamespace(config=types.SimpleNamespace(**base), training=True, bn=bn, conv_seg=torch.nn.Conv2d(8, 1, 1),
                                 backbone=types.SimpleNamespace(embed_dim=8), patch_size=14)


def test_supported_refuses_each_unsupported_case(monkeypatch):
    import fused_uncertainty as fu
    x = torch.rand(1, 3, 28, 42)
    why = lambda model, a=x, b=x: fu._unsupported(model, a, b)
    for mode in ("l2reg", "l1reg", "dino+mssim"):
        assert "mode" in why(_model_stub(uncertainty_mode=mode))
    assert "max_size" in why(_model_stub(uncertainty_dino_max_size=504))
    stub = _model_stub()
    stub.training = False
    assert "training" in why(stub)
    stub = _model_stub()
    stub.bn.eval()
    assert "BatchNorm" in why(stub)
    assert "[1, 3, H, W]" in why(_model_stub(), x.expand(2, 3, 28, 42), x.expand(2, 3, 28, 42))
    assert "fp32" in why(_model_stub(), x.double(), x.double())
    assert "CUDA" in why(_model_stub())                          # CPU tensors
    assert not fu.supported(_model_stub(), x, x)
    monkeypatch.setattr(torch.distributed, "is_available", lambda: True)
    monkeypatch.setattr(torch.distributed, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.distributed, "get_world_size", lambda group=None: 2)
    assert "across processes" in why(_model_stub())


def test_enable_installs_and_disable_restores_the_instance_attribute_and_cpu_falls_back():
    import wg_uncertainty as wu
    import wildgaussians_fused as wf
    m, Config = import_method()
    model, _ = wu.make_uncertainty_model(m, Config, "dino", "cpu", seed=1)
    probe = probe_for(m, model)
    gt = torch.rand(3, 56, 70, generator=torch.Generator().manual_seed(1))
    pred = (gt + 0.1).clamp(0, 1)
    want = wu.compute_losses(model, gt, pred, seed=4)
    wf.enable(probe, optimizer=False)
    assert "_compute_losses" not in model.__dict__                   # default: untouched
    wf.enable(probe, optimizer=False, uncertainty=True)
    hooked = model.__dict__["_compute_losses"]
    wf.enable(probe, optimizer=False, uncertainty=True)               # idempotent
    assert model.__dict__["_compute_losses"] is hooked
    got = wu.compute_losses(model, gt, pred, seed=4)                 # CPU input: the reference runs
    assert torch.equal(got[0], want[0]) and got[1] == want[1] and torch.equal(got[2], want[2])
    wf.disable(probe)
    assert "_compute_losses" not in model.__dict__
    assert model._compute_losses.__func__ is type(model)._compute_losses


@pytest.mark.parametrize("p", [0.5, 0.2, 0.0, 1.0])
def test_channel_mask_draw_matches_dropout2d_on_the_feature_map(p):
    C = 384
    x = torch.rand(1, C, 7, 9) + 0.5
    torch.manual_seed(11)
    y = F.dropout2d(x, p=p, training=True)
    after_ref = torch.get_rng_state()
    torch.manual_seed(11)
    mask = F.dropout2d(torch.ones(1, C, 1, 1), p=p, training=True)
    after = torch.get_rng_state()
    assert torch.equal(y, x * mask)
    assert torch.equal(after, after_ref)


# ---------------------------------------------------------------------------------------------------------------- GPU

class no_tf32:
    def __enter__(self):
        self.was = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.was


def images(H, W, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    gt = F.interpolate(torch.rand(1, 3, H // 8 + 2, W // 8 + 2, generator=g, device=dev), size=(H, W), mode="bilinear")
    pred = (gt + 0.05 * torch.randn(gt.shape, generator=g, device=dev)).clamp(0, 1)
    pred[..., : H // 3, : W // 4] = 1 - pred[..., : H // 3, : W // 4]
    return gt, pred


def make_model(dev, seed=3):
    import wg_uncertainty as wu
    m, Config = import_method()
    model, cfg = wu.make_uncertainty_model(m, Config, "dino", dev, seed=seed)
    g = torch.Generator(device=dev).manual_seed(seed + 50)
    with torch.no_grad():                                            # away from the initial values
        model.conv_seg.weight.normal_(0, 0.05, generator=g)
        model.conv_seg.bias.fill_(0.1)
        model.bn.weight.add_(0.2 * torch.randn(model.bn.weight.shape, generator=g, device=dev))
        model.bn.bias.add_(0.1 * torch.randn(model.bn.bias.shape, generator=g, device=dev))
    return m, model


HEAD = ("conv_seg.weight", "conv_seg.bias", "bn.weight", "bn.bias")


def snapshot(model):
    return {k: v.detach().clone() for k, v in model.state_dict().items() if not k.startswith("backbone.")}


def restore(model, snap):
    model.load_state_dict(snap, strict=False)


def run(model, fn, gt, pred, seed=5, cache_entry=None):
    """One call and its backward: (loss, metrics, loss_mult, grads, running_mean, running_var, nbt, cuda rng after)."""
    for p in model.parameters():
        p.grad = None
    torch.manual_seed(seed)
    loss, metrics, loss_mult = fn(gt, pred, _cache_entry=cache_entry)
    rng = torch.cuda.get_rng_state()
    loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if n in HEAD}
    bn = model.bn
    return dict(loss=loss.detach().clone(), metrics=metrics, loss_mult=loss_mult.clone(), grads=grads,
                running_mean=bn.running_mean.clone(), running_var=bn.running_var.clone(),
                nbt=int(bn.num_batches_tracked), rng=rng)


def oracle_arm(model, m, gt, pred, seed=5):
    """The float64 oracle on the features, mask and image statistics both arms see."""
    import fused_uncertainty as fu
    with torch.no_grad():
        x, _ = fu._normalised_padded(model, gt)
        feat = fu._features(model, x, None)
        gd, pd = m.dino_downsample(gt, max_size=350), m.dino_downsample(pred, max_size=350)
        fgd = fu._features(model, fu._normalised_padded(model, gd)[0], None)
        fpd = fu._features(model, fu._normalised_padded(model, pd)[0], None)
        torch.manual_seed(seed)
        mask = F.dropout2d(torch.ones(1, feat.shape[1], 1, 1, device=gt.device), p=model.config.uncertainty_dropout,
                           training=True).reshape(-1)
        ssim = m.ssim_down(gt, pred, max_size=400)
        msssim = m.msssim(gt, pred, max_size=400, min_size=80)
    bn, conv = model.bn, model.conv_seg
    return uo.compute(feat, fgd, fpd, mask, conv.weight, conv.bias, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                      gt, pred, ssim, msssim, clip_min=model.config.uncertainty_clip_min,
                      reg_weight=model.config.uncertainty_regularizer_weight, eps=bn.eps, momentum=bn.momentum)


def check_against_oracle(ref, fused, want, what):
    """Every output of the fused arm within twice the reference's own fp32 error against float64 (plus one fp32 ulp of
    the quantity's scale, the floor of test_fused_sh_colors.py)."""
    def bar(name, got, r, w):
        w = torch.as_tensor(w, dtype=torch.float64, device="cpu")
        got, r = torch.as_tensor(got).double().cpu(), torch.as_tensor(r).double().cpu()
        e, e_ref = float((got - w).abs().max()), float((r - w).abs().max())
        floor = 2.0 ** -23 * max(float(w.abs().max()), 1e-30)
        print(f"{what} {name}: fused {e:.3e}, reference fp32 {e_ref:.3e}")
        assert e <= 2 * e_ref + floor, (what, name, e, e_ref)

    bar("loss", fused["loss"], ref["loss"], want["loss"])
    for i, k in enumerate(uo.METRICS):
        bar(k, fused["metrics"][k], ref["metrics"][k], want["metrics"][i])
    bar("loss_mult", fused["loss_mult"], ref["loss_mult"], want["loss_mult"])
    names = dict(zip(HEAD, ("conv_w", "conv_b", "bn_w", "bn_b")))
    for n, k in names.items():
        bar(n + ".grad", fused["grads"][n], ref["grads"][n], want["grads"][k].reshape(fused["grads"][n].shape))
    bar("running_mean", fused["running_mean"], ref["running_mean"], want["running_mean"])
    bar("running_var", fused["running_var"], ref["running_var"], want["running_var"])
    assert fused["nbt"] == ref["nbt"]
    assert torch.equal(fused["rng"], ref["rng"])


def compare(H, W, dino=False):
    import fused_uncertainty as fu
    import wildgaussians_fused as wf
    dev = torch.device("cuda:0")
    m, model = make_model(dev)
    gt, pred = images(H, W, 9, dev)
    probe = probe_for(m, model)
    if dino:
        wf.enable(probe, optimizer=False, dino=True)
    try:
        snap = snapshot(model)
        with no_tf32():
            ref = run(model, model._compute_losses, gt, pred)
            restore(model, snap)
            fused = run(model, lambda *a, **k: fu.compute_losses(model, *a, **k), gt, pred)
            restore(model, snap)
            want = oracle_arm(model, m, gt, pred)
    finally:
        wf.disable(probe)
    assert fu.supported(model, gt, pred)
    assert set(fused["metrics"]) == set(ref["metrics"]) and all(type(v) is float for v in fused["metrics"].values())
    assert fused["loss"].dim() == 0 and fused["loss_mult"].shape == (1, 1, H, W)
    assert float(fused["loss_mult"].max()) <= 3
    check_against_oracle(ref, fused, want, f"{H}x{W}")


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(1080, 1920), (101, 157), (200, 301)])
def test_compute_losses_against_reference_and_float64(H, W):
    compare(H, W)


@pytest.mark.gpu
def test_compute_losses_at_4k_with_the_fused_backbone_on_both_arms():
    compare(2160, 4096, dino=True)


def counting_backbone(model):
    calls = []
    bb = model.backbone
    inner = bb.__dict__.get("get_intermediate_layers") or types.MethodType(type(bb).get_intermediate_layers, bb)

    def counted(x, *a, **k):
        calls.append(tuple(x.shape))
        return inner(x, *a, **k)

    bb.get_intermediate_layers = counted
    return calls


def same(a, b):
    assert torch.equal(a["loss"], b["loss"]) and a["metrics"] == b["metrics"] and torch.equal(a["loss_mult"], b["loss_mult"])
    assert all(torch.equal(a["grads"][k], b["grads"][k]) for k in HEAD)


@pytest.mark.gpu
def test_feature_cache_hits_and_is_shared_with_the_shipped_path():
    import fused_uncertainty as fu
    dev = torch.device("cuda:0")
    m, model = make_model(dev)
    gt, pred = images(420, 616, 10, dev)
    key = ("train", 3)
    fused_fn = lambda *a, **k: fu.compute_losses(model, *a, **k)
    snap = snapshot(model)
    calls = counting_backbone(model)
    run(model, model._compute_losses, gt, pred, cache_entry=key)          # the shipped path: stores, never hits
    shipped = dict(model._images_cache)
    assert len(shipped) == 2 and len(calls) == 3
    model._images_cache.clear()
    calls.clear()
    restore(model, snap)
    first = run(model, fused_fn, gt, pred, cache_entry=key)
    assert len(calls) == 3
    assert model._images_cache.keys() == shipped.keys()
    assert all(torch.equal(model._images_cache[k], shipped[k]) for k in shipped)
    calls.clear()
    restore(model, snap)
    second = run(model, fused_fn, gt, pred, cache_entry=key)
    assert len(calls) == 1 and calls[0][2] <= 350 + 13 and calls[0][3] <= 350 + 13   # the prediction at 350 px
    same(first, second)
    model._images_cache.clear()
    model._images_cache.update(shipped)
    calls.clear()
    restore(model, snap)
    third = run(model, fused_fn, gt, pred, cache_entry=key)
    assert len(calls) == 1
    same(first, third)


@pytest.mark.gpu
def test_two_runs_are_bitwise_identical_and_launch_count_is_pinned():
    import fused_uncertainty as fu
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    m, model = make_model(dev)
    fused_fn = lambda *a, **k: fu.compute_losses(model, *a, **k)
    for H, W in ((1080, 1920), (200, 301)):
        gt, pred = images(H, W, 11, dev)
        snap = snapshot(model)
        n0 = _C.launch_count()
        a = run(model, fused_fn, gt, pred)
        assert _C.launch_count() - n0 == LAUNCHES                     # statistics and backbone unhooked: PyTorch
        restore(model, snap)
        b = run(model, fused_fn, gt, pred)
        same(a, b)
        assert torch.equal(a["running_mean"], b["running_mean"]) and torch.equal(a["running_var"], b["running_var"])


@pytest.mark.gpu
def test_host_synchronisations_on_a_cache_hit():
    import wildgaussians_fused as wf
    dev = torch.device("cuda:0")
    m, model = make_model(dev)
    probe = probe_for(m, model)
    gt, pred = images(1080, 1920, 12, dev)
    wf.enable(probe, optimizer=False, msssim=True, dino=True, uncertainty=True)
    try:
        model.get_loss(gt[0], pred[0], _cache_entry=("train", 0))         # miss: fills the cache
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                loss, metrics, _ = model.get_loss(gt[0], pred[0], _cache_entry=("train", 0))
            finally:
                torch.cuda.set_sync_debug_mode(0)
        syncs = [str(w.message) for w in rec if "called a synchronizing" in str(w.message)]
        print("synchronisations on a hit:", len(syncs), syncs)
        assert len(syncs) <= 2, syncs
        assert np.isfinite(metrics["uncertainty_loss"]) and "ssim" not in metrics
    finally:
        wf.disable(probe)


@pytest.mark.gpu
def test_short_training_loop_matches_the_shipped_path():
    import wildgaussians_fused as wf
    dev = torch.device("cuda:0")
    res = {}
    for arm in ("shipped", "fused"):
        m, model = make_model(dev)
        probe = probe_for(m, model)
        if arm == "fused":
            wf.enable(probe, optimizer=False, msssim=True, dino=True, uncertainty=True)
        opt = torch.optim.Adam(model.parameters(), lr=model.config.uncertainty_lr)
        views = [images(540, 960, 20 + i, dev) for i in range(2)]
        torch.manual_seed(1)
        try:
            with no_tf32():
                for step in range(4):
                    gt, pred = views[step % 2]
                    opt.zero_grad()
                    loss, _, _ = model.get_loss(gt[0], pred[0], _cache_entry=("train", step % 2))
                    loss.backward()
                    opt.step()
        finally:
            wf.disable(probe)
        res[arm] = {n: p.detach().clone() for n, p in model.named_parameters() if n in HEAD}
        res[arm + "_start"] = snapshot(make_model(dev)[1])
    for n in HEAD:
        moved = float((res["shipped"][n] - res["shipped_start"][n]).abs().max())
        d = float((res["fused"][n] - res["shipped"][n]).abs().max())
        print(f"{n}: moved {moved:.3e}, fused - shipped {d:.3e}")
        assert d <= 1e-3 * moved + 1e-7, (n, d, moved)
