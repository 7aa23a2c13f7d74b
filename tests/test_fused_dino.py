"""Fused attention and early exit for the DINOv2 backbone (csrc/attention.cu, fused_dino.py,
wildgaussians_fused.enable(dino=True)).

CPU: the float64 oracle against the reference's own goldens, the C entry points' argument checks, the wrapper's
refusals and the hook's fall-back.  GPU: the attention against the oracle (goldens, N from 1 to 45420, sharp scores, the
row maximum in the last key tile) and the backbone's features against a float64 backbone, each within twice the error
of the reference's fp32 statements; the early exit's structure and the blocks it runs; fall-back, determinism, no host
synchronisation, launch counts, peak memory at 1080p and 4K; ``UncertaintyModel._compute_losses`` of the unmodified
``method.py`` hooked against unhooked.
"""
import ctypes
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import attention_oracle as ao

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["attention_tiny", "attention_odd", "attention_n200", "attention_sharp"]
# the random backbone's qkv weights (std 0.02) give near-uniform attention; q and k rows scaled by this factor give
# every query row a score spread (max - min over the keys) of at least about 10 (checked in the feature test)
SHARPEN = 5.0


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return torch.from_numpy(z["qkv"]), int(z["num_heads"]), torch.from_numpy(z["rows"]), torch.from_numpy(z["out"])


def import_method():
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    return m, Config


class Probe:
    """What ``enable`` needs of a model: its ``uncertainty_model`` (the ``dino`` hook's target)."""

    def __init__(self, backbone):
        self.uncertainty_model = types.SimpleNamespace(backbone=backbone)


# ---------------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_goldens(name):
    qkv, H, rows, out = load(name)
    got = ao.attention(qkv, H, rows=rows)
    assert got.shape == out.shape
    assert float((got - out).abs().max()) <= 1e-12


def test_c_entry_points_reject_bad_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib
    p = ctypes.c_void_p(256)                     # never dereferenced: every call below fails its checks first
    assert lib.gsr_attention_scratch_bytes(0, 5, 1) == 0
    assert lib.gsr_attention_scratch_bytes(1, 65, 6) == 6 * 2 * 80 * 1024
    for B, N, H in [(0, 5, 1), (1, 0, 1), (1, 5, 0), (-1, 5, 1), (1, -3, 1)]:
        assert lib.gsr_attention_forward(B, N, H, p, p, p, None) == -1
        assert b"bad sizes" in lib.gsr_last_error()
    for B, N, H in [(70000, 5, 1), (1, 5, 70000), (65535, 2 ** 31 - 1, 65535)]:
        assert lib.gsr_attention_scratch_bytes(B, N, H) == 0
        assert lib.gsr_attention_forward(B, N, H, p, p, p, None) == -1
        assert b"too large" in lib.gsr_last_error()
    for i in range(3):
        args = [p, p, p]
        args[i] = None
        assert lib.gsr_attention_forward(1, 5, 1, *args, None) == -1
        assert b"NULL" in lib.gsr_last_error()


def test_wrapper_refuses_cpu_tensors():
    import fused_dino
    with pytest.raises(RuntimeError, match="CUDA"):
        fused_dino.attention(torch.zeros(1, 5, 3 * 64), 1)


def test_hook_falls_back_to_the_original_on_cpu_and_disable_restores():
    import fused_dino
    import wildgaussians_fused as wf
    m, _ = import_method()
    torch.manual_seed(0)
    bb = m.dinov2.vit_small(patch_size=14, num_register_tokens=4, img_size=56)
    x = torch.randn(1, 3, 56, 70)
    probe = Probe(bb)
    assert not fused_dino.supported(bb, x, [5])
    with pytest.raises(RuntimeError, match="CUDA"):
        fused_dino.get_intermediate_layers(bb, x, [5])
    with torch.no_grad():
        want = bb.get_intermediate_layers(x, n=[5], reshape=True)
        wf.enable(probe, optimizer=False)
        assert "get_intermediate_layers" not in bb.__dict__           # default: untouched
        wf.enable(probe, optimizer=False, ssim=False, msssim=False, dino=True)
        hooked = bb.__dict__["get_intermediate_layers"]
        wf.enable(probe, optimizer=False, dino=True)                  # idempotent
        assert bb.__dict__["get_intermediate_layers"] is hooked
        got = bb.get_intermediate_layers(x, n=[5], reshape=True)      # CPU input: the original runs
    assert len(got) == 1 and torch.equal(got[0], want[0])
    wf.disable(probe)
    assert "get_intermediate_layers" not in bb.__dict__
    assert bb.get_intermediate_layers.__func__ is type(bb).get_intermediate_layers


# ---------------------------------------------------------------------------------------------------------------- GPU

class no_tf32:
    def __enter__(self):
        self.was = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.was


def max_err(a, b):
    return float((a.double() - b.to(device=a.device, dtype=torch.float64)).abs().max())


def check_attention(qkv, H, rows=None, want=None, what=""):
    """Fused vs float64 (the oracle or ``want``): max error <= 2x that of the reference's fp32 statements."""
    import fused_dino
    got = fused_dino.attention(qkv, H)
    assert got.shape == (qkv.shape[0], qkv.shape[1], H * 64) and got.dtype == torch.float32
    with no_tf32():
        if want is None:
            want = ao.attention(qkv, H, rows=rows)
        f32 = ao.attention(qkv, H, rows=rows, dtype=torch.float32)
    if rows is not None:
        got = got[:, rows.to(got.device)]
    e_ours, e_ref = max_err(got, want), max_err(f32, want)
    print(f"attention {what}: fused {e_ours:.3e}, reference fp32 {e_ref:.3e}")
    assert e_ours <= 2 * e_ref, (what, e_ours, e_ref)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_attention_against_reference_goldens(name):
    qkv, H, rows, out = load(name)
    dev = torch.device("cuda:0")
    check_attention(qkv.to(dev), H, rows=rows.to(dev), want=out.to(dev), what=name)


def random_qkv(B, N, H, seed, dev, qk_scale=1.0):
    g = torch.Generator(device=dev).manual_seed(seed)
    qkv = torch.randn(B, N, 3, H, 64, generator=g, device=dev)
    qkv[:, :, :2] *= qk_scale
    return qkv.reshape(B, N, 3 * H * 64)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 5, 37, 355, 10769])
@pytest.mark.parametrize("B,H", [(1, 6), (2, 6), (1, 12), (2, 12)])
def test_attention_against_oracle(N, B, H):
    dev = torch.device("cuda:0")
    check_attention(random_qkv(B, N, H, N + 7 * B + H, dev), H, what=(B, N, H))


@pytest.mark.gpu
def test_attention_sharp_scores_and_maximum_in_the_last_tile():
    dev = torch.device("cuda:0")
    N, H = 355, 6
    qkv = random_qkv(1, N, H, 21, dev, qk_scale=2.9)                 # |q.k / 8| up to about 40
    s = torch.einsum("nhd,mhd->hnm", qkv.view(N, 3, H, 64)[:, 0] / 8, qkv.view(N, 3, H, 64)[:, 1])
    assert float(s.abs().max()) > 30
    check_attention(qkv, H, what="sharp")
    # every query shares a direction u; the last key is 3 u: each row's maximum is key N - 1, in the last (partial) tile
    qkv = random_qkv(1, N, H, 22, dev).view(N, 3, H, 64)
    u = torch.randn(H, 64, generator=torch.Generator(device=dev).manual_seed(23), device=dev)
    qkv[:, 0] += u
    qkv[N - 1, 1] = 3 * u
    s = torch.einsum("nhd,mhd->hnm", qkv[:, 0] / 8, qkv[:, 1])
    assert bool((s.argmax(-1) == N - 1).all())
    check_attention(qkv.reshape(1, N, 3 * H * 64), H, what="last tile")


@pytest.mark.gpu
def test_attention_at_4k_on_sampled_rows():
    dev = torch.device("cuda:0")
    N, H = 45420, 6                                                 # 155 x 293 patches + 5 tokens
    qkv = random_qkv(1, N, H, 31, dev)
    g = torch.Generator(device=dev).manual_seed(32)
    rows = torch.cat([torch.tensor([0, N - 1], device=dev), torch.randperm(N - 2, generator=g, device=dev)[:2046] + 1])
    check_attention(qkv, H, rows=rows, what="4K")


def sharpened_backbone(dev, seed=3, mode="dino"):
    """The random-weight ViT-S/14 (4 registers) of an offline ``UncertaintyModel``, q and k rows scaled by SHARPEN."""
    import wg_uncertainty as wu
    m, Config = import_method()
    model, _ = wu.make_uncertainty_model(m, Config, mode, dev, seed=seed)
    bb = model.backbone
    with torch.no_grad():
        for blk in bb.blocks:
            C = blk.attn.qkv.in_features
            blk.attn.qkv.weight[:2 * C] *= SHARPEN
    return m, bb


def dino_input(H, W, seed, dev):
    """A smooth random image, normalised and padded as UncertaintyModel does, [1, 3, H, W] with H, W multiples of 14."""
    g = torch.Generator(device=dev).manual_seed(seed)
    img = torch.rand(1, 3, H // 8 + 1, W // 8 + 1, generator=g, device=dev)
    img = F.interpolate(img, size=(H, W), mode="bilinear", align_corners=False)
    return (img - 0.45) / 0.23


def leaves(result):
    return [t for item in result for t in (item if isinstance(item, tuple) else (item,))]


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(196, 350), (1092, 1932)])
def test_backbone_features_against_float64(H, W):
    import fused_dino
    dev = torch.device("cuda:0")
    _, bb = sharpened_backbone(dev)
    x = dino_input(H, W, 5, dev)
    with torch.no_grad(), no_tf32():
        blk = bb.blocks[0]
        t = bb.prepare_tokens_with_masks(x)
        qkv = blk.attn.qkv(blk.norm1(t)).view(t.shape[1], 3, 6, 64)
        s = torch.einsum("nhd,mhd->hnm", qkv[::max(1, t.shape[1] // 64), 0] / 8, qkv[:, 1])
        spread = s.amax(-1) - s.amin(-1)
        assert float(spread.min()) >= 10, float(spread.min())
        got = fused_dino.get_intermediate_layers(bb, x, n=[5], reshape=True)
        ref = bb.get_intermediate_layers(x, n=[5], reshape=True)
        want = ao.float64_backbone(bb).get_intermediate_layers(x.double(), n=[5], reshape=True)
    assert len(got) == 1 and got[0].shape == ref[0].shape == (1, 384, H // 14, W // 14)
    e_ours, e_ref = max_err(got[0], want[0]), max_err(ref[0], want[0])
    print(f"features {H}x{W}: fused {e_ours:.3e}, reference fp32 {e_ref:.3e}")
    assert e_ours <= 2 * e_ref, (e_ours, e_ref)


@pytest.mark.gpu
def test_early_exit_structure_values_and_blocks_run():
    import fused_dino
    dev = torch.device("cuda:0")
    _, bb = sharpened_backbone(dev)
    x = dino_input(196, 350, 6, dev)
    b64 = ao.float64_backbone(bb)
    cases = [dict(n=[5], reshape=True), dict(n=1), dict(n=[0, 3]), dict(n=[5], norm=False),
             dict(n=[5], return_class_token=True), dict(n=[0, 3], reshape=False, return_class_token=True)]
    with torch.no_grad(), no_tf32():
        for kw in cases:
            got = fused_dino.get_intermediate_layers(bb, x, **kw)
            ref = bb.get_intermediate_layers(x, **kw)
            want = b64.get_intermediate_layers(x.double(), **kw)
            assert type(got) is tuple and len(got) == len(ref)
            assert [type(i) for i in got] == [type(i) for i in ref]
            for g_, r_, w_ in zip(leaves(got), leaves(ref), leaves(want)):
                assert g_.shape == r_.shape, (kw, g_.shape, r_.shape)
                assert max_err(g_, w_) <= 2 * max_err(r_, w_), kw
        calls = {}
        handles = [mod.register_forward_hook(lambda mod_, i_, o_, k=(i, name): calls.__setitem__(k, calls.get(k, 0) + 1))
                   for i, blk in enumerate(bb.blocks) for name, mod in (("block", blk), ("qkv", blk.attn.qkv), ("mlp", blk.mlp))]
        try:
            fused_dino.get_intermediate_layers(bb, x, n=[0, 3])
        finally:
            for hd in handles:
                hd.remove()
    assert all(i <= 3 for i, _ in calls), calls
    assert all(calls.get((i, name)) == 1 for i in range(4) for name in ("qkv", "mlp")), calls


@pytest.mark.gpu
def test_hook_falls_back_for_unsupported_input_on_the_gpu(monkeypatch):
    import fused_dino
    import wildgaussians_fused as wf
    dev = torch.device("cuda:0")
    m, bb = sharpened_backbone(dev)
    calls = []
    cls = type(bb)

    def spy(self, x, n=1, reshape=False, return_class_token=False, norm=True):
        calls.append(x.dtype)
        return "original"

    monkeypatch.setattr(cls, "get_intermediate_layers", spy)
    x = dino_input(196, 350, 7, dev)
    probe = Probe(bb)
    wf.enable(probe, optimizer=False, dino=True)
    with torch.no_grad():
        got = bb.get_intermediate_layers(x, n=[5], reshape=True)
        assert torch.equal(got[0], fused_dino.get_intermediate_layers(bb, x, n=[5], reshape=True)[0]) and calls == []
        assert bb.get_intermediate_layers(x.double(), n=[5]) == "original"
        assert bb.get_intermediate_layers(x, n=[12]) == "original"      # the reference's assertion decides
    xg = x.clone().requires_grad_(True)
    assert bb.get_intermediate_layers(xg, n=[5]) == "original"
    assert calls == [torch.float64, torch.float32, torch.float32]
    small = m.dinov2.DinoVisionTransformer(img_size=56, patch_size=14, embed_dim=64, depth=2, num_heads=2,
                                         block_chunks=0).to(dev)
    monkeypatch.setattr(type(small), "get_intermediate_layers", spy)
    sprobe = Probe(small)
    wf.enable(sprobe, optimizer=False, dino=True)
    with torch.no_grad():
        assert not fused_dino.supported(small, x[..., :56, :56], 1)
        assert small.get_intermediate_layers(x[..., :56, :56], n=1) == "original"    # head dimension 32
    wf.disable(probe)
    wf.disable(sprobe)
    assert "get_intermediate_layers" not in bb.__dict__ and "get_intermediate_layers" not in small.__dict__


@pytest.mark.gpu
def test_two_runs_are_bitwise_identical_without_host_synchronisation():
    import fused_dino
    dev = torch.device("cuda:0")
    _, bb = sharpened_backbone(dev)
    x = dino_input(196, 350, 8, dev)
    with torch.no_grad():
        r1 = fused_dino.get_intermediate_layers(bb, x, n=[5], reshape=True)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            r2 = fused_dino.get_intermediate_layers(bb, x, n=[5], reshape=True)
            a = fused_dino.attention(random_qkv(1, 355, 6, 9, dev), 6)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        b = fused_dino.attention(random_qkv(1, 355, 6, 9, dev), 6)
    torch.cuda.synchronize()
    assert torch.equal(r1[0], r2[0]) and torch.equal(a, b)


@pytest.mark.gpu
def test_launch_count_per_attention_call():
    import fused_dino
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    for N in (1, 355, 10769):
        qkv = random_qkv(1, N, 6, 10, dev)
        n0 = _C.launch_count()
        fused_dino.attention(qkv, 6)
        assert _C.launch_count() - n0 == 2


def peak_above(fn):
    """(result, peak allocation above what was allocated before the call, in bytes)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


@pytest.mark.gpu
def test_peak_memory_of_the_full_resolution_backbone_at_1080p():
    import fused_dino
    dev = torch.device("cuda:0")
    _, bb = sharpened_backbone(dev)
    x = dino_input(1092, 1932, 11, dev)
    with torch.no_grad():
        _, fused = peak_above(lambda: fused_dino.get_intermediate_layers(bb, x, n=[5], reshape=True))
        _, ref = peak_above(lambda: bb.get_intermediate_layers(x, n=[5], reshape=True))
    print(f"peak above inputs at 1092x1932: fused {fused / 2 ** 20:.0f} MiB, reference {ref / 2 ** 20:.0f} MiB")
    assert fused < 2 ** 30


@pytest.mark.gpu
def test_compute_losses_at_4k_runs_within_2_gib():
    """``_compute_losses`` in ``dino`` mode at 4096x2160 with ``dino=True`` and ``msssim=True``.  The unhooked reference
    cannot run here: at N = 45420 tokens one [1, 6, N, N] fp32 score tensor is 49.5 GB, and softmax allocates a second
    (99 GB)."""
    import wg_uncertainty as wu
    import wildgaussians_fused as wf
    m, Config = import_method()
    dev = torch.device("cuda:0")
    model, _ = wu.make_uncertainty_model(m, Config, "dino", dev, seed=3)
    g = torch.Generator(device=dev).manual_seed(12)
    gt = F.interpolate(torch.rand(1, 3, 271, 513, generator=g, device=dev), size=(2160, 4096), mode="bilinear")[0]
    pred = (gt + 0.05 * torch.randn(gt.shape, generator=g, device=dev)).clamp(0, 1)
    probe = type("Probe", (), {"__module__": m.__name__})()
    probe.uncertainty_model = model
    wf.enable(probe, optimizer=False, msssim=True, dino=True)
    try:
        (loss, metrics, loss_mult, grads), peak = peak_above(lambda: wu.compute_losses(model, gt, pred, seed=5))
    finally:
        wf.disable(probe)
    print(f"4K _compute_losses (dino): peak above inputs {peak / 2 ** 20:.0f} MiB")
    assert bool(torch.isfinite(loss)) and bool(torch.isfinite(loss_mult).all())
    assert all(np.isfinite(v) for v in metrics.values()) and all(bool(torch.isfinite(t).all()) for t in grads.values())
    assert peak < 2 * 2 ** 30


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["l2reg", "dino+mssim", "dino"])
def test_compute_losses_through_the_unmodified_method_py(mode):
    """`enable(model, dino=True)`: ``UncertaintyModel._compute_losses`` (method.py:363-433) with a random-weight backbone,
    hooked against the reference's own backbone (TF32 off), and a third arm with the float64 backbone."""
    import wg_uncertainty as wu
    import wildgaussians_fused as wf
    m, Config = import_method()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(17)
    gt = F.interpolate(torch.rand(1, 3, 53, 78, generator=g, device=dev), size=(420, 616), mode="bilinear")
    pred = (gt + 0.05 * torch.randn(gt.shape, generator=g, device=dev)).clamp(0, 1)
    model, _ = wu.make_uncertainty_model(m, Config, mode, dev, seed=3)
    bb = model.backbone
    b64 = ao.float64_backbone(bb)
    probe = Probe(bb)
    res = {}
    with no_tf32():
        for arm in ("reference", "fused", "float64"):
            if arm == "fused":
                wf.enable(probe, optimizer=False, dino=True)
            elif arm == "float64":
                bb.get_intermediate_layers = lambda x, **kw: tuple(t.float() for t in b64.get_intermediate_layers(x.double(), **kw))
            try:
                res[arm] = wu.compute_losses(model, gt[0], pred[0], seed=5)
            finally:
                wf.disable(probe)
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
