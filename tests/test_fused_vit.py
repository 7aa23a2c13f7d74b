"""The DINOv2 backbone's token-wise layers as kernels (csrc/vit.cu, ``fused_dino.get_intermediate_layers(...,
blocks=True)``, ``wildgaussians_fused.enable(dino_blocks=True)``).

CPU: the C entry points' argument checks, ``supported(..., blocks=True)``'s refusals, the hook's fall-back and its
installation rules.  GPU: features and every option against a float64 backbone, each within twice the error of the
reference's fp32 statements (TF32 off); ``_compute_losses`` of the unmodified ``method.py`` and one ``fused_train`` step;
peak memory at 4K; determinism, no host synchronisation, the launch budget and no kernel outside the library; weight
edits seen by the next call.
"""
import ctypes
import copy
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import attention_oracle as ao
from test_fused_dino import Probe, dino_input, import_method, leaves, max_err, no_tf32, peak_above, sharpened_backbone


def small_backbone(m, dev="cpu", **kw):
    """A random two-block ViT with 64-wide heads (C = 128, 2 heads, 2 registers) that ``blocks=True`` accepts on CUDA."""
    args = dict(img_size=56, patch_size=14, embed_dim=128, depth=2, num_heads=2, num_register_tokens=2, block_chunks=0,
                init_values=1e-5)
    args.update(kw)
    torch.manual_seed(0)
    return m.dinov2.DinoVisionTransformer(**args).to(dev)


# ---------------------------------------------------------------------------------------------------------------- CPU

def test_c_entry_points_reject_bad_arguments():
    from diff_gaussian_rasterization import _C
    lib = _C._lib
    p = ctypes.c_void_p(256)                     # never dereferenced: every call below fails its checks first
    odd = ctypes.c_void_p(260)

    def tokens(B=1, H=28, W=42, C=64, patch=14, R=4, ptrs=None):
        ptrs = ptrs or [p] * 7
        return lib.gsr_vit_tokens(B, H, W, C, patch, R, *ptrs, None)

    for kw in [dict(B=0), dict(H=0), dict(W=-14), dict(C=0), dict(patch=0), dict(R=-1), dict(H=30), dict(W=43),
               dict(C=96), dict(C=1088), dict(patch=7, H=28, W=42)]:
        assert tokens(**kw) == -1 and b"bad sizes" in lib.gsr_last_error(), kw
    for kw in [dict(B=70000), dict(B=65535, H=14 * 200, W=14 * 200)]:
        assert tokens(**kw) == -1 and b"too large" in lib.gsr_last_error(), kw
    for i in range(7):
        ptrs = [p] * 7
        ptrs[i] = None
        assert tokens(ptrs=ptrs) == -1 and b"NULL" in lib.gsr_last_error(), i
    ptrs = [p] * 7
    ptrs[1] = odd
    assert tokens(ptrs=ptrs) == -1 and b"aligned" in lib.gsr_last_error()

    def linear(op=0, M=5, K=64, N=64, ptrs=None, eps=1e-6):     # ptrs: x, ln_w, ln_b, weight, bias, gamma, resid, out
        ptrs = ptrs or [p] * 8
        return lib.gsr_vit_linear(op, M, K, N, ptrs[0], ptrs[1], ptrs[2], eps, *ptrs[3:], None)

    assert linear(op=3) == -1 and b"unknown op" in lib.gsr_last_error()
    for kw in [dict(M=0), dict(K=0), dict(N=0), dict(K=66), dict(N=96), dict(M=-1)]:
        assert linear(**kw) == -1 and b"bad sizes" in lib.gsr_last_error(), kw
    for kw in [dict(K=4100), dict(N=4160)]:
        assert linear(**kw) == -1 and b"too large" in lib.gsr_last_error(), kw
    for op, required in [(0, (0, 1, 2, 3, 4, 7)), (1, (0, 1, 2, 3, 4, 7)), (2, (0, 3, 4, 6, 7))]:
        for i in required:
            ptrs = [p] * 8
            ptrs[i] = None
            assert linear(op=op, ptrs=ptrs) == -1 and b"NULL" in lib.gsr_last_error(), (op, i)
    ptrs = [p] * 8
    ptrs[3] = odd
    assert linear(ptrs=ptrs) == -1 and b"aligned" in lib.gsr_last_error()
    assert linear(eps=0.0) == -1 and b"eps" in lib.gsr_last_error()

    def output(B=1, T=10, C=64, R=4, layout=0, ptrs=None, eps=1e-6):
        ptrs = ptrs or [p] * 5
        return lib.gsr_vit_output(B, T, C, R, layout, ptrs[0], ptrs[1], ptrs[2], eps, ptrs[3], ptrs[4], None)

    for kw in [dict(B=0), dict(T=5), dict(C=48), dict(C=2048), dict(R=-1)]:
        assert output(**kw) == -1 and b"bad sizes" in lib.gsr_last_error(), kw
    assert output(layout=2) == -1 and b"unknown layout" in lib.gsr_last_error()
    assert output(B=70000) == -1 and b"too large" in lib.gsr_last_error()
    for i in (0, 1, 2, 3):
        ptrs = [p] * 5
        ptrs[i] = None
        assert output(ptrs=ptrs) == -1 and b"NULL" in lib.gsr_last_error(), i
    assert output(eps=-1.0) == -1 and b"eps" in lib.gsr_last_error()


class Cudaish(torch.Tensor):
    """A CPU tensor that reports ``is_cuda``: ``supported``'s structural checks, on a machine without a GPU."""

    @property
    def is_cuda(self):
        return True


def test_supported_refuses_each_unsupported_case():
    import fused_dino
    m, _ = import_method()
    bb = small_backbone(m)
    x = torch.zeros(1, 3, 56, 70)
    xc = x.as_subclass(Cudaish)
    with torch.no_grad():
        assert not fused_dino.supported(bb, x, 1, blocks=True)               # CPU tensors
        assert fused_dino.supported(bb, xc, 1, blocks=True)
        assert fused_dino.supported(bb, xc, [0], blocks=True)
        assert not fused_dino.supported(bb, xc.double(), 1, blocks=True)    # fp64 input
        assert not fused_dino.supported(bb, xc[..., :55], 1, blocks=True)   # not a multiple of the patch size
        assert not fused_dino.supported(bb, xc, [2], blocks=True)            # no such block
    assert not fused_dino.supported(bb, xc, 1, blocks=True)                  # parameters want a gradient
    refused = {
        "swiglu": small_backbone(m, ffn_layer="swiglufused"),
        "head dim 32": small_backbone(m, num_heads=4),
        "chunked blocks": small_backbone(m, block_chunks=2),
        "C not a multiple of 64": small_backbone(m, embed_dim=96, num_heads=1, ffn_layer="mlp"),
        "no LayerScale module": small_backbone(m),
        "tanh GELU": small_backbone(m),
        "patch-embed norm": small_backbone(m),
        "fp16 weights": small_backbone(m).half(),
        "LayerNorm without affine": small_backbone(m),
        "no bias": small_backbone(m),
    }
    refused["no LayerScale module"].blocks[0].ls2 = torch.nn.Dropout(0.0)
    refused["tanh GELU"].blocks[1].mlp.act = torch.nn.GELU(approximate="tanh")
    refused["patch-embed norm"].patch_embed.norm = torch.nn.LayerNorm(128)
    refused["LayerNorm without affine"].blocks[0].norm1 = torch.nn.LayerNorm(128, elementwise_affine=False)
    refused["no bias"].blocks[0].attn.qkv.bias = None
    with torch.no_grad():
        for what, v in refused.items():
            assert not fused_dino.supported(v, xc, 1, blocks=True), what
        assert fused_dino.supported(refused["tanh GELU"], xc, 1)            # blocks=False still takes it
        assert fused_dino.supported(refused["tanh GELU"], xc, [0], blocks=True)   # block 1 does not run for n=[0]


def test_hook_chooses_the_path_by_token_count(monkeypatch):
    """``dino_blocks``'s hook takes ``blocks=True`` up to ``BLOCKS_MAX_TOKENS`` tokens per call (the 350-px call of
    every feature-cache hit) and ``blocks=False`` above (the full-resolution call of a miss), where it measured slower."""
    import fused_dino
    import wildgaussians_fused as wf
    m, _ = import_method()
    bb = small_backbone(m, num_register_tokens=4)
    seen = []
    monkeypatch.setattr(fused_dino, "get_intermediate_layers", lambda *a, blocks=False: seen.append(blocks) or "fused")
    probe = Probe(bb)
    wf.enable(probe, optimizer=False, dino_blocks=True)
    try:
        for p in bb.parameters():
            p.requires_grad_(False)
        small, large = torch.zeros(1, 3, 196, 350), torch.zeros(1, 3, 1092, 1932)
        assert fused_dino.blocks_preferred(bb, small) and not fused_dino.blocks_preferred(bb, large)
        assert not fused_dino.blocks_preferred(bb, torch.zeros(11, 3, 196, 350))     # 11 x 355 tokens
        for x in (small, large):
            assert bb.get_intermediate_layers(x.as_subclass(Cudaish), n=[1], reshape=True) == "fused"
    finally:
        wf.disable(probe)
    assert seen == [True, False]


def test_hook_installation_fall_back_and_disable():
    import fused_dino
    import wildgaussians_fused as wf
    m, _ = import_method()
    bb = small_backbone(m)
    x = torch.randn(1, 3, 56, 70)
    probe = Probe(bb)
    with torch.no_grad():
        want = bb.get_intermediate_layers(x, n=[1], reshape=True)
        with pytest.raises(RuntimeError, match="CUDA"):
            fused_dino.get_intermediate_layers(bb, x, [1], blocks=True)
        wf.enable(probe, optimizer=False, dino=True)
        assert bb.__dict__["get_intermediate_layers"].__func__ is wf.dino_get_intermediate_layers
        wf.enable(probe, optimizer=False, dino_blocks=True)                  # replaces the dino hook
        hooked = bb.__dict__["get_intermediate_layers"]
        assert hooked.__func__ is wf.dino_blocks_get_intermediate_layers
        wf.enable(probe, optimizer=False, dino_blocks=True)                  # idempotent
        assert bb.__dict__["get_intermediate_layers"] is hooked
        wf.enable(probe, optimizer=False, dino=True)                         # not downgraded
        assert bb.__dict__["get_intermediate_layers"] is hooked
        got = bb.get_intermediate_layers(x, n=[1], reshape=True)             # CPU input: the class's method runs
    assert len(got) == 1 and torch.equal(got[0], want[0])
    wf.disable(probe)
    assert "get_intermediate_layers" not in bb.__dict__
    assert bb.get_intermediate_layers.__func__ is type(bb).get_intermediate_layers
    wf.enable(probe, optimizer=False, dino=True, dino_blocks=True)           # both in one call: blocks wins
    assert bb.__dict__["get_intermediate_layers"].__func__ is wf.dino_blocks_get_intermediate_layers
    wf.disable(probe)
    own = lambda *a, **k: "own"                                              # a user's own instance attribute stays
    bb.get_intermediate_layers = own
    wf.enable(probe, optimizer=False, dino_blocks=True)
    assert bb.__dict__["get_intermediate_layers"] is own
    wf.disable(probe)


def test_enable_method_passes_dino_blocks_through():
    import wildgaussians_fused as wf
    m, _ = import_method()
    bb = small_backbone(m)
    model = Probe(bb)
    method = types.SimpleNamespace(model=model)
    wf.enable_method(method, dino_blocks=True, optimizer=False)
    assert bb.__dict__["get_intermediate_layers"].__func__ is wf.dino_blocks_get_intermediate_layers
    wf.disable_method(method)
    assert "get_intermediate_layers" not in bb.__dict__


# ---------------------------------------------------------------------------------------------------------------- GPU

def check_call(bb, x, b64=None, what="", **kw):
    """blocks=True against the float64 backbone, within twice the reference fp32 statements' error, leaf by leaf."""
    import fused_dino
    b64 = b64 or ao.float64_backbone(bb)
    with torch.no_grad(), no_tf32():
        assert fused_dino.supported(bb, x, kw.get("n", 1), blocks=True)
        got = fused_dino.get_intermediate_layers(bb, x, blocks=True, **kw)
        ref = bb.get_intermediate_layers(x, **kw)
        want = b64.get_intermediate_layers(x.double(), **kw)
    assert type(got) is tuple and len(got) == len(ref)
    assert [type(i) for i in got] == [type(i) for i in ref]
    for g_, r_, w_ in zip(leaves(got), leaves(ref), leaves(want)):
        assert g_.shape == r_.shape and g_.dtype == torch.float32, (what, kw, g_.shape, r_.shape)
        e_ours, e_ref = max_err(g_, w_), max_err(r_, w_)
        print(f"{what} {kw}: fused {e_ours:.3e}, reference fp32 {e_ref:.3e}")
        assert e_ours <= 2 * e_ref, (what, kw, e_ours, e_ref)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W", [(1, 14, 14), (1, 42, 70), (1, 196, 350), (1, 1092, 1932), (2, 196, 350)])
def test_features_against_float64(B, H, W):
    dev = torch.device("cuda:0")
    _, bb = sharpened_backbone(dev)
    x = torch.cat([dino_input(H, W, 5 + i, dev) for i in range(B)])
    got = check_call(bb, x, what=f"{B}x{H}x{W}", n=[5], reshape=True)
    assert got[0].shape == (B, 384, H // 14, W // 14) and got[0].is_contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["vitb", "no_registers"])
def test_other_widths_and_no_registers(variant):
    m, _ = import_method()
    dev = torch.device("cuda:0")
    torch.manual_seed(4)
    if variant == "vitb":                                        # ViT-B/14 with registers, random weights
        bb = m.dinov2.vit_base(patch_size=14, num_register_tokens=4, img_size=518, init_values=1.0, block_chunks=0)
    else:
        bb = m.dinov2.vit_small(patch_size=14, num_register_tokens=0, img_size=518, init_values=1.0, block_chunks=0)
    bb = bb.to(dev).eval()
    with torch.no_grad():
        for blk in bb.blocks:
            blk.ls1.gamma.normal_(1.0, 0.2)
            blk.ls2.gamma.normal_(1.0, 0.2)
    x = dino_input(196, 350, 13, dev)
    check_call(bb, x, what=variant, n=[5], reshape=True)
    check_call(bb, x, what=variant, n=2, return_class_token=True)


@pytest.mark.gpu
def test_every_option_and_no_block_after_the_last_taken_one_runs():
    import fused_dino
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    _, bb = sharpened_backbone(dev)
    x = dino_input(196, 350, 6, dev)
    b64 = ao.float64_backbone(bb)
    cases = [dict(n=[5], reshape=True), dict(n=1), dict(n=[0, 3]), dict(n=[5], norm=False),
             dict(n=[5], return_class_token=True), dict(n=[0, 3], reshape=False, return_class_token=True),
             dict(n=[0, 3], reshape=True, return_class_token=True, norm=False)]
    for kw in cases:
        check_call(bb, x, b64, what="options", **kw)
    with torch.no_grad():
        for n, last, taken in (([0, 3], 3, 2), ([1], 1, 1), (2, 11, 2)):
            fused_dino.get_intermediate_layers(bb, x, n=n, blocks=True)
            n0 = _C.launch_count()
            fused_dino.get_intermediate_layers(bb, x, n=n, blocks=True)
            assert _C.launch_count() - n0 == 1 + 6 * (last + 1) + taken, n


def uncertainty_probe(m, model):
    probe = type("Probe", (), {"__module__": m.__name__})()
    probe.uncertainty_model = model
    return probe


@pytest.mark.gpu
def test_compute_losses_through_the_unmodified_method_py_with_cache_miss_and_hit():
    """``enable(model, uncertainty=True, dino_blocks=True)``: ``UncertaintyModel._compute_losses`` (method.py:363-433) in
    ``dino`` mode, on a cache miss (three backbone calls) and a cache hit (one).  All three arms run the fused head, so
    that only the backbone differs: the reference's own blocks (TF32 off), a float64 copy of the backbone, and
    ``dino_blocks``.  Every output is held within twice the reference arm's error against the float64 arm, plus one
    fp32 ulp of the quantity's scale: the bar of tests/test_fused_uncertainty.py."""
    import fused_dino
    import wildgaussians_fused as wf
    from test_fused_uncertainty import HEAD, images, make_model, restore, run, snapshot
    dev = torch.device("cuda:0")
    m, model = make_model(dev)
    gt, pred = images(420, 616, 9, dev)
    bb = model.backbone
    b64 = ao.float64_backbone(bb)
    probe = uncertainty_probe(m, model)
    calls = []
    inner = fused_dino._vit_layers

    def counted(*a, **k):
        calls.append(1)
        return inner(*a, **k)

    snap = snapshot(model)
    res = {}
    wf.enable(probe, optimizer=False, uncertainty=True)
    try:
        with no_tf32():
            for arm in ("reference", "float64", "fused"):
                if arm == "float64":
                    bb.get_intermediate_layers = lambda x, **kw: tuple(
                        t.float() for t in b64.get_intermediate_layers(x.double(), **kw))
                elif arm == "fused":
                    del bb.get_intermediate_layers
                    wf.enable(probe, optimizer=False, uncertainty=True, dino_blocks=True)
                    fused_dino._vit_layers = counted
                for hit in (False, True):
                    model._images_cache.clear()
                    if hit:                                       # the stored features come from the same arm
                        restore(model, snap)
                        run(model, model._compute_losses, gt, pred, cache_entry=("train", 1))
                    restore(model, snap)
                    calls.clear()
                    res[arm, hit] = run(model, model._compute_losses, gt, pred, cache_entry=("train", 1) if hit else None)
                    if arm == "fused":
                        assert len(calls) == (1 if hit else 3), (hit, len(calls))
    finally:
        fused_dino._vit_layers = inner
        wf.disable(probe)
        bb.__dict__.pop("get_intermediate_layers", None)
    for hit in (False, True):
        ref, want, fused = res["reference", hit], res["float64", hit], res["fused", hit]

        def bar(name, got, r, w):
            got, r, w = (torch.as_tensor(t).double().cpu() for t in (got, r, w))
            e, e_ref = float((got - w).abs().max()), float((r - w).abs().max())
            floor = 2.0 ** -23 * max(float(w.abs().max()), 1e-30)
            print(f"hit={hit} {name}: fused {e:.3e}, reference fp32 {e_ref:.3e}")
            assert e <= 2 * e_ref + floor, (hit, name, e, e_ref)

        bar("loss", fused["loss"], ref["loss"], want["loss"])
        for k in ref["metrics"]:
            bar(k, fused["metrics"][k], ref["metrics"][k], want["metrics"][k])
        bar("loss_mult", fused["loss_mult"], ref["loss_mult"], want["loss_mult"])
        for n in HEAD:
            bar(n, fused["grads"][n], ref["grads"][n], want["grads"][n])
        bar("running_mean", fused["running_mean"], ref["running_mean"], want["running_mean"])
        bar("running_var", fused["running_var"], ref["running_var"], want["running_var"])


@pytest.mark.gpu
def test_one_fused_train_step_runs_the_backbone_on_the_kernels():
    import fused_dino
    import diff_gaussian_rasterization as ours
    import wg_harness as wh
    import wildgaussians_fused as wf
    from test_fused_train import _method
    dev = torch.device("cuda:0")
    m, method = _method("uncertainty_masks", dev)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    wf.enable_method(method, train=True, ssim=True, msssim=True, uncertainty=True, dino_blocks=True)
    calls = []
    inner = fused_dino._vit_layers
    fused_dino._vit_layers = lambda *a, **k: calls.append(1) or inner(*a, **k)
    try:
        with no_tf32():
            metrics = method.train_iteration(1000)
    finally:
        fused_dino._vit_layers = inner
        wf.disable_method(method)
    assert len(calls) >= 1
    assert all(torch.isfinite(torch.as_tensor(float(v))) for v in metrics.values() if isinstance(v, (int, float)))


@pytest.mark.gpu
def test_compute_losses_at_4k_runs_within_2_gib():
    """``_compute_losses`` at 4096x2160 through the ``dino_blocks`` hook.  The full-resolution call has 45420 tokens,
    above ``BLOCKS_MAX_TOKENS``, so the hook runs it with ``blocks=False``; only the 350-px calls run vit.cu.  This is a
    bound on the hook's memory at 4K, not on ``blocks=True`` at 45420 tokens (that one is
    test_blocks_path_at_4k_within_2_gib)."""
    import wg_uncertainty as wu
    import wildgaussians_fused as wf
    m, Config = import_method()
    dev = torch.device("cuda:0")
    model, _ = wu.make_uncertainty_model(m, Config, "dino", dev, seed=3)
    g = torch.Generator(device=dev).manual_seed(12)
    gt = F.interpolate(torch.rand(1, 3, 271, 513, generator=g, device=dev), size=(2160, 4096), mode="bilinear")[0]
    pred = (gt + 0.05 * torch.randn(gt.shape, generator=g, device=dev)).clamp(0, 1)
    probe = uncertainty_probe(m, model)
    wf.enable(probe, optimizer=False, msssim=True, dino_blocks=True)
    try:
        (loss, metrics, loss_mult, grads), peak = peak_above(lambda: wu.compute_losses(model, gt, pred, seed=5))
    finally:
        wf.disable(probe)
    print(f"4K _compute_losses (dino_blocks): peak above inputs {peak / 2 ** 20:.0f} MiB")
    assert bool(torch.isfinite(loss)) and bool(torch.isfinite(loss_mult).all())
    assert all(bool(torch.isfinite(t).all()) for t in grads.values())
    assert peak < 2 * 2 ** 30


@pytest.mark.gpu
def test_determinism_no_host_synchronisation_launch_budget_and_only_library_kernels():
    import fused_dino
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    _, bb = sharpened_backbone(dev)
    x = dino_input(196, 350, 8, dev)
    call = lambda: fused_dino.get_intermediate_layers(bb, x, n=[5], reshape=True, blocks=True)
    with torch.no_grad():
        r1 = call()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            n0 = _C.launch_count()
            r2 = call()
            launches = _C.launch_count() - n0
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        assert torch.equal(r1[0], r2[0])
        assert launches <= 6 * 6 + 2, launches
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
             and "Memset" not in e.name}
    assert names and all(("vit_" in n or "attention_" in n) for n in names), names


@pytest.mark.gpu
def test_weight_edits_and_load_state_dict_are_seen_by_the_next_call():
    import fused_dino
    dev = torch.device("cuda:0")
    _, bb = sharpened_backbone(dev)
    x = dino_input(196, 350, 14, dev)
    b64 = ao.float64_backbone(bb)
    kw = dict(n=[5], reshape=True)
    with torch.no_grad():
        before = fused_dino.get_intermediate_layers(bb, x, blocks=True, **kw)[0].clone()
        saved = copy.deepcopy(bb.state_dict())
        bb.blocks[2].mlp.fc1.weight.mul_(1.5)                         # in place
        b64.blocks[2].mlp.fc1.weight.mul_(1.5)
    edited = check_call(bb, x, b64, what="fc1 edit", **kw)[0]
    assert max_err(edited, before) > 1e-3
    with torch.no_grad():
        bb.load_state_dict(saved)
        bb.pos_embed.add_(0.5)                                        # the position-embedding cache follows the version
        b64.pos_embed.add_(0.5)
        b64.blocks[2].mlp.fc1.weight.div_(1.5)
    check_call(bb, x, b64, what="load_state_dict + pos_embed edit", **kw)


@pytest.mark.gpu
def test_blocks_path_at_4k_within_2_gib():
    """``blocks=True`` itself at 4096x2160 (45420 tokens): finite, and within 2 GiB above its inputs."""
    import fused_dino
    dev = torch.device("cuda:0")
    _, bb = sharpened_backbone(dev)
    x = dino_input(2156, 4088, 15, dev)
    with torch.no_grad():
        got, peak = peak_above(lambda: fused_dino.get_intermediate_layers(bb, x, n=[5], reshape=True, blocks=True))
    print(f"blocks=True at 2156x4088: peak above inputs {peak / 2 ** 20:.0f} MiB")
    assert got[0].shape == (1, 384, 154, 292) and bool(torch.isfinite(got[0]).all())
    assert peak < 2 * 2 ** 30


@pytest.mark.gpu
def test_inputs_that_need_staging_copies():
    """Every operand ``blocks=True`` has to copy before a launch: a channels_last image, a channels_last patch-conv
    weight, and Linear weights and biases that are misaligned views into one flat buffer.  The copies are made in the
    same stream one after the other, so a copy released too early would be overwritten by the next one."""
    dev = torch.device("cuda:0")
    _, bb = sharpened_backbone(dev)
    bb.patch_embed.proj.to(memory_format=torch.channels_last)
    assert not bb.patch_embed.proj.weight.is_contiguous()
    with torch.no_grad():
        for blk in bb.blocks[:6]:
            for lin in (blk.attn.qkv, blk.attn.proj, blk.mlp.fc1, blk.mlp.fc2):
                w, b = lin.weight.detach(), lin.bias.detach()
                flat = torch.empty(1 + w.numel() + b.numel(), device=dev)
                flat[1:1 + w.numel()] = w.reshape(-1)
                flat[1 + w.numel():] = b
                lin.weight = torch.nn.Parameter(flat[1:1 + w.numel()].view_as(w), requires_grad=False)
                lin.bias = torch.nn.Parameter(flat[1 + w.numel():], requires_grad=False)
                assert lin.weight.data_ptr() % 16 and lin.bias.data_ptr() % 16
    x = dino_input(196, 350, 16, dev).contiguous(memory_format=torch.channels_last)
    assert not x.is_contiguous()
    check_call(bb, x, what="staged copies", n=[5], reshape=True)
    check_call(bb, x, what="staged copies", n=[0, 3], return_class_token=True)
