"""DINOv2 backbone of the uncertainty loss: the reference's ``get_intermediate_layers`` (wildgaussians/dinov2.py:789-813,
unmodified, from oracle/_ref/py) against ``fused_dino`` (csrc/attention.cu + early exit).

    python tools/bench_dino.py [--steps 5] [--rounds 5] [--out result.json]

Arms alternate round by round; medians over rounds with the spread:
  * backbone ``get_intermediate_layers(x, n=[5], reshape=True)`` at 1092x1932 (10769 tokens, the full-resolution
    uncertainty forward at C3) and 196x350 (355 tokens, ``_compute_cosine_similarity``): the reference as shipped, the
    reference's own blocks 0..5 only (early exit with the reference's attention, built here and nowhere else), hooked;
  * the attention kernel alone (split pre-pass included) at N = 10769 and 45420 with 6 heads: useful TFLOP/s counting
    4 N^2 64 H per call, executed TFLOP/s counting the split's MMAs on the padded tiles (3 per product in S = QK^T,
    4 in O = PV), and the executed rate's share of the 495 TFLOP/s dense TF32 data-sheet peak;
  * ``UncertaintyModel._compute_losses`` in ``dino`` mode, both arms with ``msssim=True``: reference against
    ``dino=True`` at C3, ``dino=True`` only at C5 (the reference's two [1, 6, 45420, 45420] fp32 tensors would need 99 GB);
  * the train step of tools/bench_msssim.py (uncertainty ``dino``, fused caller, ``ssim=True``, ``msssim=True``) without
    and with ``dino=True`` at C3, with it at C5;
  * errors against float64 (the chunked oracle, oracle/attention_oracle.py) of the fused results and of the reference's
    fp32 statements (TF32 off).
The random backbone's q and k weight rows are scaled by 5 (tests/test_fused_dino.py) so that attention is not uniform.
Prints the device name and its power limit / max SM clock (nvidia-smi, query only).  Needs a GPU; does not fall back.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "wild-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_msssim import Hooks, run_arms, textured_pair  # noqa: E402
from bench_ssim import device_info  # noqa: E402

TF32_PEAK = 495e12                    # H100 SXM data sheet, dense TF32
SHARPEN = 5.0


class DinoHook:
    """Switches one backbone's ``get_intermediate_layers`` between the class's own and the fused path."""

    def __init__(self, backbone):
        self.probe = type("Probe", (), {})()
        self.probe.uncertainty_model = type("U", (), {})()
        self.probe.uncertainty_model.backbone = backbone

    def set(self, on):
        import wildgaussians_fused as wf
        if on:
            wf.enable(self.probe, optimizer=False, dino=True)
        else:
            wf.disable(self.probe)


def early_exit_reference(bb, x, last=5):
    """The reference's own modules, blocks 0..last only, then the statements of dinov2.py:801-810 for n=[last]."""
    t = bb.prepare_tokens_with_masks(x)
    for blk in bb.blocks[:last + 1]:
        t = blk(t)
    t = bb.norm(t)[:, 1 + bb.num_register_tokens:]
    B, _, w, h = x.shape
    return (t.reshape(B, w // bb.patch_size, h // bb.patch_size, -1).permute(0, 3, 1, 2).contiguous(),)


def sharpened_uncertainty_model(m, Config, mode, dev):
    import wg_uncertainty as wu
    model, _ = wu.make_uncertainty_model(m, Config, mode, dev, seed=3)
    with torch.no_grad():
        for blk in model.backbone.blocks:
            C = blk.attn.qkv.in_features
            blk.attn.qkv.weight[:2 * C] *= SHARPEN
    return model


def dino_input(H, W, dev):
    g = torch.Generator(device=dev).manual_seed(5)
    img = torch.rand(1, 3, H // 8 + 1, W // 8 + 1, generator=g, device=dev)
    return (torch.nn.functional.interpolate(img, size=(H, W), mode="bilinear", align_corners=False) - 0.45) / 0.23


def max_err(a, b):
    return float((a.double() - b.double()).abs().max())


def backbone_case(bb, hook, H, W, steps, rounds, dev):
    import fused_dino
    from oracle import attention_oracle as ao
    x = dino_input(H, W, dev)

    def arm(kind):
        def run():
            with torch.no_grad():
                hook.set(kind == "hooked")
                if kind == "early_exit_reference":
                    early_exit_reference(bb, x)
                else:
                    bb.get_intermediate_layers(x, n=[5], reshape=True)
                hook.set(False)
        return run

    res = {"H": H, "W": W, "tokens": (H // 14) * (W // 14) + 1 + bb.num_register_tokens,
           "times": run_arms({k: arm(k) for k in ("reference", "early_exit_reference", "hooked")}, steps, rounds, warmup=2)}
    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        want = ao.float64_backbone(bb).get_intermediate_layers(x.double(), n=[5], reshape=True)[0]
        res["error_vs_fp64"] = {"fused": max_err(fused_dino.get_intermediate_layers(bb, x, n=[5], reshape=True)[0], want),
                                "reference_fp32": max_err(bb.get_intermediate_layers(x, n=[5], reshape=True)[0], want)}
    torch.backends.cudnn.allow_tf32 = True
    del want
    torch.cuda.empty_cache()
    return res


def attention_case(N, H, steps, rounds, dev):
    import fused_dino
    from oracle import attention_oracle as ao
    g = torch.Generator(device=dev).manual_seed(N)
    qkv = torch.randn(1, N, 3 * H * 64, generator=g, device=dev)
    times = run_arms({"attention": lambda: fused_dino.attention(qkv, H)}, steps, rounds, warmup=2)
    t = times["attention"]["device"]["median_ms"] * 1e-3
    useful = 4.0 * N * N * 64 * H
    mpad, npad = -(-N // 128) * 128, -(-N // 64) * 64
    executed = 2.0 * mpad * npad * 64 * H * (3 + 4)
    rows = None if N <= 20000 else torch.cat([torch.tensor([0, N - 1], device=dev),
                                              torch.randperm(N - 2, generator=g, device=dev)[:2046] + 1])
    want = ao.attention(qkv, H, rows=rows)
    got = fused_dino.attention(qkv, H)
    ref = ao.attention(qkv, H, rows=rows, dtype=torch.float32)
    got = got if rows is None else got[:, rows]
    res = {"N": N, "heads": H, "times": times, "useful_tflops": useful / t / 1e12, "executed_tflops": executed / t / 1e12,
           "share_of_tf32_peak": executed / t / TF32_PEAK, "bound": "tensor-core math (bytes moved are < 1% of the time at 3.35 TB/s)",
           "error_vs_fp64": {"rows": "all" if rows is None else "2048 sampled incl. first and last",
                             "fused": max_err(got, want), "reference_fp32": max_err(ref, want)}}
    del qkv, want, got, ref
    torch.cuda.empty_cache()
    return res


def losses_case(m, Config, hooks, H, W, steps, rounds, dev, with_reference):
    import wg_uncertainty as wu
    gt, pred = textured_pair(H, W, dev)
    model = sharpened_uncertainty_model(m, Config, "dino", dev)
    hook = DinoHook(model.backbone)

    def run_with(dino):
        def run():
            hooks.set(ssim=True, msssim=True)
            hook.set(dino)
            wu.compute_losses(model, gt[0], pred[0], seed=5)
            hook.set(False)
        return run

    arms = {"compute_losses_dino_hooked": run_with(True)}
    if with_reference:
        arms = {"compute_losses_dino_reference": run_with(False), **arms}
    try:
        times = run_arms(arms, steps, rounds, warmup=1)
    finally:
        hooks.restore()
    del model
    torch.cuda.empty_cache()
    return {"H": H, "W": W, "times": times}


def train_step_case(m, Config, hooks, cfg_name, arms_wanted, steps, rounds, dev):
    """method.py:1909-1966 with the uncertainty model (dino) on the wg_harness model with the fused caller, ssim and
    msssim on; ``dino`` off and / or on."""
    import synthetic
    import wg_harness as wh
    import wildgaussians_fused as wf
    import diff_gaussian_rasterization as ours
    kw = dict(synthetic.CONFIGS[cfg_name]); kw["seed"] = 0; kw["sh_degree"] = 3
    scene = synthetic.make_scene(**kw)
    model, cfg = wh.make_model(m, Config, scene, dev)
    unc = sharpened_uncertainty_model(m, Config, "dino", dev)
    hook = DinoHook(unc.backbone)
    cam = wh.make_camera(scene)
    H, W = scene["image_height"], scene["image_width"]
    gt_image = torch.rand(3, H, W, generator=torch.Generator().manual_seed(5)).to(dev)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    ours._C.set_geometry_cache(True)
    wf.enable(model, optimizer=False)

    def step(dino):
        def run():
            hooks.set(ssim=True, msssim=True)
            hook.set(dino)
            for p in list(model.parameters()) + list(unc.parameters()):
                p.grad = None
            embedding = model.appearance_embeddings[0]
            render_pkg = model._render_internal(cam, config=cfg, embedding=embedding, kernel_size=cfg.kernel_size)
            image_toned, image = render_pkg["render"], render_pkg["raw_render"]
            uncertainty_loss, metrics, loss_mult = unc.get_loss(gt_image, image_toned.detach(), _cache_entry=("train", 0))
            loss_mult = (loss_mult > 1).to(dtype=loss_mult.dtype)        # past the warm-up (method.py:1934-1940)
            Ll1 = torch.nn.functional.l1_loss(image_toned, gt_image, reduction="none")
            ssim_value = m.ssim(image, gt_image, size_average=False)
            loss = ((1.0 - cfg.lambda_dssim) * (Ll1 * loss_mult).mean() +
                    cfg.lambda_dssim * ((1.0 - ssim_value) * loss_mult).mean() + uncertainty_loss)
            loss.backward()
            hook.set(False)
        return run

    try:
        times = run_arms({f"train_step_dino_{'on' if d else 'off'}": step(d) for d in arms_wanted}, steps, rounds, warmup=1)
    finally:
        hooks.restore()
        wf.disable(model)
        ours._C.set_geometry_cache(False)
    del model, unc
    torch.cuda.empty_cache()
    return {"config": cfg_name, "H": H, "W": W, "P": kw["P"], "times": times}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dino.py needs a GPU")
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        raise SystemExit("the reference python package is not present (oracle/_ref/py); run __graft_entry__.build() first")
    dev = torch.device("cuda:0")
    hooks = Hooks(m)
    res = device_info()
    print(json.dumps(res), flush=True)
    bb = sharpened_uncertainty_model(m, Config, "dino", dev).backbone
    hook = DinoHook(bb)
    for name, (H, W) in (("backbone_10769", (1092, 1932)), ("backbone_355", (196, 350))):
        res[name] = backbone_case(bb, hook, H, W, a.steps, a.rounds, dev)
        print(json.dumps({name: res[name]}), flush=True)
    del bb
    for N in (10769, 45420):
        res[f"attention_{N}"] = attention_case(N, 6, a.steps, a.rounds, dev)
        print(json.dumps({f"attention_{N}": res[f"attention_{N}"]}), flush=True)
    for name, (H, W), ref in (("C3", (1080, 1920), True), ("C5", (2160, 4096), False)):
        res[f"{name}_compute_losses"] = losses_case(m, Config, hooks, H, W, a.steps, a.rounds, dev, ref)
        print(json.dumps({f"{name}_compute_losses": res[f"{name}_compute_losses"]}), flush=True)
    for name, arms in (("C3", (False, True)), ("C5", (True,))):
        res[f"{name}_train_step"] = train_step_case(m, Config, hooks, name, arms, a.steps, a.rounds, dev)
        print(json.dumps({f"{name}_train_step": res[f"{name}_train_step"]}), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
