"""Uncertainty loss in ``dino`` mode: ``UncertaintyModel._compute_losses`` (wildgaussians/method.py:363-433, unmodified,
from oracle/_ref/py) as shipped, with ``enable(msssim=True, dino=True)``, and with ``uncertainty=True`` on top
(``fused_uncertainty``: the head and loss as kernels, a feature cache that hits).

    python tools/bench_uncertainty.py [--steps 5] [--rounds 5] [--out result.json]

Arms alternate round by round; medians over rounds with [min, max], device time (CUDA events) and host time:
  * ``_compute_losses`` + backward at C3 (1920x1080) and 4096x2160: as shipped (C3 only: at 4K the shipped backbone's
    dense attention needs 99 GB), ``msssim + dino``, ``+ uncertainty`` on a miss (no cache entry: three backbone calls),
    ``+ uncertainty`` on a hit (cache entry filled in the warm-up: one backbone call, the prediction at 350 px);
  * the train step of tools/bench_dino.py at C3 (fused caller, ``ssim``, ``msssim``, ``dino``) without and with
    ``uncertainty`` (its cache entry hits after the warm-up, as in training).
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

from bench_dino import DinoHook, sharpened_uncertainty_model  # noqa: E402
from bench_msssim import Hooks, run_arms, textured_pair  # noqa: E402
from bench_ssim import device_info  # noqa: E402


class UncertaintyHook:
    """Switches one uncertainty model's ``_compute_losses`` between the class's own and the fused path."""

    def __init__(self, model):
        self.probe = type("Probe", (), {})()
        self.probe.uncertainty_model = model

    def set(self, on):
        import wildgaussians_fused as wf
        if on:
            wf.enable(self.probe, optimizer=False, uncertainty=True)
        else:
            self.probe.uncertainty_model.__dict__.pop("_compute_losses", None)


def losses_case(m, Config, hooks, H, W, steps, rounds, dev, with_shipped):
    gt, pred = textured_pair(H, W, dev)
    model = sharpened_uncertainty_model(m, Config, "dino", dev)
    dino, unc = DinoHook(model.backbone), UncertaintyHook(model)

    def arm(fast, fused, entry):
        def run():
            hooks.set(msssim=fast)
            dino.set(fast)
            unc.set(fused)
            for p in model.parameters():
                p.grad = None
            loss, _, _ = model._compute_losses(gt, pred, _cache_entry=entry)
            loss.backward()
            unc.set(False)
            dino.set(False)
        return run

    arms = {"msssim_dino": arm(True, False, None), "uncertainty_miss": arm(True, True, None),
            "uncertainty_hit": arm(True, True, ("train", 0))}
    if with_shipped:
        arms = {"shipped": arm(False, False, None), **arms}
    try:
        times = run_arms(arms, steps, rounds, warmup=1)
    finally:
        hooks.restore()
    del model
    torch.cuda.empty_cache()
    return {"H": H, "W": W, "times": times}


def train_step_case(m, Config, hooks, cfg_name, steps, rounds, dev):
    """The train step of tools/bench_dino.py (method.py:1909-1966 with ``ssim``, ``msssim`` and ``dino`` on), without and
    with ``uncertainty``."""
    import synthetic
    import wg_harness as wh
    import wildgaussians_fused as wf
    import diff_gaussian_rasterization as ours
    kw = dict(synthetic.CONFIGS[cfg_name]); kw["seed"] = 0; kw["sh_degree"] = 3
    scene = synthetic.make_scene(**kw)
    model, cfg = wh.make_model(m, Config, scene, dev)
    unc_model = sharpened_uncertainty_model(m, Config, "dino", dev)
    dino, unc = DinoHook(unc_model.backbone), UncertaintyHook(unc_model)
    cam = wh.make_camera(scene)
    H, W = scene["image_height"], scene["image_width"]
    gt_image = torch.rand(3, H, W, generator=torch.Generator().manual_seed(5)).to(dev)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    ours._C.set_geometry_cache(True)
    wf.enable(model, optimizer=False)

    def step(fused):
        def run():
            hooks.set(ssim=True, msssim=True)
            dino.set(True)
            unc.set(fused)
            for p in list(model.parameters()) + list(unc_model.parameters()):
                p.grad = None
            embedding = model.appearance_embeddings[0]
            render_pkg = model._render_internal(cam, config=cfg, embedding=embedding, kernel_size=cfg.kernel_size)
            image_toned, image = render_pkg["render"], render_pkg["raw_render"]
            uncertainty_loss, metrics, loss_mult = unc_model.get_loss(gt_image, image_toned.detach(), _cache_entry=("train", 0))
            loss_mult = (loss_mult > 1).to(dtype=loss_mult.dtype)        # past the warm-up (method.py:1934-1940)
            Ll1 = torch.nn.functional.l1_loss(image_toned, gt_image, reduction="none")
            ssim_value = m.ssim(image, gt_image, size_average=False)
            loss = ((1.0 - cfg.lambda_dssim) * (Ll1 * loss_mult).mean() +
                    cfg.lambda_dssim * ((1.0 - ssim_value) * loss_mult).mean() + uncertainty_loss)
            loss.backward()
            unc.set(False)
            dino.set(False)
        return run

    try:
        times = run_arms({"train_step_msssim_dino": step(False), "train_step_uncertainty": step(True)}, steps, rounds,
                         warmup=1)
    finally:
        hooks.restore()
        wf.disable(model)
        ours._C.set_geometry_cache(False)
    del model, unc_model
    torch.cuda.empty_cache()
    return {"config": cfg_name, "H": H, "W": W, "P": kw["P"], "times": times}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_uncertainty.py needs a GPU")
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        raise SystemExit("the reference python package is not present (oracle/_ref/py); run __graft_entry__.build() first")
    dev = torch.device("cuda:0")
    hooks = Hooks(m)
    res = device_info()
    print(json.dumps(res), flush=True)
    for name, (H, W), shipped in (("C3", (1080, 1920), True), ("4K", (2160, 4096), False)):
        res[f"{name}_compute_losses"] = losses_case(m, Config, hooks, H, W, a.steps, a.rounds, dev, shipped)
        print(json.dumps({f"{name}_compute_losses": res[f"{name}_compute_losses"]}), flush=True)
    res["C3_train_step"] = train_step_case(m, Config, hooks, "C3", a.steps, a.rounds, dev)
    print(json.dumps({"C3_train_step": res["C3_train_step"]}), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
