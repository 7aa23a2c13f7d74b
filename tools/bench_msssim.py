"""Image-quality statistics of the uncertainty loss: the reference's ``msssim`` + ``ssim_down`` (wildgaussians/method.py:
126-187, unmodified, from oracle/_ref/py) against ``fused_ssim.msssim`` / ``fused_ssim.ssim_down`` (csrc/msssim.cu).

    python tools/bench_msssim.py [--steps 20] [--rounds 5] [--train-steps 10] [--out result.json]

Per image size (C3 1920x1080, C5 4096x2160), arms alternating round by round, medians over rounds:
  * one step = ``ssim_down(gt, pred, max_size=400)`` + ``msssim(gt, pred, max_size=400, min_size=80)`` (method.py:368-369):
    the reference as shipped, the reference with ``enable(model, ssim=True)`` only (``ssim_down`` then runs the fused SSIM),
    and both fused.  Device time (CUDA events) and host wall time (perf_counter around the steps, ended by a
    synchronise: the reference's window copies block the host);
  * at C3, ``UncertaintyModel._compute_losses`` (method.py:363-433, random-weight backbone, offline) in ``dino`` and
    ``l2reg`` modes, reference against ``enable(model, msssim=True)``;
  * the fused results' error against the float64 oracle and the reference's own fp32 error (TF32 off).
At C3 also the train-step statements method.py:1909-1966 with the uncertainty model on (``dino``): the
tests/wg_harness.py model with the fused caller and ``ssim=True``, with and without ``msssim=True``.
Prints the device name and its power limit / max SM clock (nvidia-smi, query only).  Needs a GPU; does not fall back.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "wild-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_ssim import SIZES, device_info, summary  # noqa: E402


def time_both(fn, steps):
    """(device ms, host ms) per call over `steps` calls: CUDA events, and a host clock ended by a synchronise."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    host = (time.perf_counter() - t0) * 1e3 / steps
    return a.elapsed_time(b) / steps, host


def run_arms(arms, steps, rounds, warmup=3):
    """{name: {"device": [...], "host": [...]}} with the arms alternating inside every round."""
    out = {name: {"device": [], "host": []} for name in arms}
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for name, fn in arms.items():
            d, h = time_both(fn, steps)
            out[name]["device"].append(d)
            out[name]["host"].append(h)
    return {name: {k: summary(v) for k, v in t.items()} for name, t in out.items()}


class Hooks:
    """Switches the method module's ``ssim`` / ``msssim`` / ``ssim_down`` between the originals and the fused wrappers."""

    def __init__(self, m):
        import wildgaussians_fused as wf
        self.m = m
        self.orig = (m.ssim, m.msssim, m.ssim_down)
        probe = type("Probe", (), {"__module__": m.__name__})()
        wf.enable(probe, optimizer=False, ssim=True, msssim=True)
        self.fused = (m.ssim, m.msssim, m.ssim_down)
        wf.disable(probe)

    def set(self, ssim=False, msssim=False):
        self.m.ssim = self.fused[0] if ssim else self.orig[0]
        self.m.msssim, self.m.ssim_down = (self.fused[1:] if msssim else self.orig[1:])

    def restore(self):
        self.set()


def textured_pair(H, W, dev, seed=1):
    g = torch.Generator(device=dev).manual_seed(seed)
    gt = torch.rand(1, 3, H // 8 + 1, W // 8 + 1, generator=g, device=dev)
    gt = torch.nn.functional.interpolate(gt, size=(H, W), mode="bilinear", align_corners=False)
    pred = (gt + 0.05 * torch.randn(1, 3, H, W, generator=g, device=dev)).clamp(0, 1)
    return gt, pred


def stats_case(m, Config, hooks, H, W, steps, rounds, dev, with_losses):
    import wg_uncertainty as wu
    from oracle import msssim_oracle
    gt, pred = textured_pair(H, W, dev)

    def stats(ssim, msssim):
        def run():
            hooks.set(ssim=ssim, msssim=msssim)
            with torch.no_grad():
                m.ssim_down(gt, pred, max_size=400)
                m.msssim(gt, pred, max_size=400, min_size=80)
        return run

    arms = {"stats_reference": stats(False, False), "stats_ssim_only": stats(True, False), "stats_fused": stats(True, True)}
    res = {"H": H, "W": W, "steps_per_round": steps, "rounds": rounds, "times": run_arms(arms, steps, rounds)}
    # the DINO backbone runs at full resolution (uncertainty_dino_max_size is None by default): 4K is left out
    models = {mode: wu.make_uncertainty_model(m, Config, mode, dev, seed=3)[0] for mode in (("dino", "l2reg") if with_losses else ())}

    def losses(mode, fused):
        def run():
            hooks.set(msssim=fused)
            wu.compute_losses(models[mode], gt[0], pred[0], seed=5)
        return run

    arms = {f"compute_losses_{mode}_{'fused' if f else 'reference'}": losses(mode, f) for mode in models for f in (False, True)}
    if arms:
        res["times"].update(run_arms(arms, max(2, steps // 4), rounds, warmup=2))
    hooks.restore()
    torch.backends.cudnn.allow_tf32 = False
    want = (msssim_oracle.msssim(gt, pred, 400, 80), msssim_oracle.ssim_down(gt, pred, 400))
    err = {}
    for arm, msssim in (("reference_fp32", False), ("fused", True)):
        hooks.set(msssim=msssim)
        got = (m.msssim(gt, pred, max_size=400, min_size=80), m.ssim_down(gt, pred, max_size=400))
        err[arm] = {name: {"max_abs": float((g.double() - w).abs().max()), "mean_abs": abs(float(g.double().mean() - w.mean()))}
                    for name, g, w in zip(("msssim", "ssim_down"), got, want)}
    hooks.restore()
    torch.backends.cudnn.allow_tf32 = True
    res["error_vs_fp64_oracle"] = err
    del models, want
    torch.cuda.empty_cache()
    return res


def train_step_case(m, Config, hooks, steps, rounds, dev):
    """C3: method.py:1909-1966 with the uncertainty model (dino) on the wg_harness model with the fused caller."""
    import synthetic
    import wg_harness as wh
    import wg_uncertainty as wu
    import wildgaussians_fused as wf
    import diff_gaussian_rasterization as ours
    kw = dict(synthetic.CONFIGS["C3"]); kw["seed"] = 0; kw["sh_degree"] = 3
    scene = synthetic.make_scene(**kw)
    model, cfg = wh.make_model(m, Config, scene, dev)
    unc, _ = wu.make_uncertainty_model(m, Config, "dino", dev, seed=3)
    cam = wh.make_camera(scene)
    H, W = scene["image_height"], scene["image_width"]
    gt_image = torch.rand(3, H, W, generator=torch.Generator().manual_seed(5)).to(dev)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    ours._C.set_geometry_cache(True)
    wf.enable(model, optimizer=False)

    def step(msssim):
        def run():
            hooks.set(ssim=True, msssim=msssim)
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
        return run

    try:
        times = run_arms({"train_step_ssim": step(False), "train_step_ssim_msssim": step(True)}, steps, rounds, warmup=2)
    finally:
        hooks.restore()
        wf.disable(model)
        ours._C.set_geometry_cache(False)
    res = {"what": "wg_harness GaussianModel (C3: P=3M, 1920x1080, SH 3, appearance on) with the fused caller and ssim=True, "
                   "UncertaintyModel 'dino' (random ViT-S/14 weights): method.py:1909-1966 + backward; ms per step",
           "P": kw["P"], "times": times}
    res["difference_device_ms"] = (times["train_step_ssim"]["device"]["median_ms"] -
                                   times["train_step_ssim_msssim"]["device"]["median_ms"])
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--train-steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_msssim.py needs a GPU")
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        raise SystemExit("the reference python package is not present (oracle/_ref/py); run __graft_entry__.build() first")
    dev = torch.device("cuda:0")
    hooks = Hooks(m)
    res = device_info()
    for name, (H, W) in SIZES.items():
        res[name] = stats_case(m, Config, hooks, H, W, a.steps, a.rounds, dev, with_losses=name == "C3")
        print(json.dumps({name: res[name]}), flush=True)
    res["C3_train_step"] = train_step_case(m, Config, hooks, a.train_steps, a.rounds, dev)
    print(json.dumps({"C3_train_step": res["C3_train_step"]}), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
