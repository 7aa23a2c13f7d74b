"""Uncertainty loss in the modes ``fused_uncertainty`` does not take: ``UncertaintyModel._compute_losses``
(wildgaussians/method.py:363-433, unmodified, from oracle/_ref/py) in ``l2reg``, ``l1reg`` and ``dino+mssim`` mode, and the
evaluation-mode ``get_loss(gt, gt)`` that ``optimize_embedding`` makes (method.py:1781-1785).

    python tools/bench_uncertainty_modes.py [--steps 5] [--rounds 5] [--out result.json]

Arms alternate round by round; medians over rounds with [min, max], device time (CUDA events) and host time:
  * ``_compute_losses`` + backward per mode at C3 (1920x1080) and 4096x2160: as shipped (C3 only: at 4K the shipped
    backbone's dense attention needs 99 GB), with ``enable(msssim=True, dino=True, uncertainty=True)`` (which falls
    back to the class's method for these modes), and with ``uncertainty_modes=True`` on top on a miss (no cache entry)
    and on a hit (cache entry filled in the warm-up);
  * ``get_loss(gt, gt)`` in evaluation mode under ``torch.enable_grad()`` (no backward, as ``optimize_embedding``) in
    ``dino`` mode (the default configuration) and ``l2reg`` mode, the same arms without the cache entry (the reference
    passes none).
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


class ModesHook:
    """Switches one uncertainty model's ``_compute_losses`` between the class's own, ``enable(uncertainty=True)`` and
    ``enable(uncertainty=True, uncertainty_modes=True)``."""

    def __init__(self, model):
        self.probe = type("Probe", (), {})()
        self.probe.uncertainty_model = model

    def set(self, uncertainty=False, modes=False):
        import wildgaussians_fused as wf
        um = self.probe.uncertainty_model
        um.__dict__.pop("_compute_losses", None)
        um.__dict__.pop(wf._MODES_MARK, None)
        if uncertainty or modes:
            wf.enable(self.probe, optimizer=False, uncertainty=uncertainty, uncertainty_modes=modes)


def case(m, Config, hooks, mode, H, W, steps, rounds, dev, with_shipped, evaluation):
    gt, pred = textured_pair(H, W, dev)
    model = sharpened_uncertainty_model(m, Config, mode, dev)
    model.train(not evaluation)
    dino, unc = DinoHook(model.backbone), ModesHook(model)

    def arm(fast, fused, modes, entry):
        def run():
            hooks.set(msssim=fast)
            dino.set(fast)
            unc.set(fused, modes)
            for p in model.parameters():
                p.grad = None
            if evaluation:
                with torch.enable_grad():
                    model.get_loss(gt[0], gt[0])
            else:
                loss, _, _ = model._compute_losses(gt, pred, _cache_entry=entry)
                loss.backward()
            unc.set()
            dino.set(False)
        return run

    arms = {"msssim_dino_uncertainty": arm(True, True, False, None), "modes_miss": arm(True, True, True, None)}
    if not evaluation:
        arms["modes_hit"] = arm(True, True, True, ("train", 0))
    if with_shipped:
        arms = {"shipped": arm(False, False, False, None), **arms}
    try:
        times = run_arms(arms, steps, rounds, warmup=1)
    finally:
        hooks.restore()
    del model
    torch.cuda.empty_cache()
    return {"mode": mode, "eval": evaluation, "H": H, "W": W, "times": times}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_uncertainty_modes.py needs a GPU")
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        raise SystemExit("the reference python package is not present (oracle/_ref/py); run __graft_entry__.build() first")
    dev = torch.device("cuda:0")
    hooks = Hooks(m)
    res = device_info()
    print(json.dumps(res), flush=True)
    runs = [(mode, False) for mode in ("l2reg", "l1reg", "dino+mssim")] + [("dino", True), ("l2reg", True)]
    for name, (H, W), shipped in (("C3", (1080, 1920), True), ("4K", (2160, 4096), False)):
        for mode, evaluation in runs:
            key = f"{name}_{mode}_{'eval_get_loss' if evaluation else 'compute_losses'}"
            res[key] = case(m, Config, hooks, mode, H, W, a.steps, a.rounds, dev, shipped, evaluation)
            print(json.dumps({key: res[key]}), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
