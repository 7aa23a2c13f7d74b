"""Resident against staged training data in the fused training iteration, per ordinary step, two arms alternated in
rounds on two identically seeded methods:

  staged    ``enable_method(method, train=True, ssim=True, msssim=True, dino=True, uncertainty=True)``
  resident  the same with ``resident=True``: images as device bytes, device feature cache

The setup is that of tools/bench_train.py (appearance on, uncertainty ``dino``, the random-weight ViT-S): S1 (150 k
Gaussians, 640x400) with 300 cameras and C3 (3 M, 1920x1080) with 100, so the data stays far above one camera's worth.
A first epoch on each arm visits every camera (feature cache filled), then steps past ``densify_until_iter`` that
avoid every 100th iteration are timed by the host clock (each step ends in its metric read-back).  Reported: median
[min, max] ms per step over the rounds, the device's idle time per step and the host-to-device copies per step from a
separate profiler run, and the first-call start-up of each arm (the host byte check of every image, or the device
store's upload, check and pack) with the card's name and power limit read in the same process.

    python tools/bench_resident.py [--scenes S1,C3] [--rounds 5] [--steps 10] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "wild-gaussians_b200"), ROOT, os.path.join(ROOT, "tests"), os.path.dirname(__file__)):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_ssim import device_info  # noqa: E402
from bench_train import FIRST_STEP, build, profile_arm, run_steps, steps_from  # noqa: E402

CAMERAS = {"S1": 300, "C3": 100}
FLAGS = dict(train=True, ssim=True, msssim=True, dino=True, uncertainty=True)


def startup_s(method, arm, dev):
    """Seconds of the one-time data preparation the arm's first step makes."""
    import fused_train
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if arm == "resident":
        fused_train._resident(method, dev)
    else:
        fused_train._stager(method, dev)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def case(scene_name, rounds, n_steps, dev):
    import wildgaussians_fused as wf
    cameras = CAMERAS[scene_name]
    methods, startup = {}, {}
    for arm in ("staged", "resident"):
        torch.manual_seed(0)
        methods[arm] = m = build(scene_name, True, dev, cameras)
        wf.enable_method(m, resident=(arm == "resident"), **FLAGS)
        startup[arm] = startup_s(m, arm, dev)
    step_iter = {a: iter(steps_from(FIRST_STEP, 100_000)) for a in methods}
    take = lambda a, n: [next(step_iter[a]) for _ in range(n)]
    random.seed(0)
    for arm, m in methods.items():                      # one epoch: every camera drawn, every feature cached
        run_steps(m, take(arm, cameras))
    times = {a: [] for a in methods}
    for _ in range(rounds):
        for arm, m in methods.items():
            run_steps(m, take(arm, 1))
            steps = take(arm, n_steps)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run_steps(m, steps)
            torch.cuda.synchronize()
            times[arm].append((time.perf_counter() - t0) * 1000.0 / n_steps)
    prof = {}
    for arm, m in methods.items():
        run_steps(m, take(arm, 2))
        prof[arm] = profile_arm(m, take(arm, 3))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as p:
            run_steps(m, take(arm, 3))
            torch.cuda.synchronize()
        prof[arm]["h2d_copies_per_step"] = sum("HtoD" in e.name for e in p.events()) / 3
    resident = methods["resident"]
    import fused_train
    store = fused_train._stores[resident]
    cache = resident.model.uncertainty_model._images_cache
    held = {"images_resident": len(store.entries), "images_staged": len(store.staged),
            "store_mb": sum(e.img.nbytes + (0 if e.mask is None else e.mask.nbytes) for e in store.entries.values()) / 2**20,
            "features_on_device": sum(v.is_cuda for v in cache.values()), "features_on_host": sum(not v.is_cuda for v in cache.values()),
            "features_mb": sum(v.nbytes for v in cache.values() if v.is_cuda) / 2**20}
    for m in methods.values():
        wf.disable_method(m)
    del methods, resident, store, cache
    torch.cuda.empty_cache()
    return {"scene": scene_name, "cameras": cameras, "startup_s": startup, "held": held,
            "ms_per_step": {a: {"median": statistics.median(t), "min": min(t), "max": max(t)} for a, t in times.items()},
            "profile": prof}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--scenes", default="S1,C3")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resident needs a GPU")
    dev = torch.device("cuda:0")
    res = {"device": device_info(), "rounds": args.rounds, "steps_per_round": args.steps, "cases": []}
    for name in args.scenes.split(","):
        r = case(name, args.rounds, args.steps, dev)
        res["cases"].append(r)
        print(json.dumps(r), flush=True)
    res["device_after"] = device_info()
    print(json.dumps(res["device"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
