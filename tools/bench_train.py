"""Whole ``WildGaussians.train_iteration`` per step on ordinary (non-densifying) steps, three arms alternated in rounds:

  shipped      the reference's ``train_iteration`` on the drop-in rasterizer
  fused        ``enable_method(method, ssim=True, msssim=True, dino=True, uncertainty=True)``
  fused_train  the same with ``train=True`` (``fused_train.train_iteration``)

Scenes S1 (150 k Gaussians, 640x400) and C3 (3 M, 1920x1080), each with the uncertainty model (``dino`` mode, the
random-weight ViT-S of tools/bench_dino.py) in two configurations: appearance on (the default preset) and appearance off
(NeRF On-the-go).  ``--cameras`` training cameras and images (a first epoch visits every camera, so every
feature-cache entry is warm before timing); the steps are past ``densify_until_iter`` and avoid every 100th iteration
(3D-filter recomputation), so no step densifies, resets the opacity or raises the SH degree.  Each step ends in its
metric read-back, so the host clock times it.  Also reported: the one-time staging of the training images at the first
fused call (the byte-exactness check and the uint8 copies), and the host time per step of filling the pinned slot and
enqueueing the copy (``upload``).  A separate profiler run per arm counts the synchronising runtime calls per step and
the device's idle time between kernels over three steps.

    python tools/bench_train.py [--scenes S1,C3] [--cameras 4] [--rounds 5] [--steps 10] [--out results.json]
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

from bench_dino import SHARPEN  # noqa: E402
from bench_ssim import device_info  # noqa: E402

SCENES = {"S1": dict(P=150_000, W=640, H=400, seed=5), "C3": dict(P=3_000_000, W=1920, H=1080, seed=3)}
FIRST_STEP = 20_000          # iteration 20 001: past densify_until_iter (15 000) and the uncertainty warm-up
SYNC_CALLS = ("cudaStreamSynchronize", "cudaEventSynchronize", "cudaMemcpy")     # the profiler itself calls cudaDeviceSynchronize


def steps_from(start, n):
    """n steps from `start` whose iteration (step + 1) is not a multiple of 100."""
    out, s = [], start
    while len(out) < n:
        if (s + 1) % 100:
            out.append(s)
        s += 1
    return out


def build(scene_name, appearance, dev, cameras):
    import synthetic
    import wg_harness as wh
    import wg_train
    import diff_gaussian_rasterization as ours
    m, Config = wh.import_method()
    if m is None:
        raise SystemExit("reference python package not present (oracle/_ref/py): run __graft_entry__.build() first")
    sc = SCENES[scene_name]
    scene = synthetic.to_device(synthetic.make_scene(sc["P"], sc["W"], sc["H"], sh_degree=3, seed=sc["seed"]), dev)
    method = wg_train.make_method(m, Config, scene, dev, uncertainty=True, appearance=appearance, n_cameras=cameras)
    with torch.no_grad():
        for blk in method.model.uncertainty_model.backbone.blocks:
            C = blk.attn.qkv.in_features
            blk.attn.qkv.weight[:2 * C] *= SHARPEN
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    return method


def set_arm(method, arm):
    import wildgaussians_fused as wf
    wf.disable_method(method)
    if arm != "shipped":
        wf.enable_method(method, train=(arm == "fused_train"), ssim=True, msssim=True, dino=True, uncertainty=True)


def run_steps(method, steps):
    for s in steps:
        method.train_iteration(s)


def profile_arm(method, steps):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run_steps(method, steps)
        torch.cuda.synchronize()
    evs = prof.events()
    syncs = sum(e.name in SYNC_CALLS for e in evs)
    pageable = sum("Pageable" in e.name and "HtoD" in e.name for e in evs)
    busy = sorted((e.time_range.start, e.time_range.end) for e in evs
                  if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.end > e.time_range.start)
    idle, end = 0.0, None
    for a, b in busy:
        if end is not None and a > end:
            idle += a - end
        end = b if end is None else max(end, b)
    return {"syncs_per_step": syncs / len(steps), "pageable_h2d_per_step": pageable / len(steps),
            "device_idle_ms_per_step": idle / 1000.0 / len(steps)}


class UploadClock:
    """Host seconds spent in ``fused_train._Stager.upload`` (filling a pinned slot, enqueueing its copy), and whether
    the compute stream still had the previous step's work (densification statistics, Adam) queued when it returned:
    if so, the device did not wait for the host's copy."""

    def __init__(self):
        import fused_train
        self.cls, self.orig, self.samples, self.busy = fused_train._Stager, fused_train._Stager.upload, [], []
        clock = self

        def timed(stager, cid):
            t0 = time.perf_counter()
            out = clock.orig(stager, cid)
            clock.samples.append(time.perf_counter() - t0)
            clock.busy.append(not torch.cuda.current_stream(stager.device).query())
            return out
        self.cls.upload = timed

    def restore(self):
        self.cls.upload = self.orig


def case(scene_name, appearance, rounds, n_steps, cameras, dev):
    import fused_train
    method = build(scene_name, appearance, dev, cameras)
    arms = ("shipped", "fused", "fused_train")
    random.seed(0)
    torch.manual_seed(0)
    step_iter = iter(steps_from(FIRST_STEP, 100_000))
    take = lambda n: [next(step_iter) for _ in range(n)]
    t0 = time.perf_counter()
    fused_train._stager(method, dev)                                # what the first fused call does once
    staging_s = time.perf_counter() - t0
    # warm-up: one epoch on a fused arm visits every camera (feature cache filled), then every arm
    set_arm(method, "fused")
    run_steps(method, take(cameras))
    for arm in arms:
        set_arm(method, arm)
        run_steps(method, take(8))
    clock = UploadClock()
    times = {a: [] for a in arms}
    for _ in range(rounds):
        for arm in arms:
            set_arm(method, arm)
            run_steps(method, take(1))
            steps = take(n_steps)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run_steps(method, steps)
            torch.cuda.synchronize()
            times[arm].append((time.perf_counter() - t0) * 1000.0 / n_steps)
    clock.restore()
    prof = {}
    for arm in arms:
        set_arm(method, arm)
        run_steps(method, take(2))
        prof[arm] = profile_arm(method, take(3))
    set_arm(method, "shipped")
    P = len(method.model.xyz)
    del method
    torch.cuda.empty_cache()
    return {"scene": scene_name, "appearance": appearance, "P": P, "cameras": cameras,
            "staging_s_once": staging_s, "upload_host_ms_per_step": 1000.0 * statistics.median(clock.samples),
            "device_busy_after_upload": sum(clock.busy) / len(clock.busy),
            "ms_per_step": {a: {"median": statistics.median(t), "min": min(t), "max": max(t)} for a, t in times.items()},
            "profile": prof}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--scenes", default="S1,C3")
    ap.add_argument("--cameras", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train needs a GPU")
    dev = torch.device("cuda:0")
    res = {"device": device_info(), "rounds": args.rounds, "steps_per_round": args.steps, "cases": []}
    for name in args.scenes.split(","):
        for appearance in (True, False):
            r = case(name, appearance, args.rounds, args.steps, args.cameras, dev)
            res["cases"].append(r)
            print(json.dumps(r), flush=True)
    print(json.dumps(res["device"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
