"""Inference render (``WildGaussians.render``, wildgaussians/method.py:1832-1866; once per evaluation image, video frame and
viewer frame): as shipped, with the fused caller, and with the fused render.

    python tools/bench_render.py [--scenes S1,C3] [--calls N] [--rounds R] [--out F]

Arms, alternating round by round, each timed over whole ``render`` calls with the host clock (the call returns numpy
arrays, so it ends synchronised):
  * ``shipped``: the unmodified method (oracle/_ref/py) on the drop-in rasterizer;
  * ``enable``: the same after ``wildgaussians_fused.enable_method(method)``;
  * ``render``: after ``enable_method(method, render=True)`` (``fused_render.render``).
Cases: S1 (150 k Gaussians, 640x400) and C3 (3 M, 1920x1080) from ``synthetic.make_scene``, appearance on and off, depth
off and on.  Per case: median and spread of the call time per arm, whether ``render`` equals ``enable`` bit for bit (colour,
accumulation) and its largest depth difference against the largest visible distance, device-to-host bytes per call from
the shapes.  A separate ``torch.profiler`` run per arm gives per-kernel device times, the device-side copies (kind and
count) and the synchronising calls of one call.  For context, one NeRF-W protocol image (optimise the embedding, render,
metrics with LPIPS stubbed) with every fused path on.  Prints the card name and its power limit / max SM clock
(nvidia-smi, query only).  Needs a GPU; does not fall back.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "wild-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_ssim import device_info  # noqa: E402

SCENES = {"S1": dict(P=150_000, W=640, H=400, seed=5), "C3": dict(P=3_000_000, W=1920, H=1080, seed=3)}
ARMS = ("shipped", "enable", "render")
SYNC_CALLS = ("cudaStreamSynchronize", "cudaEventSynchronize", "cudaDeviceSynchronize", "cudaMemcpy")


def make_method(m, Config, sc, appearance):
    import synthetic
    import wg_train
    scene = synthetic.make_scene(sc["P"], sc["W"], sc["H"], sh_degree=3, seed=sc["seed"])
    return wg_train.make_method(m, Config, scene, torch.device("cuda:0"), appearance=appearance, seed=sc["seed"])


def camera(m, method, i=0):
    from wildgaussians.types import new_cameras
    c = method.train_cameras[i]
    return new_cameras(poses=c.poses[None].astype(np.float32), intrinsics=c.intrinsics[None].astype(np.float32),
                       camera_models=np.array([m.camera_model_to_int("pinhole")], np.int32),
                       distortion_parameters=np.zeros((1, 0), np.float32), image_sizes=c.image_sizes[None])


def arm_call(m, method, arm):
    import wildgaussians_fused as wf
    wf.disable_method(method)
    if arm == "shipped":
        return lambda cam, options: m.WildGaussians.render(method, cam, options)
    wf.enable_method(method, render=(arm == "render"))
    return lambda cam, options: method.render(cam, options)


def profile_call(fn, cam, options):
    from torch.profiler import ProfilerActivity, profile
    fn(cam, options)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn(cam, options)
    kernels, copies = collections.defaultdict(float), collections.Counter()
    syncs = collections.Counter()
    for e in prof.events():
        if e.name in SYNC_CALLS:
            syncs[e.name] += 1
        if e.device_type == torch.autograd.DeviceType.CUDA:
            t = getattr(e, "device_time", None)
            t = e.cuda_time if t is None else t
            if e.name.startswith("Memcpy") or e.name.startswith("Memset"):
                copies[e.name] += 1
            else:
                kernels[e.name[:90]] += t / 1000.0
    top = sorted(kernels.items(), key=lambda kv: -kv[1])
    return {"kernels_ms": {k: round(v, 4) for k, v in top[:14]}, "kernel_total_ms": round(sum(kernels.values()), 4),
            "copies": dict(copies), "sync_calls": dict(syncs)}


def run_case(m, Config, name, sc, appearance, calls, rounds):
    import fused_render as fr
    import wildgaussians_fused as wf
    method = make_method(m, Config, sc, appearance)
    cam = camera(m, method)
    res = {"case": name, "P": sc["P"], "W": sc["W"], "H": sc["H"], "appearance": appearance}
    emb = np.linspace(-0.5, 0.5, 32).astype(np.float32)
    for depth in (False, True):
        options = {"embedding": emb, "outputs": ("color", "depth") if depth else ("color",)}
        times = {a: [] for a in ARMS}
        for a in ARMS:                                   # warm-up: modules, camera constants, allocator pools
            fn = arm_call(m, method, a)
            for _ in range(3):
                fn(cam, options)
        for _ in range(rounds):
            for a in ARMS:
                fn = arm_call(m, method, a)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(calls):
                    fn(cam, options)
                times[a].append((time.perf_counter() - t0) * 1000.0 / calls)
        ref = arm_call(m, method, "enable")(cam, options)
        ours = arm_call(m, method, "render")(cam, options)
        wf.disable_method(method)
        HW = sc["W"] * sc["H"]
        row = {"ms_median": {a: round(statistics.median(v), 4) for a, v in times.items()},
               "ms_min_max": {a: [round(min(v), 4), round(max(v), 4)] for a, v in times.items()},
               "d2h_bytes_per_call": 4 * HW * (5 if depth else 4),
               "color_bitwise": bool(np.array_equal(ours["color"], ref["color"])),
               "accumulation_bitwise": bool(np.array_equal(ours["accumulation"], ref["accumulation"]))}
        row["speedup_vs_enable"] = round(row["ms_median"]["enable"] / row["ms_median"]["render"], 3)
        row["speedup_vs_shipped"] = round(row["ms_median"]["shipped"] / row["ms_median"]["render"], 3)
        if depth:
            model = method.model
            cc = wf._camera_constants(sys.modules[type(model).__module__], cam.item(), model.xyz.device)
            with torch.no_grad():
                radii = wf.render_internal(model, cam.item(), method.config, kernel_size=method.config.kernel_size,
                                           embedding=model.get_embedding(None), return_raw=False)["radii"]
                dmax = float(torch.norm(model.xyz - cc["cam_center"][None], dim=-1)[radii > 0].max())
            row["depth_bitwise"] = bool(np.array_equal(ours["depth"], ref["depth"]))
            row["depth_max_abs_diff"] = float(np.abs(ours["depth"].astype(np.float64) - ref["depth"]).max())
            row["depth_rel_to_max_visible_distance"] = row["depth_max_abs_diff"] / dmax
        row["profile"] = {a: profile_call(arm_call(m, method, a), cam, options) for a in ARMS}
        wf.disable_method(method)
        assert fr.supported(method, cam, options)
        res["depth" if depth else "no_depth"] = row
    del method
    torch.cuda.empty_cache()
    return res


def nerfw_image(m, Config, sc):
    """One NeRF-W protocol image at this case with every fused path on (embedding, render, metrics; LPIPS stubbed)."""
    import wildgaussians.evaluation as ev
    import wildgaussians_fused as wf
    from wildgaussians.datasets.phototourism import NerfWEvaluationProtocol

    class ZeroLPIPS(torch.nn.Module):
        def forward(self, a, b):
            return a.new_zeros((a.shape[0], 1, 1, 1))

    ev._LPIPS_CACHE["alex"] = ZeroLPIPS()
    method = make_method(m, Config, sc, True)
    method.config.appearance_optim_type = "dssim+l1"
    gt = np.clip(method.train_images[2].permute(1, 2, 0).numpy(), 0, 1)
    ds = {"cameras": camera(m, method, 2), "images": [gt], "masks": None, "metadata": {"color_space": "srgb"}}
    wf.enable_method(method, render=True, ssim=True)
    wf.enable_metrics(ev)
    proto = NerfWEvaluationProtocol()
    out = {}
    try:
        for i in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pred = proto.render(method, ds)
            t1 = time.perf_counter()
            metrics = proto.evaluate(pred, ds)
            t2 = time.perf_counter()
            if i == 2:
                out = {"optimize_and_render_ms": round((t1 - t0) * 1000, 3), "metrics_ms": round((t2 - t1) * 1000, 3),
                       "psnr": float(metrics["psnr"])}
    finally:
        wf.disable_metrics(ev)
        wf.disable_method(method)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="S1,C3")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_render.py needs a GPU"
    import wg_harness as wh
    m, Config = wh.import_method()
    assert m is not None, "the reference package (oracle/_ref/py) is needed for the shipped arm"
    import diff_gaussian_rasterization as ours
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    result = {"device": device_info(), "cases": []}
    print(json.dumps(result["device"]), flush=True)
    for name in args.scenes.split(","):
        for appearance in (True, False):
            r = run_case(m, Config, name, SCENES[name], appearance, args.calls, args.rounds)
            print(json.dumps(r), flush=True)
            result["cases"].append(r)
    result["nerfw_image_C3"] = nerfw_image(m, Config, SCENES["C3"]) if "C3" in args.scenes else None
    print(json.dumps({"nerfw_image_C3": result["nerfw_image_C3"]}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
