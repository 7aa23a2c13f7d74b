"""Test-time appearance optimisation (``optimize_embedding``, wildgaussians/method.py:1755-1830, 128 Adam iterations on
the image embedding per test image): the unmodified method against ``fused_embedding``.

    python tools/bench_embedding.py [--rounds 5] [--iters 128] [--scenes C3,S1] [--out result.json] [--trace-dir DIR]

Arms, alternating round by round, each timed over a whole call (host clock ending in a device synchronise):
  * ``reference``: ``WildGaussians.optimize_embedding`` as shipped (oracle/_ref/py) on the drop-in rasterizer;
  * ``reference+enable``: the same with ``wildgaussians_fused.enable(model, ssim=True)`` (fused caller and SSIM);
  * ``fused``: ``fused_embedding.optimize_embedding``.
Scenes: C3 (3 M Gaussians, 1920x1080) and S1 (150 k, 640x400), both from ``synthetic.make_scene``; the target image is
the render at another training embedding, the start embedding is zero, the loss is the default ``dssim+l1-scaled``
with a mask and no uncertainty model.  Reports per arm the median and spread of the call time, ms per iteration, the
final PSNR and V/P.  A separate ``torch.profiler`` run of the fused arm gives per-kernel device times of one iteration
and the number of device-to-host copies between the first and the last iteration (expected 0).  Prints the device
name and its power limit / max SM clock (nvidia-smi, query only).  Needs a GPU; does not fall back.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "wild-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_ssim import device_info  # noqa: E402

SCENES = {"C3": dict(P=3_000_000, W=1920, H=1080, seed=3), "S1": dict(P=150_000, W=640, H=400, seed=5)}


def make_case(m, Config, name, iters):
    import diff_gaussian_rasterization as ours
    import synthetic
    import wg_harness as wh
    import wildgaussians_fused as wf
    kw = SCENES[name]
    dev = torch.device("cuda:0")
    scene = synthetic.make_scene(kw["P"], kw["W"], kw["H"], sh_degree=3, seed=kw["seed"])
    model, cfg = wh.make_model(m, Config, scene, dev, seed=kw["seed"])
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    cfg.appearance_embedding_optim_iters = iters
    cam = wh.make_camera(scene)
    cam.camera_models = m.camera_model_to_int("pinhole")
    cam.item = lambda: cam
    with torch.no_grad():
        gt = wf.render_internal(model, cam, cfg, kernel_size=cfg.kernel_size, embedding=model.appearance_embeddings[1],
                                return_raw=False)["render"]
    mask = np.ones((kw["H"], kw["W"]), dtype=np.float32)
    mask[: kw["H"] // 4] = 0.0
    ds = {"cameras": cam, "images": [gt.clamp(0, 1).permute(1, 2, 0).cpu().numpy().astype(np.float32)], "masks": [mask]}
    return model, cfg, ds


def arms(m, model, cfg):
    import fused_embedding as fe
    import wildgaussians_fused as wf
    ns = types.SimpleNamespace(model=model, config=cfg)

    def reference(ds):
        wf.disable(model)
        out = m.WildGaussians.optimize_embedding(ns, ds)
        for p in model.parameters():
            p.grad = None
        return out

    def reference_enable(ds):
        wf.enable(model, optimizer=False, ssim=True)
        try:
            out = m.WildGaussians.optimize_embedding(ns, ds)
        finally:
            wf.disable(model)
        for p in model.parameters():
            p.grad = None
        return out

    def fused(ds):
        return fe.optimize_embedding(ns, ds)

    return {"reference": reference, "reference+enable": reference_enable, "fused": fused}


def timed(fn, ds):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn(ds)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def profile_fused(model, cfg, ds, trace_dir):
    """Per-kernel device time of one fused iteration (the middle one of the call) and the device-to-host copies
    between the first and the last iteration."""
    import fused_embedding as fe
    from torch.profiler import ProfilerActivity, profile, record_function
    ns = types.SimpleNamespace(model=model, config=cfg)
    loop = fe.EmbeddingLoop(ns, ds)
    torch.cuda.synchronize()
    mid = loop.iters // 2
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(loop.iters):
            if i == mid:
                torch.cuda.synchronize()              # the window holds this iteration's kernels only
                with record_function("one_iteration"):
                    loop.step(i)
                    torch.cuda.synchronize()
            else:
                loop.step(i)
        torch.cuda.synchronize()
    loop.result()
    if trace_dir:
        os.makedirs(trace_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(trace_dir, "fused_embedding_trace.json"))
    events = prof.events()
    win = [e for e in events if e.name == "one_iteration"]
    t0, t1 = (win[0].time_range.start, win[0].time_range.end) if win else (None, None)
    kernels, d2h = {}, 0
    for e in events:
        dt = getattr(e, "device_type", None)
        if dt is None or "CUDA" not in str(dt):
            continue
        if "Memcpy DtoH" in e.name or "Memcpy D2H" in e.name:
            d2h += 1
        if t0 is not None and t0 <= e.time_range.start <= t1 and e.name != "one_iteration":
            kernels[e.name] = kernels.get(e.name, 0.0) + e.time_range.elapsed_us() / 1e3
    top = dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:16])
    return {"iteration_kernels_ms": {k[:90]: round(v, 4) for k, v in top.items()},
            "iteration_device_ms_total": round(sum(kernels.values()), 4), "d2h_copies_during_loop": d2h}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=128)
    ap.add_argument("--scenes", default="S1,C3")
    ap.add_argument("--out", default=None)
    ap.add_argument("--trace-dir", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_embedding needs a GPU"
    import wg_harness as wh
    m, Config = wh.import_method()
    assert m is not None, "the reference python package (oracle/_ref/py) is needed for the reference arms"
    result = {"device": device_info(), "rounds": args.rounds, "iters": args.iters, "scenes": {}}
    for name in args.scenes.split(","):
        model, cfg, ds = make_case(m, Config, name, args.iters)
        fns = arms(m, model, cfg)
        for fn in fns.values():                       # warm-up: module loads, allocator, algorithm choice
            timed(fn, ds)
        times = {k: [] for k in fns}
        outs = {}
        for r in range(args.rounds):
            order = list(fns) if r % 2 == 0 else list(fns)[::-1]
            for k in order:
                t, outs[k] = timed(fns[k], ds)
                times[k].append(t)
        import fused_embedding as fe
        loop = fe.EmbeddingLoop(types.SimpleNamespace(model=model, config=cfg), ds)
        P = int(model.xyz.shape[0])
        row = {"P": P, "V": loop.num_visible, "V/P": round(loop.num_visible / P, 4)}
        del loop
        for k in fns:
            med = statistics.median(times[k])
            row[k] = {"call_ms_median": round(med, 2), "call_ms_min": round(min(times[k]), 2),
                      "call_ms_max": round(max(times[k]), 2), "ms_per_iteration": round(med / args.iters, 3),
                      "final_psnr": round(outs[k]["metrics"]["psnr"][-1], 4),
                      "first_psnr": round(outs[k]["metrics"]["psnr"][0], 4)}
        row["speedup_vs_reference"] = round(row["reference"]["call_ms_median"] / row["fused"]["call_ms_median"], 2)
        row["speedup_vs_reference+enable"] = round(row["reference+enable"]["call_ms_median"] / row["fused"]["call_ms_median"], 2)
        row["profile_fused"] = profile_fused(model, cfg, ds, args.trace_dir)
        result["scenes"][name] = row
        print(json.dumps({name: row}), flush=True)
        del model, fns
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
