"""``GaussianModel.densify_and_prune`` plus the ``compute_3D_filter`` that ``train_iteration`` runs after it, per call,
two arms alternated in rounds:

  shipped  the class's own ``densify_and_prune`` (``enable(model)``: the fused 3D filter)
  fused    ``enable(model, densify=True)`` (``fused_densify``, same fused 3D filter)

Scenes S1 (150 k Gaussians) and C3 (3 M), appearance on (the default preset), Adam moments present, with statistics that
select a few % of the Gaussians for cloning and for splitting and prune a few %, as in a real run.  Each call starts from
the same restored state (outside the timed window) and ends in a device synchronisation, so the host clock times it.
Also reported per arm: the peak allocation above the model's own tensors during the call, the synchronising runtime
calls per call (a separate profiler run), and the fused path alone at about 20 M Gaussians (appearance off, SH degree 3),
where torch.quantile refuses the reference's input.

    python tools/bench_densify.py [--scenes S1,C3] [--rounds 5] [--big 20000000] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "wild-gaussians_b200"), ROOT, os.path.join(ROOT, "tests"), os.path.dirname(__file__)):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_ssim import device_info  # noqa: E402

SCENES = {"S1": dict(P=150_000, seed=5), "C3": dict(P=3_000_000, seed=3)}
MAX_GRAD, MIN_OPACITY, EXTENT = 0.0002, 0.005, 1.5
SYNC_CALLS = ("cudaStreamSynchronize", "cudaEventSynchronize", "cudaMemcpy")


def set_stats(model, dev, seed=3):
    """A few % clone and split candidates, a few % transparent or very large Gaussians (pruned)."""
    P = int(model.xyz.shape[0])
    g = torch.Generator(device=dev).manual_seed(seed)
    with torch.no_grad():
        denom = torch.randint(0, 6, (P, 1), generator=g, device=dev).float()
        model.denom.copy_(denom)
        model.xyz_grad.copy_(torch.exp(torch.randn(P, 1, generator=g, device=dev) * 0.8) * MAX_GRAD * 0.2 * denom)
        if model.xyz_gradient_accum_abs is not None:
            model.xyz_gradient_accum_abs.copy_(torch.exp(torch.randn(P, 1, generator=g, device=dev)) * MAX_GRAD * 0.1 * denom)
        model.scales[torch.rand(P, generator=g, device=dev) < 0.005] = -1.2
        model.opacities[torch.rand(P, generator=g, device=dev) < 0.02] = -6.2


def state_of(model):
    opt = model.optimizer
    saved = {}
    for n in model._dynamically_sized_props:
        t = getattr(model, n, None)
        if t is not None:
            st = opt.state.get(t, None)
            saved[n] = (t.detach().clone(), None if st is None else (st["exp_avg"].clone(), st["exp_avg_sq"].clone()))
    return saved


def restore(model, saved):
    opt = model.optimizer
    groups = {g["name"]: g for g in opt.param_groups}
    for n, (t, mom) in saved.items():
        if n in groups:
            old = groups[n]["params"][0]
            p = torch.nn.Parameter(t.clone())
            st = opt.state.pop(old, None)
            if mom is not None:
                st = st or {"step": torch.tensor(3.0)}
                st["exp_avg"], st["exp_avg_sq"] = mom[0].clone(), mom[1].clone()
                opt.state[p] = st
            groups[n]["params"][0] = p
            setattr(model, n, p)
        else:
            model.register_buffer(n, t.clone())


def add_moments(model, dev):
    for grp in model.optimizer.param_groups:
        if grp["name"] in model._dynamically_sized_props:
            p = grp["params"][0]
            model.optimizer.state[p] = {"step": torch.tensor(3.0), "exp_avg": torch.zeros_like(p) + 1e-3,
                                        "exp_avg_sq": torch.zeros_like(p) + 1e-6}


def build(name, dev):
    import synthetic
    import wg_harness as wh
    import wg_train
    m, Config = wh.import_method()
    if m is None:
        raise SystemExit("reference python package not present (oracle/_ref/py): run __graft_entry__.build() first")
    sc = SCENES[name]
    scene = synthetic.to_device(synthetic.make_scene(sc["P"], 640, 400, sh_degree=3, seed=sc["seed"]), dev)
    method = wg_train.make_method(m, Config, scene, dev)
    del scene
    add_moments(method.model, dev)
    set_stats(method.model, dev)
    return method


def model_bytes(model):
    n = sum(t.numel() * 4 for t in [getattr(model, k) for k in model._dynamically_sized_props] if t is not None)
    for st in model.optimizer.state.values():
        n += sum(v.numel() * v.element_size() for k, v in st.items() if k != "step")
    return n


def one_call(method, fused):
    import wildgaussians_fused as wf
    model = method.model
    wf.enable(model, optimizer=False, densify=fused)
    try:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        out = model.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, enable_size_pruning=True)
        model.compute_3D_filter(cameras=method.train_cameras)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        peak = torch.cuda.max_memory_allocated() - base
    finally:
        wf.disable(model)
    return ms, peak, out


def kernel_ms(prof, name):
    """Device time of the kernels whose name contains `name` in a profiler run, ms."""
    tot = 0.0
    for e in prof.key_averages():
        if name in e.key:
            tot += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
    return tot / 1e3


def syncs(method, fused):
    """Synchronising runtime calls of one call and the apply kernel's device time (fused arm)."""
    import wildgaussians_fused as wf
    from torch.profiler import ProfilerActivity, profile
    model = method.model
    wf.enable(model, optimizer=False, densify=fused)
    try:
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            model.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, enable_size_pruning=True)
    finally:
        wf.disable(model)
    n = sum(e.name in SYNC_CALLS for e in prof.events())
    return n, kernel_ms(prof, "densify_apply_kernel")


def med(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def bench_scene(name, dev, rounds):
    import contextlib
    import io
    method = build(name, dev)
    model = method.model
    saved = state_of(model)
    res = {"P": int(model.xyz.shape[0]), "model_bytes": model_bytes(model)}
    times = {False: [], True: []}
    peaks = {False: [], True: []}
    outs = {}
    with contextlib.redirect_stdout(io.StringIO()):
        for r in range(rounds + 1):                                    # round 0 is the warm-up
            for fused in ((False, True) if r % 2 == 0 else (True, False)):
                restore(model, saved)
                ms, peak, out = one_call(method, fused)
                outs[fused] = out
                if r:
                    times[fused].append(ms)
                    peaks[fused].append(peak)
        n_sync = {}
        for fused in (False, True):
            restore(model, saved)
            n_sync[fused] = syncs(method, fused)
    assert outs[False] == outs[True], outs
    C, S, pruned = outs[True]
    res.update(clone=C, split=S, pruned=pruned, clone_pct=100 * C / res["P"], split_pct=100 * S / res["P"],
               prune_pct=100 * pruned / res["P"])
    for fused, arm in ((False, "shipped"), (True, "fused")):
        res[arm] = {"ms": med(times[fused]), "peak_above_model_bytes": max(peaks[fused]), "sync_calls": n_sync[fused][0]}
    # the apply kernel reads every dynamically sized float once (parameters, moments, buffers) and writes each output
    # row once, plus 16 B of positions per source row; its share of the H100 SXM's 3.35 TB/s HBM3 bandwidth
    rows_out = res["P"] + C + S - pruned
    per_row = res["model_bytes"] / res["P"]
    moved = res["model_bytes"] + per_row * rows_out + 16 * res["P"]
    res["apply"] = {"bytes_per_source_row": per_row, "bytes": moved, "kernel_ms_profiled": n_sync[True][1],
                    "share_of_3.35TBps": moved / (n_sync[True][1] * 1e-3) / 3.35e12 if n_sync[True][1] else None}
    del method, model, saved
    torch.cuda.empty_cache()
    return res


def bench_big(P, dev, rounds):
    """The fused path alone on a lean model (appearance off, SH degree 3 storage) of P Gaussians."""
    import fused_densify as fd
    import wg_harness as wh
    m, Config = wh.import_method()
    free = torch.cuda.mem_get_info(dev)[0]
    need = P * 65 * 4 * 3 + P * 40            # parameters + buffers, a saved copy, the new tensors, the scratch
    if free < need * 1.3:
        return {"skipped": f"needs about {need / 2**30:.0f} GB free, {free / 2**30:.0f} GB free"}
    cfg = Config(source_path="", model_path="", uncertainty_mode="disabled", appearance_enabled=False)
    model = m.GaussianModel(cfg, training_setup=False).to(dev)
    model._resize_parameters(P)
    g = torch.Generator(device=dev).manual_seed(1)
    with torch.no_grad():
        model.xyz.normal_(generator=g)
        model.rotations.normal_(generator=g)
        model.scales.copy_(torch.log(0.015 * torch.exp(0.3 * torch.randn(P, 3, generator=g, device=dev))))
        model.opacities.normal_(generator=g)
    model.spatial_lr_scale.fill_(1.0)
    model._setup_optimizers()                 # no Adam moments: they would triple the footprint
    set_stats(model, dev)
    saved = state_of(model)
    times = []
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):
        for r in range(rounds + 1):
            restore(model, saved)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fd.densify_and_prune(model, MAX_GRAD, MIN_OPACITY, EXTENT, True)
            torch.cuda.synchronize()
            if r:
                times.append((time.perf_counter() - t0) * 1e3)
    return {"P": P, "out": list(out), "ms": med(times)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="S1,C3")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--big", type=int, default=20_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"device": device_info(), "scenes": {}}
    for name in args.scenes.split(","):
        res["scenes"][name] = bench_scene(name, dev, args.rounds)
        print(name, json.dumps(res["scenes"][name]), flush=True)
    if args.big:
        res["big"] = bench_big(args.big, dev, max(2, args.rounds // 2))
        print("big", json.dumps(res["big"]), flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
