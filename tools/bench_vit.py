"""DINOv2 backbone of the uncertainty loss with its token-wise layers as kernels (csrc/vit.cu,
``enable(model, dino_blocks=True)``) against the fused attention alone (``dino=True``) and the reference's own blocks
with the early exit.

    python tools/bench_vit.py [--steps 10] [--rounds 5] [--train-rounds 5] [--train-steps 10] [--out result.json]

Arms alternate round by round after a warm-up; every row is a median with [min, max] over rounds:
  * the backbone call ``get_intermediate_layers(x, n=[5], reshape=True)`` at 196x350 (355 tokens: the prediction's
    features on every feature-cache hit), 686x700 and 980x980 (2455 and 4905 tokens, on either side of
    ``fused_dino.BLOCKS_MAX_TOKENS``) and 1092x1932 (10769 tokens: a cache miss at C3), device time from CUDA
    events, on the random-weight ViT-S/14 with 4 registers of tools/bench_dino.py (q and k rows sharpened).  Arms: the
    reference's blocks with the early exit, the ``dino`` hook, the ``dino_blocks`` hook (which picks ``blocks=True``
    up to ``fused_dino.BLOCKS_MAX_TOKENS``), and ``blocks=True`` called directly at every size;
  * kernel times at 10769 tokens from a separate ``torch.profiler`` run, with the FLOP count computed here from the
    shapes: the useful 24 C^2 FLOP per token per block, and what the 3xTF32 kernels execute (three products on the
    64-padded rows and the 32-padded contraction), as a share of the 495 TFLOP/s dense TF32 data-sheet rate;
  * ``fused_train`` steps at S1 and C3 (tools/bench_train.py's scenes, appearance on, ``ssim``, ``msssim``,
    ``uncertainty`` on) with ``dino=True`` against ``dino_blocks=True``, host clock over steps that end in their metric
    read-back;
  * a profiler run of its own: kernels launched per backbone call (library counter and profiler) and the synchronising
    runtime calls per ordinary ``fused_train`` step with ``dino_blocks=True``.
Prints the device name and its power limit / max SM clock (nvidia-smi, query only).  Needs a GPU; does not fall back.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import re
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "wild-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_dino import TF32_PEAK, dino_input, early_exit_reference, sharpened_uncertainty_model  # noqa: E402
from bench_msssim import run_arms  # noqa: E402
from bench_ssim import device_info  # noqa: E402
from bench_train import SYNC_CALLS, build, run_steps, steps_from  # noqa: E402

HBM_PEAK = 3.35e12                    # H100 SXM data sheet, bytes/s
SIZES = (("355", (196, 350)), ("2455", (686, 700)), ("4905", (980, 980)), ("10769", (1092, 1932)))


def set_backbone(backbone, arm):
    import wildgaussians_fused as wf
    probe = type("Probe", (), {})()
    probe.uncertainty_model = type("U", (), {})()
    probe.uncertainty_model.backbone = backbone
    wf.disable(probe)
    if arm == "dino":
        wf.enable(probe, optimizer=False, dino=True)
    elif arm == "dino_blocks":
        wf.enable(probe, optimizer=False, dino_blocks=True)


def gemm_flops(bb, tokens, take_last=5):
    """(useful, executed) FLOP of the token-wise GEMMs of one call: blocks 0..take_last and the patch embedding."""
    C, p = bb.embed_dim, bb.patch_size
    pad = lambda v, q: -(-v // q) * q
    shapes = [(tokens - 1 - bb.num_register_tokens, 3 * p * p, C)]
    shapes += [(tokens, C, 3 * C), (tokens, C, C), (tokens, C, 4 * C), (tokens, 4 * C, C)] * (take_last + 1)
    useful = sum(2.0 * M * K * N for M, K, N in shapes)
    executed = sum(3 * 2.0 * pad(M, 64) * pad(K, 32) * N for M, K, N in shapes)
    moved = sum(4.0 * (M * K + K * N + 2 * M * N) for M, K, N in shapes)      # operands once, output (and residual)
    return useful, executed, moved


def backbone_case(bb, H, W, steps, rounds, dev):
    x = dino_input(H, W, dev)

    import fused_dino

    def arm(kind):
        def run():
            with torch.no_grad():
                if kind == "early_exit_reference":
                    early_exit_reference(bb, x)
                elif kind == "blocks_always":
                    fused_dino.get_intermediate_layers(bb, x, n=[5], reshape=True, blocks=True)
                else:
                    bb.get_intermediate_layers(x, n=[5], reshape=True)
        return run

    fns = {k: arm(k) for k in ("early_exit_reference", "dino", "dino_blocks", "blocks_always")}
    # each call selects its arm's hook first (a dictionary update on the host)
    wrapped = {k: (lambda k=k: (set_backbone(bb, k if k in ("dino", "dino_blocks") else "off"), fns[k]())) for k in fns}
    times = run_arms(wrapped, steps, rounds, warmup=3)
    set_backbone(bb, "off")
    return {"H": H, "W": W, "tokens": (H // 14) * (W // 14) + 1 + bb.num_register_tokens, "times": times}


def kernel_share(bb, H, W, dev):
    """Kernel times of one dino_blocks call (profiler, mean over 5 calls) and the GEMMs' share of the TF32 rate."""
    from torch.profiler import ProfilerActivity, profile
    import fused_dino
    x = dino_input(H, W, dev)
    call = lambda: fused_dino.get_intermediate_layers(bb, x, n=[5], reshape=True, blocks=True)
    calls = 5
    with torch.no_grad():
        call()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                call()
            torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            found = re.search(r"(\w+_kernel)(<[^>]*>)?", e.name)
            name = "".join(g or "" for g in found.groups()) if found else e.name
            per[name] = per.get(name, 0.0) + e.device_time / 1000.0 / calls
    tokens = (H // 14) * (W // 14) + 1 + bb.num_register_tokens
    useful, executed, moved = gemm_flops(bb, tokens)
    gemm_ms = sum(v for k, v in per.items() if "vit_gemm" in k)
    math_s, bytes_s = executed / TF32_PEAK, moved / HBM_PEAK
    return {"tokens": tokens, "kernel_ms_per_call": per, "gemm_ms": gemm_ms,
            "useful_gflop": useful / 1e9, "executed_tf32_gflop": executed / 1e9,
            "executed_tflops": executed / (gemm_ms * 1e-3) / 1e12,
            "share_of_tf32_peak": math_s / (gemm_ms * 1e-3), "bytes_bound_share": bytes_s / (gemm_ms * 1e-3),
            "bound": "tensor-core math" if math_s >= bytes_s else "HBM bytes"}


def launches_per_call(bb, dev):
    from diff_gaussian_rasterization import _C
    from torch.profiler import ProfilerActivity, profile
    x = dino_input(196, 350, dev)
    set_backbone(bb, "dino_blocks")
    with torch.no_grad():
        bb.get_intermediate_layers(x, n=[5], reshape=True)
        torch.cuda.synchronize()
        n0 = _C.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            bb.get_intermediate_layers(x, n=[5], reshape=True)
            torch.cuda.synchronize()
        lib = _C.launch_count() - n0
    set_backbone(bb, "off")
    kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return {"library_launches": lib, "profiler_kernels": len(kernels),
            "non_library_kernels": sorted({k for k in kernels if "vit_" not in k and "attention_" not in k})}


def set_train_arm(method, arm):
    import wildgaussians_fused as wf
    wf.disable_method(method)
    wf.enable_method(method, train=True, ssim=True, msssim=True, uncertainty=True,
                     dino=(arm == "dino"), dino_blocks=(arm == "dino_blocks"))


def train_case(scene, rounds, n_steps, dev, cameras=4):
    method = build(scene, True, dev, cameras)
    arms = ("dino", "dino_blocks")
    random.seed(0)
    torch.manual_seed(0)
    it = iter(steps_from(20_000, 100_000))
    take = lambda n: [next(it) for _ in range(n)]
    for arm in arms:                                   # one epoch per arm: every feature-cache entry is warm
        set_train_arm(method, arm)
        run_steps(method, take(cameras + 4))
    times = {a: [] for a in arms}
    for _ in range(rounds):
        for arm in arms:
            set_train_arm(method, arm)
            run_steps(method, take(1))
            steps = take(n_steps)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run_steps(method, steps)
            torch.cuda.synchronize()
            times[arm].append((time.perf_counter() - t0) * 1000.0 / n_steps)
    from torch.profiler import ProfilerActivity, profile
    set_train_arm(method, "dino_blocks")
    run_steps(method, take(2))
    steps = take(3)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run_steps(method, steps)
        torch.cuda.synchronize()
    syncs = sum(e.name in SYNC_CALLS for e in prof.events()) / len(steps)
    import wildgaussians_fused as wf
    wf.disable_method(method)
    del method
    torch.cuda.empty_cache()
    return {"scene": scene, "ms_per_step": {a: {"median": statistics.median(t), "min": min(t), "max": max(t)}
                                            for a, t in times.items()},
            "dino_blocks_syncs_per_step": syncs}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--train-rounds", type=int, default=5)
    ap.add_argument("--train-steps", type=int, default=10)
    ap.add_argument("--scenes", default="S1,C3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vit.py needs a GPU")
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        raise SystemExit("the reference python package is not present (oracle/_ref/py); run __graft_entry__.build() first")
    dev = torch.device("cuda:0")
    res = device_info()
    print(json.dumps(res), flush=True)
    bb = sharpened_uncertainty_model(m, Config, "dino", dev).backbone
    for name, (H, W) in SIZES:
        res[f"backbone_{name}"] = backbone_case(bb, H, W, a.steps, a.rounds, dev)
        print(json.dumps({f"backbone_{name}": res[f"backbone_{name}"]}), flush=True)
    res["kernels_10769"] = kernel_share(bb, 1092, 1932, dev)
    print(json.dumps({"kernels_10769": res["kernels_10769"]}), flush=True)
    res["launches_355"] = launches_per_call(bb, dev)
    print(json.dumps({"launches_355": res["launches_355"]}), flush=True)
    del bb
    torch.cuda.empty_cache()
    for scene in [s for s in a.scenes.split(",") if s]:
        res[f"train_{scene}"] = train_case(scene, a.train_rounds, a.train_steps, dev)
        print(json.dumps({f"train_{scene}": res[f"train_{scene}"]}), flush=True)
    print(json.dumps(device_info()))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
