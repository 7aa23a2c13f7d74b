"""Cost of ``torch.use_deterministic_algorithms(True)``: flag off against flag on, alternated in rounds.

  backward   ``_C.rasterize_gaussians_backward`` (backward composite + chain rule; with the flag, the slot stores, the
             instance scan and the fixed-order gather)
  colour op  ``fused_colors`` backward (with the flag, per-CTA rows and their CTA-order sum)

Scenes S1 (150 k Gaussians, 640x400) and C3 (3 M, 1920x1080) of ``synthetic.make_scene``.  Each timed call is bracketed
by CUDA events; a round times ``--steps`` calls of one arm after ``--warmup`` untimed ones, the arms alternate, and the
median of the per-round means is reported with [min, max].  Peak device memory is read per arm around one call.

    python tools/bench_deterministic.py [--scenes S1,C3] [--rounds 5] [--steps 20] [--warmup 3] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "wild-gaussians_b200"), ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden"),
          os.path.dirname(__file__)):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_ssim import device_info  # noqa: E402

SCENES = {"S1": dict(P=150_000, W=640, H=400, seed=5), "C3": dict(P=3_000_000, W=1920, H=1080, seed=3)}


def backward_case(name, dev):
    import synthetic
    from diff_gaussian_rasterization import _C
    from make_golden import backward_args, call_args
    kw = SCENES[name]
    d = synthetic.to_device(synthetic.make_scene(kw["P"], kw["W"], kw["H"], sh_degree=3, seed=kw["seed"]), dev)
    _C.set_geometry_cache(False)
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(*call_args(d))
    args = backward_args(d, radii, geom, R, binning, img)
    return lambda: _C.rasterize_gaussians_backward(*args), int(R)


def colour_case(name, dev):
    import fused_colors as fc
    import test_colour_op_exact as tc
    P = SCENES[name]["P"]
    s = tc.random_scene(P, 11, dev)
    dLr, dLt = tc.loss_grads(P, 3, dev)
    mlp = tc._mlp(s)
    leaves = [s[k].clone().requires_grad_(True) for k in ("dc", "rest", "gemb", "aemb", "means")]
    params = [mlp[i].weight for i in (0, 2, 4)] + [mlp[i].bias for i in (0, 2, 4)]

    def call():
        raw, toned = fc.fused_colors(leaves[0], leaves[1], leaves[2], leaves[3], mlp, leaves[4], s["campos"], 3)
        torch.autograd.grad([raw, toned], leaves + params, [dLr, dLt])
    return call


def timed(fn, det, steps, warmup):
    torch.use_deterministic_algorithms(det)
    try:
        for _ in range(warmup):
            fn()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for a, b in ev:
            a.record()
            fn()
            b.record()
        torch.cuda.synchronize()
        return statistics.mean(a.elapsed_time(b) for a, b in ev)
    finally:
        torch.use_deterministic_algorithms(False)


def peak(fn, det):
    torch.use_deterministic_algorithms(det)
    try:
        fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn()
        torch.cuda.synchronize()
        return (torch.cuda.max_memory_allocated() - base) / 2**20
    finally:
        torch.use_deterministic_algorithms(False)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--scenes", default="S1,C3")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic needs a CUDA device")
    dev = torch.device("cuda:0")
    out = {"device": device_info(), "cases": {}}
    for name in a.scenes.split(","):
        fn_b, R = backward_case(name, dev)
        cases = {"backward": fn_b, "colour_op": colour_case(name, dev)}
        for what, fn in cases.items():
            ms = {False: [], True: []}
            for _ in range(a.rounds):
                for det in (False, True):
                    ms[det].append(timed(fn, det, a.steps, a.warmup))
            res = {}
            for det in (False, True):
                v = ms[det]
                res["on" if det else "off"] = dict(ms_median=statistics.median(v), ms_min=min(v), ms_max=max(v),
                                                   peak_extra_MiB=peak(fn, det))
            res["R"] = R
            out["cases"][f"{name} {what}"] = res
            print(json.dumps({f"{name} {what}": res}), flush=True)
    print(json.dumps(out["device"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
