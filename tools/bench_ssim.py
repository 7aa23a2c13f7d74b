"""SSIM of the photometric loss: the reference's ``ssim`` (wildgaussians/method.py:644-673, unmodified, from
oracle/_ref/py) against ``fused_ssim`` (csrc/ssim.cu), on one GPU.

    python tools/bench_ssim.py [--steps 20] [--rounds 5] [--out result.json]

Per image size (C3 1920x1080, C5 4096x2160), arms alternating round by round, CUDA events around `steps` calls:
  * ssim forward only (no gradient): reference with TF32 at PyTorch's default and with TF32 off, fused;
  * the loss block of method.py:1948-1966 (lambda_dssim = 0.2, loss_mult = 1, [1,H,W]-shaped map) forward + backward:
    same three arms; plus the fused SSIM forward + backward alone (kernel-level bytes over time);
  * the fused result's error against the float64 oracle (map, mean, dL/dimg1 relative to its largest magnitude), and
    the reference's own errors with TF32 on and off.
At C3 also the train step of tests/wg_harness.py with the fused caller (wildgaussians_fused.enable) and the real loss block
in place of the synthetic one, once with the reference's ``ssim`` and once with ``enable(..., ssim=True)``.
Prints the device name and its power limit / max SM clock (nvidia-smi, query only).  Needs a GPU; does not fall back.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "wild-gaussians_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM_PEAK = 3.35e12          # H100 SXM data sheet, bytes/s
SIZES = {"C3": (1080, 1920), "C5": (2160, 4096)}
# algorithmic HBM bytes per pixel of csrc/ssim.cu (fp32): forward reads both [3] images (24 B), writes the map (4 B) and,
# when a backward follows, the 9 factors (36 B); the backward reads both images, the factors and dL/dmap, writes dL/dimg1
FWD_NOGRAD_B, FWD_B, BWD_B = 28, 64, 24 + 36 + 4 + 12


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = r.stdout.strip()
    except Exception as e:          # reporting only
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def time_ms(fn, steps):
    """ms per call over `steps` calls, CUDA events."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def run_arms(arms, steps, rounds, warmup=3):
    """{name: [ms per round]} with the arms alternating inside every round; TF32 set per arm."""
    out = {name: [] for name in arms}
    for name, (fn, tf32) in arms.items():
        torch.backends.cudnn.allow_tf32 = tf32
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for name, (fn, tf32) in arms.items():
            torch.backends.cudnn.allow_tf32 = tf32
            out[name].append(time_ms(fn, steps))
    return out


def summary(times):
    return {"median_ms": statistics.median(times), "min_ms": min(times), "max_ms": max(times)}


def loss_block(ssim_fn, image, gt_image, lambda_dssim=0.2):
    """method.py:1948-1966 with loss_mult = 1 and no uncertainty model."""
    Ll1 = torch.nn.functional.l1_loss(image, gt_image, reduction="none")
    ssim_value = ssim_fn(image, gt_image, size_average=False)
    loss = (1.0 - lambda_dssim) * (Ll1 * 1.0).mean() + lambda_dssim * ((1.0 - ssim_value) * 1.0).mean() + 0
    loss.backward()
    return loss


def errors(ssim_fn, img, gt, G, want, tf32):
    torch.backends.cudnn.allow_tf32 = tf32
    x = img.clone().requires_grad_(True)
    smap = ssim_fn(x, gt, size_average=False)
    (smap * G).sum().backward()
    mean = ssim_fn(img, gt, size_average=True)
    wmap, wmean, wgrad = want
    return {"map_max_abs": float((smap.double() - wmap).abs().max()), "mean_abs": abs(float(mean) - float(wmean)),
            "grad_max_abs_over_max": float((x.grad.double() - wgrad).abs().max()) / float(wgrad.abs().max())}


def size_case(m, name, H, W, steps, rounds, dev):
    import fused_ssim
    from oracle import ssim_oracle
    g = torch.Generator(device=dev).manual_seed(1)
    gt = torch.rand(1, 3, H, W, generator=g, device=dev)[0]
    img = (torch.nn.functional.avg_pool2d(gt[None], 5, 1, 2)[0] + 0.05 * torch.randn(3, H, W, generator=g, device=dev)).clamp(0, 1)
    G = torch.randn(H, W, generator=g, device=dev)
    leaf = img.clone().requires_grad_(True)

    def fwd(fn):
        def run():
            with torch.no_grad():
                fn(img, gt, size_average=False)
        return run

    def block(fn):
        def run():
            leaf.grad = None
            loss_block(fn, leaf, gt)
        return run

    def fused_fwd_bwd():
        leaf.grad = None
        fused_ssim.ssim(leaf, gt, size_average=False).backward(G)

    arms = {"reference_fwd_tf32_default": (fwd(m.ssim), True), "reference_fwd_tf32_off": (fwd(m.ssim), False),
            "fused_fwd": (fwd(fused_ssim.ssim), False),
            "reference_loss_block_tf32_default": (block(m.ssim), True), "reference_loss_block_tf32_off": (block(m.ssim), False),
            "fused_loss_block": (block(fused_ssim.ssim), False), "fused_ssim_fwd_bwd": (fused_fwd_bwd, False)}
    times = run_arms(arms, steps, rounds)
    res = {"H": H, "W": W, "steps_per_round": steps, "rounds": rounds, "times": {k: summary(v) for k, v in times.items()}}
    px = H * W
    for arm, nbytes in (("fused_fwd", FWD_NOGRAD_B * px), ("fused_ssim_fwd_bwd", (FWD_B + BWD_B) * px)):
        t = res["times"][arm]["median_ms"] * 1e-3
        res[arm + "_alg_bytes"] = nbytes
        res[arm + "_frac_of_3.35TBps"] = nbytes / t / HBM_PEAK
    t = res["times"]
    for pre in ("fwd", "loss_block"):
        f = t[f"fused_{pre}"]["median_ms"]
        res[f"speedup_{pre}_vs_tf32_default"] = t[f"reference_{pre}_tf32_default"]["median_ms"] / f
        res[f"speedup_{pre}_vs_tf32_off"] = t[f"reference_{pre}_tf32_off"]["median_ms"] / f
    torch.backends.cudnn.allow_tf32 = False
    want = ssim_oracle.ssim_and_grad(img, gt, G)
    res["error_vs_fp64_oracle"] = {"fused": errors(fused_ssim.ssim, img, gt, G, want, False),
                                   "reference_tf32_off": errors(m.ssim, img, gt, G, want, False),
                                   "reference_tf32_default": errors(m.ssim, img, gt, G, want, True)}
    torch.backends.cudnn.allow_tf32 = True
    del want
    torch.cuda.empty_cache()
    return res


def train_step_case(m, Config, steps, rounds, dev):
    """C3: wg_harness model + fused caller, `_render_internal` + the real loss block + backward, original vs fused ssim."""
    import synthetic
    import wg_harness as wh
    import wildgaussians_fused as wf
    import diff_gaussian_rasterization as ours
    kw = dict(synthetic.CONFIGS["C3"]); kw["seed"] = 0; kw["sh_degree"] = 3
    scene = synthetic.make_scene(**kw)
    model, cfg = wh.make_model(m, Config, scene, dev)
    cam = wh.make_camera(scene)
    H, W = scene["image_height"], scene["image_width"]
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(5)).to(dev)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    ours._C.set_geometry_cache(True)
    original = m.ssim
    wf.enable(model, optimizer=False, ssim=True)
    hooked = m.ssim

    def step(fused):
        def run():
            m.ssim = hooked if fused else original
            for p in model.parameters():
                p.grad = None
            out = model._render_internal(cam, cfg, kernel_size=cfg.kernel_size, embedding=model.appearance_embeddings[0])
            loss_block(m.ssim, out["render"], gt)
        return run

    try:
        arms = {"train_step_reference_ssim": (step(False), True), "train_step_fused_ssim": (step(True), True)}
        times = run_arms(arms, steps, rounds)
    finally:
        wf.disable(model)
        m.ssim = original
        ours._C.set_geometry_cache(False)
    res = {"what": "wg_harness GaussianModel (C3: P=3M, 1920x1080, SH 3, appearance on) with the fused caller: "
                   "_render_internal + method.py:1948-1966 loss block + backward, TF32 default; ms per step",
           "P": kw["P"], "times": {k: summary(v) for k, v in times.items()}}
    res["difference_ms"] = (res["times"]["train_step_reference_ssim"]["median_ms"] -
                            res["times"]["train_step_fused_ssim"]["median_ms"])
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--train-steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ssim.py needs a GPU")
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        raise SystemExit("the reference python package is not present (oracle/_ref/py); run __graft_entry__.build() first")
    dev = torch.device("cuda:0")
    res = device_info()
    res["tf32_default"] = bool(torch.backends.cudnn.allow_tf32)
    for name, (H, W) in SIZES.items():
        res[name] = size_case(m, name, H, W, a.steps, a.rounds, dev)
        print(json.dumps({name: res[name]}), flush=True)
    res["C3_train_step"] = train_step_case(m, Config, a.train_steps, a.rounds, dev)
    print(json.dumps({"C3_train_step": res["C3_train_step"]}), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
