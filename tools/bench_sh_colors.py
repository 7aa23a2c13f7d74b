"""SH colours of models without appearance (the NeRF On-the-go preset: ``appearance_enabled: false``, SH degree 3):
``fused_colors.fused_sh_colors`` (csrc/sh_colors.cu) against the PyTorch statements it replaces, and the train step
of such a model with and without ``wildgaussians_fused.enable``.

    python tools/bench_sh_colors.py [--rows 3000000] [--steps 20] [--train-steps 10] [--rounds 5] [--out result.json]

(a) The colour op at `rows` rows, active degree 3, CUDA events around `steps` calls, arms alternating round by round:
    the kernels alone (forward; backward) on preallocated buffers, the autograd op forward (no gradient) and
    forward + backward, and method.py:1555-1565 (cat, clamp_max, normalize, transpose copy, eval_sh, clamp_min) the
    same two ways.  Bytes from the per-row budget of csrc/sh_colors.cu (forward 204 B read + 12 B written, backward
    216 B read + 204 B written) over the median kernel time, and the share of 3.35 TB/s.
(b) At C3 (3 M Gaussians, 1920x1080) and S1 (150 k, 640x400): ``_render_internal`` + the loss block of
    ``train_iteration`` (L1 on ``render``, 0.2 DSSIM on ``raw_render``, loss_mult 1, no uncertainty model) + backward,
    ms per step, arms alternating: an appearance-off model as shipped on the drop-in rasterizer; the same model with
    ``enable(model, ssim=True)``; an appearance-on model (wg_harness) with ``enable(model, ssim=True)`` for context.
Prints the device name and its power limit / max SM clock (nvidia-smi, query only).  Needs a GPU; does not fall back.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "wild-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_ssim import HBM_PEAK, device_info, summary, time_ms  # noqa: E402

FWD_BYTES, BWD_BYTES = 204 + 12, 216 + 204          # per row, csrc/sh_colors.cu
SCENES = {"C3": dict(P=3_000_000, W=1920, H=1080, seed=3), "S1": dict(P=150_000, W=640, H=400, seed=5)}


def run_arms(arms, steps, rounds, warmup=3):
    """{name: [ms per step, one per round]}; each arm is (setup, step) and the arms alternate inside every round."""
    out = {name: [] for name in arms}
    for setup, fn in arms.values():
        setup()
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    for r in range(rounds):
        names = list(arms) if r % 2 == 0 else list(arms)[::-1]
        for name in names:
            setup, fn = arms[name]
            setup()
            out[name].append(time_ms(fn, steps))
    return out


def statements(features_dc, features_rest, means3D, campos, deg):
    """method.py:1555-1565 (features from get_gaussians :1061-1064)."""
    from oracle import color_torch as ct
    features = torch.cat((features_dc, features_rest), dim=-1).clamp_max(1.0)
    dirs = torch.nn.functional.normalize(means3D - campos.repeat(features.shape[0], 1), dim=1)
    shs = features.view(-1, 16, 3).transpose(1, 2).contiguous()
    return torch.clamp_min(ct.eval_sh(deg, shs, dirs) + 0.5, 0.0)


def colour_op_case(P, steps, rounds, dev):
    import fused_colors as fc
    from diff_gaussian_rasterization import _C
    g = torch.Generator(device=dev).manual_seed(1)
    dc = torch.randn(P, 3, device=dev, generator=g) * 0.5
    rest = torch.randn(P, 45, device=dev, generator=g) * 0.3
    means = torch.randn(P, 3, device=dev, generator=g) * 2.0
    campos = torch.tensor([0.1, -0.2, 0.3], device=dev)
    dL = torch.randn(P, 3, device=dev, generator=g)
    leaves = [t.clone().requires_grad_(True) for t in (dc, rest, means)]
    colors, d_dc, d_rest, d_means = (torch.empty_like(t) for t in (dc, dc, rest, means))
    stream = torch.cuda.current_stream(dev).cuda_stream

    def kernel_fwd():
        _C._lib.gsr_sh_colors_forward(P, 3, dc.data_ptr(), rest.data_ptr(), means.data_ptr(), campos.data_ptr(),
                                      colors.data_ptr(), stream)

    def kernel_bwd():
        _C._lib.gsr_sh_colors_backward(P, 3, dc.data_ptr(), rest.data_ptr(), means.data_ptr(), campos.data_ptr(), dL.data_ptr(),
                                       d_dc.data_ptr(), d_rest.data_ptr(), d_means.data_ptr(), stream)

    def fwd(fn):
        def run():
            with torch.no_grad():
                fn(dc, rest, means, campos, 3)
        return run

    def fwd_bwd(fn):
        def run():
            for t in leaves:
                t.grad = None
            fn(*leaves, campos, 3).backward(dL)
        return run

    nop = lambda: None
    arms = {"kernel_fwd": (nop, kernel_fwd), "kernel_bwd": (nop, kernel_bwd),
            "fused_fwd": (nop, fwd(fc.fused_sh_colors)), "torch_fwd": (nop, fwd(statements)),
            "fused_fwd_bwd": (nop, fwd_bwd(fc.fused_sh_colors)), "torch_fwd_bwd": (nop, fwd_bwd(statements))}
    times = run_arms(arms, steps, rounds)
    res = {"P": P, "active_degree": 3, "steps_per_round": steps, "rounds": rounds,
           "times": {k: summary(v) for k, v in times.items()}}
    t = res["times"]
    for arm, per_row in (("kernel_fwd", FWD_BYTES), ("kernel_bwd", BWD_BYTES), ("fused_fwd", FWD_BYTES),
                         ("fused_fwd_bwd", FWD_BYTES + BWD_BYTES)):
        sec = t[arm]["median_ms"] * 1e-3
        res[arm + "_bytes"] = per_row * P
        res[arm + "_TBps"] = per_row * P / sec / 1e12
        res[arm + "_frac_of_3.35TBps"] = per_row * P / sec / HBM_PEAK
    res["speedup_fwd"] = t["torch_fwd"]["median_ms"] / t["fused_fwd"]["median_ms"]
    res["speedup_fwd_bwd"] = t["torch_fwd_bwd"]["median_ms"] / t["fused_fwd_bwd"]["median_ms"]
    with torch.no_grad():
        res["max_abs_colour_difference"] = float((fc.fused_sh_colors(dc, rest, means, campos, 3)
                                                  - statements(dc, rest, means, campos, 3)).abs().max())
    return res


def loss_block(m, out, gt, lambda_dssim=0.2):
    """method.py:1948-1966 with loss_mult = 1 and no uncertainty model (``m.ssim`` as currently bound)."""
    image_toned, image = out["render"], out["raw_render"]
    Ll1 = torch.nn.functional.l1_loss(image_toned, gt, reduction="none")
    ssim_value = m.ssim(image, gt, size_average=False)
    loss = (1.0 - lambda_dssim) * Ll1.mean() + lambda_dssim * (1.0 - ssim_value).mean() + 0
    loss.backward()


def step_case(m, Config, name, steps, rounds, dev):
    import diff_gaussian_rasterization as ours
    import synthetic
    import wg_harness as wh
    import wildgaussians_fused as wf
    from test_fused_sh_colors import make_model_off
    kw = SCENES[name]
    scene = synthetic.make_scene(kw["P"], kw["W"], kw["H"], sh_degree=3, seed=kw["seed"])
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    ours._C.set_geometry_cache(True)
    off, cfg_off = make_model_off(m, Config, scene, dev, seed=kw["seed"])
    on, cfg_on = wh.make_model(m, Config, scene, dev, seed=kw["seed"])
    cam = wh.make_camera(scene)
    gt = torch.rand(3, kw["H"], kw["W"], generator=torch.Generator().manual_seed(5)).to(dev)
    del scene

    def step(model, cfg):
        def run():
            for p in model.parameters():
                p.grad = None
            out = model._render_internal(cam, config=cfg, embedding=model.get_embedding(0), kernel_size=cfg.kernel_size)
            loss_block(m, out, gt)
        return run

    def shipped():
        wf.disable(on)
        wf.disable(off)

    def enabled(model):
        def setup():
            shipped()
            wf.enable(model, optimizer=False, ssim=True)
        return setup

    arms = {"appearance_off_as_shipped": (shipped, step(off, cfg_off)),
            "appearance_off_enable_ssim": (enabled(off), step(off, cfg_off)),
            "appearance_on_enable_ssim": (enabled(on), step(on, cfg_on))}
    try:
        times = run_arms(arms, steps, rounds)
    finally:
        shipped()
        ours._C.set_geometry_cache(False)
    res = {"what": f"{name}: P={kw['P']}, {kw['W']}x{kw['H']}; _render_internal + train_iteration loss block + backward, "
                   "ms per step", "steps_per_round": steps, "rounds": rounds,
           "times": {k: summary(v) for k, v in times.items()}}
    t = res["times"]
    res["speedup_enable_vs_shipped"] = t["appearance_off_as_shipped"]["median_ms"] / t["appearance_off_enable_ssim"]["median_ms"]
    del off, on
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=3_000_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--train-steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--scenes", default="S1,C3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sh_colors.py needs a GPU")
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        raise SystemExit("the reference python package is not present (oracle/_ref/py); run __graft_entry__.build() first")
    dev = torch.device("cuda:0")
    res = device_info()
    res["colour_op"] = colour_op_case(a.rows, a.steps, a.rounds, dev)
    print(json.dumps({"colour_op": res["colour_op"]}), flush=True)
    torch.cuda.empty_cache()
    for name in a.scenes.split(","):
        res["step_" + name] = step_case(m, Config, name, a.train_steps, a.rounds, dev)
        print(json.dumps({"step_" + name: res["step_" + name]}), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
