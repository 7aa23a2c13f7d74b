"""Benchmark of the evaluation metrics: the reference's ``compute_metrics`` (wildgaussians/evaluation.py:331-352, numpy
on the host) against ``fused_metrics.compute_metrics`` on one GPU.

    python tools/bench_metrics.py [--rounds 5] [--kernel-iters 200]

Workloads: the NeRF-W protocol's right half of a 1080x1920 image (uint8, a non-contiguous slice, what
``NerfWEvaluationProtocol.evaluate`` passes) and a full 1080x1920 float32 ``[1, H, W, 3]`` image (what
``DefaultEvaluationProtocol.evaluate`` passes).  For each, the two arms alternate, each call timed on the host clock
(every call ends in a host read), once with LPIPS replaced by a network that returns zeros and once with a seeded
random-weight AlexNet LPIPS in ``_LPIPS_CACHE`` (pretrained weights would need a download).  Then the two kernels
alone are timed with CUDA events over ``--kernel-iters`` calls; the fp64 FLOPs and the bytes they need are computed
from the shapes, and the share of the larger of the two H100 SXM data-sheet bounds (34 TFLOP/s non-tensor FP64,
3.35 TB/s HBM3) is reported with the bound's name.  Prints one JSON line per workload and the card's name and power
limit.  Needs ``oracle/_ref/py`` (``__graft_entry__.build()``) and a GPU.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "wild-gaussians_b200"), os.path.join(ROOT, "oracle", "_ref", "py")):
    if p not in sys.path:
        sys.path.insert(0, p)

FP64_PEAK = 34e12          # H100 SXM data sheet, non-tensor FP64
HBM_PEAK = 3.35e12         # H100 SXM data sheet, HBM3


class ZeroLPIPS(torch.nn.Module):
    def forward(self, a, b):
        return a.new_zeros((a.shape[0], 1, 1, 1))


def workloads(rng):
    H, W = 1080, 1920
    y, x = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    base = 0.5 + 0.25 * np.sin(x / 17.0)[..., None] * np.cos(y[..., None] / 23.0 + np.arange(3))
    gt = np.clip(base * 255 + rng.normal(0, 6, (H, W, 3)), 0, 255).astype(np.uint8)
    pred = np.clip(gt + rng.normal(0, 10, gt.shape), 0, 255).astype(np.uint8)
    yield "nerfw_half_1080x1920_u8", pred[:, W // 2:], gt[:, W // 2:]
    yield "full_1080x1920_f32", pred[None].astype(np.float32) / 255, gt[None].astype(np.float32) / 255


def work(shape, a_bytes, b_bytes):
    """fp64 FLOPs and DRAM bytes the two kernels need: the x pass over H rows and the y pass over the valid map, 5 maps
    x 11 taps x one fma (2 FLOPs) each, plus about 20 FLOPs per output for the map; the inputs read once, the two fp32
    LPIPS tensors written once (partials and sums are negligible)."""
    *batch, H, W, C = shape
    B = int(np.prod(batch)) if batch else 1
    Ho, Wo = H - 10, W - 10
    flops = B * C * (5 * 11 * 2 * (H * Wo + Ho * Wo) + 20 * Ho * Wo)
    nbytes = a_bytes + b_bytes + 2 * 4 * B * H * W * C
    return flops, nbytes


def time_calls(fn, rounds):
    ts = []
    for _ in range(rounds):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return ts


def kernel_ms(pred, gt, iters):
    """CUDA-event time of gsr_metrics_forward (both launches) on already-staged device inputs."""
    import fused_metrics as fm
    from diff_gaussian_rasterization import _C
    pred = pred[..., :gt.shape[-1]]
    *batch, H, W, C = gt.shape
    B = int(np.prod(batch)) if batch else 1
    dev = torch.device("cuda")
    a = torch.from_numpy(np.ascontiguousarray(gt)).to(dev)
    b = torch.from_numpy(np.ascontiguousarray(pred)).to(dev)
    lp = torch.empty((2,) + gt.shape, dtype=torch.float32, device=dev)
    sums = torch.empty((B, 3), dtype=torch.float64, device=dev)
    scratch = torch.empty(_C._lib.gsr_metrics_scratch_bytes(B, H, W, C) // 8, dtype=torch.float64, device=dev)
    args = _C.GsrMetricsArgs(B=B, H=H, W=W, C=C, a_u8=int(gt.dtype == np.uint8), b_u8=int(pred.dtype == np.uint8),
                             a=a.data_ptr(), b=b.data_ptr(), c1=fm._C1, c2=fm._C2, lpips_a=lp[0].data_ptr(),
                             lpips_b=lp[1].data_ptr(), sums=sums.data_ptr(), scratch=scratch.data_ptr())
    args.taps[:] = fm.dmpix_taps().tolist()
    s = torch.cuda.current_stream().cuda_stream

    def run():
        _C._check(_C._lib.gsr_metrics_forward(ctypes.byref(args), s), "gsr_metrics_forward")

    for _ in range(10):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, int(gt.nbytes), int(pred.nbytes)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_metrics needs a GPU"
    import fused_metrics as fm
    import wildgaussians.evaluation as ev
    from wildgaussians._metrics_lpips import LPIPS

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print(json.dumps({"card": card[0] if card else torch.cuda.get_device_name()}))
    torch.manual_seed(0)
    nets = {"zero": ZeroLPIPS(), "alex_random": LPIPS(pretrained=False, net="alex", pnet_rand=True, verbose=False)}
    rng = np.random.default_rng(0)
    for name, pred, gt in workloads(rng):
        row = {"workload": name}
        for lp_name, net in nets.items():
            ev._LPIPS_CACHE.clear()
            ev._LPIPS_CACHE["alex"] = net
            ref_fn = lambda: ev.compute_metrics(pred, gt)                                  # noqa: E731
            fused_fn = lambda: fm.compute_metrics(pred, gt, evaluation=ev)                  # noqa: E731
            r0, f0 = ref_fn(), fused_fn()                                                   # warm-up, and a check
            assert abs(r0["ssim"] - f0["ssim"]) <= 1e-10 and abs(r0["lpips"] - f0["lpips"]) <= 1e-6, (r0, f0)
            tr, tf = [], []
            for _ in range(args.rounds):
                tr += time_calls(ref_fn, 1)
                tf += time_calls(fused_fn, 1)
            row[f"ref_s_{lp_name}"] = float(np.median(tr))
            row[f"fused_ms_{lp_name}"] = 1e3 * float(np.median(tf))
            row[f"fused_ms_{lp_name}_minmax"] = [1e3 * min(tf), 1e3 * max(tf)]
            row[f"speedup_{lp_name}"] = float(np.median(tr) / np.median(tf))
        ms, a_bytes, b_bytes = kernel_ms(pred, gt, args.kernel_iters)
        flops, nbytes = work(gt.shape, a_bytes, b_bytes)
        t_fp64, t_hbm = flops / FP64_PEAK, nbytes / HBM_PEAK
        row.update(kernel_ms=ms, fp64_gflop=flops / 1e9, dram_mb=nbytes / 1e6, h2d_bytes_per_call=a_bytes + b_bytes,
                   bound="fp64" if t_fp64 >= t_hbm else "hbm", share_of_bound=max(t_fp64, t_hbm) / (ms * 1e-3),
                   rounds=args.rounds)
        print(json.dumps(row))


if __name__ == "__main__":
    main()
