#!/usr/bin/env python
"""bench.py -- forward+backward rasterization throughput on synthetic Gaussian clouds (BASELINE.json metric).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--config C3] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...

One *step* = one forward + one backward rasterization of the named workload (default C3: 3M Gaussians,
1920x1080, colours precomputed -- the path wildgaussians/method.py uses; SURVEY.md 8d).  Inputs are synthetic
(seeded generator, wild-gaussians_b200/synthetic.py) and resident in HBM when the timed region starts.
Rank 0 prints ONE JSON line:

  value / ms_per_step   Gaussians*pixels/s = P*N / t_step, device-timed (CUDA events), max over ranks
  e2e                   the same metric through the public Python API (GaussianRasterizer + autograd) with every
                        tensor argument copied from pinned host memory each step and the image + all gradients read
                        back to the host, copies inside the timed region; value = consecutive steps software-pipelined
                        (same harness for both arms), plus the one-step-in-flight and serial-copy forms
  roofline              dominant kernel: algorithmic bytes / its event-timed duration vs MEASURED_PEAKS.json
  roofline_path         SURVEY.md 8(d) whole-path formula (B_fwd + B_bwd) / (t_fwd + t_bwd)
  stages                per-stage device times (events inside libgsrast, averaged over K profiled steps run right
                        after the timed region) and their algorithmic bytes
  cpu_baseline          the CPU oracle (oracle/oracle.c, OpenMP) on a bounded sample of the workload, rank 0, N=1

--dump-outputs DIR writes what the timed path returned in its last timed step (image, radii, every gradient) as
float32 DIR/<name>.npy: arrays with one row per Gaussian on a fixed seeded sample of rows, arrays above 8 M elements
on a fixed seeded sample of elements (<= 64 MB in all).  Inputs are seeded, so two builds run with the same arguments
can be compared output for output.

--impl reference times the UNMODIFIED reference rasterizer compiled for sm_90a (oracle/_ref/libdgr_ref.so; the
reference has no CPU implementation of this path, its own implementation IS CUDA) on the same tensors; if that
library did not travel with the snapshot it falls back to the CPU oracle port.  Rank 0 only.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "wild-gaussians_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import synthetic  # noqa: E402

FALLBACK_HBM_GBS = 3350.0     # H100 SXM data sheet (HBM3), for a card allowed 700 W
E2E_NOTE = ("value / ms_per_step = the FASTEST of the forms below (both arms).  ms_per_step_pipelined: public API (GaussianRasterizer + autograd) on pinned HOST buffers, every step copies all of its "
            "inputs host->device and its image + all gradients device->host inside the timed region; steps are software-pipelined "
            "(<= 3 in flight: step i's read-back overlaps step i+1's uploads on the other PCIe direction; the closing event waits "
            "for the last read-back) -- the SAME harness times both arms.  ms_per_step_one_step_in_flight (ours): copies "
            "overlapped only inside a step, host waits for the step's result before starting the next.  "
            "ms_per_step_serial_copies: every copy on the compute stream, one step in flight")


# ----------------------------------------------------------------------------------------------------------
# helpers
# ----------------------------------------------------------------------------------------------------------
def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
        except Exception:
            pass
    return FALLBACK_HBM_GBS, "fallback (H100 SXM data sheet 3.35 TB/s)"


class ClockSampler:
    """Samples nvidia-smi clocks / throttle reasons during the timed regions."""
    Q = "index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown," \
        "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, gpu_index=0):
        self.gpu, self.rows, self.proc, self.th = gpu_index, [], None, None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "20", "-i", str(self.gpu)], stdout=subprocess.PIPE, text=True)
        except Exception:
            self.proc = None
            return
        def pump():
            for line in self.proc.stdout:
                self.rows.append(line.strip())
        self.th = threading.Thread(target=pump, daemon=True)
        self.th.start()

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        for r in self.rows:
            f = [x.strip() for x in r.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        busy = [s for s in sm if s > 0]
        return {"sm_mhz": float(np.median(busy)) if busy else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


DUMP_ROWS = 65536              # per-Gaussian rows kept by --dump-outputs
DUMP_MAX_ELEMS = 8 * 1024 * 1024


def dump_outputs(out_dir, P, arrays):
    """Writes `arrays` ({name: tensor or None}) as float32 .npy files under `out_dir`, sampled as the module doc says."""
    os.makedirs(out_dir, exist_ok=True)
    rows = np.sort(np.random.default_rng(2024).choice(P, size=min(P, DUMP_ROWS), replace=False)) if P else None
    for name, t in arrays.items():
        if t is None or t.numel() == 0:
            continue
        a = t.detach().float().cpu().numpy()
        if a.ndim >= 1 and a.shape[0] == P and P > DUMP_ROWS:
            a = a[rows]
        elif a.size > DUMP_MAX_ELEMS:
            a = a.reshape(-1)[np.sort(np.random.default_rng(2025).choice(a.size, size=DUMP_MAX_ELEMS, replace=False))]
        np.save(os.path.join(out_dir, f"{name}.npy"), np.ascontiguousarray(a, dtype=np.float32))


def step_outputs(color, radii, grads):
    from golden_util import GRAD_NAMES
    return dict({"out_color": color, "radii": radii}, **dict(zip(GRAD_NAMES, grads)))


def call_args(d):
    e = torch.Tensor([])
    return (d["bg"], d["means3D"], d.get("colors_precomp", e), d["opacities"], d.get("scales", e),
            d.get("rotations", e), d["scale_modifier"], d.get("cov3D_precomp", e), d["viewmatrix"], d["projmatrix"],
            d["tanfovx"], d["tanfovy"], d["kernel_size"], d["subpixel_offset"], d["image_height"], d["image_width"],
            d.get("shs", e), d["sh_degree"], d["campos"], False, False)


def backward_args(d, radii, geom, R, binning, img):
    e = torch.Tensor([])
    return (d["bg"], d["means3D"], radii, d.get("colors_precomp", e), d.get("scales", e), d.get("rotations", e),
            d["scale_modifier"], d.get("cov3D_precomp", e), d["viewmatrix"], d["projmatrix"], d["tanfovx"],
            d["tanfovy"], d["kernel_size"], d["subpixel_offset"], d["dL_dpix"], d.get("shs", e), d["sh_degree"],
            d["campos"], geom, R, binning, img, False)


def path_bytes(P, V, R, N, sh_M):
    """SURVEY.md 8(d): algorithmic (compulsory) bytes of one forward and one backward."""
    A_in = 44 + (12 if sh_M == 0 else 12 * sh_M)
    A_g = 56 + (12 if sh_M == 0 else 12 * sh_M)
    B_fwd = P * (A_in + 4) + V * 40 + R * 8 + R * 36 + N * 28
    B_bwd = R * 40 + N * 28 + V * 40 + P * (A_in + A_g)
    return B_fwd, B_bwd


def stage_bytes(P, V, R, N, T, sh_M, visited, N1=0):
    """Algorithmic bytes per stage (DESIGN.md "kernels" table).  `visited` = sum over tiles of the instances the
    composite actually walks (<= R; the rest of each tile's list is occluded and never read); N1 = coarse items."""
    col = 12 if sh_M == 0 else 12 * sh_M
    return {
        "preprocess_fwd": P * (44 + (0 if sh_M == 0 else col) + 4 + 4 + 8 + 8) + V * (32 + 4),
        "depth_sort": P * 16 * 4 + P * 24,       # 4 passes, each one read + one write of the (key, id) pairs; last pass
                                                 # also delivers cell counts + rectangles in depth order
        "offset_scan": P * 8,
        "emit_cells": P * (4 + 8 + 4) + N1 * 8,
        "cell_sort": N1 * 16,                    # one pass over the coarse items (<= 256 cells)
        "cell_count": N1 * 4,
        "tile_offsets": T * 16,
        "tile_scatter": R * 4 + N1 * 8,          # the per-tile instance list itself + one read of the coarse items
        "render_fwd": visited * (4 + 32 + 12) + N * (8 + 12 + 4 + 4) + T * 8,
        "render_bwd": visited * (4 + 32 + 12 + 48) + N * (8 + 12 + 4 + 4) + T * 8,
        "preprocess_bwd": P * (4 + 44 + 56 + 12) + V * (48 + 32),
    }


# ----------------------------------------------------------------------------------------------------------
# arms
# ----------------------------------------------------------------------------------------------------------
def time_steps(step, steps, warmup, dev, world, finish=None):
    """`finish` (optional) is called after the warm-up and after the last timed step, BEFORE the closing event: a
    software-pipelined step uses it to make the timing stream wait for every copy still in flight on its side streams."""
    import torch.distributed as dist
    for _ in range(warmup):
        step()
    if finish is not None:
        finish()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    if finish is not None:
        finish()
    e1.record()
    torch.cuda.synchronize(dev)
    if world > 1:
        dist.barrier()
    ms = e0.elapsed_time(e1)
    if world > 1:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    return ms / steps


def make_e2e_step_sharded(scene, dev, settings_cls, bands):
    """Multi-GPU e2e: the host buffers hold the data once per rank (same bytes); rank r moves only the r-th 1/world of
    every tensor over PCIe in either direction (parallel.upload_sharded / download_sharded), NVLink does the rest."""
    import parallel
    keys = [k for k in ("means3D", "opacities", "scales", "rotations", "colors_precomp", "shs", "bg", "viewmatrix",
                        "projmatrix", "campos", "subpixel_offset", "dL_dpix") if k in scene]
    host = {k: scene[k].contiguous().pin_memory() for k in keys}
    leaves_k = [k for k in ("means3D", "opacities", "scales", "rotations", "colors_precomp", "shs") if k in scene]
    H, W, P = scene["image_height"], scene["image_width"], scene["means3D"].shape[0]
    out_host = {"image": torch.empty((3, H, W)).pin_memory(), "means2D": torch.empty((P, 3)).pin_memory()}
    for k in leaves_k:
        out_host[k] = torch.empty_like(scene[k]).pin_memory()
    h2d = sum(v.numel() * 4 for v in host.values())
    d2h = sum(v.numel() * 4 for v in out_host.values())

    def step():
        d = {k: parallel.upload_sharded(v, dev) for k, v in host.items()}
        st = settings_cls(image_height=H, image_width=W, tanfovx=scene["tanfovx"], tanfovy=scene["tanfovy"],
                          kernel_size=scene["kernel_size"], subpixel_offset=d["subpixel_offset"], bg=d["bg"],
                          scale_modifier=1.0, viewmatrix=d["viewmatrix"], projmatrix=d["projmatrix"],
                          sh_degree=scene["sh_degree"], campos=d["campos"], prefiltered=False, debug=False,
                          return_accumulation=True)
        leaves = {k: d[k].requires_grad_(True) for k in leaves_k}
        means2D = torch.zeros((P, 3), device=dev, requires_grad=True)
        rast = parallel.ShardedGaussianRasterizer(st, bands=bands)
        img, radii, acc = rast(means3D=leaves["means3D"], means2D=means2D, opacities=leaves["opacities"],
                               shs=leaves.get("shs"), colors_precomp=leaves.get("colors_precomp"),
                               scales=leaves.get("scales"), rotations=leaves.get("rotations"))
        (img * d["dL_dpix"]).sum().backward()
        parallel.download_sharded(img.detach(), out_host["image"])
        parallel.download_sharded(means2D.grad, out_host["means2D"])
        for k in leaves_k:
            parallel.download_sharded(leaves[k].grad, out_host[k])
        torch.cuda.current_stream(dev).synchronize()     # this rank's share of the step's result is on the host
    return step, h2d, d2h


def make_e2e_step_overlapped(mod_api, scene, dev, settings_cls, defer):
    """Public-API step with host buffers, copies overlapped with compute (this repo's arm): the H2D copies run on a copy
    stream in the order the forward needs them -- the geometry stage starts when means / scales / rotations / opacities /
    camera have landed while colours, sub-pixel offsets and the upstream gradient are still in flight
    (`defer_composite_inputs`); the image goes back to the host on a third stream while the backward runs.  Same bytes,
    same public calls (GaussianRasterizer + autograd), every copy inside the timed region."""
    geo_k = [k for k in ("means3D", "opacities", "scales", "rotations", "viewmatrix", "projmatrix", "campos") if k in scene]
    col_k = [k for k in ("colors_precomp", "shs", "bg", "subpixel_offset") if k in scene]
    host = {k: scene[k].contiguous().pin_memory() for k in geo_k + col_k + ["dL_dpix"]}
    leaves_k = [k for k in ("means3D", "opacities", "scales", "rotations", "colors_precomp", "shs") if k in scene]
    H, W, P = scene["image_height"], scene["image_width"], scene["means3D"].shape[0]
    out_host = {"image": torch.empty((3, H, W)).pin_memory(), "means2D": torch.empty((P, 3)).pin_memory()}
    for k in leaves_k:
        out_host[k] = torch.empty_like(scene[k]).pin_memory()
    h2d = sum(v.numel() * 4 for v in host.values())
    d2h = sum(v.numel() * 4 for v in out_host.values())
    up, down = torch.cuda.Stream(dev), torch.cuda.Stream(dev)

    def step():
        main = torch.cuda.current_stream(dev)
        ev_geo, ev_col, ev_dl, ev_img = (torch.cuda.Event() for _ in range(4))
        d = {}
        up.wait_stream(main)
        with torch.cuda.stream(up):
            for k in geo_k:
                d[k] = host[k].to(dev, non_blocking=True)
            ev_geo.record(up)
            for k in col_k:
                d[k] = host[k].to(dev, non_blocking=True)
            ev_col.record(up)
            d["dL_dpix"] = host["dL_dpix"].to(dev, non_blocking=True)
            ev_dl.record(up)
        main.wait_event(ev_geo)
        st = settings_cls(image_height=H, image_width=W, tanfovx=scene["tanfovx"], tanfovy=scene["tanfovy"],
                          kernel_size=scene["kernel_size"], subpixel_offset=d["subpixel_offset"], bg=d["bg"],
                          scale_modifier=1.0, viewmatrix=d["viewmatrix"], projmatrix=d["projmatrix"],
                          sh_degree=scene["sh_degree"], campos=d["campos"], prefiltered=False, debug=False,
                          return_accumulation=True)
        leaves = {k: d[k].requires_grad_(True) for k in leaves_k}
        means2D = torch.zeros((P, 3), device=dev, requires_grad=True)
        defer(ev_col)                           # colours / bg / subpixel_offset are awaited right before the composite
        img, radii, acc = mod_api(st)(means3D=leaves["means3D"], means2D=means2D, opacities=leaves["opacities"],
                                      shs=leaves.get("shs"), colors_precomp=leaves.get("colors_precomp"),
                                      scales=leaves.get("scales"), rotations=leaves.get("rotations"))
        ev_img.record(main)
        with torch.cuda.stream(down):
            down.wait_event(ev_img)
            out_host["image"].copy_(img.detach(), non_blocking=True)
        main.wait_event(ev_dl)
        (img * d["dL_dpix"]).sum().backward()
        out_host["means2D"].copy_(means2D.grad, non_blocking=True)
        for k in leaves_k:
            out_host[k].copy_(leaves[k].grad, non_blocking=True)
        main.synchronize()                      # the step's result is on the host
        down.synchronize()
    return step, h2d, d2h


def make_e2e_step_pipelined(mod_api, scene, dev, settings_cls, defer=None, depth=3, bands=None):
    """Public-API step with host buffers, software-pipelined over consecutive steps (throughput form of `e2e`).

    PCIe is full duplex and the GPU has separate copy engines per direction, so step i's device-to-host read-back
    (image + every gradient, 229 MB at C3) can overlap step i+1's host-to-device copies (209 MB) and its compute.  Every
    step still performs ALL of its copies inside the timed region, through the same public calls (GaussianRasterizer +
    autograd) as the serial form; what changes is only WHEN the host waits: it blocks on step i's completion event when
    the slot is reused `depth` steps later (and at the end of the timed region, via `finish`), not at the end of step i.
    H2D copies run on `up` in the order the forward needs them (`defer`, when the backend offers it, lets the composite
    wait for the colour inputs while the geometry stage already runs), D2H copies on `down`.  The same harness is used for
    both arms (`defer` is None for the reference).  With `bands` (multi-GPU): the tile-row sharded rasterizer, and every rank
    moves only its 1/world share of each tensor over its own PCIe link (parallel.upload_sharded / download_sharded)."""
    if bands is not None:
        import parallel
        to_dev = lambda v: parallel.upload_sharded(v, dev)
        to_host = lambda t, out: parallel.download_sharded(t, out)
        make_rast = lambda st: parallel.ShardedGaussianRasterizer(st, bands=bands)
    else:
        to_dev = lambda v: v.to(dev, non_blocking=True)
        to_host = lambda t, out: out.copy_(t, non_blocking=True)
        make_rast = mod_api
    geo_k = [k for k in ("means3D", "opacities", "scales", "rotations", "viewmatrix", "projmatrix", "campos") if k in scene]
    col_k = [k for k in ("colors_precomp", "shs", "bg", "subpixel_offset") if k in scene]
    host = {k: scene[k].contiguous().pin_memory() for k in geo_k + col_k + ["dL_dpix"]}
    leaves_k = [k for k in ("means3D", "opacities", "scales", "rotations", "colors_precomp", "shs") if k in scene]
    H, W, P = scene["image_height"], scene["image_width"], scene["means3D"].shape[0]

    def out_buffers():
        o = {"image": torch.empty((3, H, W)).pin_memory(), "means2D": torch.empty((P, 3)).pin_memory()}
        for k in leaves_k:
            o[k] = torch.empty_like(scene[k]).pin_memory()
        return o
    slots = [{"out": out_buffers(), "done": None, "keep": None} for _ in range(depth)]
    h2d = sum(v.numel() * 4 for v in host.values())
    d2h = sum(v.numel() * 4 for v in slots[0]["out"].values())
    up, down = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    count = [0]

    def step():
        slot = slots[count[0] % depth]
        count[0] += 1
        if slot["done"] is not None:
            slot["done"].synchronize()          # the result of the step that used this slot is on the host
            slot["keep"] = None
        main = torch.cuda.current_stream(dev)
        ev_geo, ev_col, ev_dl, ev_img, ev_grad, ev_done = (torch.cuda.Event() for _ in range(6))
        d = {}
        with torch.cuda.stream(up):
            for k in geo_k:
                d[k] = to_dev(host[k])
            ev_geo.record(up)
            for k in col_k:
                d[k] = to_dev(host[k])
            ev_col.record(up)
            d["dL_dpix"] = to_dev(host["dL_dpix"])
            ev_dl.record(up)
        main.wait_event(ev_geo)
        if defer is None:
            main.wait_event(ev_col)
        st = settings_cls(image_height=H, image_width=W, tanfovx=scene["tanfovx"], tanfovy=scene["tanfovy"],
                          kernel_size=scene["kernel_size"], subpixel_offset=d["subpixel_offset"], bg=d["bg"],
                          scale_modifier=1.0, viewmatrix=d["viewmatrix"], projmatrix=d["projmatrix"],
                          sh_degree=scene["sh_degree"], campos=d["campos"], prefiltered=False, debug=False,
                          return_accumulation=True)
        leaves = {k: d[k].requires_grad_(True) for k in leaves_k}
        means2D = torch.zeros((P, 3), device=dev, requires_grad=True)
        if defer is not None:
            defer(ev_col)
        img, radii, acc = make_rast(st)(means3D=leaves["means3D"], means2D=means2D, opacities=leaves["opacities"],
                                        shs=leaves.get("shs"), colors_precomp=leaves.get("colors_precomp"),
                                        scales=leaves.get("scales"), rotations=leaves.get("rotations"))
        ev_img.record(main)
        out = slot["out"]
        with torch.cuda.stream(down):
            down.wait_event(ev_img)
            to_host(img.detach(), out["image"])
        main.wait_event(ev_dl)
        (img * d["dL_dpix"]).sum().backward()
        ev_grad.record(main)
        with torch.cuda.stream(down):
            down.wait_event(ev_grad)
            to_host(means2D.grad, out["means2D"])
            for k in leaves_k:
                to_host(leaves[k].grad, out[k])
            ev_done.record(down)
        slot["done"] = ev_done
        slot["keep"] = (d, leaves, means2D, img, radii, acc)     # device buffers stay alive until the copies have run

    def finish():
        main = torch.cuda.current_stream(dev)
        main.wait_stream(up)
        main.wait_stream(down)                  # the closing event is recorded after every read-back has landed
        for s_ in slots:
            if s_["done"] is not None:
                s_["done"].synchronize()
                s_["done"], s_["keep"] = None, None
    return step, finish, h2d, d2h


def make_e2e_step(mod_api, scene, dev, settings_cls, sharded=None):
    """Public-API step with host buffers: H2D of every tensor argument from pinned memory, forward, backward,
    D2H of the image and of every gradient into pinned memory."""
    keys = [k for k in ("means3D", "opacities", "scales", "rotations", "colors_precomp", "shs", "bg", "viewmatrix",
                        "projmatrix", "campos", "subpixel_offset", "dL_dpix") if k in scene]
    host = {k: scene[k].contiguous().pin_memory() for k in keys}
    leaves_k = [k for k in ("means3D", "opacities", "scales", "rotations", "colors_precomp", "shs") if k in scene]
    H, W, P = scene["image_height"], scene["image_width"], scene["means3D"].shape[0]
    out_host = {"image": torch.empty((3, H, W)).pin_memory(), "means2D": torch.empty((P, 3)).pin_memory()}
    for k in leaves_k:
        out_host[k] = torch.empty_like(scene[k]).pin_memory()
    h2d = sum(v.numel() * 4 for v in host.values())
    d2h = sum(v.numel() * 4 for v in out_host.values())

    def step():
        d = {k: v.to(dev, non_blocking=True) for k, v in host.items()}
        st = settings_cls(image_height=H, image_width=W, tanfovx=scene["tanfovx"], tanfovy=scene["tanfovy"],
                          kernel_size=scene["kernel_size"], subpixel_offset=d["subpixel_offset"], bg=d["bg"],
                          scale_modifier=1.0, viewmatrix=d["viewmatrix"], projmatrix=d["projmatrix"],
                          sh_degree=scene["sh_degree"], campos=d["campos"], prefiltered=False, debug=False,
                          return_accumulation=True)
        leaves = {k: d[k].requires_grad_(True) for k in leaves_k}
        means2D = torch.zeros((P, 3), device=dev, requires_grad=True)
        rast = mod_api(st) if sharded is None else sharded(st)
        img, radii, acc = rast(means3D=leaves["means3D"], means2D=means2D, opacities=leaves["opacities"],
                               shs=leaves.get("shs"), colors_precomp=leaves.get("colors_precomp"),
                               scales=leaves.get("scales"), rotations=leaves.get("rotations"))
        (img * d["dL_dpix"]).sum().backward()
        out_host["image"].copy_(img.detach(), non_blocking=True)
        out_host["means2D"].copy_(means2D.grad, non_blocking=True)
        for k in leaves_k:
            out_host[k].copy_(leaves[k].grad, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()     # the step's result is on the host
    return step, h2d, d2h


def cpu_baseline(cfg_name, kw, threads=None, frac=None):
    """The CPU oracle on a bounded sample of the workload: same camera / image, a seeded subsample of the cloud."""
    from oracle import cpu_oracle
    P_full = kw["P"]
    frac = frac or min(1.0, 300_000 / P_full)
    kw2 = dict(kw); kw2["P"] = max(1000, int(P_full * frac))
    scene = synthetic.make_scene(**kw2)
    if threads:
        cpu_oracle.set_num_threads(threads)
    nthreads = cpu_oracle.num_threads()
    cpu_oracle.forward(synthetic.make_scene(P=2000, W=64, H=64, sh_degree=None, seed=0))   # load + warm
    runs = []
    for _ in range(3):                                   # median of 3: a single run varies 3x between boxes / moments
        t0 = time.perf_counter(); st = cpu_oracle.forward(scene); t1 = time.perf_counter()
        cpu_oracle.backward(st, scene["dL_dpix"]); t2 = time.perf_counter()
        runs.append((t2 - t0, t1 - t0, t2 - t1))
    runs.sort()
    tot, tf, tb = runs[1]
    N = scene["image_width"] * scene["image_height"]
    return {"value": kw2["P"] * N / tot, "unit": "gaussians*pixels/s", "cores": nthreads, "kind": "port",
            "sample": f"{cfg_name} camera/image, seeded cloud of P={kw2['P']} ({frac:.3f} of the workload), "
                      f"median of 3 fwd+bwd: fwd {1e3 * tf:.0f} ms, bwd {1e3 * tb:.0f} ms, R={st['num_rendered']}",
            "host_cores": os.cpu_count()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="C3", choices=list(synthetic.CONFIGS))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-train-step", action="store_true")
    ap.add_argument("--no-other-configs", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last timed step to DIR/<name>.npy (float32, sampled, <= 64 MB)")
    a = ap.parse_args()
    a.warmup = max(a.warmup, 3)

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if a.impl == "reference" and rank != 0:
        return 0                                    # the reference has no multi-GPU path: rank 0 alone runs it
    assert torch.cuda.is_available(), "bench.py needs a GPU (no CPU fallback for the product path)"
    dev = torch.device(f"cuda:{local_rank}")
    torch.cuda.set_device(dev)
    import torch.distributed as dist
    if world > 1 and a.impl == "ours":
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)

    kw = dict(synthetic.CONFIGS[a.config]); kw["seed"] = 0
    scene = synthetic.make_scene(**kw)
    d = synthetic.to_device(scene, dev)
    P, W, H = kw["P"], kw["W"], kw["H"]
    N = W * H
    T = ((W + 15) // 16) * ((H + 15) // 16)
    sh_M = scene["shs"].shape[1] if "shs" in scene else 0
    peak, peak_src = peaks()
    workload = f"{a.config}: {P} Gaussians, {W}x{H}, " + ("colors_precomp" if sh_M == 0 else f"SH deg {scene['sh_degree']} in-kernel")

    line = {"metric": "gaussians_pixels_per_s (forward+backward rasterize)", "unit": "gaussians*pixels/s",
            "n_gpus": world if a.impl == "ours" else 1, "steps": a.steps, "warmup": a.warmup,
            "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic (seeded, SURVEY.md 8d generator)",
            "config": {"workload": workload, "P": P, "W": W, "H": H, "tiles": T,
                       "l2": "inputs_larger_than_l2 (per-step working set >= 0.5 GB vs 50 MB L2)",
                       "parallelism": "single GPU" if world == 1 else f"tile-row bands x{world}, " + {
                           "0": "NCCL all-gather (image) + all-reduce (partials)",
                           "1": "image all-gather fused into the forward composite (peer stores) and partial-gradient reduction fused "
                                "into the backward composite (peer red.add into every rank's accumulator) over NVLink symmetric memory",
                           "2": "image all-gather fused into the forward composite (peer stores), partial-gradient reduction through "
                                "the NVSwitch multicast address (multimem.red) from inside the backward composite",
                           "3": "image all-gather fused into the forward composite (peer stores); backward: local sums + marks, the "
                                "chain-rule kernel pulls the other ranks' marked rows over NVLink (no remote atomics)",
                       }.get(os.environ.get("GSR_PEER_REDUCE", "3" if world >= 3 else "1"), "?")}}     # parallel.peer_mode()

    sampler = ClockSampler(local_rank)

    # ------------------------------------------------------------------ reference arm
    if a.impl == "reference":
        from oracle import ref_cuda
        line["impl"] = "reference"
        if ref_cuda.available():
            mod = ref_cuda
            last = {}
            def step():
                R, color, radii, geom, binning, img = mod.rasterize_gaussians(*call_args(d))
                grads = mod.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))
                last.update(out=(color, radii, grads))
            sampler.start()
            ms = time_steps(step, a.steps, a.warmup, dev, 1)
            if a.dump_outputs:
                dump_outputs(a.dump_outputs, P, step_outputs(*last["out"]))
                last.clear()
            line.update(value=P * N / (ms * 1e-3), ms_per_step=ms,
                        reference_kind="unmodified reference CUDA rasterizer compiled for sm_90a (oracle/_ref/libdgr_ref.so), "
                                       "legacy default stream, run on the GPU: the reference has no CPU implementation of this path")
            # e2e with the same host-buffer harness, through the reference's own Python surface re-created around its _C
            if not a.no_e2e:
                api = make_reference_api(mod)
                p_step, p_fin, h2d, d2h = make_e2e_step_pipelined(api["GaussianRasterizer"], scene, dev,
                                                                  api["GaussianRasterizationSettings"], None)
                e_ms = time_steps(p_step, max(4, a.steps // 2), 3, dev, 1, finish=p_fin)
                del p_step, p_fin
                torch.cuda.empty_cache()
                s_step, _, _ = make_e2e_step(api["GaussianRasterizer"], scene, dev, api["GaussianRasterizationSettings"])
                s_ms = time_steps(s_step, max(3, a.steps // 2), 3, dev, 1)
                best = min(e_ms, s_ms)      # the reference gets the better of the two forms (its 15 ms of compute hide little)
                line["e2e"] = {"value": P * N / (best * 1e-3), "unit": line["unit"], "ms_per_step": best,
                               "ms_per_step_pipelined": e_ms, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                               "ms_per_step_serial_copies": s_ms,
                               "note": E2E_NOTE + ".  Reference arm: value = the FASTER of its pipelined and serial forms"}
            if a.config == "C3" and not a.no_other_configs:
                def factory(dd):
                    st = {}
                    def stp():
                        R_, color_, radii_, geom_, binning_, img_ = mod.rasterize_gaussians(*call_args(dd))
                        mod.rasterize_gaussians_backward(*backward_args(dd, radii_, geom_, R_, binning_, img_))
                        st.update(R=R_, radii=radii_)
                    return stp, (lambda: (int(st["R"]), int((st["radii"] > 0).sum())))
                try:
                    line["other_configs"] = other_config_lines(factory, dev, max(3, a.steps // 4), peaks()[0])
                except Exception as e:
                    line["other_configs"] = {"unavailable": f"{type(e).__name__}: {e}"}
            line["clocks"] = sampler.stop()
            line["gpu_launches"] = None
            line["cpu_baseline"] = {"value": line["value"], "unit": line["unit"], "kind": "reference", "cores": 0,
                                    "sample": "the line's own value: the reference has no CPU implementation of this path, this "
                                              "arm ran its unmodified CUDA implementation (oracle/_ref/libdgr_ref.so) on the GPU"}
        else:
            cb = cpu_baseline(a.config, kw)
            line.update(value=cb["value"], ms_per_step=None, cpu_baseline=cb,
                        reference_kind="oracle/_ref/libdgr_ref.so not present: CPU oracle port on the host cores",
                        e2e={"value": cb["value"], "unit": cb["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0})
        print(json.dumps(line))
        return 0

    # ------------------------------------------------------------------ our arm
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer, _C
    import parallel
    line["impl"] = "ours"
    # every timed step is a FULL forward (projection + binning + composite): the geometry reuse between consecutive
    # calls on identical tensors (SURVEY 8f-1) is switched off here and measured separately ("two_pass" below)
    _C.set_geometry_cache(False)
    bands = None
    if world > 1:
        rows = (H + 15) // 16
        bands = parallel.partition_tile_rows(rows, world)
        band = bands[rank]

    if world == 1:
        state = {}
        def step():
            R, color, radii, geom, binning, img = _C.rasterize_gaussians(*call_args(d))
            grads = _C.rasterize_gaussians_backward_lean(*backward_args(d, radii, geom, R, binning, img))
            state.update(R=R, radii=radii, geom=geom, binning=binning, img=img, color=color, grads=grads)
    else:
        state = {}
        def step():
            full, R, radii, geom, binning, img = parallel.sharded_forward(call_args(d), bands)
            grads = parallel.sharded_backward(backward_args(d, radii, geom, R, binning, img), bands)
            state.update(R=R, radii=radii, geom=geom, binning=binning, img=img, full=full, grads=grads)

    check = None
    if world > 1:
        # SCALE carries its own correctness: the sharded result of THIS run against the single-GPU result on the same
        # tensors (image bit for bit, gradients within the atomics tolerance), on every rank
        step()
        torch.cuda.synchronize(dev)
        R1, color1, radii1, geom1, binning1, img1 = _C.rasterize_gaussians(*call_args(d))
        g1 = _C.rasterize_gaussians_backward_lean(*backward_args(d, radii1, geom1, R1, binning1, img1))
        torch.cuda.synchronize(dev)
        ok_img = bool(torch.equal(state["full"][:3], color1)) and bool(torch.equal(state["radii"], radii1))
        worst = 0.0
        for a_, b_ in zip(state["grads"], g1):
            if a_ is None or b_ is None or b_.numel() == 0:
                continue
            worst = max(worst, float((a_ - b_).abs().max()) / (float(b_.abs().max()) + 1e-30))
        flags = torch.tensor([1.0 if ok_img else 0.0, worst], dtype=torch.float64, device=dev)
        mn = flags.clone(); dist.all_reduce(mn, op=dist.ReduceOp.MIN)
        mx = flags.clone(); dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        check = {"image_and_radii_bit_identical_to_single_gpu_on_every_rank": bool(mn[0].item() == 1.0),
                 "max_gradient_rel_err_over_ranks": float(mx[1].item()), "gradient_tolerance": 1e-3,
                 "passed": bool(mn[0].item() == 1.0 and mx[1].item() < 1e-3)}
        del R1, color1, radii1, geom1, binning1, img1, g1
    launches0 = _C.launch_count()
    sampler.start()
    ms = time_steps(step, a.steps, a.warmup, dev, world)
    launches = (_C.launch_count() - launches0) // (a.steps + a.warmup) * a.steps
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, P, step_outputs(state["color"] if world == 1 else state["full"], state["radii"],
                                                     state["grads"]))
    state.pop("color", None); state.pop("grads", None); state.pop("full", None)

    # separate fwd / bwd times and per-stage times: K profiled steps right after the timed region
    R = state["R"]
    V = int((state["radii"] > 0).sum())
    if world == 1:
        views = _C.debug_views(state["geom"], state["binning"], state["img"], P, sh_M, W, H, R)
        ncontrib = views["n_contrib"].view(-1)
        # instances each tile's composite walks = max n_contrib over the tile's pixels
        nc = views["n_contrib"].float()
        pad_h, pad_w = (16 - H % 16) % 16, (16 - W % 16) % 16
        ncp = torch.nn.functional.pad(nc, (0, pad_w, 0, pad_h))
        tile_max = ncp.view((H + pad_h) // 16, 16, (W + pad_w) // 16, 16).amax(dim=(1, 3))
        visited = int(tile_max.sum())
        blended_sum = int(ncontrib.long().sum())
    else:
        visited, blended_sum = 0, 0
    _C.profile_enable(True)
    acc, tf, tb = {}, [], []
    for _ in range(a.steps):
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        if world == 1:
            e0.record()
            Rr, color, radii, geom, binning, img = _C.rasterize_gaussians(*call_args(d))
            e1.record()
            _C.rasterize_gaussians_backward_lean(*backward_args(d, radii, geom, Rr, binning, img))
            e2.record()
        else:
            e0.record(); step(); e1.record(); e2.record()
        torch.cuda.synchronize(dev)
        tf.append(e0.elapsed_time(e1)); tb.append(e1.elapsed_time(e2))
        for k, v in _C.profile_read().items():
            acc.setdefault(k, []).append(v)
    _C.profile_enable(False)
    clocks = sampler.stop()      # sampled over warm-up + timed steps + the profiled steps (same kernels, GPU busy throughout)
    stage_ms = {k: float(np.mean(v)) for k, v in acc.items()}

    value = P * N / (ms * 1e-3)
    line.update(value=value, ms_per_step=ms, gpu_launches=int(launches), clocks=clocks,
                fwd_ms=float(np.median(tf)), bwd_ms=float(np.median(tb)) if world == 1 else None,
                counts={"P": P, "V": V, "R": int(R), "N": N, "tiles": T, "visited_instances": visited,
                        "sum_n_contrib": blended_sum})
    if world == 1:
        N1 = int(_C.stats(state["geom"], P, sh_M).get("num_coarse", 0))
        sb = stage_bytes(P, V, R, N, T, sh_M, visited, N1)
        stages = {k: {"ms": stage_ms[k], "alg_bytes": int(sb[k]), "gbs": sb[k] / (stage_ms[k] * 1e-3) / 1e9,
                      "frac_of_hbm_peak": sb[k] / (stage_ms[k] * 1e-3) / 1e9 / peak} for k in stage_ms if k in sb}
        dom = max(stages, key=lambda k: stages[k]["ms"])
        line["stages"] = stages
        line["roofline"] = {"bound": "hbm", "kernel": dom, "achieved": stages[dom]["gbs"], "peak": peak, "unit": "GB/s",
                            "frac": stages[dom]["gbs"] / peak, "peak_source": peak_src,
                            "alg_bytes_per_launch": stages[dom]["alg_bytes"], "launch_ms": stages[dom]["ms"]}
        Bf, Bb = path_bytes(P, V, R, N, sh_M)
        # second reading: the formula charges R * (36 + 40) B of per-instance delivery, but only `visited` of the R list
        # entries are ever walked before the pixels saturate (the rest is never read): delivery terms with `visited`
        Bw = (Bf - R * 36 + visited * 36) + (Bb - R * 40 + visited * 40)
        line["roofline_path"] = {"bound": "hbm", "B_fwd": int(Bf), "B_bwd": int(Bb), "achieved": (Bf + Bb) / (ms * 1e-3) / 1e9,
                                 "peak": peak, "unit": "GB/s", "frac": (Bf + Bb) / (ms * 1e-3) / 1e9 / peak,
                                 "formula": "SURVEY.md 8(d)",
                                 "bytes_with_walked_instances": int(Bw),
                                 "frac_with_walked_instances": Bw / (ms * 1e-3) / 1e9 / peak}
    else:
        # rank 0's stages against the per-GPU HBM peak (rank-local algorithmic bytes: its band's instances and
        # pixels, all P Gaussians for the replicated per-Gaussian stages); whole-path figure against N x peak
        vis_local, hb = 0, 0
        try:
            views = _C.debug_views(state["geom"], state["binning"], state["img"], P, sh_M, W, H, R)
            r0, r1 = min(H, 16 * band[0]), min(H, 16 * band[1])
            nc = views["n_contrib"][r0:r1].float()
            hb = r1 - r0
            pad_h, pad_w = (16 - hb % 16) % 16, (16 - W % 16) % 16
            ncp = torch.nn.functional.pad(nc, (0, pad_w, 0, pad_h))
            vis_local = int(ncp.view((hb + pad_h) // 16, 16, (W + pad_w) // 16, 16).amax(dim=(1, 3)).sum()) if hb > 0 else 0
        except Exception:
            pass
        # the collective is unconditional (every rank reaches it whatever happened above)
        tot = torch.tensor([float(R), float(vis_local)], dtype=torch.float64, device=dev)
        dist.all_reduce(tot)
        try:
            R_tot, vis_tot = int(tot[0].item()), int(tot[1].item())
            N1 = int(_C.stats(state["geom"], P, sh_M).get("num_coarse", 0))
            T_band = ((W + 15) // 16) * max(0, band[1] - band[0])
            sb = stage_bytes(P, V, R, hb * W, T_band, sh_M, vis_local, N1)
            stages = {k: {"ms": stage_ms[k], "alg_bytes": int(sb[k]), "gbs": sb[k] / (stage_ms[k] * 1e-3) / 1e9,
                          "frac_of_hbm_peak": sb[k] / (stage_ms[k] * 1e-3) / 1e9 / peak} for k in stage_ms if k in sb}
            dom = max(stages, key=lambda k: stages[k]["ms"])
            line["stages"] = stages
            line["roofline"] = {"bound": "hbm", "kernel": dom, "rank": 0, "achieved": stages[dom]["gbs"], "peak": peak,
                                "unit": "GB/s", "frac": stages[dom]["gbs"] / peak, "peak_source": peak_src,
                                "alg_bytes_per_launch": stages[dom]["alg_bytes"], "launch_ms": stages[dom]["ms"]}
            Bf, Bb = path_bytes(P, V, R_tot, N, sh_M)
            line["roofline_path"] = {"bound": "hbm", "B_fwd": int(Bf), "B_bwd": int(Bb),
                                     "achieved": (Bf + Bb) / (ms * 1e-3) / 1e9, "peak": peak * world, "unit": "GB/s",
                                     "frac": (Bf + Bb) / (ms * 1e-3) / 1e9 / (peak * world),
                                     "formula": "SURVEY.md 8(d), whole job, against world x per-GPU peak"}
            line["counts"].update(R=R_tot, R_rank0=int(R), visited_instances=vis_tot)
        except Exception as e:                       # reporting only: never lose the timing line
            line["stages"] = {k: {"ms": v} for k, v in stage_ms.items()}
            line["roofline"] = None
            line["roofline_note"] = f"not computed: {type(e).__name__}: {e}"
        line["bands"] = bands
        line["check"] = check

    # SURVEY 8f-1: wild-gaussians' step composites the same Gaussians twice (raw + appearance-toned colours,
    # method.py:1573-1611): two forwards + two backwards, with and without reuse of the first pass's geometry/binning
    if world == 1:
        d2 = dict(d); d2["colors_precomp"] = (1.0 - d["colors_precomp"]).contiguous() if "colors_precomp" in d else None
        if d2["colors_precomp"] is not None:
            def two_pass():
                _C.clear_geometry_cache()
                f1 = _C.rasterize_gaussians(*call_args(d))
                f2 = _C.rasterize_gaussians(*call_args(d2))
                _C.rasterize_gaussians_backward_lean(*backward_args(d2, f2[2], f2[3], f2[0], f2[4], f2[5]))
                _C.rasterize_gaussians_backward_lean(*backward_args(d, f1[2], f1[3], f1[0], f1[4], f1[5]))
            tp = {}
            for name, on in (("ms_reuse_geometry", True), ("ms_independent_passes", False)):
                _C.set_geometry_cache(on)
                tp[name] = time_steps(two_pass, max(3, a.steps // 2), 3, dev, 1)
            _C.set_geometry_cache(False)
            tp["what"] = "2 forwards (different colours, same geometry) + 2 backwards, device-timed"
            line["two_pass"] = tp

    # BASELINE config 3's "full train step": the reference's own, unmodified wildgaussians/method.py
    # (GaussianModel._render_internal: appearance MLP + SH colours in PyTorch, two rasterizer passes) + loss + backward
    if world == 1 and not a.no_train_step and sh_M == 0:
        try:
            line["train_step"] = full_train_step(kw, dev, max(3, a.steps // 4), a.impl)
        except Exception as e:          # reporting only: never lose the timing line
            line["train_step"] = {"unavailable": f"{type(e).__name__}: {e}"}

    if world == 1 and a.config == "C3" and not a.no_other_configs:
        def factory(dd):
            st = {}
            def stp():
                R_, color_, radii_, geom_, binning_, img_ = _C.rasterize_gaussians(*call_args(dd))
                _C.rasterize_gaussians_backward_lean(*backward_args(dd, radii_, geom_, R_, binning_, img_))
                st.update(R=R_, radii=radii_)
            return stp, (lambda: (int(st["R"]), int((st["radii"] > 0).sum())))
        try:
            line["other_configs"] = other_config_lines(factory, dev, max(3, a.steps // 4), peak)
        except Exception as e:
            line["other_configs"] = {"unavailable": f"{type(e).__name__}: {e}"}

    if world == 1 and not a.no_train_step and sh_M == 0:
        try:
            line["colour_op"] = colour_op_bench(P, dev, max(3, a.steps // 4))
        except Exception as e:
            line["colour_op"] = {"unavailable": f"{type(e).__name__}: {e}"}

    # e2e through the public API with host buffers
    if not a.no_e2e:
        if world > 1:
            e_step, h2d, d2h = make_e2e_step_sharded(scene, dev, GaussianRasterizationSettings, bands)
        else:
            import diff_gaussian_rasterization as dgr
            e_step, h2d, d2h = make_e2e_step_overlapped(GaussianRasterizer, scene, dev, GaussianRasterizationSettings,
                                                        dgr.defer_composite_inputs)
        # headline: software-pipelined over consecutive steps (throughput); the same harness times the reference arm
        if world == 1:
            p_step, p_fin, h2d, d2h = make_e2e_step_pipelined(GaussianRasterizer, scene, dev, GaussianRasterizationSettings,
                                                              dgr.defer_composite_inputs)
        else:
            p_step, p_fin, h2d, d2h = make_e2e_step_pipelined(None, scene, dev, GaussianRasterizationSettings, None, bands=bands)
        p_ms = time_steps(p_step, max(4, a.steps // 2), 3, dev, world, finish=p_fin)
        del p_step, p_fin
        torch.cuda.empty_cache()
        e_ms = time_steps(e_step, max(3, a.steps // 2), 3, dev, world)
        best = min(p_ms, e_ms)          # every arm reports the faster of its forms (the reference arm does the same)
        line["e2e"] = {"value": P * N / (best * 1e-3), "unit": line["unit"], "ms_per_step": best, "ms_per_step_pipelined": p_ms,
                       "ms_per_step_one_step_in_flight": e_ms, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h}
        if world == 1:
            s_step, _, _ = make_e2e_step(GaussianRasterizer, scene, dev, GaussianRasterizationSettings, None)
            line["e2e"]["ms_per_step_serial_copies"] = time_steps(s_step, max(3, a.steps // 2), 3, dev, 1)
            line["e2e"]["note"] = E2E_NOTE
        if world > 1:
            line["e2e"]["note"] = E2E_NOTE + (".  Multi-GPU: whole-job bytes per step; each rank moves 1/world of every tensor over "
                                              "its own PCIe link (parallel.upload_sharded / download_sharded), NVLink all-gathers the inputs")

    if rank == 0 and world == 1 and not a.no_cpu_baseline:
        line["cpu_baseline"] = cpu_baseline(a.config, kw)
        # BASELINE.json config 1 (10k Gaussians, 256x256, SH degree 0: "the reference's own CPU-runnable case") in full, not sampled
        kw1 = dict(synthetic.CONFIGS["C1"]); kw1["seed"] = 0
        c1 = cpu_baseline("C1", kw1, frac=1.0)
        line["cpu_baseline"]["config1"] = {"value": c1["value"], "unit": c1["unit"], "cores": c1["cores"], "sample": c1["sample"]}
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    if rank == 0:
        print(json.dumps(line))
    return 0


def other_config_lines(impl_step_factory, dev, steps, peak, names=("C2", "C5")):
    """BASELINE.json configs 2 (500k, 800x800, SH degree 3 in-kernel) and 5 on ONE GPU (6M, 4096x2160): device-timed
    forward+backward ms with the same timing loop as the headline, so that the driver's record carries them too."""
    out = {}
    for name in names:
        kw = dict(synthetic.CONFIGS[name]); kw["seed"] = 0
        scene = synthetic.make_scene(**kw)
        d = synthetic.to_device(scene, dev)
        P, W, H = kw["P"], kw["W"], kw["H"]
        sh_M = scene["shs"].shape[1] if "shs" in scene else 0
        step, info = impl_step_factory(d)
        ms = time_steps(step, steps, 3, dev, 1)
        R, V = info()
        Bf, Bb = path_bytes(P, V, R, W * H, sh_M)
        out[name] = {"workload": f"{P} Gaussians, {W}x{H}, " + ("colors_precomp" if sh_M == 0 else f"SH deg {scene['sh_degree']} in-kernel"),
                     "ms_per_step": ms, "value": P * W * H / (ms * 1e-3), "R": R, "V": V,
                     "roofline_path_frac": (Bf + Bb) / (ms * 1e-3) / 1e9 / peak}
        del d, scene
        torch.cuda.empty_cache()
    return out


def colour_op_bench(P, dev, steps):
    """SURVEY 8f-2: the fused per-Gaussian colour op (csrc/appearance.cu, wgmma) on P rows next to the PyTorch statements
    it replaces (oracle/color_torch.py = method.py:1570-1598 in fp32), forward and forward+backward, CUDA events."""
    import fused_colors as fc
    from oracle import color_torch as ct
    g = torch.Generator().manual_seed(11)
    R = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(dev)
    dc, rest, gemb, aemb = R(P, 3), R(P, 45, scale=0.3), R(P, 24, scale=0.5), R(32, scale=0.5)
    means, campos = R(P, 3, scale=2.0), torch.tensor([0.1, -0.2, 0.3], device=dev)
    torch.manual_seed(3)
    mlp = torch.nn.Sequential(torch.nn.Linear(59, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128), torch.nn.ReLU(),
                              torch.nn.Linear(128, 6)).to(dev)
    with torch.no_grad():
        mlp[4].bias[3:] = 80.0
    dLr, dLt = R(P, 3), R(P, 3)
    leaves = [t.clone().requires_grad_(True) for t in (dc, rest, gemb, aemb, means)]
    lin = [mlp[0], mlp[2], mlp[4]]

    def zero():
        for t in leaves + list(mlp.parameters()):
            t.grad = None

    def fused_fwd():
        with torch.no_grad():
            fc.fused_colors(*leaves[:4], mlp, leaves[4], campos, 3)

    def fused_fb():
        zero()
        raw, toned = fc.fused_colors(*leaves[:4], mlp, leaves[4], campos, 3)
        torch.autograd.backward([raw, toned], [dLr, dLt])

    def torch_fwd():
        with torch.no_grad():
            ct.colors(*leaves[:4], lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias, lin[2].weight, lin[2].bias, leaves[4],
                      campos, 3)

    def torch_fb():
        zero()
        raw, toned = ct.colors(*leaves[:4], lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias, lin[2].weight, lin[2].bias,
                               leaves[4], campos, 3)
        torch.autograd.backward([raw, toned], [dLr, dLt])

    res = {"P": P, "what": "raw + toned colours of P Gaussians (59->128->128->6 MLP + SH degree 3 + clamps), CUDA events, ms"}
    for name, fn in (("fused_fwd_ms", fused_fwd), ("fused_fwd_bwd_ms", fused_fb), ("torch_fp32_fwd_ms", torch_fwd),
                     ("torch_fp32_fwd_bwd_ms", torch_fb)):
        res[name] = time_steps(fn, steps, 3, dev, 1)
    zero()
    fwd_flop = 2.0 * P * (32 * 128 + 144 * 128 + 144 * 16)
    bwd_flop = fwd_flop + 2.0 * P * (16 * 128 + 128 * 128 + 128 * 32) + 2.0 * P * (128 * 16 + 128 * 144 + 128 * 32)
    try:
        pk = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["bf16_tflops_sustained"])
    except Exception:
        pk = None
    bwd_ms = res["fused_fwd_bwd_ms"] - res["fused_fwd_ms"]
    res["roofline"] = {"bound": "tensor", "unit": "TFLOP/s", "peak": pk, "peak_source": "MEASURED_PEAKS.json bf16_tflops_sustained",
                       "fwd_achieved": fwd_flop / (res["fused_fwd_ms"] * 1e-3) / 1e12,
                       "bwd_achieved": bwd_flop / (max(bwd_ms, 1e-6) * 1e-3) / 1e12,
                       "fwd_frac": None if not pk else fwd_flop / (res["fused_fwd_ms"] * 1e-3) / 1e12 / pk,
                       "hbm_bytes_fwd": P * (3 + 45 + 24 + 3 + 6) * 4, "hbm_bytes_bwd": P * (3 + 45 + 24 + 3 + 6 + 3 + 45 + 24 + 3) * 4,
                       "note": "MMA flops as issued (K padded to 32 / 144, N to 16); the op is bounded by the CUDA-core epilogues "
                               "(ReLU + bf16 pack + SH) and by HBM, not by the tensor pipe"}
    return res


def full_train_step(kw, dev, steps, impl="ours"):
    """ms per step of `GaussianModel._render_internal` + loss + backward (unmodified wildgaussians/method.py from
    oracle/_ref/py, see tests/wg_harness.py) on a cloud of the workload's size with SH degree 3 + 32-d appearance
    embedding (BASELINE.json config 3), on this repo's rasterizer and on the reference's compiled CUDA core."""
    import wg_harness as wh
    m, Config = wh.import_method()
    if m is None:
        return {"unavailable": "reference python package not present (oracle/_ref/py)"}
    import diff_gaussian_rasterization as ours
    from oracle import ref_cuda
    kw3 = dict(kw); kw3["sh_degree"] = 3
    scene = synthetic.make_scene(**kw3)
    model, cfg = wh.make_model(m, Config, scene, dev)
    cam = wh.make_camera(scene)
    H, W = scene["image_height"], scene["image_width"]
    g = torch.Generator().manual_seed(5)
    G1, G2 = torch.randn(3, H, W, generator=g).to(dev), torch.randn(3, H, W, generator=g).to(dev)
    res = {"what": "unmodified wildgaussians/method.py GaussianModel._render_internal (appearance on, uncertainty off, two "
                   "rasterizer passes) + (render*G1).sum() + (raw_render*G2).sum() + backward; CUDA events, ms per step",
           "P": kw3["P"], "W": W, "H": H, "steps": steps}
    arms = [("ours_ms", ours.GaussianRasterizer, ours.GaussianRasterizationSettings)]
    if ref_cuda.available():
        api = make_reference_api(ref_cuda)
        arms.append(("reference_rasterizer_ms", api["GaussianRasterizer"], api["GaussianRasterizationSettings"]))
    ours._C.set_geometry_cache(True)
    try:
        for name, rcls, scls in arms:
            wh.use_backend(m, rcls, scls)
            res[name] = time_steps(lambda: wh.train_step(model, cfg, cam, G1, G2), steps, 3, dev, 1)
        # opt-in fused caller (wildgaussians_fused.enable): fused wgmma colour op + cached camera constants, same
        # rasterizer, method.py still unmodified
        import wildgaussians_fused as wf
        wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
        wf.enable(model)
        res["ours_fused_caller_ms"] = time_steps(lambda: wh.train_step(model, cfg, cam, G1, G2), steps, 3, dev, 1)
        wf.disable(model)
        # SURVEY 8f-4: the optimizer step of the iteration (method.py:2019) on the optimizer the unmodified
        # `_setup_optimizers` (method.py:1029-1053) builds: PyTorch's Adam (foreach path) vs the same object adopted by
        # fused_adam (one kernel, csrc/adam.cu); gradients = those of the last train step, kept alive across the timed steps
        try:
            import fused_adam
            model.spatial_lr_scale.fill_(1.7)
            model._setup_optimizers()
            wh.train_step(model, cfg, cam, G1, G2)
            n_el = sum(p.numel() for g_ in model.optimizer.param_groups for p in g_["params"] if p.grad is not None)
            opt = {"elements": n_el, "alg_bytes": 28 * n_el,
                   "what": "model.optimizer.step() (Adam, 10 parameter groups incl. the appearance MLP), CUDA events, ms"}
            opt["torch_adam_ms"] = time_steps(model.optimizer.step, steps, 3, dev, 1)
            fused_adam.adopt(model.optimizer)
            opt["fused_adam_ms"] = time_steps(model.optimizer.step, steps, 3, dev, 1)
            opt["fused_gbs"] = opt["alg_bytes"] / (opt["fused_adam_ms"] * 1e-3) / 1e9
            opt["fused_frac_of_hbm_peak"] = opt["fused_gbs"] / peaks()[0]
            res["optimizer_step"] = opt
        except Exception as e:          # reporting only
            res["optimizer_step"] = {"unavailable": f"{type(e).__name__}: {e}"}
    finally:
        wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
        ours._C.set_geometry_cache(False)
    return res


def make_reference_api(_C):
    """The reference's Python surface (autograd.Function + nn.Module, __init__.py:46-241) re-created around a
    `_C`-like module, so that the reference arm's e2e goes through the same kind of public call as ours."""
    from typing import NamedTuple

    class Settings(NamedTuple):
        image_height: int; image_width: int; tanfovx: float; tanfovy: float; kernel_size: float
        subpixel_offset: torch.Tensor; bg: torch.Tensor; scale_modifier: float; viewmatrix: torch.Tensor
        projmatrix: torch.Tensor; sh_degree: int; campos: torch.Tensor; prefiltered: bool; debug: bool
        return_accumulation: bool

    class Fn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, means3D, means2D, sh, colors, opac, scales, rots, cov, s):
            R, color, radii, geom, binning, img = _C.rasterize_gaussians(
                s.bg, means3D, colors, opac, scales, rots, s.scale_modifier, cov, s.viewmatrix, s.projmatrix,
                s.tanfovx, s.tanfovy, s.kernel_size, s.subpixel_offset, s.image_height, s.image_width, sh,
                s.sh_degree, s.campos, s.prefiltered, s.debug)
            ctx.s, ctx.R = s, R
            ctx.save_for_backward(colors, means3D, scales, rots, cov, radii, sh, geom, binning, img)
            off = (128 - img.data_ptr()) % 128
            n = 4 * s.image_height * s.image_width
            acc = img[off:off + n].view(torch.float32).clone().mul_(-1).add_(1).view(s.image_height, s.image_width)
            return color, radii, acc

        @staticmethod
        def backward(ctx, g, _1, _2):
            s = ctx.s
            colors, means3D, scales, rots, cov, radii, sh, geom, binning, img = ctx.saved_tensors
            gm2, gc, go, gm3, gcov, gsh, gs, gr = _C.rasterize_gaussians_backward(
                s.bg, means3D, radii, colors, scales, rots, s.scale_modifier, cov, s.viewmatrix, s.projmatrix,
                s.tanfovx, s.tanfovy, s.kernel_size, s.subpixel_offset, g, sh, s.sh_degree, s.campos, geom, ctx.R,
                binning, img, s.debug)
            return gm3, gm2, gsh, gc, go, gs, gr, gcov, None

    class Rasterizer(torch.nn.Module):
        def __init__(self, raster_settings):
            super().__init__()
            self.raster_settings = raster_settings

        def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                    cov3D_precomp=None):
            e = torch.Tensor([])
            return Fn.apply(means3D, means2D, e if shs is None else shs, e if colors_precomp is None else colors_precomp,
                            opacities, e if scales is None else scales, e if rotations is None else rotations,
                            e if cov3D_precomp is None else cov3D_precomp, self.raster_settings)

    return {"GaussianRasterizationSettings": Settings, "GaussianRasterizer": Rasterizer}


if __name__ == "__main__":
    sys.exit(main())
