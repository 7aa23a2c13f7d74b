"""Diagnostic (run on the GPU box): ours (libgsrast.so) vs the compiled reference (oracle/_ref/libdgr_ref.so)
vs the CPU oracle, stage by stage, plus A/B timings.  Not part of the product; the pytest parity tests in
tests/test_gpu_parity.py are the gate, this prints the detail needed to debug a mismatch.

usage: python tools/gpu_compare.py [--cases small|all] [--time C2,C3] [--out compare.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "wild-gaussians_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import synthetic  # noqa: E402
from make_golden import CASES, backward_args, call_args  # noqa: E402


def bits_equal(a, b):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    if a.shape != b.shape:
        return False, -1
    av = a.view(np.uint32) if a.dtype == np.float32 else a
    bv = b.view(np.uint32) if b.dtype == np.float32 else b
    ne = int((av != bv).sum())
    return ne == 0, ne


def run_ours(d):
    from diff_gaussian_rasterization import _C
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(*call_args(d))
    P = d["means3D"].shape[0]
    M = d["shs"].shape[1] if "shs" in d else 0
    v = _C.debug_views(geom, binning, img, P, M, d["image_width"], d["image_height"], R)
    grads = _C.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))
    torch.cuda.synchronize()
    return R, color, radii, v, grads, (geom, binning, img)


def run_ref(d):
    from oracle import ref_cuda
    R, color, radii, geom, binning, img = ref_cuda.rasterize_gaussians(*call_args(d))
    P = d["means3D"].shape[0]
    v = ref_cuda.debug_views(geom, binning, img, P, d["image_width"], d["image_height"], R)
    grads = ref_cuda.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))
    torch.cuda.synchronize()
    return R, color, radii, v, grads, (geom, binning, img)


GRAD_NAMES = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales",
              "dL_drotations")


def compare_case(name, kw, dev, with_oracle=True):
    scene = synthetic.make_scene(**kw)
    d = synthetic.to_device(scene, dev)
    rep = {"case": name}
    Ro, co, ro, vo, go, _ = run_ours(d)
    Rr, cr, rr, vr, gr, _ = run_ref(d)
    Rr2, cr2, rr2, vr2, gr2, _ = run_ref(d)
    rep["R"] = [int(Ro), int(Rr)]
    vis = (rr > 0)
    rep["V"] = int(vis.sum())
    rep["radii_equal"] = bool(torch.equal(ro, rr))
    rep["tiles_touched_ne"] = int((vo["tiles_touched"][vis] != vr["tiles_touched"][vis]).sum())
    visn = vis.cpu().numpy()
    for ours_k, ref_k, sl in (("depths", "depths", None), ("xy", "means2D", slice(0, 2)),
                              ("conic_opacity", "conic_opacity", None)):
        if ours_k == "depths":
            a = vo["depths"].cpu().numpy()[visn]; b = vr["depths"].cpu().numpy()[visn]
        elif ours_k == "xy":
            a = vo["records"].cpu().numpy()[visn][:, 0:2]; b = vr["means2D"].cpu().numpy()[visn]
        else:
            rec = vo["records"].cpu().numpy()[visn]
            a = np.ascontiguousarray(rec[:, [4, 5, 6, 7]]); b = vr["conic_opacity"].cpu().numpy()[visn]
        ok, ne = bits_equal(a, b)
        rep[ours_k + "_bits_ne"] = ne
        if ne:
            rep[ours_k + "_maxabs"] = float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())
    if "shs" in d:
        ok, ne = bits_equal(vo["rgb"].cpu().numpy()[visn], vr["rgb"].cpu().numpy()[visn])
        rep["rgb_bits_ne"] = ne
    if Ro == Rr:
        rep["point_list_ne"] = int((vo["point_list"] != vr["point_list"]).sum())
        rep["ranges_ne"] = int((vo["ranges"] != vr["ranges"]).sum())
    rep["n_contrib_ne"] = int((vo["n_contrib"] != vr["n_contrib"]).sum())
    rep["final_T_bits_ne"] = bits_equal(vo["final_T"].cpu().numpy(), vr["final_T"].cpu().numpy())[1]
    rep["color_bits_ne"] = bits_equal(co.cpu().numpy(), cr.cpu().numpy())[1]
    rep["color_maxabs"] = float((co - cr).abs().max())
    rep["n_contrib_mean_max"] = [float(vr["n_contrib"].float().mean()), int(vr["n_contrib"].max())]
    for n, a, b, b2 in zip(GRAD_NAMES, go, gr, gr2):
        if b.numel() == 0:
            continue
        scale = float(b.abs().max()) + 1e-30
        rep["g_" + n] = dict(max=scale, ours_vs_ref=float((a - b).abs().max()) / scale,
                             ref_vs_ref=float((b2 - b).abs().max()) / scale)
    if with_oracle:
        from oracle import cpu_oracle
        st = cpu_oracle.forward(scene)
        g = cpu_oracle.backward(st, scene["dL_dpix"])
        o = {"R": int(st["num_rendered"])}
        o["radii_ne"] = int((st["radii"] != rr.cpu().numpy()).sum())
        o["depths_bits_ne"] = bits_equal(st["depths"][visn], vr["depths"].cpu().numpy()[visn])[1]
        o["means2D_bits_ne"] = bits_equal(st["means2D"][visn], vr["means2D"].cpu().numpy()[visn])[1]
        o["cov3D_bits_ne"] = bits_equal(st["cov3D"][visn], vr["cov3D"].cpu().numpy()[visn])[1] if "scales" in d else 0
        o["conic_opacity_bits_ne"] = bits_equal(st["conic_opacity"][visn], vr["conic_opacity"].cpu().numpy()[visn])[1]
        if "shs" in d:
            o["rgb_bits_ne"] = bits_equal(st["rgb"][visn], vr["rgb"].cpu().numpy()[visn])[1]
        if st["num_rendered"] == Rr:
            o["point_list_ne"] = int((st["point_list"].astype(np.int32) != vr["point_list"].cpu().numpy()).sum())
            o["ranges_ne"] = int((st["ranges"].astype(np.int32) != vr["ranges"].cpu().numpy()).sum())
        o["n_contrib_ne"] = int((st["n_contrib"].astype(np.int32) != vr["n_contrib"].cpu().numpy()).sum())
        o["color_maxabs"] = float(np.abs(st["out_color"] - cr.cpu().numpy()).max())
        names = dict(dL_dmeans2D="dL_dmeans2D", dL_dcolors="dL_dcolors", dL_dopacity="dL_dopacity",
                     dL_dmeans3D="dL_dmeans3D", dL_dcov3D="dL_dcov3D", dL_dsh="dL_dsh", dL_dscales="dL_dscales",
                     dL_drotations="dL_drotations")
        for n, b in zip(GRAD_NAMES, gr):
            if b.numel() == 0:
                continue
            bb = b.cpu().numpy()
            scale = float(np.abs(bb).max()) + 1e-30
            o["g_" + n] = float(np.abs(g[names[n]].reshape(bb.shape) - bb).max()) / scale
        rep["oracle_vs_ref"] = o
    return rep


def time_config(name, dev, iters=10, warm=3):
    kw = dict(synthetic.CONFIGS[name]); kw["seed"] = 0
    scene = synthetic.make_scene(**kw)
    d = synthetic.to_device(scene, dev)
    from diff_gaussian_rasterization import _C
    from oracle import ref_cuda
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    res = {"config": name}
    for label, mod in (("ours", _C), ("ref", ref_cuda)):
        tf, tb = [], []
        for it in range(warm + iters):
            flush.zero_()
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e0.record()
            R, color, radii, geom, binning, img = mod.rasterize_gaussians(*call_args(d))
            e1.record()
            grads = mod.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))
            e2.record()
            torch.cuda.synchronize()
            if it >= warm:
                tf.append(e0.elapsed_time(e1)); tb.append(e1.elapsed_time(e2))
            del geom, binning, img, grads
        res[label] = dict(R=int(R), V=int((radii > 0).sum()), fwd_ms=float(np.median(tf)), bwd_ms=float(np.median(tb)))
    res["speedup_fwd_bwd"] = (res["ref"]["fwd_ms"] + res["ref"]["bwd_ms"]) / (res["ours"]["fwd_ms"] + res["ours"]["bwd_ms"])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="all")
    ap.add_argument("--time", default="")
    ap.add_argument("--extra", default="", help="comma list of P:W:H[:deg] random scenes for the integer parity check")
    ap.add_argument("--out", default="compare.json")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    print("host:", os.cpu_count(), "cores;", torch.cuda.get_device_name(0))
    out = {"cases": [], "timing": []}
    names = list(CASES) if a.cases == "all" else [c for c in a.cases.split(",") if c]
    for n in names:
        t = time.time()
        rep = compare_case(n, CASES[n], dev)
        rep["sec"] = round(time.time() - t, 2)
        print(json.dumps(rep)); sys.stdout.flush()
        out["cases"].append(rep)
    for spec in [s for s in a.extra.split(",") if s]:
        f = spec.split(":")
        kw = dict(P=int(f[0]), W=int(f[1]), H=int(f[2]), sh_degree=(int(f[3]) if len(f) > 3 and f[3] != "n" else None), seed=11)
        rep = compare_case("extra_" + spec, kw, dev, with_oracle=False)
        print(json.dumps(rep)); sys.stdout.flush()
        out["cases"].append(rep)
    for c in [c for c in a.time.split(",") if c]:
        r = time_config(c, dev)
        print(json.dumps(r)); sys.stdout.flush()
        out["timing"].append(r)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
