"""Generates tests/golden/*.npz by running the UNMODIFIED reference CUDA rasterizer
(oracle/_ref/libdgr_ref.so, built by oracle/Makefile from the reference checkout) on a GPU.

The reference has no golden vectors of its own (SURVEY.md section 8c: "parity unpinned by the reference's
own tests"), so these files pin the CPU oracle (tests/test_oracle_golden.py, runs without a GPU) and the
CUDA path (tests/test_gpu_parity.py).  Inputs are not stored: they are regenerated from
``synthetic.make_scene(**case)``; a checksum of the inputs is stored to detect RNG drift.

Run on the GPU box:   python tests/golden/make_golden.py gpurun_out/golden
then copy gpurun_out/golden/*.npz into tests/golden/.
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "wild-gaussians_b200"))

CASES = {
    # name: make_scene kwargs
    "c1_deg0": dict(P=10_000, W=256, H=256, sh_degree=0, max_sh_degree=0, seed=0),
    "precomp_small": dict(P=3_000, W=200, H=120, sh_degree=None, seed=1, scale_range=(0.004, 0.06)),
    "sh3_small": dict(P=3_000, W=144, H=112, sh_degree=3, seed=2, scale_range=(0.004, 0.06), bg=(0.3, 0.1, 0.7)),
    "sh1_jitter": dict(P=2_000, W=100, H=90, sh_degree=1, seed=3, subpixel_jitter=0.5, scale_range=(0.004, 0.08)),
    "unnorm_quat": dict(P=2_000, W=128, H=96, sh_degree=None, seed=4, normalize_rot=False, scale_range=(0.002, 0.04)),
    "cov3d_precomp": dict(P=2_000, W=128, H=96, sh_degree=None, seed=5, cov3D_precomp=True, scale_range=(0.004, 0.06)),
    "big_splats": dict(P=400, W=256, H=192, sh_degree=None, seed=6, scale_range=(0.05, 0.4)),
}

INPUT_KEYS = ("means3D", "opacities", "scales", "rotations", "cov3D_precomp", "colors_precomp", "shs",
              "viewmatrix", "projmatrix", "campos", "bg", "subpixel_offset", "dL_dpix")


def input_digest(scene) -> str:
    h = hashlib.sha256()
    for k in INPUT_KEYS:
        if k in scene:
            h.update(k.encode())
            h.update(scene[k].contiguous().numpy().tobytes())
    return h.hexdigest()


def call_args(d):
    """Positional argument tuples of _C.rasterize_gaussians for a scene on some device."""
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


def run_reference(scene, dev):
    import synthetic
    from oracle import ref_cuda
    d = synthetic.to_device(scene, dev)
    R, color, radii, geom, binning, img = ref_cuda.rasterize_gaussians(*call_args(d))
    P, W, H = d["means3D"].shape[0], d["image_width"], d["image_height"]
    v = ref_cuda.debug_views(geom, binning, img, P, W, H, R)
    grads = ref_cuda.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))
    torch.cuda.synchronize()
    vis = (radii > 0).cpu().numpy()
    out = dict(num_rendered=np.int64(R), out_color=color.cpu().numpy(), radii=radii.cpu().numpy(),
               final_T=v["final_T"].cpu().numpy(), n_contrib=v["n_contrib"].cpu().numpy(),
               ranges=v["ranges"].cpu().numpy(), point_list=v["point_list"].cpu().numpy(),
               tiles_touched=v["tiles_touched"].cpu().numpy())
    # per-Gaussian state is only defined for rendered Gaussians (SURVEY N6): zero the rest
    for k in ("depths", "means2D", "conic_opacity", "cov3D", "rgb"):
        a = v[k].cpu().numpy().copy()
        a[~vis] = 0
        out[k] = a
    out["tiles_touched"] = out["tiles_touched"] * vis
    names = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales",
             "dL_drotations")
    for n, g in zip(names, grads):
        out[n] = g.cpu().numpy()
    return out


def main(outdir):
    import synthetic
    os.makedirs(outdir, exist_ok=True)
    dev = torch.device("cuda:0")
    for name, kw in CASES.items():
        scene = synthetic.make_scene(**kw)
        out = run_reference(scene, dev)
        out["input_digest"] = np.array(input_digest(scene))
        path = os.path.join(outdir, name + ".npz")
        np.savez_compressed(path, **out)
        print(f"{name}: R={int(out['num_rendered'])} V={(out['radii'] > 0).sum()} "
              f"n_contrib max={out['n_contrib'].max()} -> {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "gpurun_out", "golden"))
