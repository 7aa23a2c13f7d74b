"""Generates the posed-camera / guard-band golden vectors (tests/golden/<name>.npz and <name>.inputs.npz) by running the
UNMODIFIED reference CUDA rasterizer (oracle/_ref/libdgr_ref.so) on a GPU.  The scenes come from the builders in
tests/test_adversarial_scenes.py; their tensors AND scalars are stored in the .inputs.npz, because regenerating the
tensors from the seeds is not bit-reproducible across host CPUs.

Run on a GPU machine:   python tests/golden/make_golden_posed.py <outdir>
then copy <outdir>/*.npz into tests/golden/.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "wild-gaussians_b200"), HERE, os.path.dirname(HERE)):
    if p not in sys.path:
        sys.path.insert(0, p)

from make_golden import INPUT_KEYS, run_reference  # noqa: E402


def main(outdir):
    """Writes <name>.inputs.npz and <name>.npz for every posed case into `outdir`."""
    import test_adversarial_scenes as adv
    os.makedirs(outdir, exist_ok=True)
    dev = torch.device("cuda:0")
    for name in adv.POSED_GOLDEN:
        scene = adv.golden_posed_scene(name)
        inputs = {k: scene[k].contiguous().numpy() for k in INPUT_KEYS if k in scene}
        inputs.update({k: np.array(scene[k]) for k in adv.SCALARS})
        np.savez_compressed(os.path.join(outdir, name + ".inputs.npz"), **inputs)
        scene = adv.load_posed_inputs(name, outdir)           # exactly what is stored
        out = run_reference(scene, dev)
        path = os.path.join(outdir, name + ".npz")
        np.savez_compressed(path, **out)
        print(f"{name}: R={int(out['num_rendered'])} V={(out['radii'] > 0).sum()} -> {path}")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: python tests/golden/make_golden_posed.py <outdir>")
    main(sys.argv[1])
