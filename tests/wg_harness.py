"""TEST / BENCH INFRASTRUCTURE -- runs the reference's own, UNMODIFIED ``wildgaussians/method.py`` on a rasterizer backend.

``GaussianModel._render_internal`` (method.py:1479-1632) is the caller of the hot path: it builds the camera matrices,
evaluates the appearance MLP + SH colours in PyTorch and calls ``GaussianRasterizer`` two (or three) times per step.
This module imports that file as shipped (from ``oracle/_ref/py``, the copy of the reference's package made by
``__graft_entry__.build()`` where the reference checkout can be read), stubs its three third-party imports
that this path never touches (omegaconf, plyfile, simple_knn), fills a ``GaussianModel`` with a seeded synthetic
cloud and executes one train-step-like forward + backward:

    out = model._render_internal(camera, config, kernel_size=0.1, embedding=model.appearance_embeddings[0])
    loss = (out["render"] * G1).sum() + (out["raw_render"] * G2).sum();  loss.backward()

The rasterizer backend is whatever ``diff_gaussian_rasterization`` resolves to (this repo's drop-in package, since
``wild-gaussians_b200`` is on sys.path) or, for the comparison run, the reference's compiled CUDA core behind the
same two names (``use_backend``) -- method.py's source is not touched either way.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CANDIDATES = [os.path.join(ROOT, "oracle", "_ref", "py")]


def reference_root():
    for c in CANDIDATES:
        if os.path.exists(os.path.join(c, "wildgaussians", "method.py")):
            return c
    return None


def import_method():
    """(wildgaussians.method module, Config class); None, None when the reference package is not available."""
    root = reference_root()
    if root is None:
        return None, None
    for p in (os.path.join(ROOT, "wild-gaussians_b200"), root):
        if p not in sys.path:
            sys.path.insert(0, p)
    try:                                        # this repo's drop-in for the reference's simple-knn submodule
        import simple_knn._C  # noqa: F401
    except Exception:
        pass
    for name in ("omegaconf", "plyfile", "simple_knn", "simple_knn._C"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["omegaconf"].OmegaConf = getattr(sys.modules["omegaconf"], "OmegaConf", object)
    sys.modules["plyfile"].PlyData = getattr(sys.modules["plyfile"], "PlyData", object)
    sys.modules["plyfile"].PlyElement = getattr(sys.modules["plyfile"], "PlyElement", object)
    if not hasattr(sys.modules["simple_knn._C"], "distCUDA2"):
        sys.modules["simple_knn._C"].distCUDA2 = None
    for p in (os.path.join(ROOT, "wild-gaussians_b200"), root):
        if p not in sys.path:
            sys.path.insert(0, p)
    import wildgaussians.method as m
    from wildgaussians.config import Config
    return m, Config


def use_backend(m, rasterizer_cls, settings_cls):
    """Point method.py's two imported names at another backend (module attributes, not source)."""
    m.GaussianRasterizer = rasterizer_cls
    m.GaussianRasterizationSettings = settings_cls


def make_model(m, Config, scene, device, seed=0, trained_like=True, filter_3d=0.002):
    """A ``GaussianModel`` (appearance on, uncertainty off) holding the synthetic cloud of `scene`
    (synthetic.make_scene with sh_degree=3): parameters are the INVERSE activations of the scene's values, so that
    ``get_gaussians()`` (method.py:1060-1086) reproduces them (up to the 3D filter)."""
    cfg = Config(source_path="", model_path="", uncertainty_mode="disabled")
    torch.manual_seed(seed)
    model = m.GaussianModel(cfg, training_setup=False).to(device)
    P = scene["means3D"].shape[0]
    model._resize_parameters(P)
    shs = scene["shs"]                                         # [P, 16, 3]
    with torch.no_grad():
        model.xyz.copy_(scene["means3D"])
        model.features_dc.copy_(shs[:, 0, :])
        model.features_rest.copy_(shs[:, 1:, :].reshape(P, -1))
        model.scales.copy_(torch.log(scene["scales"]))
        model.rotations.copy_(scene["rotations"])
        model.opacities.copy_(torch.special.logit(scene["opacities"].clamp(1e-4, 1 - 1e-4)))
        model.filter_3D.fill_(filter_3d)
        g = torch.Generator().manual_seed(seed + 7)
        model.embeddings.copy_(torch.randn(P, model.embeddings.shape[1], generator=g) * 0.3)
        model.set_num_training_images(4)
        model.appearance_embeddings.copy_(torch.randn(4, cfg.appearance_embedding_dim, generator=g) * 0.3)
        model.active_sh_degree.fill_(cfg.sh_degree)
        if trained_like:
            # at initialisation `mul` (0.01 x MLP output) is ~0 and every toned colour is ~0.5; a trained model has
            # mul ~ 1: emulate it through the last layer's bias (same device as tests/golden/make_golden_colors.py)
            model.appearance_mlp.mlp[-1].bias[3:] = 100.0
    model.train()
    return model, cfg


def make_camera(scene):
    """Single pinhole camera matching synthetic.make_scene: world->camera = identity, fx = fy = 0.9 W."""
    W, H = int(scene["image_width"]), int(scene["image_height"])
    fx = W / (2.0 * scene["tanfovx"])
    fy = H / (2.0 * scene["tanfovy"])
    pose = np.concatenate([np.eye(3, dtype=np.float32), np.zeros((3, 1), dtype=np.float32)], axis=1)   # camera-to-world
    return types.SimpleNamespace(poses=pose, image_sizes=np.array([W, H], dtype=np.int32),
                                 intrinsics=np.array([fx, fy, W / 2.0, H / 2.0], dtype=np.float32))


PARAMS = ("xyz", "features_dc", "features_rest", "scales", "rotations", "opacities", "embeddings",
          "appearance_embeddings")


def train_step(model, cfg, camera, G1, G2, zero=True):
    """One forward + backward through the unmodified ``_render_internal``; returns its output dict."""
    if zero:
        for p in model.parameters():
            p.grad = None
    out = model._render_internal(camera, cfg, kernel_size=cfg.kernel_size, embedding=model.appearance_embeddings[0],
                                 return_raw=True)
    loss = (out["render"] * G1).sum() + (out["raw_render"] * G2).sum()
    loss.backward()
    return out


def collect(model, out):
    """Images and every gradient of the step as a dict of detached tensors."""
    res = {"render": out["render"].detach(), "raw_render": out["raw_render"].detach(), "radii": out["radii"],
           "accumulation": out["accumulation"].detach(), "viewspace_grad": out["viewspace_points"].grad.detach().clone()}
    for n in PARAMS:
        res["g_" + n] = getattr(model, n).grad.detach().clone()
    for i, p in enumerate(model.appearance_mlp.parameters()):
        res[f"g_mlp{i}"] = p.grad.detach().clone()
    return res
