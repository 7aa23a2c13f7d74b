"""TEST / BENCH INFRASTRUCTURE -- a ``WildGaussians`` ready for ``train_iteration``, built without a dataset.

``make_method`` fills a ``GaussianModel`` (optimizer set up, uncertainty model offline when asked for) with the
synthetic cloud of ``synthetic.make_scene`` and wraps it in a ``WildGaussians`` made through ``__new__``, with
``n_cameras`` (four by default) seeded cameras around the scene's camera and seeded training images stored the way
method.py:1716-1723 stores them ([3,H,W] fp32 views of HWC arrays, masks [1,H,W]).  Image 1 is not byte-exact (a value off the k / 255 grid); the others
are.  Mask 2 is fractional (k / 255 values); the others are 0 / 1.
"""
from __future__ import annotations

import types

import numpy as np
import torch

N_CAMERAS = 4


class Cameras:
    """What train_iteration and compute_3D_filter use of a ``Cameras`` batch: len, indexing, iteration, image_sizes."""

    def __init__(self, cams):
        self.cams = list(cams)
        self.image_sizes = np.stack([c.image_sizes for c in self.cams])

    def __len__(self):
        return len(self.cams)

    def __getitem__(self, i):
        return self.cams[i]


def _images(H, W, n, seed, masks):
    rng = np.random.default_rng(seed)
    imgs, msks = [], []
    for i in range(n):
        base = rng.random((H // 8 + 2, W // 8 + 2, 3))
        up = np.kron(base, np.ones((8, 8, 1)))[:H, :W]
        img = np.rint(up * 255).astype(np.uint8).astype(np.float32) / np.float32(255)
        if i == 1:
            img[H // 2, W // 3, 1] = np.float32(0.123456789)          # not on the byte grid
        imgs.append(torch.from_numpy(np.moveaxis(img, -1, 0)))
        if masks:
            mk = np.ones((H, W), dtype=np.float32)
            mk[: H // 3, : W // 4] = 0.0
            if i == 2:
                mk[H // 2:, W // 2:] = np.float32(128) / np.float32(255)
            msks.append(torch.from_numpy(mk[None]))
    return imgs, (msks if masks else None)


def make_method(m, Config, scene, dev, *, uncertainty=False, masks=False, seed=0, active_sh_degree=3, appearance=True,
                n_cameras=N_CAMERAS, **overrides):
    import wg_uncertainty as wu
    cfg = Config(source_path="", model_path="", uncertainty_mode="dino" if uncertainty else "disabled",
                 appearance_enabled=appearance, **overrides)
    torch.manual_seed(seed)
    with wu.offline(m, cfg.uncertainty_backbone):
        model = m.GaussianModel(cfg, training_setup=False).to(dev)
    P = scene["means3D"].shape[0]
    model._resize_parameters(P)
    shs = scene["shs"]
    with torch.no_grad():
        model.xyz.copy_(scene["means3D"])
        model.features_dc.copy_(shs[:, 0, :])
        model.features_rest.copy_(shs[:, 1:, :].reshape(P, -1))
        model.scales.copy_(torch.log(scene["scales"]))
        model.rotations.copy_(scene["rotations"])
        model.opacities.copy_(torch.special.logit(scene["opacities"].clamp(1e-4, 1 - 1e-4)))
        model.filter_3D.fill_(0.002)
        g = torch.Generator().manual_seed(seed + 7)
        if appearance:
            model.embeddings.copy_(torch.randn(P, model.embeddings.shape[1], generator=g) * 0.3)
            model.set_num_training_images(n_cameras)
            model.appearance_embeddings.copy_(torch.randn(n_cameras, cfg.appearance_embedding_dim, generator=g) * 0.3)
            model.appearance_mlp.mlp[-1].bias[3:] = 100.0
        model.active_sh_degree.fill_(active_sh_degree)
        model.spatial_lr_scale.fill_(1.0)
        for n in ("xyz_grad", "denom", "max_radii2D", "xyz_gradient_accum_abs", "xyz_gradient_accum_abs_max"):
            if getattr(model, n, None) is not None:
                getattr(model, n).zero_()
    model._setup_optimizers()
    model.eval()

    W, H = int(scene["image_width"]), int(scene["image_height"])
    fx = W / (2.0 * scene["tanfovx"])
    fy = H / (2.0 * scene["tanfovy"])
    cams = []
    for i in range(n_cameras):
        j = i % 8
        pose = np.concatenate([np.eye(3, dtype=np.float32), np.array([[0.03 * j], [-0.02 * j], [0.01 * j]], np.float32)],
                              axis=1)
        cams.append(types.SimpleNamespace(poses=pose, image_sizes=np.array([W, H], dtype=np.int32),
                                          intrinsics=np.array([fx, fy, W / 2.0, H / 2.0], dtype=np.float32)))
    method = m.WildGaussians.__new__(m.WildGaussians)
    method.model, method.config = model, cfg
    method.train_cameras = Cameras(cams)
    method.train_images, method.train_masks = _images(H, W, n_cameras, seed + 11, masks)
    method._viewpoint_stack = []
    method.cameras_extent = 4.0
    method._sky_distance = None
    method.step = 0
    return method
