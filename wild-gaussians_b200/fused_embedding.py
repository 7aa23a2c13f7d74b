"""Test-time appearance optimisation on one geometry pass: a drop-in for ``WildGaussians.optimize_embedding``
(wildgaussians/method.py:1755-1830), which runs once per test image before it is rendered (the wild-gaussians
evaluation protocol).

The reference runs ``appearance_embedding_optim_iters`` (128) Adam iterations on the 32-float image embedding, and every
iteration re-renders through ``_render_internal`` -- projection, depth sort, binning, a raw and a toned composite -- and
runs the full backward into every model parameter.  Only the embedding changes between iterations, so here:

* the geometry, depth order, tile lists and blend masks are computed once (``_C.rasterize_gaussians``) and every
  iteration re-composites the toned colours on them (``gsr_forward_recolor``);
* the colour op runs on the V visible Gaussians only (``radii > 0``; the others are never blended), compacted once;
* the composite's backward produces only dL/dcolour (``gsr_backward_colors``) and the colour op's backward only
  dL/d(embedding) (``gsr_appearance_embedding_backward`` + ``gsr_appearance_unpack_grads``);
* loss, MSE and PSNR stay on the device until the end: no host synchronisation inside the loop.

The loss statements are the reference's (``scale_grads`` of the method module, ``mse_loss`` / ``l1_loss``), with the SSIM
term through ``fused_ssim.ssim``; the optimizer is the reference's ``torch.optim.Adam``.  Model parameters are never
written.  Known difference: when ``model.optimizer`` is None the reference leaves 128 iterations of accumulated
gradients in every model parameter's ``.grad``; this path does not touch ``.grad``.

    import fused_embedding
    out = fused_embedding.optimize_embedding(method, dataset)             # same arguments and result as the method
    wildgaussians_fused.enable_method(method)                             # or: route method.optimize_embedding here

Anything outside the accelerated configuration (see ``supported``) runs the reference method itself.
"""
from __future__ import annotations

import math
import sys
from ctypes import byref

import numpy as np
import torch

import fused_ssim
import wildgaussians_fused as wgf
from diff_gaussian_rasterization import _C
from fused_colors import fused_activations

_lib = _C._lib
_MLP_SHAPES = ((128, 59), (128, 128), (6, 128))


def _method_module(method):
    return sys.modules[type(method.model).__module__]


def _mlp_linears(model):
    mlp = getattr(getattr(model, "appearance_mlp", None), "mlp", None)
    if mlp is None:
        return None
    lin = [x for x in mlp if isinstance(x, torch.nn.Linear)]
    return lin if len(lin) == 3 and tuple(tuple(x.weight.shape) for x in lin) == _MLP_SHAPES else None


def _optim_type(config):
    t = str(config.appearance_optim_type)
    return (t[:-7], True) if t.endswith("-scaled") else (t, False)


def supported(method, dataset, embedding=None) -> bool:
    """True when the fused loop computes what ``optimize_embedding`` of the method would: the accelerated model
    configuration (``wildgaussians_fused._supported`` and the default MLP shape), an ``mse`` or ``dssim+l1`` loss
    (optionally ``-scaled``), a pinhole camera, CUDA fp32 parameters, an fp32 start embedding, no tile-row shard."""
    model, config = method.model, method.config
    if not wgf._supported(model, config) or _mlp_linears(model) is None:
        return False
    if _optim_type(config)[0] not in ("mse", "dssim+l1"):
        return False
    tens = [model.xyz, model.features_dc, model.features_rest, model.embeddings, model.scales, model.opacities,
            model.rotations, model.filter_3D] + [p for x in _mlp_linears(model) for p in (x.weight, x.bias)]
    if not all(t.is_cuda and t.dtype == torch.float32 for t in tens):
        return False
    if embedding is not None and not (isinstance(embedding, np.ndarray) and embedding.dtype == np.float32
                                      and embedding.size == int(config.appearance_embedding_dim)):
        return False
    if embedding is None and model.appearance_embeddings.dtype != torch.float32:
        return False
    if _C.get_tile_row_shard() != (0, 0):
        return False
    camera = dataset["cameras"].item()
    return camera.camera_models == _method_module(method).camera_model_to_int("pinhole")


def _reference(method):
    cls = type(method)
    if not hasattr(cls, "optimize_embedding"):       # e.g. a namespace holding (model, config)
        cls = _method_module(method).WildGaussians
    return cls.optimize_embedding


class EmbeddingLoop:
    """The state of one fused ``optimize_embedding`` call: ``step(i)`` runs iteration i without a host synchronisation,
    ``result()`` reads everything back once."""

    def __init__(self, method, dataset, embedding=None):
        model, config = method.model, method.config
        m = _method_module(method)
        dev = model.xyz.device
        self.model, self.config, self.iters = model, config, int(config.appearance_embedding_optim_iters)
        camera = dataset["cameras"].item()
        model.eval()
        start = torch.from_numpy(embedding).to(dev) if embedding is not None else model.get_embedding(None)
        self.param = torch.nn.Parameter(start.detach().clone().requires_grad_(True))
        self.optimizer = torch.optim.Adam([self.param], lr=config.appearance_embedding_optim_lr)
        self.gt = torch.tensor(m.convert_image_dtype(dataset["images"][0], np.float32), dtype=torch.float32,
                               device=dev).permute(2, 0, 1)
        masks = dataset["masks"]
        self.mask = (torch.tensor(m.convert_image_dtype(masks[0], np.float32), dtype=torch.float32, device=dev)[..., None]
                     .permute(2, 0, 1).float() if masks is not None else None)
        self.kind, scaled = _optim_type(config)
        self.lambda_dssim = float(config.lambda_dssim)
        self.scale_grads = m.scale_grads
        self.loss_mult = None
        if scaled and model.uncertainty_model is not None:
            with torch.enable_grad():
                _, _, loss_mult = model.uncertainty_model.get_loss(self.gt, self.gt)
            self.loss_mult = (loss_mult > 1).to(dtype=loss_mult.dtype)

        # one geometry pass (what _render_internal of wildgaussians_fused feeds the rasterizer)
        cc = wgf._camera_constants(m, camera, dev)
        H, W = cc["height"], cc["width"]
        self.deg = wgf._active_degree(model)
        with torch.no_grad():
            scales, opacity, rotations = fused_activations(model.scales, model.opacities, model.rotations, model.filter_3D)
        P = int(model.xyz.shape[0])
        f32 = dict(dtype=torch.float32, device=dev)
        self.colors = torch.zeros((P, 3), **f32)
        bg, sub = torch.zeros((3,), **f32), torch.zeros((H, W, 2), **f32)
        empty = torch.Tensor([])
        R, _, radii, self.geom, self.binning, self.img = _C.rasterize_gaussians(
            bg, model.xyz.detach(), self.colors, opacity, scales, rotations, 1.0, empty, cc["world_view"], cc["full_proj"],
            cc["tanfovx"], cc["tanfovy"], float(config.kernel_size), sub, H, W, empty, self.deg, cc["cam_center"], False, False)
        _C.clear_geometry_cache()            # this object holds the buffers it needs
        self.radii = radii
        self.vis = torch.nonzero(radii > 0).squeeze(1)
        V = int(self.vis.numel())
        self.num_visible = V
        self.image = torch.empty((3, H, W), **f32)
        self.img2 = torch.empty_like(self.img)
        self.dcolor = torch.empty((P, 3), **f32)
        self._keep = (bg, sub, scales, opacity, rotations, cc)
        stream = torch.cuda.current_stream(dev).cuda_stream
        self.stream = stream

        self.fwd_args = _C.forward_args(
            background=bg, means3D=model.xyz, colors=self.colors, opacities=opacity, scales=scales, rotations=rotations,
            viewmatrix=cc["world_view"], projmatrix=cc["full_proj"], campos=cc["cam_center"], tan_fovx=cc["tanfovx"],
            tan_fovy=cc["tanfovy"], kernel_size=float(config.kernel_size), subpixel_offset=sub, H=H, W=W, radii=radii,
            out_color=self.image, degree=self.deg)
        ba = _C.GsrBackwardArgs()
        ba.P, ba.M, ba.R, ba.W, ba.H = P, 0, int(R), W, H
        ba.subpixel_offset = sub.data_ptr()
        ba.geom_buffer, ba.binning_buffer, ba.img_buffer = self.geom.data_ptr(), self.binning.data_ptr(), self.img2.data_ptr()
        ba.dL_dcolor = self.dcolor.data_ptr()
        self.bwd_args = ba

        # the colour op's inputs of the visible Gaussians, compacted once
        lin = _mlp_linears(model)
        self.w = [t.detach().contiguous() for x in lin for t in (x.weight, x.bias)]
        gather = lambda t: t.detach().index_select(0, self.vis).contiguous()
        self.dc_v, self.rest_v = gather(model.features_dc), gather(model.features_rest.reshape(P, -1))
        self.gemb_v, self.means_v = gather(model.embeddings), gather(model.xyz)
        self.toned_v = torch.empty((V, 3), **f32)
        self.dtoned_v = torch.empty((V, 3), **f32)
        self.blob = torch.empty((_lib.gsr_appearance_packed_weight_bytes(),), dtype=torch.uint8, device=dev)
        self.pack = torch.empty((_lib.gsr_appearance_grad_pack_bytes() // 4,), **f32)
        self.unpacked = [torch.empty(s, **f32) for s in ((128, 59), (128,), (128, 128), (128,), (6, 128), (6,))]
        self.status = torch.zeros((1,), dtype=torch.int32, device=dev)
        aa = _C.GsrAppearanceArgs()
        aa.P, aa.sh_degree = V, self.deg
        aa.features_dc, aa.features_rest, aa.embeddings = self.dc_v.data_ptr(), self.rest_v.data_ptr(), self.gemb_v.data_ptr()
        aa.means3D, aa.campos, aa.packed_weights = self.means_v.data_ptr(), cc["cam_center"].data_ptr(), self.blob.data_ptr()
        aa.colors_toned, aa.dL_dcolors_toned = self.toned_v.data_ptr(), self.dtoned_v.data_ptr()
        aa.grad_pack, aa.status = self.pack.data_ptr(), self.status.data_ptr()
        self.app_args = aa
        self.param.grad = torch.zeros_like(self.param)
        self.metrics = torch.zeros((self.iters, 3), **f32)    # loss, mse, log10(mse)

    def render(self):
        """The toned image at the current embedding (``self.image``)."""
        w, s = self.w, self.stream
        _C._check(_lib.gsr_appearance_pack_weights(w[0].data_ptr(), w[1].data_ptr(), w[2].data_ptr(), w[3].data_ptr(),
                                                   w[4].data_ptr(), w[5].data_ptr(), self.param.data_ptr(),
                                                   self.blob.data_ptr(), s), "gsr_appearance_pack_weights")
        _C._check(_lib.gsr_appearance_colors_forward(byref(self.app_args), s), "gsr_appearance_colors_forward")
        self.colors.index_copy_(0, self.vis, self.toned_v)
        _C._check(_lib.gsr_forward_recolor(byref(self.fwd_args), self.geom.data_ptr(), self.binning.data_ptr(),
                                           self.img.data_ptr(), self.img2.data_ptr(), s), "gsr_forward_recolor")
        return self.image

    def loss(self, image):
        """The reference's loss statements (method.py:1790-1806) on ``image``: (loss, mse)."""
        if self.mask is not None:
            image = self.scale_grads(image, self.mask)
        if self.loss_mult is not None:
            image = self.scale_grads(image, self.loss_mult)
        mse = torch.nn.functional.mse_loss(image, self.gt)
        if self.kind == "mse":
            return mse, mse
        l1 = torch.nn.functional.l1_loss(image, self.gt)
        ssim_value = fused_ssim.ssim(image, self.gt, size_average=True)
        return (1.0 - self.lambda_dssim) * l1 + self.lambda_dssim * (1.0 - ssim_value), mse

    def embedding_grad(self, dL_dimage):
        """dL/d(embedding) [32] (into ``self.param.grad``) from dL/d(toned image) [3,H,W] on the current colours."""
        s = self.stream
        self.bwd_args.dL_dpix = dL_dimage.data_ptr()
        _C._check(_lib.gsr_backward_colors(byref(self.bwd_args), s), "gsr_backward_colors")
        torch.index_select(self.dcolor, 0, self.vis, out=self.dtoned_v)
        _C._check(_lib.gsr_appearance_embedding_backward(byref(self.app_args), s), "gsr_appearance_embedding_backward")
        u = self.unpacked
        _C._check(_lib.gsr_appearance_unpack_grads(self.pack.data_ptr(), self.w[0].data_ptr(), self.param.data_ptr(),
                                                   u[0].data_ptr(), u[1].data_ptr(), u[2].data_ptr(), u[3].data_ptr(),
                                                   u[4].data_ptr(), u[5].data_ptr(), self.param.grad.data_ptr(), s),
                  "gsr_appearance_unpack_grads")
        return self.param.grad

    def step(self, i):
        image = self.render().detach().requires_grad_(True)
        with torch.enable_grad():
            loss, mse = self.loss(image)
            loss.backward()
        self.metrics[i, 0] = loss.detach()
        self.metrics[i, 1] = mse.detach()
        self.embedding_grad(image.grad.contiguous())
        self.optimizer.step()

    def result(self):
        self.metrics[:, 2] = torch.log10(self.metrics[:, 1])
        vals = self.metrics.cpu().tolist()
        if getattr(self.model, "optimizer", None) is not None:
            self.model.optimizer.zero_grad()
        return {"embedding": self.param.detach().cpu().numpy(),
                "metrics": {"psnr": [20 * math.log10(1.0) - 10 * v[2] for v in vals], "mse": [v[1] for v in vals],
                            "loss": [v[0] for v in vals]}}


def optimize_embedding(method, dataset, *, embedding=None):
    """Drop-in for ``WildGaussians.optimize_embedding``: same arguments, same result dictionary.  Reads only
    ``method.model`` and ``method.config``; unsupported configurations run the method's own implementation."""
    if not supported(method, dataset, embedding):
        return _reference(method)(method, dataset, embedding=embedding)
    with torch.cuda.device(method.model.xyz.device):
        loop = EmbeddingLoop(method, dataset, embedding)
        for i in range(loop.iters):
            loop.step(i)
        return loop.result()
