"""Golden vectors of the uncertainty head and the ``dino``-mode loss, produced by the REFERENCE ITSELF.

Runs where the reference checkout can be read (CPU torch is enough):
    python tests/golden/make_golden_uncertainty.py
builds the reference's ``UncertaintyModel`` offline (random backbone, ``tests/wg_uncertainty.py``), casts it to float64
and runs its unmodified ``_compute_losses`` (method.py:363-433) and backward on the CPU.  The backbone is replaced by a
deterministic float64 function of the 14 x 14 patch means (channels with non-zero means, so BatchNorm has work to do);
the same input gives the same features, as the frozen backbone does.  The head is rebuilt for 96 channels (the kernels
take C at run time) to keep the files small; features are values fp32 can hold, the images are 8-bit, the two image
statistics are rounded to multiples of 2^-15 (stored as int16 codes; the loss statements see the rounded values), and
``loss_mult`` is stored on every ``stride``-th row and column.  The dropout mask is the seeded draw the reference makes,
recorded by repeating it on a [1, C, 1, 1] tensor of ones.  The head parameters and running statistics are random, away
from their initial values.  Sizes: 100 x 130 (below 350 px, not a multiple of 14: no resize, the 350-px map is the
image), 351 x 60 (the 350-px map is 350 x 70, wider than the image) and 50 x 400 (the 350-px map is 56 x 350, taller
than the image).  Each file holds the inputs (features of the three backbone calls, images, the two image statistics,
mask, parameters, running statistics) and the outputs (loss, metrics, loss_mult, the four gradients, running
statistics).
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from make_golden_colors import import_reference  # noqa: E402
import wg_uncertainty as wu  # noqa: E402

CASES = [("uncertainty_small_odd", 100, 130, 1), ("uncertainty_resize", 351, 60, 2),
         ("uncertainty_tall_down", 50, 400, 3)]
C = 96
STRIDE = 3
STAT_SCALE = 2.0 ** 15                             # image statistics in [-1, 1] as int16 codes


def stub_backbone(seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(C, 3, generator=g, dtype=torch.float64)
    D = torch.randn(C, 3, generator=g, dtype=torch.float64) * 3
    bias = torch.randn(C, generator=g, dtype=torch.float64) * 2
    phase = torch.rand(C, generator=g, dtype=torch.float64) * 6.28
    calls = []

    def get_intermediate_layers(x, n=1, reshape=False, **kw):
        p = F.avg_pool2d(x, 14)
        f = torch.einsum("ck,nkhw->nchw", A, p) + bias[:, None, None] + 0.5 * torch.sin(
            torch.einsum("ck,nkhw->nchw", D, p) + phase[:, None, None])
        f = f.float().double()
        calls.append(f.clone())
        return (f,)

    return get_intermediate_layers, calls


def images(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    gt = F.interpolate(torch.rand(1, 3, H // 6 + 2, W // 6 + 2, generator=g, dtype=torch.float64), size=(H, W),
                       mode="bilinear", align_corners=False)
    pred = (gt + 0.08 * torch.randn(gt.shape, generator=g, dtype=torch.float64)).clamp(0, 1)
    pred[..., : H // 3, : W // 4] = 1 - pred[..., : H // 3, : W // 4]            # a region the backbone sees as different
    q = lambda t: (t * 255).round() / 255
    return q(gt), q(pred)


def make_case(m, Config, name, H, W, seed):
    model, cfg = wu.make_uncertainty_model(m, Config, "dino", "cpu", seed=seed)
    model.conv_seg = torch.nn.Conv2d(C, 1, kernel_size=1)
    model.bn = torch.nn.SyncBatchNorm(C)
    model = model.double()
    g = torch.Generator().manual_seed(100 + seed)
    with torch.no_grad():
        model.conv_seg.weight.copy_(torch.randn(1, C, 1, 1, generator=g, dtype=torch.float64) * 0.05)
        model.conv_seg.bias.fill_(0.1)
        model.bn.weight.copy_(1 + 0.2 * torch.randn(C, generator=g, dtype=torch.float64))
        model.bn.bias.copy_(0.1 * torch.randn(C, generator=g, dtype=torch.float64))
        model.bn.running_mean.copy_(0.1 * torch.randn(C, generator=g, dtype=torch.float64))
        model.bn.running_var.copy_(1 + torch.rand(C, generator=g, dtype=torch.float64))
    fn, calls = stub_backbone(seed)
    model.backbone.get_intermediate_layers = fn
    gt, pred = images(H, W, seed)
    inputs = dict(gt=gt, pred=pred, conv_w=model.conv_seg.weight.detach().clone(), conv_b=model.conv_seg.bias.detach().clone(),
                  bn_w=model.bn.weight.detach().clone(), bn_b=model.bn.bias.detach().clone(),
                  running_mean_in=model.bn.running_mean.clone(), running_var_in=model.bn.running_var.clone())
    q = lambda t: (t * STAT_SCALE).round().clamp(-STAT_SCALE, STAT_SCALE - 1) / STAT_SCALE
    inputs["ssim"] = q(m.ssim_down(gt, pred, max_size=400))
    inputs["msssim"] = q(m.msssim(gt, pred, max_size=400, min_size=80))
    # the loss statements see the rounded statistics stored in the file
    saved = m.ssim_down, m.msssim
    m.ssim_down = lambda *a, **k: inputs["ssim"]
    m.msssim = lambda *a, **k: inputs["msssim"]
    torch.manual_seed(7)
    inputs["mask"] = F.dropout2d(torch.ones(1, C, 1, 1, dtype=torch.float64), p=cfg.uncertainty_dropout, training=True).reshape(C)
    torch.manual_seed(7)
    try:
        loss, metrics, loss_mult = model._compute_losses(gt, pred)
    finally:
        m.ssim_down, m.msssim = saved
    loss.backward()
    assert len(calls) == 3, len(calls)
    out = dict(loss=loss.detach(), metrics=torch.tensor([metrics[k] for k in ("loss", "ssim", "msssim", "ssim_discounted",
                                                                             "mse_discounted", "psnr_discounted", "beta")],
                                 dtype=torch.float64),
               loss_mult=loss_mult[..., ::STRIDE, ::STRIDE], d_conv_w=model.conv_seg.weight.grad,
               d_conv_b=model.conv_seg.bias.grad,
               d_bn_w=model.bn.weight.grad, d_bn_b=model.bn.bias.grad, running_mean=model.bn.running_mean,
               running_var=model.bn.running_var, feat=calls[0], feat_gt_down=calls[1], feat_pred_down=calls[2])
    arrays = {k: v.detach().numpy() for k, v in {**inputs, **out}.items()}
    for k in ("feat", "feat_gt_down", "feat_pred_down"):
        arrays[k] = arrays[k].astype(np.float32)
    for k in ("ssim", "msssim"):
        arrays[k] = np.round(arrays[k] * STAT_SCALE).astype(np.int16)
    for k in ("gt", "pred"):
        arrays[k] = np.round(arrays[k] * 255).astype(np.uint8)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), clip_min=cfg.uncertainty_clip_min,
                        reg_weight=cfg.uncertainty_regularizer_weight, eps=model.bn.eps, momentum=model.bn.momentum,
                        stride=STRIDE, stat_scale=STAT_SCALE, **arrays)
    print(name, {k: round(float(v), 6) for k, v in metrics.items()}, "loss_mult", tuple(loss_mult.shape))


if __name__ == "__main__":
    m, Config = import_reference()
    for case in CASES:
        make_case(m, Config, *case)
