"""Golden vectors of the uncertainty loss in every mode, in training and evaluation mode and with a capped head input,
produced by the REFERENCE ITSELF.

Runs where the reference checkout can be read (CPU torch is enough):
    python tests/golden/make_golden_uncertainty_modes.py
As ``make_golden_uncertainty.py`` (whose stand-in backbone, images and head it reuses: float64 on the CPU, 96 channels,
8-bit images, image statistics rounded to multiples of 2^-15), it runs the reference's unmodified ``_compute_losses``
(method.py:363-433) and backward, here once per (mode, BatchNorm mode) from the same parameters and running statistics.
One file per image size holds the shared inputs (the features of the three backbone inputs, the images, the two image
statistics and the 350-px MS-SSIM map of ``dino+mssim``, the dropout mask, the parameters, the running statistics) and,
under the prefix ``<mode>_<train|eval>_``, each run's outputs (loss, metrics, loss_mult on every ``stride``-th row and
column, the four gradients, the running statistics).  The three sizes of ``make_golden_uncertainty.py`` carry ``l2reg``,
``l1reg`` and ``dino+mssim`` in both modes and ``dino`` in evaluation mode; ``uncertainty_modes_cap`` carries ``l2reg``
in both modes at 351 x 60 with ``uncertainty_dino_max_size = 200`` (a 210 x 42 head input).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_golden_colors import import_reference  # noqa: E402
from make_golden_uncertainty import C, STAT_SCALE, STRIDE, images, stub_backbone  # noqa: E402
import wg_uncertainty as wu  # noqa: E402

RUNS = [(mode, training) for mode in ("l2reg", "l1reg", "dino+mssim") for training in (True, False)] + [("dino", False)]
CASES = [("uncertainty_modes_small_odd", 100, 130, 1, None, RUNS),
         ("uncertainty_modes_resize", 351, 60, 2, None, RUNS),
         ("uncertainty_modes_tall_down", 50, 400, 3, None, RUNS),
         ("uncertainty_modes_cap", 351, 60, 4, 200, [("l2reg", True), ("l2reg", False)])]
METRICS = ("loss", "ssim", "msssim", "ssim_discounted", "mse_discounted", "psnr_discounted", "beta")


def tag(mode, training):
    return f"{mode.replace('+', '_')}_{'train' if training else 'eval'}_"


def make_case(m, Config, name, H, W, seed, cap, runs):
    model, cfg = wu.make_uncertainty_model(m, Config, "dino", "cpu", seed=seed)
    model.conv_seg = torch.nn.Conv2d(C, 1, kernel_size=1)
    model.bn = torch.nn.SyncBatchNorm(C)
    model = model.double()
    cfg.uncertainty_dino_max_size = cap
    g = torch.Generator().manual_seed(100 + seed)
    with torch.no_grad():
        model.conv_seg.weight.copy_(torch.randn(1, C, 1, 1, generator=g, dtype=torch.float64) * 0.05)
        model.conv_seg.bias.fill_(0.1)
        model.bn.weight.copy_(1 + 0.2 * torch.randn(C, generator=g, dtype=torch.float64))
        model.bn.bias.copy_(0.1 * torch.randn(C, generator=g, dtype=torch.float64))
        model.bn.running_mean.copy_(0.1 * torch.randn(C, generator=g, dtype=torch.float64))
        model.bn.running_var.copy_(1 + torch.rand(C, generator=g, dtype=torch.float64))
    start = {k: v.clone() for k, v in model.state_dict().items() if not k.startswith("backbone.")}
    fn, calls = stub_backbone(seed)
    model.backbone.get_intermediate_layers = fn
    gt, pred = images(H, W, seed)
    inputs = dict(gt=gt, pred=pred, conv_w=model.conv_seg.weight.detach().clone(), conv_b=model.conv_seg.bias.detach().clone(),
                  bn_w=model.bn.weight.detach().clone(), bn_b=model.bn.bias.detach().clone(),
                  running_mean_in=model.bn.running_mean.clone(), running_var_in=model.bn.running_var.clone())
    q = lambda t: (t * STAT_SCALE).round().clamp(-STAT_SCALE, STAT_SCALE - 1) / STAT_SCALE
    inputs["ssim"] = q(m.ssim_down(gt, pred, max_size=400))
    inputs["msssim"] = q(m.msssim(gt, pred, max_size=400, min_size=80))
    gd, pd = m.dino_downsample(gt, max_size=350), m.dino_downsample(pred, max_size=350)
    inputs["msssim_down"] = q(m.msssim(gd, pd, min_size=80))
    torch.manual_seed(7)
    inputs["mask"] = torch.nn.functional.dropout2d(torch.ones(1, C, 1, 1, dtype=torch.float64), p=cfg.uncertainty_dropout,
                                                   training=True).reshape(C)
    out = {}
    # the loss statements see the rounded statistics stored in the file
    saved = m.ssim_down, m.msssim
    m.ssim_down = lambda *a, **k: inputs["ssim"]
    m.msssim = lambda x, y, max_size=None, min_size=200: inputs["msssim"] if max_size == 400 else inputs["msssim_down"]
    try:
        for mode, training in runs:
            model.load_state_dict(start, strict=False)
            model.zero_grad(set_to_none=True)
            model.train(training)
            cfg.uncertainty_mode = mode
            calls.clear()
            torch.manual_seed(7)
            loss, metrics, loss_mult = model._compute_losses(gt, pred)
            loss.backward()
            assert len(calls) == (3 if mode.startswith("dino") else 1), (mode, len(calls))
            inputs["feat"] = calls[0]
            if len(calls) == 3:
                inputs["feat_gt_down"], inputs["feat_pred_down"] = calls[1], calls[2]
            t = tag(mode, training)
            metrics_t = torch.tensor([metrics[k] for k in METRICS], dtype=torch.float64)
            out.update({t + "loss": loss.detach(), t + "metrics": metrics_t,
                        t + "loss_mult": loss_mult[..., ::STRIDE, ::STRIDE], t + "d_conv_w": model.conv_seg.weight.grad,
                        t + "d_conv_b": model.conv_seg.bias.grad, t + "d_bn_w": model.bn.weight.grad,
                        t + "d_bn_b": model.bn.bias.grad, t + "running_mean": model.bn.running_mean.clone(),
                        t + "running_var": model.bn.running_var.clone()})
            print(name, mode, "train" if training else "eval", round(float(loss), 6), "loss_mult", tuple(loss_mult.shape))
    finally:
        m.ssim_down, m.msssim = saved
    arrays = {k: v.detach().numpy() for k, v in {**inputs, **out}.items()}
    for k in ("feat", "feat_gt_down", "feat_pred_down"):
        if k in arrays:
            arrays[k] = arrays[k].astype(np.float32)
    for k in ("ssim", "msssim", "msssim_down"):
        arrays[k] = np.round(arrays[k] * STAT_SCALE).astype(np.int16)
    for k in ("gt", "pred"):
        arrays[k] = np.round(arrays[k] * 255).astype(np.uint8)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), clip_min=cfg.uncertainty_clip_min,
                        reg_weight=cfg.uncertainty_regularizer_weight, eps=model.bn.eps, momentum=model.bn.momentum,
                        stride=STRIDE, stat_scale=STAT_SCALE, cap=-1 if cap is None else cap,
                        runs=np.array([tag(mo, tr) for mo, tr in runs]), **arrays)


if __name__ == "__main__":
    m, Config = import_reference()
    for case in CASES:
        make_case(m, Config, *case)
