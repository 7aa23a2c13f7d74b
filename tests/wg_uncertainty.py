"""TEST / BENCH INFRASTRUCTURE -- the reference's ``UncertaintyModel`` (wildgaussians/method.py:204-442) built offline.

``UncertaintyModel.__init__`` asks its backbone factory for pretrained DINOv2 weights (method.py:212), which downloads
them (dinov2.py:938-942).  ``offline()`` prevents that: inside it the factory is called with ``pretrained=False`` (random
ViT-S/14 weights; a ``functools.partial`` would not do, because the call's explicit ``pretrained=True`` overrides it) and
``torch.hub.load_state_dict_from_url`` and ``urllib.request.urlopen`` raise.  Timing and the code paths exercised do not
depend on the weights.  Dropout is active in training mode, so compared runs seed the RNG identically.
"""
from __future__ import annotations

import contextlib
import urllib.request

import torch


def _no_network(*args, **kwargs):
    raise RuntimeError("network access is disabled here")


@contextlib.contextmanager
def offline(m, backbone: str = "dinov2_vits14_reg"):
    """Inside: method module `m`'s DINOv2 factory builds random weights and the two download functions raise."""
    orig = getattr(m.dinov2, backbone)
    saved = (torch.hub.load_state_dict_from_url, urllib.request.urlopen)
    setattr(m.dinov2, backbone, lambda **kw: orig(**{**kw, "pretrained": False}))
    torch.hub.load_state_dict_from_url, urllib.request.urlopen = _no_network, _no_network
    try:
        yield
    finally:
        setattr(m.dinov2, backbone, orig)
        torch.hub.load_state_dict_from_url, urllib.request.urlopen = saved


def make_uncertainty_model(m, Config, mode: str, device, seed: int = 0):
    """An ``UncertaintyModel`` in training mode with random backbone weights and the given ``uncertainty_mode``."""
    cfg = Config(source_path="", model_path="", uncertainty_mode=mode)
    torch.manual_seed(seed)
    with offline(m, cfg.uncertainty_backbone):
        model = m.UncertaintyModel(cfg)
    model = model.to(device)
    model.train()
    return model, cfg


def compute_losses(model, gt, prediction, seed: int = 0):
    """``_compute_losses`` (method.py:363-433) on [3,H,W] images with a fixed RNG state, then its backward.
    Returns (loss, metrics, loss_mult, {head parameter name: gradient})."""
    for p in model.parameters():
        p.grad = None
    torch.manual_seed(seed)
    loss, metrics, loss_mult = model._compute_losses(gt.unsqueeze(0), prediction.unsqueeze(0))
    loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    return loss.detach(), metrics, loss_mult.detach(), grads
