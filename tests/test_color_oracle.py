"""Colour-path oracle (oracle/color_oracle.py, SURVEY 8f-2) against golden vectors produced by the reference itself
(tests/golden/make_golden_colors.py imports wildgaussians/method.py), and an import-level drop-in check."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
CASES = ["colors_deg3", "colors_deg1"]


def _load(name):
    d = dict(np.load(os.path.join(GOLD, name + ".npz")))
    w = tuple(d[k] for k in ("W1", "b1", "W2", "b2", "W3", "b3"))
    return d, w


def _colors(d, w, **over):
    from oracle import color_oracle as co
    a = dict(features=d["features"], gembedding=d["gembedding"], aembedding=d["aembedding"][None], weights=w)
    a.update(over)
    feats = np.minimum(a["features"], 1.0)          # `features = gaussians["features"].clamp_max(1.0)` (method.py:1570)
    return co.toned_colors(feats, a["gembedding"], a["aembedding"], a["weights"], d["means3D"], d["campos"],
                           int(d["active_deg"]))


@pytest.mark.parametrize("name", CASES)
def test_forward_matches_the_reference(name):
    d, w = _load(name)
    got = _colors(d, w)
    assert got.shape == d["colors"].shape
    assert np.abs(got - d["colors"]).max() < 1e-12          # fp64 on both sides
    if name == "colors_deg3":                                # the trained-like case exercises the clamp at 0
        assert (d["colors"] == 0).any() and (d["colors"] > 0).any()


@pytest.mark.parametrize("name", CASES)
def test_reference_gradients_are_the_gradients_of_the_oracle(name):
    """Central differences of loss = sum(colors * dL) through the oracle reproduce the reference's autograd gradients
    (spot-checked entries): the fixtures' gradients are usable as the parity target of a fused backward."""
    d, w = _load(name)
    dL = d["dL_dcolors"]
    rng = np.random.default_rng(0)

    def loss(**over):
        return float((_colors(d, w, **over) * dL).sum())

    eps = 1e-6
    for key, gkey in (("features", "g_features"), ("gembedding", "g_gembedding")):
        base = d[key]
        for _ in range(6):
            i, j = rng.integers(base.shape[0]), rng.integers(base.shape[1])
            if key == "features" and abs(base[i, j] - 1.0) < 1e-3:
                continue                                         # kink of clamp_max
            hi, lo = base.copy(), base.copy()
            hi[i, j] += eps; lo[i, j] -= eps
            fd = (loss(**{key: hi}) - loss(**{key: lo})) / (2 * eps)
            assert abs(fd - d[gkey][i, j]) < 1e-5 * max(1.0, abs(fd)), (key, i, j, fd, d[gkey][i, j])
    for wi, gname in ((0, "g_W1"), (2, "g_W2"), (4, "g_W3"), (5, "g_b3")):
        base = w[wi]
        idx = tuple(rng.integers(s) for s in base.shape)
        hi, lo = base.copy(), base.copy()
        hi[idx] += eps; lo[idx] -= eps
        wh, wl = list(w), list(w)
        wh[wi], wl[wi] = hi, lo
        fd = (loss(weights=tuple(wh)) - loss(weights=tuple(wl))) / (2 * eps)
        assert abs(fd - d[gname][idx]) < 1e-5 * max(1.0, abs(fd)), (gname, idx, fd, d[gname][idx])


def test_reference_method_module_imports_on_the_drop_in_package():
    """wildgaussians/method.py:26 (`from diff_gaussian_rasterization import GaussianRasterizationSettings,
    GaussianRasterizer`) resolves to this repo's package; only possible where build() copied the reference's package."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import wg_harness
    m, _ = wg_harness.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    import diff_gaussian_rasterization as ours
    assert m.GaussianRasterizer is ours.GaussianRasterizer
    assert m.GaussianRasterizationSettings is ours.GaussianRasterizationSettings
    assert m.GaussianRasterizationSettings._fields[0] == "image_height" and len(m.GaussianRasterizationSettings._fields) == 15


@pytest.mark.parametrize("name", CASES)
def test_torch_restatement_matches_the_reference_outputs_and_gradients(name):
    """oracle/color_torch.py (the oracle of the fused CUDA colour op) in fp64 against the reference's own outputs and
    autograd gradients."""
    import torch
    from oracle import color_torch as ct
    d, w = _load(name)
    t = {k: torch.tensor(d[k], dtype=torch.float64, requires_grad=True) for k in
         ("features", "gembedding", "aembedding", "W1", "b1", "W2", "b2", "W3", "b3")}
    f = t["features"]
    raw, toned = ct.colors(f[:, :3], f[:, 3:], t["gembedding"], t["aembedding"], t["W1"], t["b1"], t["W2"], t["b2"], t["W3"],
                           t["b3"], torch.tensor(d["means3D"]), torch.tensor(d["campos"]), int(d["active_deg"]))
    assert float((toned.detach() - torch.tensor(d["colors"])).abs().max()) < 1e-12
    (toned * torch.tensor(d["dL_dcolors"])).sum().backward()
    for k, g in (("features", "g_features"), ("gembedding", "g_gembedding"), ("aembedding", "g_aembedding"), ("W1", "g_W1"),
                 ("b1", "g_b1"), ("W2", "g_W2"), ("b2", "g_b2"), ("W3", "g_W3"), ("b3", "g_b3")):
        assert float((t[k].grad - torch.tensor(d[g])).abs().max()) < 1e-10 * max(1.0, float(np.abs(d[g]).max())), k
