"""CPU tests: the C restatement (oracle/oracle.c) against golden vectors produced by the UNMODIFIED reference
CUDA rasterizer on a GPU (tests/golden/make_golden.py).  This is what pins the oracle (SURVEY.md 8c)."""
import numpy as np
import pytest

from golden_util import GRAD_NAMES, GRAD_TOL, PIX_TOL, bits, load_case, rel_err
from make_golden import CASES
from oracle import cpu_oracle


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    scene, gold = load_case(request.param)
    st = cpu_oracle.forward(scene)
    return request.param, scene, gold, st


def test_integer_artefacts_bit_exact(case):
    name, scene, gold, st = case
    assert st["num_rendered"] == int(gold["num_rendered"])
    assert np.array_equal(st["radii"], gold["radii"])
    assert np.array_equal(st["tiles_touched"].astype(np.int32), gold["tiles_touched"])
    assert np.array_equal(st["point_list"].astype(np.int32), gold["point_list"]), "sorted instance list differs"
    assert np.array_equal(st["ranges"].astype(np.int32), gold["ranges"])


def test_projected_state_bit_exact(case):
    """depths / means2D / cov3D / conic+opacity / SH colours: same bits as the reference (notes N1, N2)."""
    name, scene, gold, st = case
    vis = gold["radii"] > 0
    for k in ("depths", "means2D", "conic_opacity"):
        assert np.array_equal(bits(st[k][vis]), bits(gold[k][vis])), k
    if "scales" in scene:
        assert np.array_equal(bits(st["cov3D"][vis]), bits(gold["cov3D"][vis]))
    if "shs" in scene:
        assert np.array_equal(bits(st["rgb"][vis]), bits(gold["rgb"][vis]))


def test_composite_within_tolerance(case):
    """Pixels within 1e-4 (measured: ~2e-7; expf differs from CUDA's by an ulp).  n_contrib may flip where an
    alpha sits on a threshold: allow 1e-4 of the pixels."""
    name, scene, gold, st = case
    assert np.abs(st["out_color"] - gold["out_color"]).max() < PIX_TOL
    assert np.abs(st["final_T"] - gold["final_T"]).max() < PIX_TOL
    ne = (st["n_contrib"].astype(np.int32) != gold["n_contrib"]).mean()
    assert ne <= 1e-4, f"{ne:.2e} of n_contrib differ"


def test_gradients_within_tolerance(case):
    name, scene, gold, st = case
    g = cpu_oracle.backward(st, scene["dL_dpix"])
    for n in GRAD_NAMES:
        ref = gold[n]
        if ref.size == 0:
            continue
        assert rel_err(g[n].reshape(ref.shape), ref) < GRAD_TOL, n
