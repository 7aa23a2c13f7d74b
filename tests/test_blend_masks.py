"""Blend masks (GPU): the forward records, per tile, 8x8 pixel block and list position below K = 1024, whether some
pixel of the block blended that position; the backward walks only those positions (common.cuh, render_bwd.cu).

* The masks read from the image buffer equal a float64 numpy recomputation from the projected records, the sorted
  instance list, the tile ranges and n_contrib, at every position below the block's largest n_contrib (positions
  whose alpha or power lies within a hair of a threshold are not compared).
* A scene dense enough that tile lists run past K (the footprint-box fallback of the backward) has gradients within
  the parity bar against the compiled reference.
"""
import numpy as np
import pytest
import torch

import synthetic
from golden_util import GRAD_NAMES
from make_golden import backward_args, call_args

pytestmark = pytest.mark.gpu

K = 1024
WORDS = K // 32
BLOCKS = 4

SMALL = [dict(P=20_000, W=320, H=240, sh_degree=None, seed=41),
         dict(P=30_000, W=300, H=200, sh_degree=None, seed=42, subpixel_jitter=0.3)]
# ~100k faint Gaussians over 4x4 tiles: lists of thousands of instances and n_contrib beyond K
DENSE = dict(P=100_000, W=64, H=64, sh_degree=None, seed=43)
DENSE_OPACITY = 0.01


def _scene(kw, opacity=None):
    scene = synthetic.make_scene(**kw)
    if opacity is not None:
        scene["opacities"] = torch.full_like(scene["opacities"], opacity)
    return scene


def _run(kw, opacity=None):
    """Forward + backward through the C ABI; returns numpy arrays of the artefacts the tests compare."""
    from diff_gaussian_rasterization import _C
    d = synthetic.to_device(_scene(kw, opacity), torch.device("cuda:0"))
    W, H = d["image_width"], d["image_height"]
    P = d["means3D"].shape[0]
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(*call_args(d))
    v = _C.debug_views(geom, binning, img, P, 0, W, H, R)
    grads = _C.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))
    torch.cuda.synchronize()
    T = ((W + 15) // 16) * ((H + 15) // 16)
    # the mask array follows the tile ranges in the image buffer, 256-byte aligned (api.cu carve_img)
    end = v["ranges"].data_ptr() + 8 * T
    off = ((end + 255) // 256) * 256 - img.data_ptr()
    masks = img.view(torch.uint8)[off:off + 4 * T * BLOCKS * WORDS].view(torch.int32).view(T, BLOCKS, WORDS)
    out = dict(masks=masks.cpu().numpy().view(np.uint32), color=color.cpu().numpy(), radii=radii.cpu().numpy(),
               n_contrib=v["n_contrib"].cpu().numpy().astype(np.int64), ranges=v["ranges"].cpu().numpy().astype(np.int64),
               point_list=v["point_list"].cpu().numpy().astype(np.int64), records=v["records"].cpu().numpy(),
               subpixel_offset=d["subpixel_offset"].cpu().numpy(), W=W, H=H)
    for n, g in zip(GRAD_NAMES, grads):
        out["grad_" + n] = g.cpu().numpy()
    return out


def _block_last(o):
    """[T, 4] largest n_contrib of each 8x8 block."""
    W, H = o["W"], o["H"]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    nc = np.zeros((gy * 16, gx * 16), np.int64)
    nc[:H, :W] = o["n_contrib"]
    b = nc.reshape(gy, 2, 8, gx, 2, 8).max(axis=(2, 5))          # [gy, by, gx, bx]
    return b.transpose(0, 2, 1, 3).reshape(gy * gx, 4)             # block k = bx + 2 by


def _expected_masks(o):
    """bits[T, 4, K] recomputed in float64, and a `sure` flag that is False near a threshold."""
    W, H = o["W"], o["H"]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    last = _block_last(o)
    rec = o["records"].astype(np.float64)
    so = o["subpixel_offset"].astype(np.float64)
    bits = np.zeros((gx * gy, 4, K), bool)
    sure = np.ones((gx * gy, 4, K), bool)
    for t in range(gx * gy):
        r0, r1 = o["ranges"][t]
        tx, ty = t % gx, t // gx
        for k in range(4):
            n = int(min(last[t, k], K, r1 - r0))
            if n == 0:
                continue
            x0, y0 = tx * 16 + 8 * (k % 2), ty * 16 + 8 * (k // 2)
            ys, xs = np.mgrid[y0:min(y0 + 8, H), x0:min(x0 + 8, W)]
            if ys.size == 0:
                continue
            px = (xs + so[ys, xs, 0]).ravel()
            py = (ys + so[ys, xs, 1]).ravel()
            ncp = o["n_contrib"][ys, xs].ravel()
            ids = o["point_list"][r0:r0 + n]
            g = rec[ids]
            dx = g[:, 0:1] - px[None, :]
            dy = g[:, 1:2] - py[None, :]
            power = -0.5 * (g[:, 4:5] * dx * dx + g[:, 6:7] * dy * dy) - g[:, 5:6] * dx * dy
            alpha = np.minimum(0.99, g[:, 7:8] * np.exp(power))
            live = np.arange(n)[:, None] < ncp[None, :]
            act = live & (power <= 0) & (alpha >= 1 / 255)
            near = live & ((np.abs(power) < 1e-5) | (np.abs(alpha - 1 / 255) < 1e-6))
            bits[t, k, :n] = act.any(axis=1)
            sure[t, k, :n] = ~near.any(axis=1)
            sure[t, k, n:] = False
        sure[t, :, :] &= np.arange(K)[None, :] < np.minimum(last[t], K)[:, None]
    return bits, sure


def _unpack(masks):
    return ((masks[..., :, None] >> np.arange(32, dtype=np.uint32)) & 1).astype(bool).reshape(masks.shape[0], 4, K)


def _check_masks(o):
    bits, sure = _expected_masks(o)
    got = _unpack(o["masks"])
    assert sure.sum() > 1000, "too few positions compared"
    bad = (got != bits) & sure
    assert not bad.any(), f"{int(bad.sum())} mask bits differ, first at {np.argwhere(bad)[:5].tolist()}"


@pytest.mark.parametrize("kw", SMALL, ids=lambda k: f"P{k['P']}_{k['W']}x{k['H']}_s{k['seed']}")
def test_masks_match_numpy(kw):
    _check_masks(_run(kw))


def test_fallback_beyond_k_against_compiled_reference():
    from oracle import ref_cuda
    from test_gpu_parity import check_grad
    if not ref_cuda.available():
        pytest.skip("oracle/_ref/libdgr_ref.so not present")
    o = _run(DENSE, DENSE_OPACITY)
    assert int(o["n_contrib"].max()) > K, "scene does not exercise the positions beyond K"
    d = synthetic.to_device(_scene(DENSE, DENSE_OPACITY), torch.device("cuda:0"))
    R, color, radii, geom, binning, img = ref_cuda.rasterize_gaussians(*call_args(d))
    rg = ref_cuda.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))
    rg2 = ref_cuda.rasterize_gaussians_backward(*backward_args(d, radii, geom, R, binning, img))
    torch.cuda.synchronize()
    assert np.array_equal(o["radii"], radii.cpu().numpy())
    for n, a, b in zip(GRAD_NAMES, rg, rg2):
        if a.numel() == 0:
            continue
        check_grad(n, torch.from_numpy(o["grad_" + n]).view_as(a.cpu()), a.cpu(), b.cpu())
