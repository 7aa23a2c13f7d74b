"""SURVEY 8f-4: ``compute_3D_filter`` (method.py:1140-1190) over all cameras in two kernels (csrc/filter3d.cu).

not gpu: the numpy oracle against golden outputs of the reference's own method (tests/golden/filter3d_*.npz, made by
make_golden_filter3d.py); the host-side camera table.  gpu: the kernel through wildgaussians_fused.compute_3D_filter against
the goldens, the oracle, and the unmodified method run on the same device.
Tolerance: every value is one fp32 min / divide / multiply of a camera-space depth: 2e-6 relative; the in-image test is a
discontinuity, so a Gaussian within an ulp of an image border may pick another camera -- at most 0.1 % of the entries may
differ by more (observed: none)."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import filter3d_oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load(name):
    z = np.load(os.path.join(GOLD, f"filter3d_{name}.npz"))
    cams = [types.SimpleNamespace(poses=z["poses"][i], image_sizes=z["sizes"][i], intrinsics=z["intrinsics"][i])
            for i in range(z["poses"].shape[0])]
    return z["xyz"], cams, z["filter_3D"].reshape(-1)


def check(got, want, what):
    rel = np.abs(got - want) / np.abs(want)
    bad = int((rel > 2e-6).sum())
    assert bad <= max(0, int(1e-3 * want.size)), f"{what}: {bad} of {want.size} entries differ (max rel {rel.max():.3g})"
    return bad


@pytest.mark.parametrize("name", ["small", "many_cams"])
def test_oracle_matches_reference_golden(name):
    xyz, cams, want = load(name)
    got = filter3d_oracle.compute_3d_filter(xyz, cams)
    assert got.dtype == np.float32 and got.shape == want.shape
    check(got, want, "oracle vs reference")


def test_camera_table_layout():
    import wildgaussians_fused as wf
    xyz, cams, _ = load("small")
    table, focal = wf.camera_table(cams)
    assert table.shape == (len(cams), 20) and table.dtype == np.float32
    assert focal == max(float(c.intrinsics[0]) for c in cams)
    R, T = filter3d_oracle.camera_matrices(cams[3].poses)
    assert np.array_equal(table[3, :9].reshape(3, 3), R) and np.array_equal(table[3, 9:12], T)
    W, H = cams[3].image_sizes
    assert np.array_equal(table[3, 14:], np.array([W / 2.0, H / 2.0, -0.15 * W, W * 1.15, -0.15 * H, 1.15 * H], dtype=np.float32))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "many_cams"])
def test_kernel_matches_golden_and_oracle(name):
    import wildgaussians_fused as wf
    xyz, cams, want = load(name)
    dev = torch.device("cuda:0")
    model = types.SimpleNamespace(xyz=torch.from_numpy(xyz).to(dev), filter_3D=torch.zeros((xyz.shape[0], 1), device=dev))
    model.register_buffer = lambda k, v: setattr(model, k, v)
    wf.compute_3D_filter(model, cams)
    got = model.filter_3D.cpu().numpy()
    assert got.shape == (xyz.shape[0], 1)
    check(got.reshape(-1), want, "kernel vs reference golden")
    check(got.reshape(-1), filter3d_oracle.compute_3d_filter(xyz, cams), "kernel vs oracle")


@pytest.mark.gpu
def test_kernel_matches_unmodified_method_on_the_device_and_unseen_gaussians():
    import wg_harness as wh
    import wildgaussians_fused as wf
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    dev = torch.device("cuda:0")
    P = 200_003
    cfg = Config(source_path="", model_path="", uncertainty_mode="disabled")
    model = m.GaussianModel(cfg, training_setup=False).to(dev)
    model._resize_parameters(P)
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():
        pts = torch.randn(P, 3, generator=g) * 2.5
        pts[:5000, 2] = -60.0 - pts[:5000, 2].abs()      # behind every camera below: exercises `distance[~valid] = max`
        model.xyz.copy_(pts)
    cams = []
    for k in range(40):                                  # cameras at z = -8 .. -6 looking along +z, slightly shifted
        c2w = np.concatenate([np.eye(3, dtype=np.float32), np.array([[0.05 * k - 1.0], [0.3 * (k % 3)], [-8.0 + 0.05 * k]], dtype=np.float32)], axis=1)
        W, H = 640 + 8 * k, 480 + 4 * k
        cams.append(types.SimpleNamespace(poses=c2w, image_sizes=np.array([W, H], dtype=np.int32),
                                          intrinsics=np.array([420.0 + 3 * k, 425.0 + 3 * k, W / 2.0, H / 2.0], dtype=np.float32)))
    model.compute_3D_filter(cams)                 # the reference's own statements, on the GPU
    want = model.filter_3D.detach().cpu().numpy().reshape(-1)
    wf.enable(model)
    model.compute_3D_filter(cams)
    got = model.filter_3D.detach().cpu().numpy()
    assert got.shape == (P, 1) and model.filter_3D.device.type == "cuda"
    check(got.reshape(-1), want, "kernel vs method.py on the device")
    assert len(set(got[:5000, 0].tolist())) == 1 and got[0, 0] == got.max()
    wf.disable(model)
