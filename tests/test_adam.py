"""SURVEY 8f-4: the optimizer step (method.py:2019 on the Adam built at :1033-1049).

not gpu: the numpy oracle against torch.optim.Adam itself (the reference's dependency, imported here on CPU), FusedAdam's
host logic (fallback for unsupported settings / CPU tensors).  gpu: csrc/adam.cu through the C ABI and through FusedAdam
against torch.optim.Adam on the same device and against the oracle, on parameter groups shaped like the reference's.
Tolerance: the update is a handful of fp32 operations per element; implementations differ by fma contraction only, so
|ours - torch| <= 2e-6 * lr-scaled update + 1e-7 * |param| (stated per assert below)."""
import numpy as np
import pytest
import torch

from oracle import adam_oracle


def reference_like_groups(P, device, seed=0, n_images=5):
    """Parameter groups with the shapes / learning rates / weight decay of method.py:1033-1049 (Config defaults)."""
    g = torch.Generator().manual_seed(seed)
    R = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(device).requires_grad_(True)
    mlp = [R(128, 59, scale=0.1), R(128, scale=0.1), R(128, 128, scale=0.1), R(128, scale=0.1), R(6, 128, scale=0.1), R(6, scale=0.1)]
    return [
        {"params": [R(P, 3)], "lr": 0.00016 * 1.7, "name": "xyz"},
        {"params": [R(P, 3)], "lr": 0.0025, "name": "features_dc"},
        {"params": [R(P, 1)], "lr": 0.05, "name": "opacities"},
        {"params": [R(P, 3)], "lr": 0.005, "name": "scales"},
        {"params": [R(P, 4)], "lr": 0.001, "name": "rotations"},
        {"params": [R(n_images, 32, scale=0.01)], "lr": 0.001, "name": "appearance_embeddings", "weight_decay": 0.02},
        {"params": [R(P, 24, scale=0.3)], "lr": 0.005, "name": "embeddings"},
        {"params": [R(P, 45, scale=0.3)], "lr": 0.0025 / 20.0, "name": "features_rest"},
        {"params": mlp, "lr": 0.0005, "name": "appearance_mlp"},
    ]


def clone_groups(groups):
    return [{**g, "params": [p.detach().clone().requires_grad_(True) for p in g["params"]]} for g in groups]


def set_grads(groups, seed, sparse_rows=False):
    g = torch.Generator().manual_seed(seed)
    for gr in groups:
        for p in gr["params"]:
            grad = torch.randn(p.shape, generator=g) * 0.01
            if sparse_rows and p.dim() == 2 and p.shape[0] > 64:      # most Gaussians receive no gradient in a step
                grad[torch.rand(p.shape[0], generator=g) < 0.8] = 0.0
            p.grad = grad.to(p.device)


def test_oracle_matches_torch_adam_cpu():
    groups = reference_like_groups(3000, "cpu", seed=1)
    opt = torch.optim.Adam(clone_groups(groups), lr=1.0, eps=1e-15)
    state = [[(p.detach().numpy().copy(), np.zeros(p.shape, np.float32), np.zeros(p.shape, np.float32)) for p in g["params"]]
             for g in opt.param_groups]
    for step in range(1, 6):
        set_grads(opt.param_groups, 100 + step, sparse_rows=True)
        grads = [[p.grad.numpy().copy() for p in g["params"]] for g in opt.param_groups]
        opt.step()
        for gi, g in enumerate(opt.param_groups):
            for pi, p in enumerate(g["params"]):
                p0, m0, v0 = state[gi][pi]
                p1, m1, v1 = adam_oracle.adam_step(p0, grads[gi][pi], m0, v0, step, g["lr"], eps=1e-15,
                                                   weight_decay=g.get("weight_decay", 0.0))
                state[gi][pi] = (p1, m1, v1)
                st = opt.state[p]
                # one fp32 rounding of the update (|update| <= ~lr) + one of the parameter
                tol = 4e-7 * g["lr"] * step ** 0.5 * 4 + 2e-7 * np.abs(p1).max()
                assert np.abs(p1 - p.detach().numpy()).max() <= tol, (g["name"], step)
                # moments: a few fp32 roundings relative to the tensor's scale (entries near zero come from cancellation)
                mt, vt = st["exp_avg"].numpy(), st["exp_avg_sq"].numpy()
                assert np.abs(m1 - mt).max() <= 1e-6 * np.abs(mt).max()
                assert np.abs(v1 - vt).max() <= 1e-6 * np.abs(vt).max()


def test_fused_adam_falls_back_on_cpu_tensors_and_unsupported_settings():
    import fused_adam
    groups = reference_like_groups(500, "cpu", seed=2)
    a = torch.optim.Adam(clone_groups(groups), lr=1.0, eps=1e-15)
    b = fused_adam.FusedAdam(clone_groups(groups), lr=1.0, eps=1e-15)            # CPU tensors: torch's own step runs
    c = fused_adam.adopt(torch.optim.Adam(clone_groups(groups), lr=1.0, eps=1e-15, amsgrad=True))
    assert isinstance(c, fused_adam.FusedAdam) and isinstance(c, torch.optim.Adam)
    for step in range(3):
        for o in (a, b, c):
            set_grads(o.param_groups, 7 + step)
            o.step()
    for ga, gb in zip(a.param_groups, b.param_groups):
        for pa, pb in zip(ga["params"], gb["params"]):
            assert torch.equal(pa, pb)
            assert torch.equal(a.state[pa]["exp_avg_sq"], b.state[pb]["exp_avg_sq"])
    assert "max_exp_avg_sq" in c.state[c.param_groups[0]["params"][0]]               # amsgrad really ran in torch
    with pytest.raises(TypeError):
        fused_adam.adopt(torch.optim.SGD([torch.zeros(3, requires_grad=True)], lr=0.1))


@pytest.mark.gpu
def test_fused_adam_matches_torch_adam_and_oracle():
    import fused_adam
    dev = torch.device("cuda:0")
    groups = reference_like_groups(70001, dev, seed=3)          # not a multiple of the 4096-element chunk
    ref = torch.optim.Adam(clone_groups(groups), lr=1.0, eps=1e-15)
    ours = fused_adam.FusedAdam(clone_groups(groups), lr=1.0, eps=1e-15)
    oracle_state = None
    for step in range(1, 8):
        set_grads(ref.param_groups, 50 + step, sparse_rows=True)
        for gr, go in zip(ref.param_groups, ours.param_groups):
            for pr, po in zip(gr["params"], go["params"]):
                po.grad = pr.grad.clone()
        if step == 4:                                            # per-group lr changes (method.py:1206-1209 does it every step)
            ref.param_groups[0]["lr"] *= 0.5; ours.param_groups[0]["lr"] *= 0.5
        if step == 1:
            p0 = ours.param_groups[7]["params"][0]
            oracle_state = (p0.detach().cpu().numpy().copy(), np.zeros(p0.shape, np.float32), np.zeros(p0.shape, np.float32))
        g7 = ours.param_groups[7]["params"][0].grad.cpu().numpy()
        ref.step(); ours.step()
        oracle_state = adam_oracle.adam_step(*oracle_state[:1], g7, *oracle_state[1:], step, ours.param_groups[7]["lr"], eps=1e-15)
        torch.cuda.synchronize()
        for gr, go in zip(ref.param_groups, ours.param_groups):
            for pr, po in zip(gr["params"], go["params"]):
                tol = 2e-6 * gr["lr"] + 1e-7 * float(pr.abs().max())
                assert float((pr - po).abs().max()) <= tol, (gr["name"], step)
                sr, so = ref.state[pr], ours.state[po]
                assert float((sr["exp_avg"] - so["exp_avg"]).abs().max()) <= 1e-6 * float(sr["exp_avg"].abs().max())
                assert float((sr["exp_avg_sq"] - so["exp_avg_sq"]).abs().max()) <= 1e-6 * float(sr["exp_avg_sq"].abs().max())
                assert float(sr["step"]) == float(so["step"]) == step
        p7 = ours.param_groups[7]["params"][0].detach().cpu().numpy()
        assert np.abs(p7 - oracle_state[0]).max() <= 2e-6 * ours.param_groups[7]["lr"] * step + 1e-7 * np.abs(p7).max()
    # state_dict round trip into a plain torch.optim.Adam (checkpoints stay interchangeable)
    plain = torch.optim.Adam(clone_groups(groups), lr=1.0, eps=1e-15)
    plain.load_state_dict(ours.state_dict())
    assert float(plain.state[plain.param_groups[0]["params"][0]]["step"]) == 7


@pytest.mark.gpu
def test_adam_c_abi_arguments_and_zero_grads():
    import ctypes
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda:0")
    n = 10007
    p, g = torch.randn(n, device=dev), torch.randn(n, device=dev) * 0.1
    m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    # an unaligned view exercises the scalar path
    pu, gu, mu, vu = (t.clone()[1:] for t in (p, g, m, v))
    want = adam_oracle.adam_step(p.cpu().numpy(), g.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy(), 1, 0.01, eps=1e-15, weight_decay=0.1)
    segs = (_C.GsrAdamSegment * 2)()
    for s, (a, b, c, d) in zip(segs, ((p, g, m, v), (pu, gu, mu, vu))):
        s.param, s.grad, s.exp_avg, s.exp_avg_sq, s.n, s.step, s.lr, s.weight_decay = a.data_ptr(), b.data_ptr(), c.data_ptr(), d.data_ptr(), a.numel(), 1, 0.01, 0.1
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    assert _C._lib.gsr_adam_step(segs, 2, 0.9, 0.999, 1e-15, 1, stream) == 0
    torch.cuda.synchronize()
    assert np.abs(p.cpu().numpy() - want[0]).max() <= 1e-6
    assert np.abs(pu.cpu().numpy() - want[0][1:]).max() <= 1e-6
    assert float(g.abs().max()) == 0.0 and float(gu.abs().max()) == 0.0          # zero_grads
    assert _C._lib.gsr_adam_step(segs, 33, 0.9, 0.999, 1e-15, 0, stream) != 0       # too many segments
    segs[0].step = 0
    assert _C._lib.gsr_adam_step(segs, 1, 0.9, 0.999, 1e-15, 0, stream) != 0        # step must be >= 1
    assert _C._lib.gsr_adam_step(segs, 1, 1.5, 0.999, 1e-15, 0, stream) != 0        # bad beta
    assert _C._lib.gsr_adam_step(None, 0, 0.9, 0.999, 1e-15, 0, stream) == 0        # nothing to do


@pytest.mark.gpu
def test_adopting_the_optimizer_built_by_the_unmodified_method_py():
    """`GaussianModel._setup_optimizers` (method.py:1029-1053, unmodified) builds the optimizer; `fused_adam.adopt` turns that
    very object into the fused one; three train-step-like iterations (gradients from `_render_internal` + loss.backward,
    then `optimizer.step()` as method.py:2019 calls it) give the same parameters as the untouched optimizer."""
    import copy
    import synthetic
    import wg_harness as wh
    import fused_adam
    m, Config = wh.import_method()
    if m is None:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    import diff_gaussian_rasterization as ours
    dev = torch.device("cuda:0")
    kw = dict(P=30_000, W=320, H=200, seed=71)
    scene = synthetic.make_scene(sh_degree=3, **kw)
    cam = wh.make_camera(scene)
    g = torch.Generator().manual_seed(5)
    G1, G2 = torch.randn(3, kw["H"], kw["W"], generator=g).to(dev), torch.randn(3, kw["H"], kw["W"], generator=g).to(dev)
    wh.use_backend(m, ours.GaussianRasterizer, ours.GaussianRasterizationSettings)
    models = []
    for fused in (False, True):
        model, cfg = wh.make_model(m, Config, scene, dev, seed=kw["seed"])
        model.spatial_lr_scale.fill_(1.7)
        model._setup_optimizers()
        assert type(model.optimizer) is torch.optim.Adam and len(model.optimizer.param_groups) >= 8
        if fused:
            fused_adam.adopt(model.optimizer)
            assert isinstance(model.optimizer, fused_adam.FusedAdam)
        models.append((model, cfg))
    for it in range(3):
        grads = None
        for model, cfg in models:
            wh.train_step(model, cfg, cam, G1, G2)
            if grads is None:       # the composite's float atomics are not run-to-run reproducible: both optimizers see the SAME gradients
                grads = [p.grad.clone() if p.grad is not None else None for p in model.parameters()]
            else:
                for p, gr in zip(model.parameters(), grads):
                    p.grad = None if gr is None else gr.clone()
            model.optimizer.step()
            model.optimizer.zero_grad(set_to_none=True)
        for (na, pa), (nb, pb) in zip(models[0][0].named_parameters(), models[1][0].named_parameters()):
            lr = max(g_["lr"] for g_ in models[0][0].optimizer.param_groups)
            assert float((pa - pb).abs().max()) <= 2e-6 * lr + 1e-7 * float(pa.abs().max()), (na, it)
