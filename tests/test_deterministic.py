"""Reproducible runs under ``torch.use_deterministic_algorithms(True)``: the fixed-order reductions of the backward
composite (``render_bwd.cu``), the colour-only backward (``gsr_backward_colors``) and the colour op
(``appearance.cu``), and the refusal of the multi-GPU backward reductions.

CPU tests: the shims set ``deterministic`` from the flag on every call (a recording stand-in for the library), and the
multi-GPU backward raises, or warns under ``warn_only=True``.

GPU tests: with the flag on, every accumulator entry of the backward composite stays within its ``oracle/bwd_bound.c``
bound on the scenes of ``test_backward_exact``; three runs (one after unrelated work on another stream) give the same
bits for the accumulator and the 8 gradients, which agree with the default path within ``test_gpu_parity.check_grad``'s
bars; the colour op stays within its ``oracle/color_exact.py`` bounds and repeats bit for bit, as does the
embedding-only backward; and short fused training runs and ``optimize_embedding`` calls, each made twice in a fresh
process, return the same bits.
"""
import contextlib
import ctypes
import json
import os
import subprocess
import sys
import types
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def deterministic(on=True, warn_only=False):
    was, was_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=was_warn)


# ======================================================================================================================
# CPU
# ======================================================================================================================
class _Recorder:
    """Stands in for libgsrast: records the ``deterministic`` field of every args struct it is handed, returns 0."""

    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        if name in ("gsr_last_error", "gsr_appearance_deterministic_scratch_bytes"):
            return getattr(self.real, name)

        def call(*args):
            flags = [a._obj.deterministic for a in args if hasattr(a, "_obj") and hasattr(a._obj, "deterministic")]
            self.calls.append((name, flags))
            return 0
        return call


def _embedding_loop_stub():
    from diff_gaussian_rasterization import _C
    f32 = dict(dtype=torch.float32)
    ba, aa = _C.GsrBackwardArgs(), _C.GsrAppearanceArgs()
    ba.P, ba.R, aa.P = 4, 6, 4
    return types.SimpleNamespace(stream=0, bwd_args=ba, app_args=aa, dcolor=torch.zeros((4, 3), **f32),
                                 vis=torch.arange(4), dtoned_v=torch.zeros((4, 3), **f32), det_rows=None,
                                 pack=torch.zeros(8, **f32), w=[torch.zeros(1, **f32)], param=torch.zeros(32, **f32),
                                 unpacked=[torch.zeros(1, **f32)] * 6)


def test_shims_set_the_field_from_the_flag_on_every_call(monkeypatch):
    """fused_embedding's backward calls and the rasterizer's backward carry deterministic = the flag at call time."""
    import fused_embedding as fe
    from diff_gaussian_rasterization import _C
    rec = _Recorder(_C._lib)
    monkeypatch.setattr(_C, "_lib", rec)
    monkeypatch.setattr(fe, "_lib", rec, raising=False)
    monkeypatch.setattr(_C, "_stream", lambda dev: 0)
    loop = _embedding_loop_stub()
    loop.param.grad = torch.zeros(32)
    for flag in (False, True, False):
        rec.calls.clear()
        with deterministic(flag):
            fe.EmbeddingLoop.embedding_grad(loop, torch.zeros((3, 2, 2)))
        got = {n: f for n, f in rec.calls if f}
        assert got == {"gsr_backward_colors": [int(flag)], "gsr_appearance_embedding_backward": [int(flag)]}, rec.calls

    # the rasterizer's backward: accumulator alignment and CUDA device scoping are stubbed out
    big = torch.zeros(4 * 12 + 64 + 256)
    off = (-big.data_ptr()) % 256 // 4
    monkeypatch.setattr(_C, "_zero_accumulator", lambda P, dev: big[off:])
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    e = torch.empty(0)
    z = lambda *s: torch.zeros(*s)
    args = (z(3), z(4, 3), torch.ones(4, dtype=torch.int32), z(4, 3), z(4, 3), z(4, 4), 1.0, e, z(4, 4), z(4, 4), 1.0,
            1.0, 0.3, z(2, 2, 2), z(3, 2, 2), e, 0, z(3), z(8), 6, z(8), z(8), False)
    for flag in (True, False):
        rec.calls.clear()
        with deterministic(flag):
            _C.rasterize_gaussians_backward(*args)
        assert [f for n, f in rec.calls if n == "gsr_backward"] == [[int(flag)]], rec.calls


def test_multi_gpu_backward_raises_or_warns_under_the_flag():
    import parallel
    for fn in (lambda: parallel.sharded_backward(None, None), lambda: parallel.reduced_partials(None, 1, None)):
        with deterministic(True):
            with pytest.raises(RuntimeError, match="parallel.*deterministic"):
                fn()
        with deterministic(True, warn_only=True):
            with pytest.warns(UserWarning, match="deterministic"):
                with pytest.raises((TypeError, AttributeError, ValueError)):   # it goes on (here without a process group)
                    fn()
        with deterministic(False):
            with warnings.catch_warnings():
                warnings.simplefilter("error")
                with pytest.raises((TypeError, AttributeError, ValueError)):
                    fn()


# ======================================================================================================================
# GPU: backward composite
# ======================================================================================================================
def _grads(o):
    from diff_gaussian_rasterization import _C
    from make_golden import backward_args
    R, geom, binning, img = o["bufs"]
    g = _C.rasterize_gaussians_backward(*backward_args(o["d"], o["radii"], geom, R, binning, img))
    torch.cuda.synchronize()
    return [t.clone() for t in g]


def _partials(o, shard=None):
    from diff_gaussian_rasterization import _C
    from make_golden import backward_args
    R, geom, binning, img = o["bufs"]
    P = o["P"]
    acc = _C.rasterize_gaussians_backward_partials(*backward_args(o["d"], o["radii"], geom, R, binning, img),
                                                   shard=shard)[:P * 12].view(P, 12).clone()
    torch.cuda.synchronize()
    return acc


def _other_stream_work():
    """Unrelated work on another stream while nothing else runs: it leaves the device in another state (caches, clocks,
    allocator) for the next run."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.randn((4096, 4096), device="cuda")
        for _ in range(4):
            x = (x @ x).tanh()
    s.synchronize()


def _scenes():
    import test_backward_exact as be
    from test_adversarial_scenes import scene_shape
    from test_blend_masks import DENSE, DENSE_OPACITY, _scene
    out = {k: (lambda k=k: be.ordinary_scenes()[k]) for k in ("small_320x240", "small_300x200_jitter", "posed_bg")}
    out["dense"] = lambda: _scene(DENSE, DENSE_OPACITY)
    for n in (be.K - 1, be.K, be.K + 1, 64, 65):
        out[f"stack_{n}"] = lambda n=n: be.scene_stack(n)
    for W, H in ((1, 1), (1, 37), (17, 33), (4095, 3)):
        out[f"shape_{W}x{H}"] = lambda W=W, H=H: scene_shape(W, H)
    return out


SCENES = ["small_320x240", "small_300x200_jitter", "posed_bg", "dense", "stack_1023", "stack_1024", "stack_1025",
          "stack_64", "stack_65", "shape_1x1", "shape_1x37", "shape_17x33", "shape_4095x3"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
def test_backward_composite_is_bounded_and_bitwise_repeatable(name):
    import test_backward_exact as be
    from test_gpu_parity import check_grad
    scene = _scenes()[name]()
    with deterministic():
        o, res = be._check_scene("deterministic " + name, scene, und_share=None)
        accs = [torch.as_tensor(o["acc"])]
        grads = [_grads(o)]
        _other_stream_work()
        for _ in range(2):
            accs.append(_partials(o).cpu())
            grads.append(_grads(o))
    for a in accs[1:]:
        assert torch.equal(a.view(torch.int32), accs[0].view(torch.int32)), name
    for g in grads[1:]:
        for k, (x, y) in enumerate(zip(g, grads[0])):
            if x is not None:
                assert torch.equal(x.view(torch.int32), y.view(torch.int32)), (name, k)
    # the default path, twice, gives the bar's run-to-run noise
    default = [_grads(o), _grads(o)]
    for k, (ours, ref, again) in enumerate(zip(grads[0], *default)):
        if ours is not None and ref.numel() and float(ref.abs().max()) > 0:
            check_grad(f"{name} grad {k}", ours, ref, again)


@pytest.mark.gpu
def test_tile_row_shard_takes_the_deterministic_flush():
    """The single-process tile-row shard: the rectangles are clipped to the band, so the slots are those of the band's
    instances; bounded and bitwise repeatable."""
    import test_backward_exact as be
    from test_blend_masks import SMALL, _scene
    with deterministic():
        o, res = be._check_scene("deterministic shard_3_9", _scene(SMALL[0]), shard=(3, 9))
        again = _partials(o, shard=(3, 9)).cpu()
    assert torch.equal(again.view(torch.int32), torch.as_tensor(o["acc"]).view(torch.int32))
    assert (np.abs(o["acc"]).sum(axis=1) == 0).sum() > 0 and res["blended_pairs"] > 0


@pytest.mark.gpu
def test_colour_only_backward_is_bounded_and_repeatable():
    import test_backward_exact as be
    from test_adversarial_scenes import scene_posed
    from test_fused_embedding import color_backward
    from diff_gaussian_rasterization import _C
    o = be._run(scene_posed("precomp", P=20_000, W=200, H=150))
    d, P = o["d"], o["P"]
    R, geom, binning, img = o["bufs"]
    outs = []
    for _ in range(3):
        out = torch.full((P, 3), float("nan"), device=d["means3D"].device)
        a = _C.GsrBackwardArgs()
        a.P, a.M, a.R, a.W, a.H = P, 0, int(R), int(d["image_width"]), int(d["image_height"])
        a.subpixel_offset = d["subpixel_offset"].data_ptr()
        a.geom_buffer, a.binning_buffer, a.img_buffer = geom.data_ptr(), binning.data_ptr(), img.data_ptr()
        a.dL_dpix, a.dL_dcolor = d["dL_dpix"].data_ptr(), out.data_ptr()
        scratch, marks = _C.deterministic_buffers(P, int(R), out.device)
        a.deterministic, a.det_scratch, a.det_marks = 1, scratch.data_ptr(), marks.data_ptr()
        _C._check(_C._lib.gsr_backward_colors(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "colors")
        torch.cuda.synchronize()
        _C.deterministic_done(marks)
        assert not torch.any(marks), "marks left set"
        outs.append(out.cpu())
        _other_stream_work()
    assert all(torch.equal(x.view(torch.int32), outs[0].view(torch.int32)) for x in outs[1:])
    acc_c = np.zeros((P, 10))
    acc_c[:, 7:10] = outs[0].numpy()
    be._assert_within("deterministic gsr_backward_colors", acc_c, be._oracle(o, colour_walk=True), slots=(7, 8, 9))
    ref = color_backward(d, R, geom, binning, img, d["dL_dpix"]).cpu()
    assert float((ref - outs[0]).abs().max()) <= 1e-5 * float(ref.abs().max())


# ======================================================================================================================
# GPU: colour op
# ======================================================================================================================
def _embedding_kernel_det(s, deg, dLt):
    """test_colour_op_exact.run_embedding_kernel with deterministic = 1."""
    from diff_gaussian_rasterization import _C
    lib = _C._lib
    dev = dLt.device
    st = torch.cuda.current_stream().cuda_stream
    w = [s[k].contiguous() for k in ("W1", "b1", "W2", "b2", "W3", "b3")]
    blob = torch.empty((lib.gsr_appearance_packed_weight_bytes(),), dtype=torch.uint8, device=dev)
    _C._check(lib.gsr_appearance_pack_weights(*[t.data_ptr() for t in w], s["aemb"].data_ptr(), blob.data_ptr(), st), "pack")
    pack = torch.full((lib.gsr_appearance_grad_pack_bytes() // 4,), float("nan"), device=dev)
    rows = torch.full((lib.gsr_appearance_deterministic_scratch_bytes() // 4,), float("nan"), device=dev)
    status = torch.zeros((1,), dtype=torch.int32, device=dev)
    a = _C.GsrAppearanceArgs()
    a.P, a.sh_degree = int(s["dc"].shape[0]), deg
    a.features_dc, a.features_rest, a.embeddings = s["dc"].data_ptr(), s["rest"].data_ptr(), s["gemb"].data_ptr()
    a.means3D, a.campos, a.packed_weights = s["means"].data_ptr(), s["campos"].data_ptr(), blob.data_ptr()
    a.dL_dcolors_toned, a.grad_pack, a.status = dLt.data_ptr(), pack.data_ptr(), status.data_ptr()
    a.deterministic, a.det_scratch = 1, rows.data_ptr()
    _C._check(lib.gsr_appearance_embedding_backward(ctypes.byref(a), st), "gsr_appearance_embedding_backward")
    outs = [torch.empty(sh, device=dev) for sh in ((128, 59), (128,), (128, 128), (128,), (6, 128), (6,), (32,))]
    _C._check(lib.gsr_appearance_unpack_grads(pack.data_ptr(), w[0].data_ptr(), s["aemb"].data_ptr(),
                                              *[t.data_ptr() for t in outs], st), "unpack")
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    return dict(W1=outs[0], b1=outs[1], aemb=outs[6])


@pytest.mark.gpu
@pytest.mark.parametrize("P,deg", [(100_037, 3), (100_037, 1), (4_099, 2), (4_099, 0), (77, 0), (77, 3)])
def test_colour_op_is_bounded_and_bitwise_repeatable(P, deg):
    import test_colour_op_exact as tc
    from oracle import color_exact as ce
    dev = torch.device("cuda:0")
    s = tc.random_scene(P, 1000 + P, dev)
    dLr, dLt = tc.loss_grads(P, 3, dev)
    with deterministic():
        runs = [tc.run_kernel(s, deg, dLr, dLt)]
        _other_stream_work()
        runs.append(tc.run_kernel(s, deg, dLr, dLt))
    tc.compare(runs[0], tc.oracle(s, deg, dLt, dLr), f"deterministic P={P} deg {deg}")
    for k, v in runs[0].items():
        if v is not None:
            assert torch.equal(v.view(torch.int32), runs[1][k].view(torch.int32)), k
    e = [_embedding_kernel_det(s, deg, dLt) for _ in range(2)]
    wg = ce.weight_grads(tc.oracle(s, deg, dLt, None), ctas_per_sm=2, num_sms=tc.num_sms())
    for key in ("b1", "aemb"):
        ce.check("deterministic embedding kernel d" + key, e[0][key], wg[key])
        assert torch.equal(e[0][key].view(torch.int32), e[1][key].view(torch.int32)), key


# ======================================================================================================================
# GPU: end to end, each run in a fresh process
# ======================================================================================================================
_E2E = r"""
import json, os, random, sys
ROOT = sys.argv[1]
for p in (ROOT, os.path.join(ROOT, "wild-gaussians_b200"), os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import hashlib
import numpy as np
import torch
torch.use_deterministic_algorithms(True)
digest = {}
def put(k, t):
    if t is None:
        return
    if isinstance(t, torch.Tensor):
        digest[k] = hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()
    else:
        digest[k] = repr(t)
what = sys.argv[2]
if what == "embedding":
    import test_fused_embedding as tfe
    import fused_embedding as fe
    import types
    m, model, cfg, cam, gt_np = tfe._setup(dict(P=40_000, W=333, H=211), uncertainty=True)
    cfg.appearance_optim_type = "dssim+l1-scaled"
    ns = types.SimpleNamespace(model=model, config=cfg)
    out = fe.optimize_embedding(ns, tfe._dataset(cam, gt_np), embedding=np.zeros(32, dtype=np.float32))
    put("embedding", torch.as_tensor(out["embedding"]))
    for k, v in out["metrics"].items():
        put(k, torch.as_tensor(v))
else:
    import test_fused_train as tft
    dev = torch.device("cuda:0")
    method, out = tft._run(what, True, list(range(tft.FIRST, tft.LAST + 1)), dev)
    model, opt = method.model, method.model.optimizer
    for i, (cams, metrics, n) in enumerate(out):
        put(f"step{i}", repr((cams, sorted(metrics.items()), n)))
    for grp in opt.param_groups:
        for pi, p in enumerate(grp["params"]):
            put(f"{grp['name']}.{pi}", p)
            for k, v in opt.state.get(p, {}).items():
                put(f"{grp['name']}.{pi}.{k}", v)
    for name in tft.DENSIFICATION_BUFFERS:
        put(name, getattr(model, name, None))
    um = getattr(model, "uncertainty_model", None)
    if um is not None:
        for n, b in um.named_buffers():
            put("unc." + n, b)
print("DIGEST " + json.dumps(digest))
"""


def _e2e(what):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-c", _E2E, ROOT, what], capture_output=True, text=True, env=env, timeout=1800)
    if "reference python package not present" in r.stdout + r.stderr:
        pytest.skip("reference python package not present (oracle/_ref/py)")
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    line = [x for x in r.stdout.splitlines() if x.startswith("DIGEST ")][-1]
    return json.loads(line[len("DIGEST "):])


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["plain", "uncertainty_masks", "no_appearance_scale_grad", "embedding"])
def test_two_runs_give_the_same_bits(what):
    """Fused training across a densification and an opacity reset (with appearance, with the `dino` uncertainty model,
    without appearance), and the fused optimize_embedding: every parameter, Adam moment, buffer and metric."""
    a, b = _e2e(what), _e2e(what)
    assert len(a) > 3
    diff = [k for k in a if a[k] != b.get(k)]
    assert not diff and a.keys() == b.keys(), diff
