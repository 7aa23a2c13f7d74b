"""The fused colour op (csrc/appearance.cu) entry by entry against an fp64 oracle of its rounded network
(oracle/color_exact.py): every output and gradient entry must lie within the oracle's a-priori bound.

Scenes:
  * lattice scenes (ce.lattice_scene): inputs, weights and biases on dyadic grids, so every forward GEMM sum is exact in
    fp32 in any order and the MLP output, every hidden activation and every ReLU mask are known exactly.  Exact kinks are
    hit on purpose: features equal to 1, pre-activations equal to 0, tone-map products equal to 1.
  * random scenes (the recipe of test_appearance.py) and the reference's trained-like goldens (tests/golden/colors_deg*.npz).
    Rows whose ReLU mask or colour clamp the oracle cannot decide ("undetermined") are counted, asserted below
    MAX_UNDETERMINED, and still checked against a bound that allows either choice.
Weight, bias and image-embedding gradients are checked entry-wise against bounds that include the flagged roundings,
the undetermined rows' possible contributions and the reordering of the sums over tiles and CTAs.  No cosine, no quantile.

The CPU tests check the oracle itself (against the fp64 network, the reference goldens and the bf16-emulating torch
restatement), the lattice premise, and that the comparison catches the corruptions a broken tile schedule, warpgroup split
or CTA flush would cause (mutation tests on the oracle's own outputs).
"""
import functools
import os

import numpy as np
import pytest
import torch

from oracle import color_exact as ce

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
MAX_UNDETERMINED = 0.08          # random scenes: fraction of rows with an undetermined mask (CPU estimate ~4 %)
ROW_KEYS = ("g_dc", "g_rest", "g_gemb", "g_means")
WEIGHT_KEYS = ("W1", "b1", "W2", "b2", "W3", "b3", "aemb")


# ---- scenes ----------------------------------------------------------------------------------------------------------
def random_scene(P, seed, device="cpu"):
    """test_appearance.py's recipe: some colours clamp at 0, some features > 1, mul ~ 0.8"""
    g = torch.Generator().manual_seed(seed)
    R = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale
    s = dict(dc=(torch.rand(P, 3, generator=g) * 1.6 - 0.9) / 0.28209479, rest=R(P, 45, scale=0.3),
             gemb=R(P, 24, scale=0.5), aemb=R(32, scale=0.5), means=R(P, 3, scale=2.0),
             campos=torch.tensor([0.1, -0.2, 0.3]))
    torch.manual_seed(seed)
    mlp = torch.nn.Sequential(torch.nn.Linear(59, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128), torch.nn.ReLU(),
                              torch.nn.Linear(128, 6))
    with torch.no_grad():
        mlp[4].bias[3:] = 80.0
    for k, lin in zip((1, 2, 3), (mlp[0], mlp[2], mlp[4])):
        s[f"W{k}"], s[f"b{k}"] = lin.weight.detach().clone(), lin.bias.detach().clone()
    return {k: v.float().to(device) for k, v in s.items()}


def golden_scene(name, device="cpu", dtype=torch.float32):
    d = dict(np.load(os.path.join(GOLD, name + ".npz")))
    T = lambda k: torch.tensor(d[k], dtype=dtype, device=device)
    s = dict(dc=T("features")[:, :3].contiguous(), rest=T("features")[:, 3:].contiguous(), gemb=T("gembedding"),
             aemb=T("aembedding"), means=T("means3D"), campos=T("campos"))
    for k in range(1, 4):
        s[f"W{k}"], s[f"b{k}"] = T(f"W{k}"), T(f"b{k}")
    return s, int(d["active_deg"]), T("dL_dcolors"), d


def loss_grads(P, seed, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(P, 3, generator=g).to(device), torch.randn(P, 3, generator=g).to(device)


def oracle(s, deg, dL_toned, dL_raw, **kw):
    return ce.colour_op(s["dc"], s["rest"], s["gemb"], s["aemb"], s["W1"], s["b1"], s["W2"], s["b2"], s["W3"], s["b3"],
                        s["means"], s["campos"], deg, dL_toned, dL_raw, **kw)


# ---- the kernel ------------------------------------------------------------------------------------------------------
def _mlp(s):
    mlp = torch.nn.Sequential(torch.nn.Linear(59, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128), torch.nn.ReLU(),
                              torch.nn.Linear(128, 6)).to(s["dc"].device)
    with torch.no_grad():
        for lin, k in ((mlp[0], 1), (mlp[2], 2), (mlp[4], 3)):
            lin.weight.copy_(s[f"W{k}"])
            lin.bias.copy_(s[f"b{k}"])
    return mlp


def run_kernel(s, deg, dLr, dLt, mode="both"):
    """fused_colors forward + backward.  mode: "both" (loss on raw and toned), "toned" / "raw" (loss on one output; the
    other's gradient reaches the backward as zeros), "noraw" (want_raw=False: the backward gets no raw gradient)."""
    import fused_colors as fc
    mlp = _mlp(s)
    leaves = [s[k].clone().requires_grad_(True) for k in ("dc", "rest", "gemb", "aemb", "means")]
    raw, toned = fc.fused_colors(leaves[0], leaves[1], leaves[2], leaves[3], mlp, leaves[4], s["campos"], deg,
                                 want_raw=mode != "noraw")
    outs, grads = {"both": ([raw, toned], [dLr, dLt]), "toned": ([toned], [dLt]), "raw": ([raw], [dLr]),
                   "noraw": ([toned], [dLt])}[mode]
    params = [mlp[i].weight for i in (0, 2, 4)] + [mlp[i].bias for i in (0, 2, 4)]
    gr = torch.autograd.grad(outs, leaves + params, grads)
    torch.cuda.synchronize()
    assert fc.last_status_ok()
    k = dict(raw=None if raw is None else raw.detach(), toned=toned.detach(), g_dc=gr[0], g_rest=gr[1], g_gemb=gr[2],
             aemb=gr[3], g_means=gr[4], W1=gr[5], W2=gr[6], W3=gr[7], b1=gr[8], b2=gr[9], b3=gr[10])
    return k


def run_embedding_kernel(s, deg, dLt):
    """gsr_appearance_embedding_backward + gsr_appearance_unpack_grads: (db1 [128], dW1 [128, 59], daemb [32])"""
    import ctypes

    import fused_colors as fc
    from diff_gaussian_rasterization import _C
    lib = _C._lib
    dev = dLt.device
    st = torch.cuda.current_stream().cuda_stream
    w = [s[k].contiguous() for k in ("W1", "b1", "W2", "b2", "W3", "b3")]
    blob = torch.empty((lib.gsr_appearance_packed_weight_bytes(),), dtype=torch.uint8, device=dev)
    _C._check(lib.gsr_appearance_pack_weights(*[t.data_ptr() for t in w], s["aemb"].data_ptr(), blob.data_ptr(), st), "pack")
    pack = torch.full((lib.gsr_appearance_grad_pack_bytes() // 4,), float("nan"), device=dev)
    status = torch.zeros((1,), dtype=torch.int32, device=dev)
    a = _C.GsrAppearanceArgs()
    a.P, a.sh_degree = int(s["dc"].shape[0]), deg
    a.features_dc, a.features_rest, a.embeddings = s["dc"].data_ptr(), s["rest"].data_ptr(), s["gemb"].data_ptr()
    a.means3D, a.campos, a.packed_weights = s["means"].data_ptr(), s["campos"].data_ptr(), blob.data_ptr()
    a.dL_dcolors_toned, a.grad_pack, a.status = dLt.data_ptr(), pack.data_ptr(), status.data_ptr()
    _C._check(lib.gsr_appearance_embedding_backward(ctypes.byref(a), st), "gsr_appearance_embedding_backward")
    outs = [torch.empty(sh, device=dev) for sh in ((128, 59), (128,), (128, 128), (128,), (6, 128), (6,), (32,))]
    _C._check(lib.gsr_appearance_unpack_grads(pack.data_ptr(), w[0].data_ptr(), s["aemb"].data_ptr(),
                                              *[t.data_ptr() for t in outs], st), "unpack")
    torch.cuda.synchronize()
    assert int(status.item()) == 0 and fc.last_status_ok()
    return dict(W1=outs[0], b1=outs[1], aemb=outs[6])


def num_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def compare(k, res, label, forward_keys=("raw", "toned")):
    """assert every entry within its bound; returns the worst |error| / bound per tensor (printed for the record)"""
    wg = ce.weight_grads(res, ctas_per_sm=1, num_sms=num_sms())
    worst = {}
    for key in forward_keys:
        if k.get(key) is not None:
            worst[key] = ce.ratio(k[key], res[key])
            ce.check(key, k[key], res[key])
    det = ~res["undetermined"]
    for key in ROW_KEYS:
        worst[key] = ce.ratio(k[key][det.to(k[key].device)], res[key][det])      # reported: determined rows
        ce.check(key, k[key], res[key])                                          # asserted: every row
    for key in WEIGHT_KEYS:
        worst["d" + key] = ce.ratio(k[key], wg[key])
        ce.check("d" + key, k[key], wg[key])
    und = float(res["undetermined"].double().mean())
    print(label, "undetermined rows", f"{und:.4%}", "worst error / bound", {a: round(b, 4) for a, b in worst.items()},
          res["stats"])
    return worst, und


# =====================================================================================================================
# CPU: the oracle, the lattice premise and the checker
# =====================================================================================================================
def test_lattice_premise():
    """the lattice scene's forward sums are exact in fp32 in two orders and in fp64, spans <= 20 bits"""
    spans = ce.check_lattice_premise(ce.lattice_scene(2048, 5))
    assert max(spans) <= 20, spans
    print("lattice spans (bits)", spans)


def test_lattice_oracle_is_exact_in_the_forward_and_hits_the_kinks():
    s = ce.lattice_scene(4096, 6)
    dLr, dLt = loss_grads(4096, 7)
    res = oracle(s, 3, dLt, dLr, exact_mlp=True)
    st = res["stats"]
    assert st["H1 flagged"] == 0 and st["H2 flagged"] == 0
    assert st["layer-1 masks undetermined"] == 0 and st["layer-2 masks undetermined"] == 0
    assert float(res["undetermined"].double().mean()) < 0.01
    # the kinks are hit exactly: features == 1, and channel 2's tone map is the identity (t == f)
    assert int((s["rest"] == 1).sum()) > 1000 and int((s["dc"] == 1).sum()) > 100
    assert bool((res["toned"].c[:, 2] == res["raw"].c[:, 2]).all())
    # layer-1 pre-activations exactly 0
    X = torch.cat((s["dc"].double().clamp_max(1), s["gemb"].double()), 1)
    z1 = X @ s["W1"].double()[:, :27].T + s["b1"].double() + s["W1"].double()[:, 27:] @ s["aemb"].double()
    assert int((z1 == 0).sum()) > 1000


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_oracle_without_rounding_is_the_fp64_network(deg):
    """bf16 off: the oracle's bounds contain the fp64 autograd gradients of the torch restatement (oracle/color_torch.py)
    on every row and every weight entry, at a random scene"""
    from oracle import color_torch as ct
    P = 20_011 if deg == 3 else 3_001
    s = random_scene(P, 1000 + P)
    dLr, dLt = loss_grads(P, 3)
    res = oracle(s, deg, dLt, dLr, bf16_operands=False, bf16_backward=False)
    L = [s[k].double().clone().requires_grad_(True) for k in ("dc", "rest", "gemb", "aemb", "means")]
    W = [s[k].double().clone().requires_grad_(True) for k in ("W1", "b1", "W2", "b2", "W3", "b3")]
    raw, toned = ct.colors(L[0], L[1], L[2], L[3], *W, L[4], s["campos"].double(), deg)
    ((raw * dLr.double()).sum() + (toned * dLt.double()).sum()).backward()
    k = dict(raw=raw, toned=toned, g_dc=L[0].grad, g_rest=L[1].grad, g_gemb=L[2].grad, aemb=L[3].grad,
             g_means=torch.zeros_like(L[4]) if L[4].grad is None else L[4].grad,
             W1=W[0].grad, b1=W[1].grad, W2=W[2].grad, b2=W[3].grad, W3=W[4].grad, b3=W[5].grad)
    wg = ce.weight_grads(res)
    for key in ("raw", "toned") + ROW_KEYS:
        ce.check(key, k[key], res[key])
    for key in WEIGHT_KEYS:
        ce.check(key, k[key], wg[key])
    assert float(res["undetermined"].double().mean()) < MAX_UNDETERMINED


@pytest.mark.parametrize("name", ["colors_deg3", "colors_deg1"])
def test_oracle_without_rounding_contains_the_reference_goldens(name):
    """bf16 off: the reference's own fp64 outputs and autograd gradients lie within the oracle's bounds"""
    s, deg, dLt, d = golden_scene(name, dtype=torch.float64)
    res = oracle(s, deg, dLt, None, bf16_operands=False, bf16_backward=False)
    det = ~res["undetermined"]
    ce.check("toned", torch.tensor(d["colors"]), res["toned"])
    g_feat = torch.tensor(d["g_features"])
    ce.check("g_dc", g_feat[:, :3], res["g_dc"], det)
    ce.check("g_rest", g_feat[:, 3:], res["g_rest"], det)
    ce.check("g_gemb", torch.tensor(d["g_gembedding"]), res["g_gemb"], det)
    wg = ce.weight_grads(res)
    for key in ("W1", "b1", "W2", "b2", "W3", "b3"):
        ce.check(key, torch.tensor(d["g_" + key]), wg[key])
    ce.check("aemb", torch.tensor(d["g_aembedding"]), wg["aemb"])
    assert float(det.double().mean()) > 0.9


def test_oracle_forward_contains_the_bf16_emulating_restatement():
    """bf16 on: color_torch.colors(emulate_bf16=True) in fp64 -- the rounded network evaluated exactly -- lies within the
    oracle's bounds: colours on every row; the colour stage's gradients (features_rest, means) on determined rows"""
    from oracle import color_torch as ct
    P, deg = 20_011, 3
    s = random_scene(P, 1000 + P)
    dLr, dLt = loss_grads(P, 3)
    res = oracle(s, deg, dLt, dLr)
    _, b2e, b3e = ce.effective_biases(s["W1"], s["b1"], s["W2"], s["b2"], s["W3"], s["b3"], s["aemb"])
    L = [s[k].double().clone().requires_grad_(True) for k in ("dc", "rest", "gemb", "aemb", "means")]
    W = [s["W1"].double(), s["b1"].double(), s["W2"].double(), b2e.c, s["W3"].double(), b3e.c]
    raw, toned = ct.colors(L[0], L[1], L[2], L[3], *W, L[4], s["campos"].double(), deg, emulate_bf16=True)
    ((raw * dLr.double()).sum() + (toned * dLt.double()).sum()).backward()
    ce.check("raw", raw, res["raw"])
    ce.check("toned", toned, res["toned"])
    det = ~res["undetermined"]
    ce.check("g_rest", L[1].grad, res["g_rest"], det)
    ce.check("g_means", L[4].grad, res["g_means"], det)


@functools.lru_cache(maxsize=1)
def _mutation_base():
    P, deg = 100_037, 3
    s = random_scene(P, 1000 + P)
    dLr, dLt = loss_grads(P, 3)
    res = oracle(s, deg, dLt, dLr)
    return s, deg, dLr, dLt, res


def _kernel_like(res):
    """the oracle's centres rounded to fp32: what a correct kernel could return"""
    k = {key: res[key].c.float() for key in ROW_KEYS}
    wg = ce.weight_grads(res)
    k.update({key: wg[key].c.float() for key in WEIGHT_KEYS})
    return k, wg


def _unpack_from_db1(k, res, db1):
    W1, aemb = res["W1"], res["aemb"]
    k["b1"] = db1
    k["W1"] = k["W1"].clone()
    k["W1"][:, 27:] = (db1[:, None].double() * aemb[None]).float()
    k["aemb"] = (W1[:, 27:].T @ db1.double()).float()


MUTATIONS = ["clean", "ragged_tile_zeroed", "warpgroup_rows_zeroed", "warpgroup_rows_swapped", "cta_tiles_dropped",
             "db1_slot_missing", "one_row_g_means_negated"]


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_checker_catches_corrupted_outputs(mutation):
    """The comparison functions of the GPU tests, fed the oracle's own outputs (P = 100 037, deg 3): they accept them
    as they are and reject each corruption a broken schedule could cause."""
    s, deg, dLr, dLt, res = _mutation_base()
    P = res["P"]
    k, wg = _kernel_like(res)
    tiles = (P + 127) // 128
    t = tiles // 2                                     # a full tile in the middle
    if mutation == "ragged_tile_zeroed":
        for key in ROW_KEYS:
            k[key][(tiles - 1) * 128:] = 0
    elif mutation == "warpgroup_rows_zeroed":
        for key in ROW_KEYS:
            k[key][t * 128 + 64:t * 128 + 128] = 0
    elif mutation == "warpgroup_rows_swapped":
        for key in ROW_KEYS:
            a = k[key][t * 128:t * 128 + 128].clone()
            k[key][t * 128:t * 128 + 128] = torch.cat((a[64:], a[:64]))
    elif mutation == "cta_tiles_dropped":
        grid = min(tiles, 132)
        cta = 7
        rows = torch.cat([torch.arange(tt * 128, min(P, tt * 128 + 128)) for tt in range(cta, tiles, grid)])
        sub = oracle({kk: (v[rows] if v.dim() and v.shape[0] == P else v) for kk, v in s.items()}, deg, dLt[rows], dLr[rows])
        for key, (c, _, _) in sub["sums"].items():
            k[key] = k[key].clone()
            k[key][..., :c.shape[-1]] = (k[key][..., :c.shape[-1]].double() - c).float()
        _unpack_from_db1(k, res, k["b1"])
    elif mutation == "db1_slot_missing":
        db1 = k["b1"].clone()
        db1[int(wg["b1"].c.abs().argmax())] = 0
        _unpack_from_db1(k, res, db1)
    elif mutation == "one_row_g_means_negated":
        row = int((res["g_means"].c.abs() / (res["g_means"].r + 1e-30)).max(1).values.argmax())
        k["g_means"][row] = -k["g_means"][row]
    if mutation == "clean":
        ce.check_row_grads(k, res)
        ce.check_weight_grads(k, wg)
        return
    with pytest.raises(AssertionError):
        ce.check_row_grads(k, res)
        ce.check_weight_grads(k, wg)


# =====================================================================================================================
# GPU: the kernels against the oracle
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_lattice_scene_every_entry(deg):
    dev = torch.device("cuda:0")
    P = 2 * 132 * 128 + 77
    s = ce.lattice_scene(P, 40 + deg, dev)
    dLr, dLt = loss_grads(P, 50 + deg, dev)
    k = run_kernel(s, deg, dLr, dLt)
    res = oracle(s, deg, dLt, dLr, exact_mlp=True)
    assert res["stats"]["layer-1 masks undetermined"] == 0 and res["stats"]["layer-2 masks undetermined"] == 0
    compare(k, res, f"lattice deg {deg}")
    assert float(res["undetermined"].double().mean()) < 0.01
    e = run_embedding_kernel(s, deg, dLt)
    ro = oracle(s, deg, dLt, None, exact_mlp=True)
    wg = ce.weight_grads(ro, ctas_per_sm=2, num_sms=num_sms())
    for key in ("b1", "aemb"):
        ce.check("embedding kernel d" + key, e[key], wg[key])
    ce.check("embedding kernel dW1[:, 27:]", e["W1"][:, 27:], wg["W1"][:, 27:])


@pytest.mark.gpu
@pytest.mark.parametrize("P,deg", [(100_037, 3), (4_099, 2), (77, 0)])
def test_random_scene_every_entry(P, deg):
    dev = torch.device("cuda:0")
    s = random_scene(P, 1000 + P, dev)
    dLr, dLt = loss_grads(P, 3, dev)
    k = run_kernel(s, deg, dLr, dLt)
    res = oracle(s, deg, dLt, dLr)
    _, und = compare(k, res, f"random P={P} deg {deg}")
    assert und < MAX_UNDETERMINED
    e = run_embedding_kernel(s, deg, dLt)
    ro = oracle(s, deg, dLt, None)
    wg = ce.weight_grads(ro, ctas_per_sm=2, num_sms=num_sms())
    for key in ("b1", "aemb"):
        ce.check("embedding kernel d" + key, e[key], wg[key])
    ce.check("embedding kernel dW1[:, 27:]", e["W1"][:, 27:], wg["W1"][:, 27:])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["colors_deg3", "colors_deg1"])
def test_reference_goldens_every_entry(name):
    dev = torch.device("cuda:0")
    s, deg, dLt, _ = golden_scene(name, dev)
    P = int(s["dc"].shape[0])
    k = run_kernel(s, deg, None, dLt, mode="toned")
    res = oracle(s, deg, dLt, None)
    _, und = compare(k, res, name, forward_keys=("toned",))
    assert und < MAX_UNDETERMINED


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["1", "63", "64", "65", "127", "128", "129", "sm*128+1", "2*sm*128-1", "2*sm*128+1"])
def test_shapes(case):
    """one warpgroup, both, the ragged tile; CTAs owning one or two tiles in the backward (one CTA per SM) and in the
    forward / embedding kernels (two per SM)"""
    sm = num_sms()
    P = int(eval(case, {"sm": sm}))
    dev = torch.device("cuda:0")
    s = random_scene(P, 2000 + P, dev)
    dLr, dLt = loss_grads(P, 4, dev)
    k = run_kernel(s, 3, dLr, dLt)
    res = oracle(s, 3, dLt, dLr)
    compare(k, res, f"shape P={P}")
    e = run_embedding_kernel(s, 3, dLt)
    wg = ce.weight_grads(oracle(s, 3, dLt, None), ctas_per_sm=2, num_sms=sm)
    ce.check("embedding kernel db1", e["b1"], wg["b1"])
    ce.check("embedding kernel daemb", e["aemb"], wg["aemb"])


@pytest.mark.gpu
def test_three_million_ragged():
    P = 3_000_037
    dev = torch.device("cuda:0")
    s = random_scene(P, 77, dev)
    dLr, dLt = loss_grads(P, 5, dev)
    k = run_kernel(s, 3, dLr, dLt)
    res = oracle(s, 3, dLt, dLr)
    _, und = compare(k, res, f"random P={P}")
    assert und < MAX_UNDETERMINED


@pytest.mark.gpu
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("mode", ["both", "toned", "raw", "noraw"])
def test_arguments(deg, mode):
    """SH degrees 0..3; a loss on both outputs, on one of them, and want_raw=False"""
    P = 4_099
    dev = torch.device("cuda:0")
    s = random_scene(P, 3000 + deg, dev)
    dLr, dLt = loss_grads(P, 6, dev)
    k = run_kernel(s, deg, dLr, dLt, mode)
    res = oracle(s, deg, dLt if mode != "raw" else torch.zeros_like(dLt), dLr if mode in ("both", "raw") else None)
    compare(k, res, f"args deg {deg} {mode}", forward_keys=("toned",) if mode == "noraw" else ("raw", "toned"))
    if mode == "noraw":
        assert k["raw"] is None


@pytest.mark.gpu
def test_offset_views_are_accepted_and_give_the_same_bits():
    """features_rest and embeddings as contiguous views with a storage offset (not 16-byte aligned)"""
    import fused_colors as fc
    P = 1_000
    dev = torch.device("cuda:0")
    s = random_scene(P, 11, dev)
    dLr, dLt = loss_grads(P, 12, dev)
    ref = run_kernel(s, 3, dLr, dLt)
    big_rest = torch.empty(P + 1, 45, device=dev)
    big_rest[1:] = s["rest"]
    big_gemb = torch.empty(P * 24 + 1, device=dev)
    big_gemb[1:] = s["gemb"].flatten()
    v = dict(s, rest=big_rest[1:], gemb=big_gemb[1:].view(P, 24))
    assert v["rest"].is_contiguous() and v["rest"].data_ptr() % 16 and v["gemb"].data_ptr() % 16
    got = run_kernel(v, 3, dLr, dLt)
    for key in ("raw", "toned") + ROW_KEYS:          # per-row outputs: the same bits (the weight sums use atomics)
        assert torch.equal(ref[key], got[key]), key
    compare(got, oracle(s, 3, dLt, dLr), "offset views")
    assert fc.last_status_ok()
