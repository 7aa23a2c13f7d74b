"""The multi-GPU composite epilogues on one GPU, with simulated ranks.

The tile-row sharded rasterizer (``parallel.py``) has three kernel paths that only multi-GPU training reaches:
* the forward composite's all-gather epilogue, which stores every rank's band into the images of all ranks
  (``peer_images``);
* the backward composite's peer reduction (mode 1), which adds each rank's per-Gaussian sums straight into the
  accumulators of all ranks, and the mark bytes of pull mode;
* the pull-mode chain rule (mode 3), which adds the marked rows of all ranks in rank order and clears the previous
  pass's rows and marks.

None of them needs a second GPU.  A peer pointer is an ordinary device address, so N ranks are N allocations on one
device; the protocol's barriers become stream order (part A) or a stream synchronisation plus a host barrier (part B).
The multicast mode needs an NVSwitch multicast address and is not covered here.

A. Kernel level: the ranks' ``_C`` calls in sequence on one stream, against
   * the single-GPU result: images bit-exact, accumulators and gradients within twenty times the run-to-run noise of
     the single-GPU float atomics (``test_gpu_parity.check_grad``);
   * float64: the CPU oracle's per-band sums (``cpu_oracle`` with ``tile_rows``) and gradients, which the sharded
     result must approach as closely as the single-GPU one does, up to 4x (or 1e-5).
B. ``parallel.sharded_forward`` / ``sharded_backward`` themselves, one thread and one stream per rank, with
   ``torch.distributed`` and the symmetric-memory state replaced by in-process stand-ins.

CPU tests: ``partition_tile_rows`` and ``abi_band`` never hand a rank the whole-image shard ``(0, 0)``.
"""
import threading

import numpy as np
import pytest
import torch

import parallel
import synthetic
from make_golden import backward_args, call_args
from oracle import cpu_oracle
from test_adversarial_scenes import GRAD_NAMES, fp64_gradients, rel_errors_to, scene_posed

TILE = 16


# ======================================================================================================================
# CPU: band bookkeeping
# ======================================================================================================================
def _partition_with_absolute_slack(n, w, weights):
    """``partition_tile_rows`` as it was with an absolute rounding slack of 1e-9 * max(1, total)."""
    import bisect
    cum = [0.0]
    for x in weights:
        cum.append(cum[-1] + float(x))
    total, cuts = cum[-1], [0]
    for r in range(1, w):
        cuts.append(min(n, max(bisect.bisect_left(cum, total * r / w - 1e-9 * max(1.0, total)), cuts[-1])))
    cuts.append(n)
    return [(cuts[r], cuts[r + 1]) for r in range(w)]


@pytest.mark.parametrize("scale", [1e-12, 1e-20, 1e-300])
@pytest.mark.parametrize("rows,world", [(14, 4), (3, 5), (1, 8), (68, 8)])
def test_tiny_weights_give_no_rank_the_whole_image_sentinel(rows, world, scale):
    """A total weight below about 1e-9 x world put every cut at row 0 and handed ranks the band (0, 0), which the
    C ABI reads as the whole image."""
    bands = parallel.partition_tile_rows(rows, world, [scale] * rows)
    assert (0, 0) not in bands, bands
    assert bands[0][0] == 0 and bands[-1][1] == rows
    assert all(a[1] == b[0] for a, b in zip(bands, bands[1:])) and all(y1 >= y0 for y0, y1 in bands)
    # the same split as unit weights
    assert bands == parallel.partition_tile_rows(rows, world, [1.0] * rows)


def test_partitions_of_ordinary_weights_are_unchanged():
    g = np.random.default_rng(5)
    for _ in range(300):
        rows, world = int(g.integers(1, 90)), int(g.integers(1, 10))
        w = (g.random(rows) * 10.0 ** g.uniform(-3, 6)) * (g.random(rows) < 0.8)
        old = _partition_with_absolute_slack(rows, world, w) if w.sum() > 0 else None
        new = parallel.partition_tile_rows(rows, world, list(w))
        if old is not None and (0, 0) not in old[1:]:
            assert new == old, (rows, world, list(w))


def test_abi_band_keeps_the_whole_image_sentinel_out_of_sharded_calls():
    H = 212                                                       # 14 tile rows
    assert parallel.abi_band((0, 0), H) == (14, 14)
    assert parallel.abi_band((5, 5), H) == (14, 14)
    assert parallel.abi_band((9, 3), H) == (14, 14)
    assert parallel.abi_band((0, 14), H) == (0, 14)
    assert parallel.abi_band((3, 9), H) == (3, 9)


# ======================================================================================================================
# GPU: scenes, bands, references
# ======================================================================================================================
SCENES = {
    # ragged last tile row (212 = 13 x 16 + 4) and odd width
    "precomp": lambda: synthetic.make_scene(P=40_000, W=300, H=212, sh_degree=None, seed=46),
    "sh3": lambda: synthetic.make_scene(P=20_000, W=256, H=176, sh_degree=3, seed=61, bg=(0.2, 0.1, 0.3)),
    "cov3d": lambda: synthetic.make_scene(P=20_000, W=240, H=170, sh_degree=None, seed=62, cov3D_precomp=True),
    "posed": lambda: scene_posed("precomp", seed=101, P=20_000),
    # 3 tile rows for 5 ranks: empty bands
    "short": lambda: synthetic.make_scene(P=20_000, W=300, H=40, sh_degree=None, seed=63),
}


def make_bands(kind, gy, N):
    if kind == "equal":
        return parallel.partition_tile_rows(gy, N)
    if kind == "skewed":            # the first N-1 rows weigh 50 each: one-row bands, the rest to the last rank
        bands = parallel.partition_tile_rows(gy, N, [50.0] * (N - 1) + [1.0] * (gy - N + 1))
        assert sum(1 for y0, y1 in bands if y1 - y0 == 1) >= N - 1
        return bands
    if kind == "empty_first":       # explicit bands, the first one empty in the (0, 0) form
        return [(0, 0)] + parallel.partition_tile_rows(gy, N - 1)
    raise ValueError(kind)


CASES = [("precomp", 1, "equal"), ("precomp", 2, "equal"), ("precomp", 3, "skewed"), ("precomp", 5, "equal"),
         ("precomp", 8, "skewed"), ("precomp", 2, "empty_first"), ("sh3", 3, "equal"), ("cov3d", 5, "skewed"),
         ("posed", 3, "equal"), ("short", 5, "equal")]
CASE_IDS = [f"{s}-N{n}-{b}" for s, n, b in CASES]

_cache = {}


@pytest.fixture(scope="module")
def C():
    from diff_gaussian_rasterization import _C
    _C.set_geometry_cache(False)
    yield _C
    _C.set_geometry_cache(True)


def upstream(scene, which):
    """Upstream gradients: the scene's own, one that is zero outside one tile row, another random one, all-zero."""
    g = scene["dL_dpix"]
    if which == "g":
        return g
    if which == "g_band":
        t = (scene["image_height"] + TILE - 1) // TILE // 2
        out = torch.zeros_like(g)
        out[:, TILE * t:TILE * (t + 1)] = g[:, TILE * t:TILE * (t + 1)]
        return out
    if which == "g2":
        return torch.randn(g.shape, generator=torch.Generator().manual_seed(99)).float()
    if which == "zero":
        return torch.zeros_like(g)
    raise ValueError(which)


def scene_state(name):
    """The scene on the device and its single-GPU forward."""
    key = ("scene", name)
    if key not in _cache:
        from diff_gaussian_rasterization import _C as C
        scene = SCENES[name]()
        d = synthetic.to_device(scene, torch.device("cuda:0"))
        R, color, radii, geom, binning, img = C.rasterize_gaussians(*call_args(d))
        P, W, H = d["means3D"].shape[0], d["image_width"], d["image_height"]
        M = d["shs"].shape[1] if "shs" in d else 0
        v = C.debug_views(geom, binning, img, P, M, W, H, R)
        _cache[key] = dict(scene=scene, d=d, P=P, M=M, W=W, H=H, gy=(H + TILE - 1) // TILE, R=R, radii=radii,
                           image=torch.cat([color, v["final_T"][None]]).clone(), bufs=(geom, binning, img),
                           final_T=v["final_T"].cpu().numpy(), n_contrib=v["n_contrib"].cpu().numpy())
    return _cache[key]


def with_dl(d, dl):
    d2 = dict(d)
    d2["dL_dpix"] = dl.to(d["dL_dpix"].device)
    return d2


def single_backward(name, which):
    """Single-GPU gradients and [P,12] partial sums for one upstream gradient, each computed twice (the float atomics
    make two runs differ: that difference calibrates the bars)."""
    key = ("single", name, which)
    if key not in _cache:
        from diff_gaussian_rasterization import _C as C
        s = scene_state(name)
        geom, binning, img = s["bufs"]
        bargs = backward_args(with_dl(s["d"], upstream(s["scene"], which)), s["radii"], geom, s["R"], binning, img)
        grads = [dict(zip(GRAD_NAMES, C.rasterize_gaussians_backward(*bargs))) for _ in range(2)]
        parts = [C.rasterize_gaussians_backward_partials(*bargs)[: s["P"] * 12].view(s["P"], 12).clone() for _ in range(2)]
        torch.cuda.synchronize()
        _cache[key] = dict(grads=grads, parts=[p.double().cpu().numpy() for p in parts])
    return _cache[key]


def oracle_band(band, gy):
    """The oracle reads (0, 0) as the whole image too: an empty band goes in as the empty band below the last row."""
    return (gy, gy) if band[1] <= band[0] else tuple(band)


def fp64_reference(name, bands):
    """float64 gradients of the whole image and the [P,10] sums of each band, on the kernel's forward."""
    key = ("fp64", name, tuple(bands))
    if key not in _cache:
        s = scene_state(name)
        g64, _ = fp64_gradients(s["scene"], cpu_oracle.forward(s["scene"]), s["final_T"], s["n_contrib"])
        per_band = [fp64_gradients(s["scene"], cpu_oracle.forward(s["scene"], tile_rows=oracle_band(b, s["gy"])),
                                   s["final_T"], s["n_contrib"])[0]["acc"] for b in bands]
        total = np.sum(per_band, axis=0)
        assert np.abs(total - g64["acc"]).max() <= 1e-9 * np.abs(g64["acc"]).max(), "oracle bands do not add up"
        _cache[key] = dict(grads=g64, band_acc=per_band, acc=total)
    return _cache[key]


def column_errors(x, ref):
    """Per column of a [P,10] sum array: largest absolute error relative to the column's largest magnitude."""
    return np.abs(x - ref).max(0) / (np.abs(ref).max(0) + 1e-30)


def check_sums(what, rows, single, f64):
    """``rows`` [P,12] of one accumulator against the single-GPU partials (noise-tied) and the fp64 sums (4x)."""
    x = rows[:, :10].double().cpu().numpy()
    assert not np.any(rows[:, 10:].cpu().numpy()), (what, "padding columns written")
    a, b = single["parts"][0][:, :10], single["parts"][1][:, :10]
    err, noise = column_errors(x, a), column_errors(b, a)
    assert np.all(err <= np.maximum(20.0 * noise, 1e-5)), (what, "vs single GPU", err, noise)
    e64, s64 = column_errors(x, f64), column_errors(a, f64)
    assert np.all(e64 <= np.maximum(4.0 * s64, 1e-5)), (what, "vs fp64", e64, s64)


def check_gradients(what, grads, single, g64=None):
    """The bars of the single-GPU parity tests: ``check_grad`` against the single-GPU gradients and, with ``g64``,
    element-wise relative error to fp64 within max(4 x the single-GPU error, 1e-5)."""
    from test_gpu_parity import check_grad
    ref, ref2 = single["grads"]
    for n in GRAD_NAMES:
        if grads[n] is None or ref[n] is None or ref[n].numel() == 0:
            continue
        check_grad(f"{what} {n}", grads[n].view_as(ref[n]), ref[n], ref2[n])
    if g64 is not None:
        np_of = lambda gr: {n: (None if gr[n] is None else gr[n].detach().cpu().numpy()) for n in GRAD_NAMES}
        mine, theirs = np_of(grads), np_of(ref)
        want = {n: (g64[n] if mine[n] is not None else np.zeros(0)) for n in GRAD_NAMES}
        ours_err, single_err = rel_errors_to(want, mine), rel_errors_to(want, theirs)
        for n, e in ours_err.items():
            assert e <= max(4.0 * single_err[n], 1e-5), (what, n, "element-wise relative error to fp64", e,
                                                         "single GPU", single_err[n])


# ======================================================================================================================
# A. N simulated ranks through the _C wrappers
# ======================================================================================================================
class Ranks:
    """The symmetric buffers of N ranks, as N allocations on one device: [4,H,W] images (NaN-filled), two sets of
    accumulators and mark arrays, and int64 device tables of their addresses."""

    def __init__(self, N, P, H, W, dev):
        self.N, self.P, self.H, self.W = N, P, H, W
        self.images = [torch.full((4 * H * W,), float("nan"), device=dev) for _ in range(N)]
        self.accums = [[torch.zeros(P * 12 + 64, device=dev) for _ in range(N)] for _ in range(2)]
        self.marks = [[torch.zeros(P + 256, dtype=torch.uint8, device=dev) for _ in range(N)] for _ in range(2)]
        for t in [t for s in self.accums for t in s]:
            assert t.data_ptr() % 256 == 0
        table = lambda ts: torch.tensor([t.data_ptr() for t in ts], dtype=torch.int64, device=dev)
        self.image_table = table(self.images)
        self.accum_tables = [table(s) for s in self.accums]

    def rows(self, k, r):
        return self.accums[k][r][: self.P * 12].view(self.P, 12)

    def assert_set_clear(self, k, what):
        for r in range(self.N):
            assert int(torch.count_nonzero(self.accums[k][r])) == 0, (what, "accumulator", k, "rank", r)
            assert int(torch.count_nonzero(self.marks[k][r])) == 0, (what, "marks", k, "rank", r)


def setup_case(C, name, N, kind):
    s = scene_state(name)
    bands = make_bands(kind, s["gy"], N)
    abands = [parallel.abi_band(b, s["H"]) for b in bands]
    return s, bands, abands, Ranks(N, s["P"], s["H"], s["W"], s["d"]["means3D"].device)


def forward_ranks(C, s, abands, rk, d=None):
    """Every rank's forward, the all-gather fused in; returns each rank's (R, radii, geom, binning, img)."""
    d = s["d"] if d is None else d
    out = []
    for r, band in enumerate(abands):
        R, none, radii, geom, binning, img = C.rasterize_gaussians_shard(
            band, *call_args(d), peer_images=(rk.image_table.data_ptr(), rk.N))
        assert none is None
        out.append((R, radii, geom, binning, img))
    torch.cuda.synchronize()
    return out


def rank_bargs(s, fw, r, which):
    R, radii, geom, binning, img = fw[r]
    return backward_args(with_dl(s["d"], upstream(s["scene"], which)), radii, geom, R, binning, img)


def assert_gathered(rk, want, what):
    for r in range(rk.N):
        img = rk.images[r].view(4, rk.H, rk.W)
        assert not bool(torch.isnan(img).any()), (what, "rank", r, "pixels nobody stored")
        assert torch.equal(img, want), (what, "rank", r, float((img - want).abs().max()))


@pytest.mark.gpu
@pytest.mark.parametrize("name,N,kind", CASES, ids=CASE_IDS)
def test_forward_all_gather(C, name, N, kind):
    """Every rank ends up with the single-GPU [colour; final_T] bit for bit, and for a second frame with other colours
    into the same buffers."""
    s, bands, abands, rk = setup_case(C, name, N, kind)
    fw = forward_ranks(C, s, abands, rk)
    assert_gathered(rk, s["image"], "frame 1")
    assert sum(f[0] for f in fw) == s["R"]
    for r, f in enumerate(fw):
        assert torch.equal(f[1], s["radii"]), ("radii", r)

    # a second frame with other colours, into the same buffers
    d2 = dict(s["d"])
    if "shs" in d2:
        d2["shs"] = (0.5 - d2["shs"]).contiguous()
    else:
        d2["colors_precomp"] = (1.0 - d2["colors_precomp"]).contiguous()
    R2, color2, *_ = C.rasterize_gaussians(*call_args(d2))
    want2 = torch.cat([color2, s["image"][3:]])
    assert not torch.equal(want2, s["image"])
    forward_ranks(C, s, abands, rk, d2)
    assert_gathered(rk, want2, "frame 2")


@pytest.mark.gpu
@pytest.mark.parametrize("name,N,kind", CASES, ids=CASE_IDS)
def test_peer_reduction(C, name, N, kind):
    """Mode 1: every rank adds its band's sums into the accumulators of all ranks (``red.global.add`` through the
    pointer table).  Every accumulator holds the complete sums, the chain rule on each gives the single-GPU gradients,
    and it leaves its accumulator all-zero -- also over passes that alternate the sets with other upstream gradients."""
    s, bands, abands, rk = setup_case(C, name, N, kind)
    fw = forward_ranks(C, s, abands, rk)
    f64 = fp64_reference(name, bands)
    for k, which in ((0, "g"), (1, "g_band"), (0, "zero"), (1, "g")):
        for r in range(N):
            C.rasterize_gaussians_backward_partials_peers(rk.accums[k][r], rk.accum_tables[k].data_ptr(), N, 0,
                                                          *rank_bargs(s, fw, r, which), shard=abands[r])
        torch.cuda.synchronize()
        single = single_backward(name, which)
        if which == "g":
            for r in range(N):
                check_sums(f"{which} rank {r} accumulator", rk.rows(k, r), single, f64["acc"])
        grads = [dict(zip(GRAD_NAMES, C.rasterize_gaussians_backward_finalize(
            rk.accums[k][r], *rank_bargs(s, fw, r, which), shard=abands[r]))) for r in range(N)]
        torch.cuda.synchronize()
        rk.assert_set_clear(0, f"after {which}")
        rk.assert_set_clear(1, f"after {which}")
        for r in range(N):
            if which == "zero":
                assert all(int(torch.count_nonzero(g)) == 0 for g in grads[r].values() if g is not None), r
            else:
                check_gradients(f"{which} rank {r}", grads[r], single, f64["grads"] if which == "g" else None)


def pull_pass(C, s, fw, abands, rk, k, which, order=None):
    """One pull-mode pass into set k: marked partials on every rank, then the pull chain rule on every rank (which
    clears set k^1).  Returns the gradients per rank and the rows / marks every rank left in set k."""
    N = rk.N
    for r in range(N):
        C.rasterize_gaussians_backward_partials_marked(rk.accums[k][r], rk.marks[k][r], *rank_bargs(s, fw, r, which),
                                                       shard=abands[r])
    torch.cuda.synchronize()
    rows = [rk.rows(k, r).clone() for r in range(N)]
    marks = [rk.marks[k][r][: s["P"]].clone() for r in range(N)]
    grads = [pull_finalize(C, s, fw, abands, rk, k, r, which) for r in range(N)]
    torch.cuda.synchronize()
    return grads, rows, marks


def pull_finalize(C, s, fw, abands, rk, k, r, which):
    return dict(zip(GRAD_NAMES, C.rasterize_gaussians_backward_finalize_pull(
        rk.accums[k][r], [t.data_ptr() for t in rk.accums[k]], [t.data_ptr() for t in rk.marks[k]], rk.N, r,
        rk.accums[k ^ 1][r], rk.marks[k ^ 1][r], *rank_bargs(s, fw, r, which), shard=abands[r])))


def check_pull_result(C, s, fw, abands, grads, rows, marks, what, which):
    """All ranks agree bit for bit, and they equal the chain rule applied to the rank-order sum of the rows the ranks
    left (which is what the pull kernel must compute); the marks bracket the rows."""
    N, P = len(grads), s["P"]
    for r in range(1, N):
        for n in GRAD_NAMES:
            a, b = grads[0][n], grads[r][n]
            assert (a is None) == (b is None) and (a is None or torch.equal(a, b)), (what, "rank", r, n)
    total = torch.zeros_like(rows[0])
    for r in range(N):
        total = total + rows[r]
    buf = torch.zeros(P * 12 + 64, device=total.device)
    buf[: P * 12] = total.view(-1)
    want = dict(zip(GRAD_NAMES, C.rasterize_gaussians_backward_finalize(buf, *rank_bargs(s, fw, 0, which),
                                                                        shard=abands[0])))
    for n in GRAD_NAMES:
        if want[n] is not None:
            assert torch.equal(grads[0][n], want[n]), (what, n, "not the rank-order sum of the ranks' rows")
    M = s["M"]
    for r in range(N):
        nonzero = (rows[r] != 0).any(1)
        marked = marks[r] != 0
        assert bool(marks[r].le(1).all())
        assert not bool((nonzero & ~marked).any()), (what, "rank", r, "rows added to but not marked")
        R, radii, geom, binning, img = fw[r]
        listed = torch.zeros(P, dtype=torch.bool, device=marked.device)
        pl = C.debug_views(geom, binning, img, P, M, s["W"], s["H"], R)["point_list"]
        listed[pl.long()] = True
        assert not bool((marked & ~listed).any()), (what, "rank", r, "marks outside the band's instance list")


@pytest.mark.gpu
@pytest.mark.parametrize("name,N,kind", CASES, ids=CASE_IDS)
def test_pull_mode(C, name, N, kind):
    """Mode 3 in lock-step over four passes that alternate the sets: marked partials into each rank's own set, then
    every rank's pull chain rule reads the marked rows of all ranks and clears the previous set."""
    s, bands, abands, rk = setup_case(C, name, N, kind)
    fw = forward_ranks(C, s, abands, rk)
    f64 = fp64_reference(name, bands)
    for p, which in enumerate(("g", "g_band", "g2", "g")):
        k = p & 1
        grads, rows, marks = pull_pass(C, s, fw, abands, rk, k, which)
        rk.assert_set_clear(k ^ 1, f"pass {p}: the previous pass's set after this pass's chain rule")
        check_pull_result(C, s, fw, abands, grads, rows, marks, f"pass {p}", which)
        single = single_backward(name, which)
        if which == "g":
            for r in range(N):             # each rank's own rows are its band's sums
                check_sums(f"pass {p} rank {r} own rows", rows[r], single_band(C, name, abands[r], s),
                           f64["band_acc"][r])
        check_gradients(f"pass {p}", grads[0], single, f64["grads"] if which == "g" else None)
    # the last pass's set is cleared by the next pass: an all-zero one
    pull_pass(C, s, fw, abands, rk, 0, "zero")
    rk.assert_set_clear(1, "after the closing pass")


def single_band(C, name, band, s):
    """Single-GPU partial sums of one band (the whole-image forward's buffers, the backward restricted to the band),
    twice, for the noise bar of a rank's own rows."""
    key = ("single_band", name, tuple(band))
    if key not in _cache:
        geom, binning, img = s["bufs"]
        bargs = backward_args(s["d"], s["radii"], geom, s["R"], binning, img)
        parts = [C.rasterize_gaussians_backward_partials(*bargs, shard=band)[: s["P"] * 12].view(s["P"], 12).clone()
                 for _ in range(2)]
        torch.cuda.synchronize()
        _cache[key] = dict(parts=[p.double().cpu().numpy() for p in parts])
    return _cache[key]


@pytest.mark.gpu
@pytest.mark.parametrize("name,N,kind", [("precomp", 3, "skewed"), ("precomp", 8, "equal")], ids=["N3", "N8"])
def test_pull_mode_worst_case_order(C, name, N, kind):
    """The furthest the protocol lets ranks drift apart: rank 0 finalises pass k and starts pass k+1 while the others
    are still reading its pass-k rows.  The partial sums come from float atomics, so two runs differ in their last
    bits; every pass is held bit-exact to the chain rule on the rank-order sum of the rows the ranks left, which is
    what lock-step computes, and the gradients meet the lock-step bars."""
    s, bands, abands, rk = setup_case(C, name, N, kind)
    fw = forward_ranks(C, s, abands, rk)
    f64 = fp64_reference(name, bands)
    grads, rows, marks = pull_pass(C, s, fw, abands, rk, 0, "g")          # lock-step: set 1 now has rows to clear
    for k0, (w_k, w_k1) in ((1, ("g2", "g")), (3, ("g", "g_band"))):
        k, k1 = k0 & 1, (k0 + 1) & 1
        snap = lambda kk: ([rk.rows(kk, r).clone() for r in range(N)], [rk.marks[kk][r][: s["P"]].clone() for r in range(N)])
        for r in range(N):                                                 # 1. all partials(k)
            C.rasterize_gaussians_backward_partials_marked(rk.accums[k][r], rk.marks[k][r], *rank_bargs(s, fw, r, w_k),
                                                           shard=abands[r])
        torch.cuda.synchronize()
        rows_k, marks_k = snap(k)
        g_k = [None] * N
        g_k[0] = pull_finalize(C, s, fw, abands, rk, k, 0, w_k)            # 2. finalize(k) on rank 0
        C.rasterize_gaussians_backward_partials_marked(rk.accums[k1][0], rk.marks[k1][0], *rank_bargs(s, fw, 0, w_k1),
                                                       shard=abands[0])    # 3. partials(k+1) on rank 0
        for r in range(1, N):                                              # 4. finalize(k) on the others
            g_k[r] = pull_finalize(C, s, fw, abands, rk, k, r, w_k)
        for r in range(1, N):                                              # 5. the remaining partials(k+1)
            C.rasterize_gaussians_backward_partials_marked(rk.accums[k1][r], rk.marks[k1][r],
                                                           *rank_bargs(s, fw, r, w_k1), shard=abands[r])
        torch.cuda.synchronize()
        rows_k1, marks_k1 = snap(k1)
        g_k1 = [pull_finalize(C, s, fw, abands, rk, k1, r, w_k1) for r in range(N)]    # 6. all finalize(k+1)
        torch.cuda.synchronize()
        rk.assert_set_clear(k, f"set {k} after finalize(k+1)")
        for g, rw, mk, which in ((g_k, rows_k, marks_k, w_k), (g_k1, rows_k1, marks_k1, w_k1)):
            check_pull_result(C, s, fw, abands, g, rw, mk, f"worst-case order, {which}", which)
            check_gradients(f"worst-case order, {which}", g[0], single_backward(name, which),
                            f64["grads"] if which == "g" else None)


@pytest.mark.gpu
def test_pull_mode_refuses_more_than_eight_ranks(C):
    s, bands, abands, rk = setup_case(C, "short", 1, "equal")
    fw = forward_ranks(C, s, abands, rk)
    ptr_a, ptr_m = rk.accums[0][0].data_ptr(), rk.marks[0][0].data_ptr()
    args = rank_bargs(s, fw, 0, "g")
    with pytest.raises(RuntimeError, match="bad peer arguments"):
        C.rasterize_gaussians_backward_finalize_pull(rk.accums[0][0], [ptr_a] * 9, [ptr_m] * 9, 9, 0, rk.accums[1][0],
                                                     rk.marks[1][0], *args, shard=abands[0])
    torch.cuda.synchronize()
    rk.assert_set_clear(0, "a refused call")


# ======================================================================================================================
# B. parallel.py with N threads on one GPU
# ======================================================================================================================
class _DistStandIn:
    """What parallel.py asks torch.distributed, answered per thread."""

    def __init__(self, world):
        self.world, self.local = world, threading.local()

    def get_rank(self, group=None):
        return self.local.rank

    def get_world_size(self, group=None):
        return self.world

    def get_backend(self, group=None):
        return "nccl"


class _Handle:
    """Stand-in for a symmetric-memory rendezvous handle: the ranks' buffer addresses (host list and device table) and
    a barrier that drains this rank's stream before meeting the other threads."""

    def __init__(self, bufs, rank, barrier):
        self.buffer_ptrs = [t.data_ptr() for t in bufs]
        self._table = torch.tensor(self.buffer_ptrs, dtype=torch.int64, device=bufs[0].device)
        self.buffer_ptrs_dev = self._table.data_ptr()
        self.rank, self.world_size, self._barrier = rank, len(bufs), barrier

    def barrier(self, channel=0):
        torch.cuda.current_stream().synchronize()
        self._barrier.wait()


class _FakePeerState:
    """What sharded_forward / sharded_backward read of parallel._PeerState, over buffers shared by the threads."""

    def __init__(self, shared, rank, barrier, mode):
        self.world = len(shared["images"][0])
        self.images = [shared["images"][f][rank] for f in range(2)]
        self.image_hdls = [_Handle(shared["images"][f], rank, barrier) for f in range(2)]
        self.accums = [shared["accums"][k][rank] for k in range(2)]
        self.accum_hdls = [_Handle(shared["accums"][k], rank, barrier) for k in range(2)]
        self.marks = [shared["marks"][k][rank] for k in range(2)] if mode == 3 else []
        self.mark_hdls = [_Handle(shared["marks"][k], rank, barrier) for k in range(2)] if mode == 3 else []
        self.mcs = [0, 0]
        self.frame = 0
        self.bwd = 0


@pytest.mark.gpu
@pytest.mark.parametrize("mode,N,kind", [(1, 3, "equal"), (3, 3, "skewed"), (3, 5, "equal"), (1, 2, "empty_first"),
                                         (3, 2, "empty_first")],
                         ids=["peer-N3", "pull-N3-skewed", "pull-N5", "peer-empty-first", "pull-empty-first"])
def test_parallel_sharded_steps_in_threads(C, monkeypatch, mode, N, kind):
    """Two steps of two composites each (raw and toned colours, as method.py renders), one thread per rank: every
    rank's images are the single-GPU images bit for bit, its gradients meet the single-GPU bars, and every shared
    buffer is all-zero after the last pass's buffers are cleared."""
    name = "precomp"
    s = scene_state(name)
    P, H, W, dev = s["P"], s["H"], s["W"], s["d"]["means3D"].device
    bands = make_bands(kind, s["gy"], N)
    shared = dict(images=[[torch.full((4 * H * W,), float("nan"), device=dev) for _ in range(N)] for _ in range(2)],
                  accums=[[torch.zeros(P * 12 + 64, device=dev) for _ in range(N)] for _ in range(2)],
                  marks=[[torch.zeros(P + 256, dtype=torch.uint8, device=dev) for _ in range(N)] for _ in range(2)])
    barrier = threading.Barrier(N, timeout=60)
    states = [_FakePeerState(shared, r, barrier, mode) for r in range(N)]
    stand_in = _DistStandIn(N)
    monkeypatch.setattr(parallel, "dist", stand_in)
    monkeypatch.setattr(parallel, "_peers", lambda P_, H_, W_, device, group: states[stand_in.get_rank()])
    monkeypatch.setattr(parallel, "_PEER_MODE_ENV", str(mode))

    # inputs of the two steps: the second after a small geometry update; raw and toned colours with their gradients
    d0 = s["d"]
    g = torch.Generator().manual_seed(7)
    d1 = dict(d0)
    d1["means3D"] = (d0["means3D"] + 2e-3 * torch.randn(d0["means3D"].shape, generator=g).to(dev)).contiguous()
    inputs = {}
    for step, d in enumerate((d0, d1)):
        inputs[(step, "raw")] = d
        t = dict(d)
        t["colors_precomp"] = (0.8 * d["colors_precomp"] + 0.1).contiguous()
        t["dL_dpix"] = torch.randn(d["dL_dpix"].shape, generator=g).to(dev)
        inputs[(step, "toned")] = t
    torch.cuda.synchronize()

    results = [dict() for _ in range(N)]
    errors = []

    def rank_main(r):
        stand_in.local.rank = r
        stream = torch.cuda.Stream(dev)
        try:
            with torch.cuda.stream(stream):
                for step in range(2):
                    fwd = {}
                    for comp in ("raw", "toned"):
                        full, R, radii, geom, binning, img = parallel.sharded_forward(call_args(inputs[(step, comp)]), bands)
                        fwd[comp] = (full, R, radii, geom, binning, img)
                    for comp in ("toned", "raw"):
                        full, R, radii, geom, binning, img = fwd[comp]
                        grads = parallel.sharded_backward(backward_args(inputs[(step, comp)], radii, geom, R, binning,
                                                                        img), bands)
                        results[r][(step, comp)] = (full, radii, dict(zip(GRAD_NAMES, grads)))
            stream.synchronize()
        except BaseException as e:          # noqa: BLE001 -- reported by the main thread
            errors.append((r, e))
            barrier.abort()

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(N)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(180)
    assert not any(t.is_alive() for t in threads), "a rank thread did not finish"
    if errors:
        raise errors[0][1]

    # single-GPU references
    for (step, comp), d in inputs.items():
        R, color, radii, geom, binning, img = C.rasterize_gaussians(*call_args(d))
        fT = C.debug_views(geom, binning, img, P, 0, W, H, R)["final_T"]
        want = torch.cat([color, fT[None]])
        bargs = backward_args(d, radii, geom, R, binning, img)
        single = dict(grads=[dict(zip(GRAD_NAMES, C.rasterize_gaussians_backward(*bargs))) for _ in range(2)])
        torch.cuda.synchronize()
        g64 = fp64_reference(name, bands)["grads"] if (step, comp) == (0, "raw") else None
        for r in range(N):
            full, radii_r, grads = results[r][(step, comp)]
            assert torch.equal(full, want), (step, comp, "rank", r)
            assert torch.equal(radii_r, radii), (step, comp, "rank", r)
            check_gradients(f"step {step} {comp} rank {r}", grads, single, g64)
            if mode == 3 and r > 0:
                for n in GRAD_NAMES:
                    a, b = results[0][(step, comp)][2][n], grads[n]
                    assert a is None or torch.equal(a, b), (step, comp, "rank", r, n)
    # mode 1 clears each accumulator in its chain rule; mode 3 leaves the last pass's set for the next pass to clear
    for k in range(2):
        for r in range(N):
            if mode == 1 or k == 0:
                assert int(torch.count_nonzero(shared["accums"][k][r])) == 0, ("accumulator", k, "rank", r)
                assert int(torch.count_nonzero(shared["marks"][k][r])) == 0, ("marks", k, "rank", r)
