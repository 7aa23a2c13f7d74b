"""Screen-space sharding of one rasterization across the GPUs of a box (SURVEY.md section 8e).

The reference is single-GPU (``method.py:113-117``); this is the new multi-GPU path BASELINE.json asks
for.  One process per GPU (``torch.distributed``, NCCL over NVLink/NVSwitch).  Every rank holds all P
Gaussians (replicated parameters, as in single-GPU training) and

* forward: projects all Gaussians (cheap, HBM-bound) but bins / sorts / composites only its band of tile
  rows ``[y0, y1)``; because the sort key's major field is the tile id, a band's instance list is exactly
  the corresponding slice of the single-GPU list, so its pixels are bit-identical to the single-GPU image.
  One all-gather of the colour (+ transmittance) bands assembles the full image on every rank.
* backward: the upstream gradient image is replicated (every rank evaluates the loss on the full image);
  each rank runs the backward composite on its band into a ``[P,12]`` partial-sum array; one all-reduce (sum)
  adds the partials of Gaussians that straddle bands -- a plain all-gather would be wrong -- and every rank then runs the
  per-Gaussian chain rule on the summed partials, yielding the full gradients everywhere.

The collective helpers below are backend-agnostic (tested with gloo on CPU, world_size 2).
"""
from __future__ import annotations

import os

from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist

TILE = 16


def partition_tile_rows(num_tile_rows: int, world_size: int, weights: Sequence[float] | None = None) -> List[Tuple[int, int]]:
    """Contiguous bands of tile rows, one per rank.  With ``weights`` (e.g. instances per tile row from the
    previous iteration) the bands are chosen to equalise the weight; otherwise the row counts."""
    import bisect
    n, w = int(num_tile_rows), int(world_size)
    assert n >= 0 and w >= 1
    if weights is None or float(sum(weights)) <= 0.0:
        weights = [1.0] * n
    assert len(weights) == n
    cum = [0.0]
    for x in weights:
        cum.append(cum[-1] + float(x))
    total = cum[-1]
    cuts = [0]
    for r in range(1, w):
        # first row boundary at which the running weight reaches r/w of the total; the rounding slack is relative, so
        # tiny totals do not pull every cut down to row 0
        e = bisect.bisect_left(cum, total * r / w - 1e-9 * total)
        cuts.append(min(n, max(e, cuts[-1])))
    cuts.append(n)
    return [(cuts[r], cuts[r + 1]) for r in range(w)]


def abi_band(band: Tuple[int, int], H: int) -> Tuple[int, int]:
    """A rank's band as the ``_C`` calls take it.  There ``(0, 0)`` is the single-GPU "whole image" shard, so an empty
    band -- ``(0, 0)`` included -- is handed over as the empty band below the last tile row; otherwise a rank without
    rows would composite the whole image and add its sums on top of everyone else's."""
    y0, y1 = int(band[0]), int(band[1])
    if y1 <= y0:
        gy = (int(H) + TILE - 1) // TILE
        return gy, gy
    return y0, y1


def band_pixel_rows(band: Tuple[int, int], H: int) -> Tuple[int, int]:
    return min(H, band[0] * TILE), min(H, band[1] * TILE)


def gather_image_bands(img: torch.Tensor, bands: Sequence[Tuple[int, int]], group=None) -> torch.Tensor:
    """``img`` is ``[C,H,W]`` with only this rank's band rows valid; returns the full ``[C,H,W]`` on every rank.

    A single all-gather: each rank contributes its band packed into a ``[C, hmax, W]`` slab (bands may differ
    in height by one tile row; shorter ones are zero padded)."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    C, H, W = img.shape
    rows = [band_pixel_rows(b, H) for b in bands]
    hmax = max(r1 - r0 for r0, r1 in rows)
    slab = torch.zeros((C, hmax, W), dtype=img.dtype, device=img.device)
    r0, r1 = rows[rank]
    slab[:, : r1 - r0] = img[:, r0:r1]
    out = torch.empty((world, C, hmax, W), dtype=img.dtype, device=img.device)
    try:
        dist.all_gather_into_tensor(out, slab, group=group)
    except (RuntimeError, NotImplementedError):        # backends without the fused form
        parts = [torch.empty_like(slab) for _ in range(world)]
        dist.all_gather(parts, slab, group=group)
        out = torch.stack(parts)
    full = torch.empty_like(img)
    for r, (a, b) in enumerate(rows):
        full[:, a:b] = out[r, :, : b - a]
    return full


def reduce_partials(accum: torch.Tensor, group=None) -> torch.Tensor:
    """Sum the per-Gaussian partial-gradient arrays of all bands in place (all-reduce)."""
    dist.all_reduce(accum, op=dist.ReduceOp.SUM, group=group)
    return accum


# ---- collectives fused into the composites (peer / multicast memory over NVLink-NVSwitch) --------------------------------
# Forward: every rank's composite stores its band of the [4,H,W] image (colour + final transmittance) straight into the
# symmetric image buffer of EVERY rank (peer-mapped pointers); one device-side barrier later each rank holds the full
# image -- no NCCL call, no staging copies.
# Backward: GSR_PEER_REDUCE=1 (default): every rank's backward composite adds its per-Gaussian sums straight into the
# accumulators of all ranks through peer pointers; =2: through the NVSwitch multicast address when the platform offers
# one (one multimem.red per 16 bytes, the switch updates every replica); =0: local sums + NCCL all-reduce after the kernel
# (and a NCCL all-gather of the image bands in the forward).  The accumulators stay zero between steps: the per-Gaussian
# chain-rule stage zero-fills its accumulator after consuming it (no fill + barrier in front of the reductions).  If symmetric memory cannot be set up the
# NCCL path is used.
# GSR_PEER_REDUCE=3 ("pull"): the backward composite adds into its OWN accumulator and marks the Gaussians it touched; after
# one barrier every rank's chain-rule kernel reads the marked rows of the other ranks through their peer mappings (plain
# loads, rank order -> bit-identical gradients on all ranks).  No remote atomics: peer `red` is posted cheaply but drains
# slowly, behind the barrier that follows the kernel.
# Default (GSR_PEER_REDUCE unset): 1 for two ranks, 3 from three ranks on (the remote-atomic drain grows with the rank
# count; the multi-GPU modes have not been timed on H100 machines).
_PEER_MODE_ENV = os.environ.get("GSR_PEER_REDUCE")


def peer_mode(group=None) -> int:
    """The reduction mode in effect for this process group (see above)."""
    if _PEER_MODE_ENV is not None:
        return int(_PEER_MODE_ENV)
    return 3 if dist.get_world_size(group) >= 3 else 1
_peer_state: dict = {}
_peer_warned = False


class _PeerState:
    """Symmetric buffers of one (P, H, W, device, group): the [P,12] accumulator and the [4,H,W] image."""

    def __init__(self, P, H, W, device, group):
        import torch.distributed._symmetric_memory as symm_mem
        g = group if group is not None else dist.group.WORLD
        mode = peer_mode(group)
        # two accumulators, used alternately (same argument as for the images below: with several backward passes per
        # step -- wild-gaussians composites twice -- a rank's reductions of pass k+1 must not land in a peer's accumulator
        # while that peer is still consuming pass k; pass k+2 lies behind pass k+1's barrier)
        self.accums = [symm_mem.empty(P * 12 + 64, dtype=torch.float32, device=device) for _ in range(2)]
        for t in self.accums:
            t.zero_()
        self.accum_hdls = [symm_mem.rendezvous(t, g) for t in self.accums]
        self.bwd = 0
        # pull-mode reduction (GSR_PEER_REDUCE=3): one mark byte per Gaussian next to each accumulator
        self.marks, self.mark_hdls = [], []
        if mode == 3:
            self.marks = [symm_mem.empty(P + 256, dtype=torch.uint8, device=device) for _ in range(2)]
            for t in self.marks:
                t.zero_()
            self.mark_hdls = [symm_mem.rendezvous(t, g) for t in self.marks]
        # two images, used alternately: a rank may start storing frame k+1 into its peers while a slower peer is still
        # copying frame k out of its own buffer (forward-only loops have no other barrier in between); it cannot reach
        # frame k+2 before that peer has passed frame k+1's barrier, i.e. finished the copy of frame k
        self.images = [symm_mem.empty(4 * H * W, dtype=torch.float32, device=device) for _ in range(2)]
        self.image_hdls = [symm_mem.rendezvous(t, g) for t in self.images]
        self.frame = 0
        self.mcs = [0, 0]
        if mode == 2:
            for i, h in enumerate(self.accum_hdls):
                try:
                    self.mcs[i] = int(h.multicast_ptr or 0)
                except Exception:
                    self.mcs[i] = 0
        for t, h in zip(self.accums, self.accum_hdls):
            assert t.data_ptr() % 256 == 0 and all(int(x) % 256 == 0 for x in h.buffer_ptrs)
        self.world = self.accum_hdls[0].world_size
        # every rank's accumulators are zero before anyone adds into them
        self.accum_hdls[0].barrier(channel=0)


def _peers(P, H, W, device, group):
    """The symmetric state, or None when the NCCL path has to be used."""
    global _peer_warned
    if peer_mode(group) <= 0 or P <= 0 or dist.get_backend(group) != "nccl":
        return None
    key = (int(P), int(H), int(W), str(device), id(group))
    st = _peer_state.get(key)
    if st is None and key not in _peer_state:
        try:
            st = _PeerState(P, H, W, device, group)
        except Exception as e:                      # no symmetric memory on this platform / build: NCCL path
            st = None
            if not _peer_warned:
                _peer_warned = True
                print(f"[parallel] symmetric memory unavailable ({type(e).__name__}: {e}); using NCCL collectives")
        _peer_state[key] = st
    return st


def sharded_forward(fwd_args, bands, group=None):
    """This rank's band of one forward + the image all-gather.  ``fwd_args``: the 21 positional arguments of
    ``_C.rasterize_gaussians``.  Returns ``(full [4,H,W] (colour planes + final transmittance), num_rendered, radii, geom,
    binning, img)``; the full image is identical on every rank."""
    from diff_gaussian_rasterization import _C
    rank = dist.get_rank(group)
    means3D = fwd_args[1]
    P, H, W = int(means3D.size(0)), int(fwd_args[14]), int(fwd_args[15])
    shard = abi_band(bands[rank], H)
    st = _peers(P, H, W, means3D.device, group)
    if st is not None:
        image, hdl = st.images[st.frame], st.image_hdls[st.frame]
        st.frame ^= 1
        R, _none, radii, geom, binning, img = _C.rasterize_gaussians_shard(
            shard, *fwd_args, peer_images=(hdl.buffer_ptrs_dev, st.world))
        hdl.barrier(channel=0)                      # every band has landed in every rank's image
        full = image.view(4, H, W).clone()          # the symmetric buffer is overwritten two forwards later
        return full, R, radii, geom, binning, img
    R, color, radii, geom, binning, img = _C.rasterize_gaussians_shard(shard, *fwd_args)
    offset = (128 - img.data_ptr()) % 128
    final_T = img[offset:offset + 4 * H * W].view(torch.float32).view(1, H, W)
    full = gather_image_bands(torch.cat([color, final_T], dim=0), bands, group)
    return full, R, radii, geom, binning, img


def reduced_partials(bwd_args, P: int, device, group=None, shard=None) -> torch.Tensor:
    """Backward composite of this rank's band + sum over all bands: returns the accumulator holding the complete
    per-Gaussian sums (flat fp32, first P*12 entries).  Either NCCL all-reduce of the partial arrays or, with
    GSR_PEER_REDUCE, the reduction fused into the kernel through peer / multicast memory."""
    from diff_gaussian_rasterization import _C
    _C.refuse_nondeterministic("parallel.reduced_partials (multi-GPU backward reduction: peer red, multicast or NCCL "
                               "all-reduce)")
    H, W = int(bwd_args[14].size(1)), int(bwd_args[14].size(2))
    st = _peers(P, H, W, device, group)
    if st is not None:
        # the accumulators of all ranks are zero here: cleared by the previous step's chain-rule kernel (or at creation),
        # and the forward's image barrier lies between that kernel and this one on every rank
        accum, hdl, mc = st.accums[st.bwd], st.accum_hdls[st.bwd], st.mcs[st.bwd]
        st.bwd ^= 1
        _C.rasterize_gaussians_backward_partials_peers(accum, hdl.buffer_ptrs_dev, st.world, mc, *bwd_args, shard=shard)
        hdl.barrier(channel=1)                   # all contributions have landed everywhere
        return accum
    accum = _C.rasterize_gaussians_backward_partials(*bwd_args, shard=shard)
    reduce_partials(accum[: P * 12], group)
    return accum


def sharded_backward(bwd_args, bands, group=None):
    """Backward of ``sharded_forward``: ``bwd_args`` are the 23 positional arguments of
    ``_C.rasterize_gaussians_backward`` (upstream gradient replicated); returns the 8 gradient tensors, complete on every
    rank."""
    from diff_gaussian_rasterization import _C
    _C.refuse_nondeterministic("parallel.sharded_backward (multi-GPU backward reduction: peer red, multicast, pull or "
                               "NCCL all-reduce)")
    rank = dist.get_rank(group)
    means3D = bwd_args[1]
    H, W = int(bwd_args[14].size(1)), int(bwd_args[14].size(2))
    shard = abi_band(bands[rank], H)
    if peer_mode(group) == 3:
        P = int(means3D.size(0))
        st = _peers(P, H, W, means3D.device, group)
        if st is not None and st.marks:
            # pull mode: local sums + marks, one barrier, then every rank reads the rows the others marked (no remote
            # atomics, no N-fold write amplification, the same summation order everywhere)
            k = st.bwd
            st.bwd ^= 1
            accum, hdl, marks, mhdl = st.accums[k], st.accum_hdls[k], st.marks[k], st.mark_hdls[k]
            _C.rasterize_gaussians_backward_partials_marked(accum, marks, *bwd_args, shard=shard)
            hdl.barrier(channel=1)               # every rank's sums and marks of this pass are complete
            return _C.rasterize_gaussians_backward_finalize_pull(
                accum, list(hdl.buffer_ptrs), list(mhdl.buffer_ptrs), st.world, hdl.rank, st.accums[k ^ 1], st.marks[k ^ 1],
                *bwd_args, shard=shard)
    accum = reduced_partials(bwd_args, int(means3D.size(0)), means3D.device, group, shard=shard)
    return _C.rasterize_gaussians_backward_finalize(accum, *bwd_args, shard=shard)


class _ShardedRasterize(torch.autograd.Function):
    """Tile-row sharded counterpart of ``diff_gaussian_rasterization._RasterizeGaussians``."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings, bands, group):
        s = raster_settings
        args = (s.bg, means3D, colors_precomp, opacities, scales, rotations, s.scale_modifier, cov3Ds_precomp,
                s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.kernel_size, s.subpixel_offset,
                s.image_height, s.image_width, sh, s.sh_degree, s.campos, s.prefiltered, s.debug)
        H, W = int(s.image_height), int(s.image_width)
        if int(means3D.size(0)) == 0:          # nothing to render (the reference skips everything, rasterize_points.cu:83)
            ctx.empty = True
            dev = means3D.device
            z = torch.zeros((3, H, W), dtype=torch.float32, device=dev)
            return z, torch.zeros((0,), dtype=torch.int32, device=dev), (torch.zeros((H, W), dtype=torch.float32, device=dev)
                                                                         if s.return_accumulation else None)
        ctx.empty = False
        # the band is an explicit argument of the calls (stored on ctx for the backward), not module state
        full, num_rendered, radii, geom, binning, img = sharded_forward(args, bands, group)
        ctx.raster_settings, ctx.num_rendered, ctx.bands, ctx.group = s, num_rendered, bands, group
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geom, binning, img)
        accumulation = (1.0 - full[3]) if s.return_accumulation else None
        return full[:3], radii, accumulation

    @staticmethod
    def backward(ctx, grad_out_color, _1, _2):
        s = ctx.raster_settings
        if ctx.empty:
            return (None,) * 11
        colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geom, binning, img = ctx.saved_tensors
        args = (s.bg, means3D, radii, colors_precomp, scales, rotations, s.scale_modifier, cov3Ds_precomp,
                s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.kernel_size, s.subpixel_offset,
                grad_out_color, sh, s.sh_degree, s.campos, geom, ctx.num_rendered, binning, img, s.debug)
        (g_means2D, g_colors, g_opac, g_means3D, g_cov3D, g_sh, g_scales, g_rot) = sharded_backward(args, ctx.bands, ctx.group)
        return (g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rot, g_cov3D, None, None, None)


# ---- host-buffer I/O for the sharded path: every rank moves only 1/world of the bytes over PCIe ---------------------------
def upload_sharded(host: torch.Tensor, device, group=None) -> torch.Tensor:
    """`host` is a pinned CPU tensor holding the SAME data on every rank.  Rank r copies only the r-th of `world` equal
    chunks of its bytes to the device; one all-gather (NVLink) assembles the full tensor on every rank."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    flat = host.reshape(-1)
    n = flat.numel()
    chunk = (n + world - 1) // world
    full = torch.empty((chunk * world,), dtype=host.dtype, device=device)
    lo, hi = min(n, rank * chunk), min(n, (rank + 1) * chunk)
    mine = full[rank * chunk: rank * chunk + (hi - lo)]
    if hi > lo:
        mine.copy_(flat[lo:hi], non_blocking=True)
    dist.all_gather_into_tensor(full, full[rank * chunk:(rank + 1) * chunk].clone(), group=group)
    return full[:n].view(host.shape)


def download_sharded(dev_t: torch.Tensor, host_out: torch.Tensor, group=None) -> None:
    """Counterpart of ``upload_sharded`` for results that are replicated on every rank (image, gradients): rank r copies
    only its chunk into its pinned `host_out`; the ranks' host buffers together hold the tensor exactly once."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    flat, out = dev_t.reshape(-1), host_out.reshape(-1)
    n = flat.numel()
    chunk = (n + world - 1) // world
    lo, hi = min(n, rank * chunk), min(n, (rank + 1) * chunk)
    if hi > lo:
        out[lo:hi].copy_(flat[lo:hi], non_blocking=True)


class ShardedGaussianRasterizer(torch.nn.Module):
    """Same call signature as ``GaussianRasterizer``; every rank must call it with identical arguments.
    Returns the full image, radii and accumulation on every rank."""

    def __init__(self, raster_settings, group=None, bands=None, row_weights=None):
        super().__init__()
        self.raster_settings = raster_settings
        self.group = group
        world = dist.get_world_size(group)
        rows = (int(raster_settings.image_height) + TILE - 1) // TILE
        self.bands = list(bands) if bands is not None else partition_tile_rows(rows, world, row_weights)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        if (shs is None) == (colors_precomp is None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        empty = torch.Tensor([])
        return _ShardedRasterize.apply(
            means3D, means2D, empty if shs is None else shs, empty if colors_precomp is None else colors_precomp,
            opacities, empty if scales is None else scales, empty if rotations is None else rotations,
            empty if cov3D_precomp is None else cov3D_precomp, self.raster_settings, self.bands, self.group)
