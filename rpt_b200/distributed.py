"""Multi-GPU sharding of Renderer::sample (SURVEY 8e).

The reference parallelises over image rows with rayon (src/renderer.rs:118-127); pixels
and samples are independent and the scene is read-only.  Here the image is cut into
16x8-pixel tiles dealt round-robin to ranks (tile t belongs to rank t % world), every
rank (one process per GPU) renders only its tiles into a zero-initialised full-size
float3 buffer, and ONE all-reduce(sum) over NCCL assembles the image.  Because the RNG
stream is keyed by (seed, pixel, sample) and every pixel is summed by exactly one rank,
the result is bit-identical for any world size (x + 0 is exact).

Two ways to assemble, same bits:

  * `assemble` / `render_distributed`: every rank renders into a zeroed FULL-size buffer, one all-reduce(sum).  N x the
    image in flight.
  * `gather_tiles` / `render_distributed_gather`: every rank renders ONLY its own tiles into a compact tile-major
    buffer (rptb_render_params.compact_out, 1/N of the image), one all-gather, then a fixed permutation puts the
    pixels in row-major order.  1 x the image in flight, and nothing is summed at all -- what bench.py times.

The device Buffer shards the same way (`ShardBuffer`, rptb_buffer_create_shard): every rank samples, adapts and adds
features into its own tiles with no exchange, and `ShardBuffer.gather` -- one all-gather of the ranks' exchange blocks
-- gives every rank an ordinary whole DeviceBuffer, the same bits for any world size.  `render_iterative_distributed`
is Renderer.iterative_render over a ShardBuffer; with adaptive sampling it adds one collective per batch, an
all-reduce of the ranks' active pixel counts that ends the loop.  Nothing else is exchanged.

`render_frames_distributed` is Renderer.render_frames over ShardBuffers.  A reprojected pixel needs only its own
features and the whole previous frame, which every rank already holds: the frame's gather, with features, gave it.  So
each rank reprojects that gathered buffer into its own shard (ShardBuffer.reproject_from), and a frame costs one
all-gather, the one that makes its image.  Testing the history against fresh entries (history_test,
ShardBuffer.merge_history_from) reads each pixel's own fresh state only, so it adds no exchange either.

Guided adaptive sampling (Adaptive(guide=...)) is the exception: its filter reaches about 62 pixels at 5 passes, across
other ranks' tiles, so every rank needs the whole image's state before each guided call.  A rank keeps a gathered whole
buffer current instead of re-gathering it: one full gather with features when the filter is first needed, then after
every call one all-gather of delta blocks (ShardBuffer.gather_delta) -- only the pixels that call changed, with their
new state -- applied in place.  Each rank's filter and decisions are then those of the whole buffer's call, bit for
bit, and so are its entries.  The error estimate from two half buffers (Adaptive(estimate="halves")) runs the same
way over shards with halves (ShardBuffer(halves=True)): their full and delta blocks carry HALF too, and the gathered
whole buffer has halves.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Optional

import numpy as np

from . import _capi as capi
from . import api

TILE_W, TILE_H = 16, 8  # must match rpt_b200/csrc/integrator.cuh


def tile_owner(width: int, height: int, shard_count: int) -> np.ndarray:
    """(height, width) int array: which shard renders each pixel."""
    tiles_x = (width + TILE_W - 1) // TILE_W
    ys, xs = np.mgrid[0:height, 0:width]
    tile = (ys // TILE_H) * tiles_x + (xs // TILE_W)
    return (tile % shard_count).astype(np.int32)


def shard_tiles(width: int, height: int, shard_index: int, shard_count: int) -> int:
    """How many 16x8 tiles shard `shard_index` of `shard_count` owns (RenderArgs::ntiles_mine)."""
    ntiles = ((width + TILE_W - 1) // TILE_W) * ((height + TILE_H - 1) // TILE_H)
    return (ntiles - shard_index + shard_count - 1) // shard_count if ntiles > shard_index else 0


def gather_permutation(width: int, height: int, shard_count: int) -> np.ndarray:
    """For the concatenation of the shards' compact buffers, each padded to shard 0's size (the largest):
    perm[y * width + x] = index of that pixel in the concatenation (in pixels, not floats).  Mirrors rptb_tile_pixel."""
    tiles_x = (width + TILE_W - 1) // TILE_W
    per = shard_tiles(width, height, 0, shard_count) * TILE_W * TILE_H
    ys, xs = np.mgrid[0:height, 0:width]
    tile = (ys // TILE_H) * tiles_x + (xs // TILE_W)
    lx, ly = xs % TILE_W, ys % TILE_H
    j = ((ly // 4) * 2 + lx // 8) * 32 + (ly % 4) * 8 + lx % 8   # warp (ly/4, lx/8) covers 8x4 pixels, lane = row-major inside it
    return ((tile % shard_count) * per + (tile // shard_count) * (TILE_W * TILE_H) + j).astype(np.int64).ravel()


def gather_tiles(render_compact: Callable[[int, int], "object"], width: int, height: int, perm=None, group=None):
    """All ranks call this.  `render_compact(rank, world)` -> 1-D float tensor holding this rank's tiles, tile-major
    (shard_tiles(...) * 384 values; it may be longer -- it is cut / padded to shard 0's size).  One all-gather, then
    the pixels are put in row-major order: returns (height*width, 3) on every rank."""
    import torch
    import torch.distributed as dist

    on = dist.is_available() and dist.is_initialized()
    rank = dist.get_rank(group) if on else 0
    world = dist.get_world_size(group) if on else 1
    mine = render_compact(rank, world)
    per = shard_tiles(width, height, 0, world) * TILE_W * TILE_H * 3
    if mine.numel() != per:
        padded = mine.new_zeros(per)
        padded[:min(per, mine.numel())] = mine[:per]
        mine = padded
    if world > 1:
        allv = mine.new_empty(per * world)
        dist.all_gather_into_tensor(allv, mine, group=group)
    else:
        allv = mine
    if perm is None:
        perm = torch.from_numpy(gather_permutation(width, height, world)).to(allv.device)
    return allv.view(-1, 3).index_select(0, perm)


def assemble(render_shard: Callable[[int, int], "object"], group=None):
    """The collective step, independent of what renders a shard: every rank calls
    `render_shard(rank, world)` -> a tensor holding its tiles and zeros elsewhere, then one
    all-reduce(sum).  Used with the CUDA shard renderer in production (NCCL) and with a CPU
    shard renderer in the gloo tests."""
    import torch.distributed as dist

    on = dist.is_available() and dist.is_initialized()
    rank = dist.get_rank(group) if on else 0
    world = dist.get_world_size(group) if on else 1
    out = render_shard(rank, world)
    if world > 1:
        dist.all_reduce(out, op=dist.ReduceOp.SUM, group=group)
    return out


def render_shard_device(renderer, iterations: int, out, shard_index: int, shard_count: int, first_sample: int = 0,
                        stream: Optional[int] = None, stats: Optional[capi.Stats] = None, collect_stats: int = 0,
                        compact: bool = False) -> None:
    """Launch this shard's part of Renderer::sample into `out`, a CUDA float32 tensor of
    width*height*3 elements (torch) on the renderer's device.  `stream` is a raw
    cudaStream_t; torch's default stream has handle 0, which is passed as cudaStreamLegacy
    (0x1) because NULL means "the library's own stream, synchronous" at the C ABI.  compact = True: `out` holds only
    this shard's tiles, tile-major (shard_tiles(...) * 384 floats; rptb_render_params.compact_out)."""
    ds = renderer.device_scene()
    p = renderer.params(iterations, first_sample, shard_index, shard_count, collect_stats)
    p.compact_out = 1 if compact else 0
    cam = renderer.camera.to_c()
    capi.check(
        capi.lib().rptb_render_samples_device(ds.handle, C.byref(cam), C.byref(p), C.c_void_p(out.data_ptr()),
                                              C.c_void_p(stream or 1), C.byref(stats) if stats is not None else None),
        "rptb_render_samples_device",
    )


def render_distributed(renderer, iterations: int, first_sample: int = 0, group=None, out=None):
    """All ranks call this; returns the full image as a CUDA float32 tensor (H*W, 3) on
    every rank.  One process per GPU (torchrun); NCCL over NVLink.  The kernel and the
    all-reduce are enqueued on the same stream: no host synchronisation in between."""
    import torch

    dev = torch.device("cuda", renderer._first_device())
    if out is None:
        out = torch.empty(renderer._width * renderer._height * 3, dtype=torch.float32, device=dev)

    def shard(rank: int, world: int):
        stream = torch.cuda.current_stream(dev).cuda_stream
        render_shard_device(renderer, iterations, out, rank, world, first_sample, stream)
        return out

    return assemble(shard, group).view(-1, 3)


def render_distributed_gather(renderer, iterations: int, first_sample: int = 0, group=None, scratch=None, perm=None):
    """Like render_distributed, through the all-gather of compact shards: (H*W, 3) float32 on every rank."""
    import torch

    dev = torch.device("cuda", renderer._first_device())
    w, h = renderer._width, renderer._height

    def shard(rank: int, world: int):
        n = shard_tiles(w, h, 0, world) * TILE_W * TILE_H * 3
        buf = scratch if scratch is not None and scratch.numel() == n else torch.zeros(n, dtype=torch.float32, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        render_shard_device(renderer, iterations, buf, rank, world, first_sample, stream, compact=True)
        return buf

    return gather_tiles(shard, w, h, perm, group)


# ---- the device Buffer, one shard per rank ---------------------------------------------------------------------------
SHARD_HEADER_BYTES = 256  # must match rpt_b200/csrc/api.cu (kShardHeaderBytes)


def shard_block_layout(width: int, height: int, shard_count: int, with_features: bool = False, halves: bool = False) -> dict:
    """Byte offsets of the planes in one shard's exchange block (rptb_buffer_export_shard), the same for every shard:
    a header, then sums (3 doubles a slot), M2 (1 double), with features the feature sums (8 doubles: normal 3, albedo
    3, hits 1, depth 1), then counts (1 uint32), and from a shard with halves HALF (3 doubles: the sums of the odd
    entries) at "half".  Every plane has `slots` = shard 0's tiles * 128 slots, the padding gather_tiles uses, so slot
    k * 128 + j of shard s's planes is pixel rptb_tile_pixel(width, height, s, shard_count, k, j) and
    gather_permutation(width, height, shard_count) // slots / % slots finds a pixel's shard and slot."""
    slots = shard_tiles(width, height, 0, shard_count) * TILE_W * TILE_H
    sums = SHARD_HEADER_BYTES
    m2 = sums + slots * 3 * 8
    features = m2 + slots * 8
    counts = features + (slots * 8 * 8 if with_features else 0)
    lay = {"slots": slots, "sums": sums, "m2": m2, "features": features, "counts": counts, "bytes": counts + slots * 4}
    if halves:
        lay["half"] = lay["bytes"]
        lay["bytes"] += slots * 3 * 8
    return lay


DELTA_HEADER_BYTES = 256  # must match rpt_b200/csrc/delta.h (kDeltaHeaderBytes)
DELTA_PIXELS_AT = 248  # the byte offset of the header's pixel count (DeltaHeader::pixels, a uint32)


def delta_block_layout(capacity: int, halves: bool = False) -> dict:
    """Byte offsets of the planes in one shard's delta block of `capacity` pixels (rptb_buffer_export_delta), the same for
    every shard: a header, then sums (3 doubles a pixel), M2 (1 double), counts (1 uint32) and slots (1 uint32: the
    pixel's compact slot in its shard, ascending), and from a shard with halves HALF (3 doubles) at "half"
    (rptb_delta_bytes_halves).  Only the header's pixel count of each plane is written."""
    m = int(capacity)
    sums = DELTA_HEADER_BYTES
    m2 = sums + 24 * m
    counts = m2 + 8 * m
    slots = counts + 4 * m
    lay = {"capacity": m, "sums": sums, "m2": m2, "counts": counts, "slots": slots, "bytes": slots + 4 * m}
    if halves:
        lay["half"] = lay["bytes"]
        lay["bytes"] += 24 * m
    return lay


def _all_gather_bytes(mine, world: int, group):
    """Every rank's uint8 block (the same size on every rank), concatenated in rank order: (on mine's device, on the host
    or None).  NCCL gathers GPU to GPU; any other backend (gloo) through a host tensor, which is also returned."""
    import torch
    import torch.distributed as dist

    if world == 1:
        return mine, None
    if dist.get_backend(group) == "nccl":
        gathered = torch.empty(mine.numel() * world, dtype=torch.uint8, device=mine.device)
        dist.all_gather_into_tensor(gathered, mine, group=group)
        return gathered, None
    staged = torch.empty(mine.numel() * world, dtype=torch.uint8)
    dist.all_gather_into_tensor(staged, mine.cpu(), group=group)
    return staged.to(mine.device), staged


def _rank_world(group=None):
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


class ShardBuffer(api.DeviceBuffer):
    """A DeviceBuffer holding one rank's shard of the image (rptb_buffer_create_shard): the 16x8 tiles t with
    t % world == rank, on the scene's one device.  Renderer.sample and Renderer.sample_features render and add only
    those tiles, with no exchange; an adaptive sample() returns this rank's active pixel count, and reproject_from
    takes this rank's pixels' history from a whole buffer.  Whole-image reads (image, variance, sums, pixel_stats,
    counts, features, denoise, add_samples) are refused: gather() first.  `entries` counts the calls (a bound on any
    pixel's count) until the gather reads the counts.  `halves` (rptb_buffer_create_shard_halves): the shard also keeps
    the sums of each pixel's odd entries, its blocks carry them, and gather() gives a whole buffer with halves -- what
    Adaptive(estimate="halves") needs.  Its reproject_from and merge_history_from take history with halves from a whole
    src with halves (RptbError from a plain one)."""

    def __init__(self, scene: "api.DeviceScene", width: int, height: int, filter: Optional["api.Filter"] = None, group=None,
                 rank: Optional[int] = None, world: Optional[int] = None, halves: bool = False):
        if rank is None or world is None:
            rank, world = _rank_world(group)
        self.width, self.height = int(width), int(height)
        self.filter = filter or api.Filter()
        self.devices = list(scene.devices)
        self.entries = 0
        self.feature_rays = 0
        self.shard = (int(rank), int(world))
        self.halves = bool(halves)
        self.group = group
        self._scene = scene  # the whole buffer of gather() is created on it
        self.handle = C.c_void_p()
        name = "rptb_buffer_create_shard_halves" if self.halves else "rptb_buffer_create_shard"
        capi.check(getattr(capi.lib(), name)(scene.handle, self.width, self.height, self.filter.radius, self.shard[0], self.shard[1],
                                             C.byref(self.handle)), name)

    def block_bytes(self, with_features: bool = False) -> int:
        """The size of this shard's exchange block (rptb_buffer_shard_bytes; shard_block_layout): the same on every rank."""
        return int(capi.lib().rptb_buffer_shard_bytes(self.handle, 1 if with_features else 0))

    def export(self, out, with_features: bool = False, stream: Optional[int] = None) -> None:
        """Writes this shard's exchange block into `out`, a CUDA uint8 tensor of block_bytes() on the buffer's device, on
        `stream` (a raw cudaStream_t; the current torch stream when None)."""
        import torch

        if stream is None:
            stream = torch.cuda.current_stream(out.device).cuda_stream
        capi.check(capi.lib().rptb_buffer_export_shard(self.handle, C.c_void_p(out.data_ptr()), 1 if with_features else 0,
                                                       C.c_void_p(stream or 1)), "rptb_buffer_export_shard")

    def reproject_from(self, src: "api.DeviceBuffer", params: Optional["api.Reproject"] = None) -> int:
        """DeviceBuffer.reproject_from into this shard (rptb_buffer_reproject_shard): this rank's pixels take their history
        from `src`, a whole DeviceBuffer on this rank's device -- typically the previous frame's shards gathered with
        features, prev.gather(with_features=True).  Every pixel gets the bits a whole buffer's reprojection gives it,
        HALF included for a shard with halves (whose `src` must have halves too).  Returns this rank's reused pixels;
        summed over the ranks, they are the whole call's."""
        if isinstance(src, ShardBuffer):
            raise TypeError("src is a ShardBuffer: gather() the shards into a whole buffer first")
        c = (params or api.Reproject()).to_c()
        n = C.c_uint64(0)
        capi.check(capi.lib().rptb_buffer_reproject_shard(self.handle, src.handle, C.byref(c), C.byref(n)),
                   "rptb_buffer_reproject_shard")
        self.entries = int(c.max_history)  # the bound a reprojected pixel's count keeps
        return int(n.value)

    def merge_history_from(self, src: "api.DeviceBuffer", reproject: Optional["api.Reproject"] = None,
                           test: Optional["api.HistoryTest"] = None) -> tuple:
        """DeviceBuffer.merge_history_from into this shard (rptb_buffer_reproject_merge_shard): this rank's pixels test
        the history of `src`, a whole DeviceBuffer on this rank's device (the previous frame gathered with features),
        against their own fresh entries.  Every pixel gets the bits a whole buffer's merge gives it, HALF included for a
        shard with halves (whose `src` must have halves too).  Returns this rank's (reused, rejected) pixels; summed over
        the ranks, they are the whole call's."""
        if isinstance(src, ShardBuffer):
            raise TypeError("src is a ShardBuffer: gather() the shards into a whole buffer first")
        c = (reproject or api.Reproject()).to_c()
        gamma = (test or api.HistoryTest()).gamma
        n, j = C.c_uint64(0), C.c_uint64(0)
        capi.check(capi.lib().rptb_buffer_reproject_merge_shard(self.handle, src.handle, C.byref(c), gamma, C.byref(n), C.byref(j)),
                   "rptb_buffer_reproject_merge_shard")
        self.entries += int(c.max_history)  # the fresh calls plus the history's bound
        return int(n.value), int(j.value)

    def _exchange(self, group, nbytes: int, export) -> tuple:
        """What gather and gather_delta share: check the process group against the shard, `export(out, stream)` this
        shard's block into a new CUDA uint8 tensor of `nbytes` on the buffer's device, all-gather every rank's block and
        wait for it.  Returns _all_gather_bytes' (gathered, staged)."""
        import torch

        group = self.group if group is None else group
        rank, world = self.shard
        if world > 1 and _rank_world(group) != (rank, world):
            raise ValueError(f"the shard is {rank} of {world} but the process group has rank/world {_rank_world(group)}")
        dev = torch.device("cuda", self.devices[0])
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            mine = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            export(mine, stream.cuda_stream)
            out = _all_gather_bytes(mine, world, group)
            stream.synchronize()  # the import reads the gathered bytes on the library's stream
        return out

    def gather(self, group=None, with_features: bool = False) -> "api.DeviceBuffer":
        """All ranks call this: export every shard's block, one all_gather_into_tensor, and import the blocks into a new
        whole DeviceBuffer on this rank's device -- the same bits on every rank, and those of one whole buffer given the
        same calls.  NCCL gathers GPU to GPU; any other backend (gloo) through a host tensor.  `with_features` carries
        the feature sums too (denoise and reproject need them), 100 instead of 36 bytes per pixel.  A shard with halves
        carries HALF as well (124 or 60 bytes per pixel) and gives a whole buffer with halves."""
        gathered, _ = self._exchange(group, self.block_bytes(with_features), lambda out, stream: self.export(out, with_features, stream))
        whole = api.DeviceBuffer(self._scene, self.width, self.height, self.filter, halves=self.halves)
        capi.check(capi.lib().rptb_buffer_import_shards(whole.handle, C.c_void_p(gathered.data_ptr()), self.shard[1],
                                                        1 if with_features else 0), "rptb_buffer_import_shards")
        whole.entries = int(whole.counts().max())
        whole.feature_rays = self.feature_rays if with_features else 0
        return whole

    def export_delta(self, out, capacity: int, stream: Optional[int] = None) -> int:
        """Writes this shard's delta block of `capacity` pixels (delta_block_layout(capacity, self.halves);
        rptb_buffer_export_delta) into `out`, a
        CUDA uint8 tensor on the buffer's device, on `stream` (a raw cudaStream_t; the current torch stream when None):
        the pixels this shard's last call changed, which must be an adaptive or guided call made right after an export
        (gather or gather_delta).  Returns their number."""
        import torch

        if stream is None:
            stream = torch.cuda.current_stream(out.device).cuda_stream
        n = C.c_uint32(0)
        capi.check(capi.lib().rptb_buffer_export_delta(self.handle, C.c_void_p(out.data_ptr()), int(capacity), C.c_void_p(stream or 1),
                                                       C.byref(n)), "rptb_buffer_export_delta")
        return int(n.value)

    def gather_delta(self, whole: "api.DeviceBuffer", capacity: int, group=None) -> None:
        """All ranks call this after an adaptive or guided call: export this shard's delta block, one
        all_gather_into_tensor (as gather() does), and apply every rank's block in place to `whole`
        (rptb_buffer_import_deltas) -- this rank's gathered buffer, brought to the shards' state before the call by
        gather(with_features=True) or the previous gather_delta.  Afterwards `whole` is what a new gather would give.
        `capacity`, the same on every rank: at least the largest active count of the call over the ranks."""
        import torch

        world = self.shard[1]
        lay = delta_block_layout(capacity, self.halves)
        gathered, staged = self._exchange(group, lay["bytes"], lambda out, stream: self.export_delta(out, capacity, stream))
        capi.check(capi.lib().rptb_buffer_import_deltas(whole.handle, C.c_void_p(gathered.data_ptr()), world, lay["capacity"]),
                   "rptb_buffer_import_deltas")
        # a delta only raises counts: the largest is the old one or one of the counts the blocks carry
        blocks = (staged if staged is not None else gathered).view(world, lay["bytes"])
        pixels = blocks[:, DELTA_PIXELS_AT:DELTA_PIXELS_AT + 4].contiguous().view(torch.int32)
        counts = blocks[:, lay["counts"]:lay["slots"]].contiguous().view(torch.int32)
        written = torch.arange(lay["capacity"], device=blocks.device).unsqueeze(0) < pixels
        if bool(written.any()):
            whole.entries = max(whole.entries, int(counts[written].max()))


def _count_device(buffer: ShardBuffer, group=None):
    """Where the per-batch active counts are exchanged: on the GPU under NCCL, on the host otherwise."""
    import torch
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and buffer.shard[1] > 1 and dist.get_backend(group) == "nccl":
        return torch.device("cuda", buffer.devices[0])
    return "cpu"


class _GuidedShard:
    """A rank's guided calls on its ShardBuffer and the gathered whole buffer its filter runs over, kept current: one full
    gather with features before the first call that runs the filter, then after every call one gather_delta of that
    call.  Every rank makes the same calls, and so the same collectives."""

    def __init__(self, renderer, shard: ShardBuffer, adaptive: "api.Adaptive", group=None):
        self.renderer, self.shard, self.adaptive, self.group = renderer, shard, adaptive, group
        self.whole: Optional[api.DeviceBuffer] = None
        self.count_dev = _count_device(shard, group)

    def sample(self, samples: int) -> int:
        """One guided call of `samples` samples on every rank, and its delta once the whole buffer exists; returns the
        active pixels summed over the ranks."""
        import torch
        import torch.distributed as dist

        a, s = self.adaptive, self.shard
        if self.whole is None and a.guide.iterations > 0 and s.entries >= a.min_entries:
            self.whole = s.gather(self.group, with_features=True)
        active = self.renderer.sample(samples, s, want_stats=False, adaptive=a, guide_buffer=self.whole)
        counts = [active]
        if s.shard[1] > 1:  # every rank's count: their sum ends a loop, their largest is the delta's capacity
            out = torch.empty(s.shard[1], dtype=torch.int64, device=self.count_dev)
            dist.all_gather_into_tensor(out, torch.tensor([active], dtype=torch.int64, device=self.count_dev), group=self.group)
            counts = out.tolist()
        if self.whole is not None:
            s.gather_delta(self.whole, max(counts), self.group)
        return sum(counts)

    def close(self) -> None:
        if self.whole is not None:
            self.whole.close()
            self.whole = None


def _check_guided_world(adaptive, world: int) -> None:
    """A guided loop on shards keeps a gathered whole buffer on every rank and exchanges the ranks' deltas.  On one rank
    the shard is already the whole image, so that copy and that exchange would only add work to what the whole-buffer
    loop does: refused, before any device work or collective, with the loop to use instead."""
    if adaptive is not None and adaptive.guide is not None and world < 2:
        if adaptive.estimate == "halves":
            raise ValueError('guided adaptive sampling on the error estimate (estimate="halves") on shards needs two or more '
                             "ranks (torch.distributed initialized); one process renders it on one whole buffer with halves: "
                             "Renderer.iterative_render")
        raise ValueError("guided adaptive sampling (Adaptive(guide=...)) on shards needs two or more ranks (torch.distributed "
                         "initialized); one process renders it on one whole buffer: Renderer.iterative_render / render_frames")


def render_iterative_distributed(renderer, callback_interval: int, callback: Callable[[int, ShardBuffer], None],
                                 adaptive: Optional["api.Adaptive"] = None, group=None,
                                 buffer: Optional[ShardBuffer] = None, feature_samples: int = 16) -> ShardBuffer:
    """All ranks call this: Renderer.iterative_render over this rank's ShardBuffer (`buffer`, e.g. one given features
    first; None creates one for the renderer's size and filter).  Every batch renders and adds this rank's tiles only;
    the callback receives the ShardBuffer and calls its gather() when it wants an image, so a batch exchanges nothing
    unless asked.  With `adaptive`, the loop ends after a batch in which no rank rendered a pixel: one all-reduce(sum)
    of the ranks' active counts per batch.  Returns the ShardBuffer.
    A guided criterion (adaptive.guide) mirrors iterative_render: a shard with no features first gets `feature_samples`
    feature rays per pixel; the first batch that runs the filter is preceded by one gather with features, and every
    batch after that by the gather_delta of the batch before, which runs right after it, ahead of the callback.  The
    active counts are all-gathered instead of all-reduced: their sum ends the loop, their largest is the delta's
    capacity.  With one rank, a guided criterion is refused (ValueError): the whole-buffer loop does the same work.
    The error estimate (Adaptive(guide=..., estimate="halves")) needs a shard with halves: None creates one, and a given
    buffer without halves is refused (ValueError) before any device work or collective.  The loop then gives
    iterative_render's bits on one whole buffer with halves."""
    import torch
    import torch.distributed as dist

    _check_guided_world(adaptive, buffer.shard[1] if buffer is not None else _rank_world(group)[1])
    halves = adaptive is not None and adaptive.estimate == "halves"
    if halves and buffer is not None and not buffer.halves:
        raise ValueError('estimate="halves" needs a shard buffer with halves: ShardBuffer(..., halves=True), or buffer=None')
    if buffer is None:
        buffer = ShardBuffer(renderer.device_scene(), renderer._width, renderer._height, renderer._filter, group=group,
                             halves=halves)
    if adaptive is not None and adaptive.guide is not None:
        if buffer.feature_rays == 0:
            renderer.sample_features(feature_samples, buffer)
        guided = _GuidedShard(renderer, buffer, adaptive, group)
        try:
            iteration = 0
            while iteration < renderer._num_samples:
                steps = min(renderer._num_samples - iteration, callback_interval)
                iteration += steps
                if guided.sample(steps) == 0:
                    break
                callback(iteration, buffer)
        finally:
            guided.close()
        return buffer
    on = dist.is_available() and dist.is_initialized() and buffer.shard[1] > 1
    count_dev = _count_device(buffer, group)
    iteration = 0
    while iteration < renderer._num_samples:
        steps = min(renderer._num_samples - iteration, callback_interval)
        active = renderer.sample(steps, buffer, want_stats=False, adaptive=adaptive)
        iteration += steps
        if adaptive is not None:
            if on:
                total = torch.tensor([active], dtype=torch.int64, device=count_dev)
                dist.all_reduce(total, op=dist.ReduceOp.SUM, group=group)
                active = int(total.item())
            if active == 0:
                break
        callback(iteration, buffer)
    return buffer


def render_frames_distributed(renderer, cameras, entries: int = 8, feature_samples: int = 16,
                              reproject: Optional["api.Reproject"] = api.Reproject(), adaptive: Optional["api.Adaptive"] = None,
                              denoise: Optional["api.Denoise"] = None, group=None,
                              history_test: Optional["api.HistoryTest"] = None):
    """All ranks call this: Renderer.render_frames over one ShardBuffer per frame, yielding each frame's (height, width,
    3) uint8 on every rank -- the bytes of render_frames on one whole buffer, for any world size.  Per frame: this
    rank's shard gets `feature_samples` feature rays through the frame's camera, the previous frame's gathered buffer is
    reprojected into it (unless `reproject` is None), and `entries` plain or adaptive entries are added, continuing
    the renderer's sample streams; then one gather (with features when `reproject` or `denoise` needs them) makes the
    whole buffer the frame's image() or denoised_image(denoise) comes from, and which the next frame reprojects.  That
    gather is the frame's only all-gather of full blocks.  `history_test` as in render_frames: each rank tests its own
    pixels.
    A guided criterion (adaptive.guide): the frame's guided entries run as in render_iterative_distributed, with one
    gather with features before the first that runs the filter and a gather_delta after each.  The whole buffer they keep
    current is the frame's image and the next frame's source, so a frame still makes one full gather (at its end, as
    without guidance, when no entry ran the filter).  With one rank, a guided criterion is refused (ValueError), as in
    render_iterative_distributed.  The error estimate (estimate="halves") is refused (ValueError), as render_frames
    refuses it: the loop makes no shards with halves yet (ShardBuffer.reproject_from and merge_history_from take them)."""
    _check_guided_world(adaptive, _rank_world(group)[1])
    renderer._check_frames(entries, adaptive, denoise, reproject, history_test)
    with_features = reproject is not None or denoise is not None
    own, prev = renderer.camera, None
    try:
        for cam in cameras:
            renderer.camera = cam
            buf = ShardBuffer(renderer.device_scene(), renderer._width, renderer._height, renderer._filter, group=group)
            guided = _GuidedShard(renderer, buf, adaptive, group) if adaptive is not None and adaptive.guide is not None else None
            try:
                renderer.sample_features(feature_samples, buf)
                renderer._frame_entries(buf, prev, entries, reproject, adaptive, history_test,
                                        None if guided is None else guided.sample)
                if guided is not None and guided.whole is not None:
                    whole, guided.whole = guided.whole, None
                else:
                    whole = buf.gather(group, with_features)
            finally:
                if guided is not None:
                    guided.close()
                buf.close()
            img = whole.image() if denoise is None else whole.denoised_image(denoise)
            if prev is not None:
                prev.close()
            prev = whole
            yield img
    finally:
        renderer.camera = own
        if prev is not None:
            prev.close()
