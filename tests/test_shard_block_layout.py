"""The exchange block of a shard buffer (distributed.shard_block_layout) on the host: every shard's planes are padded to
shard 0's slots, slot k * 128 + j of shard s is pixel rptb_tile_pixel(w, h, s, n, k, j), and the concatenation of the
blocks -- what the all-gather gives -- puts every pixel in exactly one slot, where gather_permutation says.  No
device: rptb_tile_pixel is host code."""
import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200.distributed import SHARD_HEADER_BYTES, gather_permutation, shard_block_layout, shard_tiles

SIZES = [(50, 27, 3), (33, 9, 2), (16, 8, 1), (20, 10, 8), (97, 61, 5), (128, 96, 8)]


@pytest.mark.parametrize("w,h,n", SIZES)
@pytest.mark.parametrize("with_features", [False, True])
def test_block_layout(w, h, n, with_features):
    lay = shard_block_layout(w, h, n, with_features)
    slots = lay["slots"]
    assert slots == max(shard_tiles(w, h, s, n) for s in range(n)) * 128 == shard_tiles(w, h, 0, n) * 128
    assert lay["sums"] == SHARD_HEADER_BYTES and SHARD_HEADER_BYTES % 256 == 0
    assert lay["m2"] == lay["sums"] + 24 * slots
    assert lay["features"] == lay["m2"] + 8 * slots
    assert lay["counts"] == lay["features"] + (64 * slots if with_features else 0)
    assert lay["bytes"] == SHARD_HEADER_BYTES + (100 if with_features else 36) * slots
    for k in ("sums", "m2", "features", "counts", "bytes"):
        assert lay[k] % 8 == 0  # every plane starts aligned for its doubles, and so does the next block


@pytest.mark.parametrize("w,h,n", SIZES)
def test_blocks_hold_every_pixel_once(w, h, n):
    """Blocks packed by the tile deal (as rptb_buffer_export_shard writes them) and read back through
    gather_permutation give every pixel its own values; the padding slots hold nothing of the image."""
    lib = capi.lib()
    lay = shard_block_layout(w, h, n, True)
    slots, nb = lay["slots"], lay["bytes"]
    gathered = np.full(nb * n, 0xEE, np.uint8)  # unwritten bytes
    owner = np.full((n, slots), -1, np.int64)
    for s in range(n):
        blk = gathered[s * nb:(s + 1) * nb]
        sums = blk[lay["sums"]:lay["m2"]].view(np.float64).reshape(slots, 3)
        m2 = blk[lay["m2"]:lay["features"]].view(np.float64)
        feat = blk[lay["features"]:lay["counts"]].view(np.float64)
        counts = blk[lay["counts"]:].view(np.uint32)
        mine = shard_tiles(w, h, s, n) * 128
        for e in range(mine):
            p = lib.rptb_tile_pixel(w, h, s, n, e // 128, e % 128)
            owner[s, e] = p
            if p < 0:
                continue
            sums[e] = (p, p + 0.25, p + 0.5)
            m2[e] = -p
            feat[6 * slots + e] = 1000 + p  # the hits plane, after the normal and albedo planes (3 a slot each)
            counts[e] = p + 7
    seen = owner[owner >= 0]
    assert np.array_equal(np.sort(seen), np.arange(w * h))  # every pixel in exactly one slot of one shard

    perm = gather_permutation(w, h, n)  # pixel -> (shard, slot) = divmod(perm, slots)
    shard, slot = np.divmod(perm, slots)
    for p in range(w * h):
        assert owner[shard[p], slot[p]] == p
    base = shard * nb
    got_sums = np.stack([gathered[b + lay["sums"] + 24 * e:b + lay["sums"] + 24 * e + 24].view(np.float64)
                         for b, e in zip(base, slot)])
    got_counts = np.array([gathered[b + lay["counts"] + 4 * e:b + lay["counts"] + 4 * e + 4].view(np.uint32)[0]
                           for b, e in zip(base, slot)])
    got_hits = np.array([gathered[b + lay["features"] + 8 * (6 * slots + e):b + lay["features"] + 8 * (6 * slots + e) + 8]
                         .view(np.float64)[0] for b, e in zip(base, slot)])
    px = np.arange(w * h, dtype=np.float64)
    assert np.array_equal(got_sums, np.stack([px, px + 0.25, px + 0.5], axis=1))
    assert np.array_equal(got_counts, np.arange(w * h) + 7)
    assert np.array_equal(got_hits, 1000 + px)


def test_exchange_sizes_at_1080p():
    """36 bytes a pixel, 100 with features: about 75 and 207 MB at 1920x1080 for one shard (world 1)."""
    assert shard_block_layout(1920, 1080, 1)["bytes"] == 256 + 36 * 1920 * 1080 == 74_649_856
    assert shard_block_layout(1920, 1080, 1, True)["bytes"] == 256 + 100 * 1920 * 1080 == 207_360_256
