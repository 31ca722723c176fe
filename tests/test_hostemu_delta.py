"""The delta exchange's per-element export and import (delta.h) in host emulation, against numpy: random changed pixels of
every shard are exported into delta blocks and the blocks, concatenated as an all-gather gives them, are scattered into
a one-part whole buffer's compact planes.  Every shard slot must land on the pixel gather_permutation and rptb_tile_pixel
give it, carry its bits, and nothing else may change -- for the sizes and shard counts of test_shard_block_layout.py,
tile-less shards included.  No device."""
import ctypes as C
import os

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200.distributed import DELTA_PIXELS_AT, delta_block_layout, gather_permutation, shard_tiles
from tests.hostemu import emu
from tests.test_shard_block_layout import SIZES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dp, u32p = capi.c_double_p, capi.c_u32_p
_lib = None


def _emu():
    """tests/hostemu/_build/libhostemu_delta.so: delta.h compiled for the host."""
    global _lib
    if _lib is not None:
        return _lib
    emu.lib()  # `make hostemu` builds every emulation library
    L = C.CDLL(os.path.join(ROOT, "tests", "hostemu", "_build", "libhostemu_delta.so"))
    L.hostemu_delta_bytes.restype = C.c_uint64
    L.hostemu_delta_bytes.argtypes = [C.c_uint32]
    L.hostemu_delta_export.restype = None
    L.hostemu_delta_export.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, dp, dp, u32p]
    L.hostemu_delta_import.restype = None
    L.hostemu_delta_import.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, dp, dp, u32p]
    L.hostemu_delta_whole_slots.restype = None
    L.hostemu_delta_whole_slots.argtypes = [C.c_uint32, C.c_uint32, u32p, C.c_uint64, C.POINTER(C.c_uint64)]
    _lib = L
    return L


def _slot_pixels(w, h, s, n):
    """Pixel of every compact slot of shard (s, n), -1 past a ragged edge (rptb_tile_pixel)."""
    lib = capi.lib()
    return np.array([lib.rptb_tile_pixel(w, h, s, n, e // 128, e % 128) for e in range(shard_tiles(w, h, s, n) * 128)], np.int64)


def _rand_state(rng, npix):
    sums = rng.standard_normal((npix, 3)) * 10.0 ** rng.integers(-300, 300, (npix, 1))
    return sums, rng.random(npix) * 1e3, rng.integers(0, 2**32, npix, dtype=np.uint64).astype(np.uint32)


@pytest.mark.parametrize("w,h,n", SIZES)
def test_delta_scatter_puts_every_slot_on_its_pixel(w, h, n):
    rng = np.random.default_rng(w * 1000 + h * 10 + n)
    L = _emu()
    npix = w * h
    whole_pix = _slot_pixels(w, h, 0, 1)  # compact slot of a one-part whole buffer -> pixel
    assert np.array_equal(gather_permutation(w, h, 1)[whole_pix[whole_pix >= 0]], np.flatnonzero(whole_pix >= 0))
    old = _rand_state(rng, whole_pix.size)  # the whole buffer's compact planes before
    new = _rand_state(rng, npix)            # the shards' state of every pixel after, row-major
    changed, lists = np.zeros(npix, bool), []
    for s in range(n):  # each shard changes a random subset of its own pixels, listed by ascending slot
        pix = _slot_pixels(w, h, s, n)
        valid = np.flatnonzero(pix >= 0)
        pick = np.sort(rng.choice(valid, size=rng.integers(0, valid.size + 1), replace=False)) if valid.size else valid
        lists.append((pix, pick.astype(np.uint32)))
        changed[pix[pick]] = True
    m = max([p.size for _, p in lists] + [0]) + 3  # spare capacity: its slots stay unwritten
    lay = delta_block_layout(m)
    assert L.hostemu_delta_bytes(m) == lay["bytes"]
    gathered = np.full(lay["bytes"] * n, 0xEE, np.uint8)
    perm = gather_permutation(w, h, n)
    slots0 = shard_tiles(w, h, 0, n) * 128
    for s, (pix, pick) in enumerate(lists):
        blk = gathered[s * lay["bytes"]:(s + 1) * lay["bytes"]]
        blk[lay["slots"]:lay["slots"] + 4 * pick.size] = pick.view(np.uint8)
        # the shard's compact planes: its pixels' new state, garbage in the ragged slots
        ps = np.where((pix >= 0)[:, None], new[0][np.maximum(pix, 0)], np.nan)
        pm = np.where(pix >= 0, new[1][np.maximum(pix, 0)], np.nan)
        pc = np.where(pix >= 0, new[2][np.maximum(pix, 0)], 0xDEAD).astype(np.uint32)
        ps, pm = np.ascontiguousarray(ps), np.ascontiguousarray(pm)
        L.hostemu_delta_export(blk.ctypes.data_as(C.c_void_p), m, pick.size, ps.ctypes.data_as(dp), pm.ctypes.data_as(dp),
                               pc.ctypes.data_as(u32p))
        assert blk[DELTA_PIXELS_AT:DELTA_PIXELS_AT + 4].view(np.uint32)[0] == pick.size
        # what the block carries, element by element, in numpy
        got_sums = blk[lay["sums"]:lay["m2"]].view(np.float64).reshape(m, 3)[:pick.size]
        assert got_sums.tobytes() == new[0][pix[pick]].tobytes()
        assert blk[lay["counts"]:lay["slots"]].view(np.uint32)[:pick.size].tobytes() == new[2][pix[pick]].tobytes()
        assert np.all(blk[lay["m2"] + 8 * pick.size:lay["counts"]] == 0xEE)  # slots past n are not written
        # the shard slot's pixel is where gather_permutation puts it, and the whole slot delta.h names holds that pixel
        assert np.array_equal(perm[pix[pick]], s * slots0 + pick.astype(np.int64))
        ws = np.empty(pick.size, np.uint64)
        L.hostemu_delta_whole_slots(s, n, pick.ctypes.data_as(u32p), pick.size, ws.ctypes.data_as(C.POINTER(C.c_uint64)))
        assert np.array_equal(whole_pix[ws.astype(np.int64)], pix[pick])
    sums, m2, counts = (np.ascontiguousarray(a.copy()) for a in old)
    L.hostemu_delta_import(gathered.ctypes.data_as(C.c_void_p), n, m, sums.ctypes.data_as(dp), m2.ctypes.data_as(dp),
                           counts.ctypes.data_as(u32p))
    # numpy: the changed pixels' slots take the new state bit for bit, every other slot keeps the old bits
    hit = (whole_pix >= 0) & changed[np.maximum(whole_pix, 0)]
    want_sums = np.where(hit[:, None], new[0][np.maximum(whole_pix, 0)], old[0])
    want_m2 = np.where(hit, new[1][np.maximum(whole_pix, 0)], old[1])
    want_counts = np.where(hit, new[2][np.maximum(whole_pix, 0)], old[2])
    assert sums.tobytes() == want_sums.tobytes()
    assert m2.tobytes() == want_m2.tobytes()
    assert counts.tobytes() == want_counts.astype(np.uint32).tobytes()
