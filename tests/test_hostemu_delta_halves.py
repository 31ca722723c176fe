"""The halves delta block's per-element export and import (delta.h) in host emulation, against numpy and against the
plain block: HALF arrives with its bits on the pixel of its slot, bytes [0, 256 + 40 m) of a halves block are those of
the plain block made from the same state, and the import writes the plain import's sums, M2 and counts -- for the sizes
and shard counts of test_shard_block_layout.py, tile-less shards included.  No device."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.hostemu import emu
from tests.test_hostemu_delta import _emu as _plain_emu
from tests.test_hostemu_delta import _rand_state, _slot_pixels
from tests.test_shard_block_layout import SIZES

from rpt_b200 import _capi as capi
from rpt_b200.distributed import delta_block_layout, shard_tiles

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dp, u32p = capi.c_double_p, capi.c_u32_p
_lib = None


def _emu():
    """tests/hostemu/_build/libhostemu_delta_halves.so: delta.h's halves functions compiled for the host."""
    global _lib
    if _lib is not None:
        return _lib
    emu.lib()  # `make hostemu` builds every emulation library
    L = C.CDLL(os.path.join(ROOT, "tests", "hostemu", "_build", "libhostemu_delta_halves.so"))
    L.hostemu_delta_halves_bytes.restype = C.c_uint64
    L.hostemu_delta_halves_bytes.argtypes = [C.c_uint32]
    L.hostemu_delta_halves_export.restype = None
    L.hostemu_delta_halves_export.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, dp, dp, u32p, dp]
    L.hostemu_delta_halves_import.restype = None
    L.hostemu_delta_halves_import.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, dp, dp, u32p, dp]
    _lib = L
    return L


def _ptr(a, t):
    return a.ctypes.data_as(t)


@pytest.mark.parametrize("w,h,n", SIZES)
def test_halves_delta_carries_half_and_keeps_the_plain_prefix(w, h, n):
    rng = np.random.default_rng(w * 7919 + h * 31 + n)
    L, P = _emu(), _plain_emu()
    npix = w * h
    whole_pix = _slot_pixels(w, h, 0, 1)
    old = _rand_state(rng, whole_pix.size)
    old_half = rng.standard_normal((whole_pix.size, 3)) * 10.0 ** rng.integers(-300, 300, (whole_pix.size, 1))
    new = _rand_state(rng, npix)
    new_half = rng.standard_normal((npix, 3)) * 10.0 ** rng.integers(-300, 300, (npix, 1))
    changed, lists = np.zeros(npix, bool), []
    for s in range(n):
        pix = _slot_pixels(w, h, s, n)
        valid = np.flatnonzero(pix >= 0)
        pick = np.sort(rng.choice(valid, size=rng.integers(0, valid.size + 1), replace=False)) if valid.size else valid
        lists.append((pix, pick.astype(np.uint32)))
        changed[pix[pick]] = True
    m = max([p.size for _, p in lists] + [0]) + 3  # spare capacity: its slots stay unwritten
    lay, plain = delta_block_layout(m, halves=True), delta_block_layout(m)
    assert L.hostemu_delta_halves_bytes(m) == lay["bytes"] == capi.lib().rptb_delta_bytes_halves(m)
    gathered = np.full(lay["bytes"] * n, 0xEE, np.uint8)
    gathered_plain = np.full(plain["bytes"] * n, 0xEE, np.uint8)
    assert sum(shard_tiles(w, h, s, n) for s in range(n)) * 128 >= npix
    for s, (pix, pick) in enumerate(lists):
        blk = gathered[s * lay["bytes"]:(s + 1) * lay["bytes"]]
        pblk = gathered_plain[s * plain["bytes"]:(s + 1) * plain["bytes"]]
        for b, lo in ((blk, lay), (pblk, plain)):
            b[:256] = 0  # the same header bytes in both
            b[lo["slots"]:lo["slots"] + 4 * pick.size] = pick.view(np.uint8)
        ok = pix >= 0
        ps = np.ascontiguousarray(np.where(ok[:, None], new[0][np.maximum(pix, 0)], np.nan))
        pm = np.ascontiguousarray(np.where(ok, new[1][np.maximum(pix, 0)], np.nan))
        pc = np.where(ok, new[2][np.maximum(pix, 0)], 0xDEAD).astype(np.uint32)
        ph = np.ascontiguousarray(np.where(ok[:, None], new_half[np.maximum(pix, 0)], np.nan))
        L.hostemu_delta_halves_export(blk.ctypes.data_as(C.c_void_p), m, pick.size, _ptr(ps, dp), _ptr(pm, dp), _ptr(pc, u32p),
                                      _ptr(ph, dp))
        P.hostemu_delta_export(pblk.ctypes.data_as(C.c_void_p), m, pick.size, _ptr(ps, dp), _ptr(pm, dp), _ptr(pc, u32p))
        # the prefix is the plain block's, byte for byte (unwritten slots included)
        assert blk[:lay["half"]].tobytes() == pblk.tobytes()
        # HALF: the listed slots' bits, then nothing
        got = blk[lay["half"]:].view(np.float64).reshape(m, 3)
        assert got[:pick.size].tobytes() == new_half[pix[pick]].tobytes()
        assert np.all(blk[lay["half"] + 24 * pick.size:] == 0xEE)
    arrays = [np.ascontiguousarray(a.copy()) for a in old]
    plain_arrays = [np.ascontiguousarray(a.copy()) for a in old]
    half = np.ascontiguousarray(old_half.copy())
    L.hostemu_delta_halves_import(gathered.ctypes.data_as(C.c_void_p), n, m, _ptr(arrays[0], dp), _ptr(arrays[1], dp),
                                  _ptr(arrays[2], u32p), _ptr(half, dp))
    P.hostemu_delta_import(gathered_plain.ctypes.data_as(C.c_void_p), n, m, _ptr(plain_arrays[0], dp), _ptr(plain_arrays[1], dp),
                           _ptr(plain_arrays[2], u32p))
    for a, b in zip(arrays, plain_arrays):
        assert a.tobytes() == b.tobytes()  # sums, M2 and counts as the plain import writes them
    hit = (whole_pix >= 0) & changed[np.maximum(whole_pix, 0)]
    want_half = np.where(hit[:, None], new_half[np.maximum(whole_pix, 0)], old_half)
    assert half.tobytes() == want_half.tobytes()
    want_sums = np.where(hit[:, None], new[0][np.maximum(whole_pix, 0)], old[0])
    assert arrays[0].tobytes() == want_sums.tobytes()
