"""The delta exchange block of a shard buffer (distributed.delta_block_layout) on the host: its size is
rptb_delta_bytes', every plane and the next block start 8-byte aligned, and the header's pixel count sits where
DELTA_PIXELS_AT says.  No device: rptb_delta_bytes is host code."""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200.distributed import DELTA_HEADER_BYTES, DELTA_PIXELS_AT, delta_block_layout
from tests.test_hostemu_delta import _emu


@pytest.mark.parametrize("m", [0, 1, 2, 3, 7, 128, 1000, 480_000, 2_073_600])
def test_delta_layout_is_the_library_size(m):
    lay = delta_block_layout(m)
    assert lay["bytes"] == capi.lib().rptb_delta_bytes(m) == 256 + 40 * m
    assert lay["sums"] == DELTA_HEADER_BYTES == 256
    assert lay["m2"] == lay["sums"] + 24 * m
    assert lay["counts"] == lay["m2"] + 8 * m
    assert lay["slots"] == lay["counts"] + 4 * m
    assert lay["bytes"] == lay["slots"] + 4 * m
    for k in ("sums", "m2", "bytes"):
        assert lay[k] % 8 == 0  # the doubles are aligned, and so is the next block of an all-gather
    for k in ("counts", "slots"):
        assert lay[k] % 4 == 0


def test_header_pixel_count_offset():
    """hostemu_delta_export writes the header's pixel count (and capacity) where the Python side reads it."""
    m = 5
    blk = np.zeros(delta_block_layout(m)["bytes"], np.uint8)  # slot list all 0: every pixel copies slot 0
    _emu().hostemu_delta_export(blk.ctypes.data_as(C.c_void_p), m, 3, np.arange(15.0).ctypes.data_as(capi.c_double_p),
                                np.arange(5.0).ctypes.data_as(capi.c_double_p), np.arange(5, dtype=np.uint32).ctypes.data_as(capi.c_u32_p))
    hdr = blk[:DELTA_HEADER_BYTES]
    assert hdr[DELTA_PIXELS_AT:DELTA_PIXELS_AT + 8].view(np.uint32).tolist() == [3, m]
    assert _emu().hostemu_delta_bytes(m) == delta_block_layout(m)["bytes"]
