"""The exchange blocks of a shard buffer with halves on the host: the delta block's size is rptb_delta_bytes_halves',
256 + 64 m, with the plain block's prefix and HALF after the slots; the full block adds HALF's 24 bytes a slot after
counts; the C ABI binds the new entry points as the header declares them; and the Python loops refuse what they cannot
do before any device work.  No device."""
import ctypes as C
import os
import re
import types

import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, distributed, scenes
from rpt_b200.distributed import DELTA_HEADER_BYTES, delta_block_layout, shard_block_layout
from tests.test_shard_block_layout import SIZES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPACITIES = [0, 1, 2, 3, 7, 128, 1000, 480_000, 2_073_600]  # those of test_delta_block_layout.py


@pytest.mark.parametrize("m", CAPACITIES)
def test_delta_halves_layout_is_the_library_size(m):
    lay, plain = delta_block_layout(m, halves=True), delta_block_layout(m)
    assert lay["bytes"] == capi.lib().rptb_delta_bytes_halves(m) == 256 + 64 * m
    assert {k: v for k, v in lay.items() if k not in ("half", "bytes")} == {k: v for k, v in plain.items() if k != "bytes"}
    assert lay["sums"] == DELTA_HEADER_BYTES
    assert lay["half"] == plain["bytes"] == 256 + 40 * m
    assert lay["bytes"] == lay["half"] + 24 * m
    for k in ("sums", "m2", "half", "bytes"):
        assert lay[k] % 8 == 0  # the doubles are aligned, and so is the next block of an all-gather
    for k in ("counts", "slots"):
        assert lay[k] % 4 == 0
    assert delta_block_layout(m, halves=False) == plain and "half" not in plain


@pytest.mark.parametrize("w,h,n", SIZES)
@pytest.mark.parametrize("with_features", [False, True])
def test_shard_halves_layout(w, h, n, with_features):
    lay, plain = shard_block_layout(w, h, n, with_features, halves=True), shard_block_layout(w, h, n, with_features)
    slots = lay["slots"]
    assert slots % 128 == 0
    assert {k: v for k, v in lay.items() if k not in ("half", "bytes")} == {k: v for k, v in plain.items() if k != "bytes"}
    assert lay["half"] == plain["bytes"] == lay["counts"] + 4 * slots
    assert lay["bytes"] == lay["half"] + 24 * slots == 256 + (124 if with_features else 60) * slots
    assert lay["half"] % 8 == 0 and lay["bytes"] % 8 == 0
    assert shard_block_layout(w, h, n, with_features, halves=False) == plain and "half" not in plain


def test_exchange_sizes_at_1080p():
    """60 bytes a pixel, 124 with features, for one shard of 1920x1080 (world 1), and a delta of every pixel."""
    assert shard_block_layout(1920, 1080, 1, halves=True)["bytes"] == 256 + 60 * 1920 * 1080
    assert shard_block_layout(1920, 1080, 1, True, halves=True)["bytes"] == 256 + 124 * 1920 * 1080
    assert delta_block_layout(1920 * 1080, halves=True)["bytes"] == 256 + 64 * 1920 * 1080


def test_abi_signatures_match_header():
    text = open(os.path.join(ROOT, "include", "rpt_b200.h")).read()
    flat = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", text, flags=re.S))
    assert ("int rptb_buffer_create_shard_halves(rptb_scene* scene, uint32_t width, uint32_t height, uint32_t box_radius, "
            "uint32_t shard_index, uint32_t shard_count, rptb_buffer** out);") in flat
    assert "uint64_t rptb_delta_bytes_halves(uint32_t capacity);" in flat
    m = re.search(r"int rptb_sample_into_guided_error_shard\(([^;]*)\);", flat)
    g = re.search(r"int rptb_sample_into_guided_shard\(([^;]*)\);", flat)
    assert m and g and m.group(1) == g.group(1)
    syms = {name: (res, args) for name, res, args in capi.SYMBOLS}
    assert syms["rptb_buffer_create_shard_halves"] == syms["rptb_buffer_create_shard"]
    assert syms["rptb_delta_bytes_halves"] == syms["rptb_delta_bytes"]
    assert syms["rptb_sample_into_guided_error_shard"] == syms["rptb_sample_into_guided_shard"]
    for name in ("rptb_buffer_create_shard_halves", "rptb_delta_bytes_halves", "rptb_sample_into_guided_error_shard"):
        assert hasattr(capi.lib(), name)


def test_abi_refusals_before_any_device_work():
    L = capi.lib()
    fake = C.c_void_p(1)  # never looked at: the arguments are refused first
    out = C.c_void_p()
    assert L.rptb_buffer_create_shard_halves(None, 8, 8, 0, 0, 2, C.byref(out)) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_create_shard_halves(fake, 0, 8, 0, 0, 2, C.byref(out)) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_create_shard_halves(fake, 8, 8, 0, 0, 2, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_create_shard_halves(fake, 8, 8, 0, 2, 2, C.byref(out)) == capi.ERR_BAD_ARG
    assert b"shard_index" in L.rptb_last_error()
    cam, p = capi.Camera(), capi.RenderParams()
    p.width, p.height, p.iterations, p.shard_count = 8, 8, 1, 2
    good_c, good_d = api.Adaptive().to_c(), api.Denoise().to_c()

    def call(crit, guide):
        return L.rptb_sample_into_guided_error_shard(fake, C.byref(cam), C.byref(p), crit, guide, fake, fake, None, None)

    assert call(C.byref(capi.Adaptive(0.02, 1e-3, 1, 0)), C.byref(good_d)) == capi.ERR_BAD_ARG
    assert call(None, C.byref(good_d)) == capi.ERR_BAD_ARG
    assert call(C.byref(good_c), None) == capi.ERR_BAD_ARG
    assert call(C.byref(good_c), C.byref(capi.Denoise(13, 128, 1.0, 4.0, 1e-3))) == capi.ERR_BAD_ARG
    assert call(C.byref(good_c), C.byref(capi.Denoise(0, 128, 1.0, 4.0, 1e-3))) == capi.ERR_BAD_ARG
    assert b"iterations" in L.rptb_last_error()


HALVES = api.Adaptive(guide=api.Denoise(), estimate="halves")


def _renderer():
    cfg = scenes.sphere_scene()
    return api.Renderer(cfg.scene, cfg.camera).width(8).height(8).num_samples(4)


def test_iterative_loop_refusals_before_device_work():
    r = _renderer()
    with pytest.raises(ValueError, match="halves"):  # one rank: the whole-buffer loop does it
        distributed.render_iterative_distributed(r, 1, lambda i, b: None, adaptive=HALVES)
    plain = types.SimpleNamespace(shard=(0, 2), halves=False, feature_rays=0)  # stands for a ShardBuffer without halves
    with pytest.raises(ValueError, match="halves"):
        distributed.render_iterative_distributed(r, 1, lambda i, b: None, adaptive=HALVES, buffer=plain)
    assert r._dev_scene is None  # nothing reached the device


def test_frame_loop_refuses_halves_on_any_world(monkeypatch):
    r = _renderer()
    monkeypatch.setattr(distributed, "_rank_world", lambda group=None: (0, 2))
    with pytest.raises(ValueError, match="halves"):
        next(distributed.render_frames_distributed(r, [r.camera], entries=2, adaptive=HALVES))
    assert r._dev_scene is None
