"""The slim lane of the packed-table kernels without counters, on the CPU.

A render given no counters of a packed-table scene (Cornell, the sphere) runs an F_NOCOUNT twin (test_render_budget.py).
Those twins keep less state per lane (integrator.cuh, slim_lane): status / dead / depth share one word, and the run of
samples is two words.  Here:
- ptxas's report holds the four twins to the register cap of RPTB_MIN_BLOCKS_FLAT and to the spill stores they have now;
- the host emulation of the twins (tests/hostemu/hostemu_slim.cu) gives the counting variant's image bit for bit, with
  one chunk, several chunks, several sample groups and shards."""
import ctypes as C
import os

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests.hostemu import emu
from tests.test_render_budget import F_FLAT, F_NOCOUNT, F_SMALL, min_blocks, ptxas_report

SLIM_LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu", "_build", "libhostemu_slim.so")

# spill stores (bytes) ptxas reports for the slim twins (sm_90a, CUDA 12.9): (FEAT, list schedule) -> bytes
SLIM_SPILL_STORES = {
    (F_FLAT | F_NOCOUNT, False): 332, (F_FLAT | F_SMALL | F_NOCOUNT, False): 308,
    (F_FLAT | F_NOCOUNT, True): 344, (F_FLAT | F_SMALL | F_NOCOUNT, True): 320,
}

_lib = None


def slim_lib():
    global _lib
    if _lib is None:
        emu.lib()  # `make hostemu` builds every emulation library
        L = C.CDLL(SLIM_LIB)
        dp = C.POINTER(C.c_double)
        L.hostemu_render_silent.argtypes = [C.c_void_p, C.POINTER(capi.Camera), C.POINTER(capi.RenderParams), dp]
        _lib = L
    return _lib


@pytest.mark.parametrize("key", sorted(SLIM_SPILL_STORES))
def test_slim_twins_keep_their_budget(key):
    rep = ptxas_report()
    assert key in rep, sorted(rep)
    regs, stores, _ = rep[key]
    assert regs <= 65536 // (128 * min_blocks("RPTB_MIN_BLOCKS_FLAT")), (key, regs)
    assert stores <= SLIM_SPILL_STORES[key], (key, stores)


def silent_and_counting(cfg, w, h, spp, mb, **kw):
    flat = api.FlatScene(cfg.scene)
    s = emu.EmuScene(flat)
    try:
        p = api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).seed(3).params(spp, **kw)
        counting, _, fc = s.render(cfg.camera, p)
        silent = np.empty_like(counting)
        cam = cfg.camera.to_c() if hasattr(cfg.camera, "to_c") else cfg.camera
        fs = slim_lib().hostemu_render_silent(s.handle, C.byref(cam), C.byref(p), silent.ctypes.data_as(C.POINTER(C.c_double)))
    finally:
        s.close()
    assert fc & F_FLAT and not fc & F_NOCOUNT
    assert fs == fc | F_NOCOUNT, (fs, fc)
    return silent, counting


@pytest.mark.parametrize("name,w,h,spp,mb", [("cornell", 20, 12, 40, 6), ("cornell", 20, 12, 150, 3), ("sphere", 24, 16, 70, 6),
                                             ("cornell", 17, 9, 300, 64)])
def test_silent_render_is_the_counting_render(name, w, h, spp, mb):
    """one chunk (40 spp); 3 chunks of 64 (150, 70); 5 chunks of 64 over ragged tiles, at max_bounces 64 (depth's
    largest value in the packed word)"""
    silent, counting = silent_and_counting(scenes.CONFIGS[name](), w, h, spp, mb)
    assert np.isfinite(silent).all()
    np.testing.assert_array_equal(silent, counting)


@pytest.mark.parametrize("groups", [2, 3, 5])
def test_silent_render_is_the_counting_render_in_sample_groups(monkeypatch, groups):
    """several sample groups per tile (RPTB_GROUPS): a lane's run of samples ends at a group's end, not the image's"""
    monkeypatch.setenv("RPTB_GROUPS", str(groups))
    silent, counting = silent_and_counting(scenes.cornell_scene(), 20, 12, 330, 4)
    np.testing.assert_array_equal(silent, counting)


def test_silent_render_with_shards_and_a_first_sample():
    cfg = scenes.cornell_scene()
    for i in range(3):
        silent, counting = silent_and_counting(cfg, 20, 12, 150, 3, first_sample=2**32 - 70, shard_index=i, shard_count=3)
        np.testing.assert_array_equal(silent, counting)
