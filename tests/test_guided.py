"""Adaptive sampling guided by the denoiser without a GPU: the criterion's per-pixel and per-slot functions (guided.h) in
host emulation, after the emulated filter, against their numpy restatement (tests/guided_ref.py) on random and edge-case
states -- counts 0, 1, 2, ..., NaN and inf sums, zero variance, inf depth, zero normals, ragged tiles and every part of
1 and of 4; api.Adaptive(guide=...)'s arguments; the C library's refusals before any device work; and the refusals of
the distributed loops before any collective."""
import ctypes as C
import os

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, distributed, scenes
from tests import guided_ref as gref
from tests.hostemu import emu
from tests.test_denoise import random_state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dp, u8p, u32p = capi.c_double_p, capi.c_u8_p, capi.c_u32_p
_lib = None


def _emu():
    """tests/hostemu/_build/libhostemu_guided.so: the denoiser's emulation plus guided.h."""
    global _lib
    if _lib is not None:
        return _lib
    emu.lib()  # `make hostemu` builds every emulation library
    L = C.CDLL(os.path.join(ROOT, "tests", "hostemu", "_build", "libhostemu_guided.so"))
    L.hostemu_demodulate.restype = None
    L.hostemu_demodulate.argtypes = [dp, dp, u32p, C.c_uint64, dp, C.c_double, dp, dp]
    L.hostemu_denoise_pass.restype = None
    L.hostemu_denoise_pass.argtypes = [dp, dp, dp, dp, dp, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(capi.Denoise), dp, dp]
    L.hostemu_guided_pixels.restype = None
    L.hostemu_guided_pixels.argtypes = [u32p, dp, dp, dp, C.c_uint64, C.c_double, C.POINTER(capi.Adaptive), u8p]
    L.hostemu_guided_part.restype = C.c_uint64
    L.hostemu_guided_part.argtypes = [dp, dp, dp, u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double,
                                      C.POINTER(capi.Adaptive), u8p, u8p]
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(dp)


def emu_passes(sums, m2, counts, nrm, z, albedo, d):
    """The device's demodulation and passes, each through the host-compiled denoise.h: (i', v')."""
    H, W = z.shape
    c = d.to_c()
    i, v = np.empty((H, W, 3)), np.empty((H, W))
    _emu().hostemu_demodulate(_p(np.ascontiguousarray(sums)), _p(np.ascontiguousarray(m2)), counts.ctypes.data_as(u32p), H * W,
                              _p(albedo), d.albedo_eps, _p(i), _p(v))
    for k in range(d.iterations):
        i2, v2 = np.empty_like(i), np.empty_like(v)
        _emu().hostemu_denoise_pass(_p(i), _p(v), _p(nrm), _p(z), _p(albedo), W, H, 1 << k, C.byref(c), _p(i2), _p(v2))
        i, v = i2, v2
    return i, v


def edge_state(seed, H, W):
    """random_state with the edge cases a buffer can hold: counts 0..9 (0 and 1 entries: a reprojected buffer), NaN and
    inf sums, zero variance, misses (inf depth, zero normal, albedo 1)."""
    rng = np.random.default_rng(seed)
    sums, m2, _, nrm, z, albedo = random_state(rng, H, W, counted=True)
    counts = rng.integers(0, 10, (H, W)).astype(np.uint32)
    mean = rng.uniform(0, 1, (H, W, 3)) * rng.choice([0.1, 1.0, 5.0], (H, W, 1))
    sums = mean * counts[..., None]
    m2 = rng.uniform(0, 0.5, (H, W)) * np.maximum(counts.astype(np.float64) - 1.0, 0.0)
    m2[rng.random((H, W)) < 0.05] = 0.0
    sums[rng.random((H, W)) < 0.01] = np.nan
    sums[rng.random((H, W)) < 0.01] = np.inf
    m2[rng.random((H, W)) < 0.01] = np.nan
    return sums, m2, counts, np.ascontiguousarray(nrm), np.ascontiguousarray(z), np.ascontiguousarray(albedo)


def _criterion(c, v, min_entries=3):
    """A criterion whose threshold splits the finite pixels about in half, so both decisions are exercised."""
    with np.errstate(invalid="ignore", divide="ignore"):
        m = ((c[..., 0] + c[..., 1]) + c[..., 2]) / 3.0
        ratio = np.sqrt(v) / np.abs(m)
    rel = float(np.nanmedian(ratio[np.isfinite(ratio)]))
    return api.Adaptive(rel_tol=rel, abs_tol=1e-4, min_entries=min_entries)


def _check_against_numpy(got, want, near, npix):
    """Equal decisions except at borderline pixels, which must be few."""
    assert near.sum() <= max(2, npix // 1000), near.sum()
    assert not np.any((got != want) & ~near), np.argwhere((got != want) & ~near)[:5]


STATES = [(1, 1, 5), (7, 9, 5), (29, 37, 5), (37, 29, 3), (24, 48, 1), (45, 61, 5), (16, 16, 12)]


@pytest.mark.parametrize("H,W,it", STATES)
def test_pixels_match_numpy(H, W, it):
    sums, m2, counts, nrm, z, albedo = edge_state(H * 1000 + W + it, H, W)
    d = api.Denoise(iterations=it)
    c, v = gref.filtered(sums, m2, counts, nrm, z, albedo, d)
    crit = _criterion(c, v)
    want = gref.active(counts, c, v, crit)
    i, ev = emu_passes(sums, m2, counts, nrm, z, albedo, d)
    got = np.empty(H * W, np.uint8)
    cc = crit.to_c()
    _emu().hostemu_guided_pixels(counts.ctypes.data_as(u32p), _p(i), _p(ev), _p(albedo), H * W, d.albedo_eps, C.byref(cc),
                                 got.ctypes.data_as(u8p))
    _check_against_numpy(got.reshape(H, W).astype(bool), want, gref.borderline(counts, c, v, crit), H * W)
    # what the definition implies: fewer than min_entries, or a NaN v' (0 or 1 entries, a NaN sum), keeps a pixel active
    assert want[counts < crit.min_entries].all()
    assert want[np.isnan(v)].all()
    assert np.isnan(v[counts <= 1]).all()
    if H * W > 100:
        assert 0.05 < want[counts >= crit.min_entries].mean() < 0.95


@pytest.mark.parametrize("H,W", [(7, 9), (29, 37), (45, 61), (8, 32), (9, 17)])
@pytest.mark.parametrize("index,count", [(0, 1), (0, 4), (1, 4), (2, 4), (3, 4)])
def test_part_slots_match_numpy(H, W, index, count):
    sums, m2, counts, nrm, z, albedo = edge_state(H * 31 + W, H, W)
    d = api.Denoise(iterations=4)
    c, v = gref.filtered(sums, m2, counts, nrm, z, albedo, d)
    crit = _criterion(c, v, min_entries=2)
    want_mask, want_flags = gref.part_decision(counts, c, v, crit, index, count)
    tiles = len(want_mask) // 128
    i, ev = emu_passes(sums, m2, counts, nrm, z, albedo, d)
    mask, flags = np.full(tiles * 128, 7, np.uint8), np.full(tiles * 4, 7, np.uint8)
    cc = crit.to_c()
    n = _emu().hostemu_guided_part(_p(i), _p(ev), _p(albedo), counts.ctypes.data_as(u32p), W, H, index, count, tiles, d.albedo_eps,
                                   C.byref(cc), mask.ctypes.data_as(u8p), flags.ctypes.data_as(u8p))
    assert set(np.unique(mask)) <= {0, 1} and set(np.unique(flags)) <= {0, 1}
    assert n == mask.sum()
    near = gref.borderline(counts, c, v, crit).reshape(-1)
    p = gref.slot_pixels(W, H, index, count)
    slot_near = np.where(p >= 0, near[np.maximum(p, 0)], False)
    _check_against_numpy(mask.astype(bool), want_mask, slot_near, H * W)
    assert not mask[p < 0].any()  # slots past a ragged edge are never active
    if not slot_near.any():
        assert np.array_equal(flags.astype(bool), want_flags)
    # the parts together mark every pixel once, as the whole-image decision does
    if count == 1:
        whole = gref.active(counts, c, v, crit).reshape(-1)
        assert np.array_equal(np.sort(p[want_mask]), np.flatnonzero(whole))


def test_slot_pixels_cover_the_image_once():
    for W, H, n in [(1, 1, 1), (17, 9, 3), (100, 60, 4), (33, 8, 5)]:
        got = np.concatenate([gref.slot_pixels(W, H, k, n) for k in range(n)])
        assert np.array_equal(np.sort(got[got >= 0]), np.arange(W * H))
        for k in range(n):
            L = capi.lib()
            p = gref.slot_pixels(W, H, k, n)
            for e in range(0, len(p), 37):
                assert L.rptb_tile_pixel(W, H, k, n, e // 128, e % 128) == p[e]


# ---- api.Adaptive ----------------------------------------------------------------------------------------------------
def test_adaptive_guide_argument():
    a = api.Adaptive()
    assert a.guide is None
    d = api.Denoise(iterations=3)
    g = api.Adaptive(0.05, 1e-3, 5, guide=d)
    assert g.guide is d and (g.rel_tol, g.abs_tol, g.min_entries) == (0.05, 1e-3, 5)
    assert api.Adaptive(0.05, 1e-3, 5, d).guide is d  # positional, after min_entries
    c, cg = a.to_c(), api.Adaptive(guide=d).to_c()
    assert bytes(c) == bytes(cg)  # the C criterion does not carry the guide
    counts, sums, m2 = np.array([1, 5, 5]), np.array([[1.0, 1, 1], [5, 5, 5], [5, 5, 5]]), np.array([0.0, 0.0, 100.0])
    assert np.array_equal(a.active(counts, sums, m2), api.Adaptive(guide=d).active(counts, sums, m2))
    with pytest.raises(TypeError):
        api.Adaptive(guide=api.Reproject())
    with pytest.raises(TypeError):
        api.Adaptive(guide=5)


# ---- the C ABI's refusals before any device work --------------------------------------------------------------------
def test_guided_errors_before_any_device_work():
    L = capi.lib()
    cam, p = capi.Camera(), capi.RenderParams()
    p.width, p.height, p.iterations, p.shard_count = 8, 8, 1, 1
    good_c, good_d = api.Adaptive().to_c(), api.Denoise().to_c()
    fake = C.c_void_p(1)  # never looked at: the arguments are refused first

    def call(crit, guide, scene=None, buf=fake):
        return L.rptb_sample_into_guided(scene, C.byref(cam), C.byref(p), crit, guide, buf, None, None)

    bad_crit = [capi.Adaptive(0.02, 1e-3, 1, 0), capi.Adaptive(float("nan"), 1e-3, 4, 0), capi.Adaptive(0.02, -1.0, 4, 0),
                capi.Adaptive(float("inf"), 1e-3, 4, 0)]
    for c in bad_crit:
        assert call(C.byref(c), C.byref(good_d), scene=fake) == capi.ERR_BAD_ARG
        assert b"min_entries" in L.rptb_last_error() or b"tolerances" in L.rptb_last_error()
    bad_d = [capi.Denoise(13, 128, 1.0, 4.0, 1e-3), capi.Denoise(5, 128, -1.0, 4.0, 1e-3), capi.Denoise(5, 128, 1.0, float("nan"), 1e-3),
             capi.Denoise(5, 128, 1.0, 4.0, float("inf")), capi.Denoise(5, 128, 1.0, 4.0, 0.0), capi.Denoise(0, 128, 1.0, 4.0, 0.0)]
    for d in bad_d:
        assert call(C.byref(good_c), C.byref(d), scene=fake) == capi.ERR_BAD_ARG
        assert b"iterations" in L.rptb_last_error() or b"finite" in L.rptb_last_error()
        assert L.rptb_buffer_denoise_variance(fake, C.byref(d), _p(np.empty(1))) == capi.ERR_BAD_ARG
    assert call(None, C.byref(good_d), scene=fake) == capi.ERR_BAD_ARG
    assert call(C.byref(good_c), None, scene=fake) == capi.ERR_BAD_ARG
    assert call(C.byref(good_c), C.byref(good_d)) == capi.ERR_BAD_ARG  # no scene
    assert call(C.byref(good_c), C.byref(good_d), scene=fake, buf=None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_variance(None, C.byref(good_d), _p(np.empty(1))) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_variance(fake, C.byref(good_d), None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_variance(fake, None, _p(np.empty(1))) == capi.ERR_BAD_ARG


# ---- distributed: refused before any collective ----------------------------------------------------------------------
def test_distributed_refuses_a_guided_criterion():
    cfg = scenes.sphere_scene()
    r = api.Renderer(cfg.scene, cfg.camera).width(8).height(8).num_samples(4)
    guided = api.Adaptive(guide=api.Denoise())
    with pytest.raises(ValueError, match="guided"):
        distributed.render_iterative_distributed(r, 1, lambda i, b: None, adaptive=guided)
    with pytest.raises(ValueError, match="guided"):
        next(distributed.render_frames_distributed(r, [cfg.camera], entries=2, adaptive=guided))
    assert r._dev_scene is None  # nothing reached the device
