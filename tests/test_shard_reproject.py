"""Reprojection into shard buffers without a GPU: reproject_slot (reproject.h), run by the host emulation over every
element of every shard's compact tiles as reproject_part_kernel runs it, and scattered back through the tile deal, is
hostemu_reproject on the whole image bit for bit -- for shard counts that leave ragged tiles and shards with no tile,
for a source of another size, and for pixels that see the environment.  Also the new entry point's argument checks."""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from rpt_b200.distributed import gather_permutation, shard_tiles
from tests.test_reproject import _emu, _p, emu_reproject, orbit, random_stats

dp = capi.c_double_p
RAYS = 3
CENTER = (0.0, 0.5, 0.0)  # above the sphere: the upper part of the view sees the environment


def _lib():
    L = _emu()
    cam = C.POINTER(capi.Camera)
    L.hostemu_reproject_part.restype = None
    L.hostemu_reproject_part.argtypes = [cam, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, dp, C.c_uint64, C.c_double, cam,
                                         C.c_uint32, C.c_uint32, dp, dp, capi.c_u32_p, dp, dp, dp, C.POINTER(capi.Reproject),
                                         dp, dp, capi.c_u32_p, C.POINTER(C.c_uint64)]
    L.hostemu_features_resolve.restype = None
    L.hostemu_features_resolve.argtypes = [dp, C.c_uint64, C.c_double, dp, dp, dp, dp]
    return L


_FEAT = {}


def _feature_sums(cam, w, h):
    """The emulated feature pass of the sphere scene (it sees the environment around the sphere) through `cam`: w*h*8
    row-major sums, the planes normal (3 per pixel), albedo (3), hits, depth."""
    key = (tuple(cam.eye), tuple(cam.direction), w, h)
    if key not in _FEAT:
        flat = api.FlatScene(scenes.sphere_scene().scene)
        L = _lib()
        handle = C.c_void_p(L.hostemu_scene_create(C.byref(flat.desc), C.create_string_buffer(512), 512))
        try:
            p = api.Renderer(api.Scene(), cam).width(w).height(h).seed(3).precision(capi.PRECISION_F64).params(RAYS)
            out = np.empty(w * h * 8)
            assert L.hostemu_features(handle, C.byref(cam.to_c()), C.byref(p), _p(out)) >= 0
        finally:
            L.hostemu_scene_destroy(handle)
        _FEAT[key] = out
    return _FEAT[key]


def _resolve(sums, w, h):
    n = w * h
    N, z, a, f = np.empty((h, w, 3)), np.empty((h, w)), np.empty((h, w, 3)), np.empty((h, w))
    _lib().hostemu_features_resolve(_p(sums), n, float(RAYS), _p(N), _p(z), _p(a), _p(f))
    return N, z, f


def _cameras():
    scam = api.Camera.look_at(api.vec3(0.3, 0.6, 4.5), np.asarray(CENTER), api.vec3(0.0, 1.0, 0.0), 0.7)
    return scam, orbit(scam, CENTER, 0.07, lift=0.05)


def _compact(rows, npix, slot, mine, nelem):
    """Shard `mine`'s compact feature sums (nelem elements a plane) from the row-major ones; elements past a ragged edge
    hold NaN, which reproject_slot must never read."""
    out = np.full(nelem * 8, np.nan)
    p = np.flatnonzero(mine)
    for base_r, base_c, k in ((0, 0, 3), (3 * npix, 3 * nelem, 3), (6 * npix, 6 * nelem, 1), (7 * npix, 7 * nelem, 1)):
        for c in range(k):
            out[base_c + k * slot[p] + c] = rows[base_r + k * p + c]
    return out


# (dst width, height), (src width, height): 20x10 is 4 tiles, so shards 4.. of 5 and 8 own none
SIZES = [((128, 96), (128, 96)), ((97, 61), (80, 70)), ((20, 10), (24, 14))]


@pytest.mark.parametrize("dsize,ssize", SIZES)
def test_shards_reproject_like_the_whole_image(dsize, ssize):
    (dw, dh), (sw, sh) = dsize, ssize
    scam, dcam = _cameras()
    L = _lib()
    drows = _feature_sums(dcam, dw, dh)
    dN, dz, df = _resolve(drows, dw, dh)
    sN, sz, sf = _resolve(_feature_sums(scam, sw, sh), sw, sh)
    ssums, sm2, scounts = random_stats(np.random.default_rng(dw), sh, sw)
    assert (df == 0).any() and (df > 0).any()  # environment pixels and surface pixels
    prm = api.Reproject()
    want_s, want_m, want_n = emu_reproject(dcam, dN, dz, df, scam, ssums, sm2, scounts, sN, sz, sf, prm)
    want_reused = int((want_n > 0).sum())
    assert 0 < want_reused < dw * dh  # history for some pixels, none for others
    assert (want_n[df == 0] > 0).any()  # the environment is reprojected too
    src = [np.ascontiguousarray(a, np.float64) for a in (ssums, sm2, sN, sz, sf)]
    sc = np.ascontiguousarray(scounts, np.uint32)
    dc, scc, pc = dcam.to_c(), scam.to_c(), prm.to_c()
    npix = dw * dh
    for n in (1, 2, 3, 5, 8):
        perm = gather_permutation(dw, dh, n)
        slots = shard_tiles(dw, dh, 0, n) * 128
        owner, slot = perm // slots, perm % slots
        got_s, got_m, got_n = np.full((npix, 3), np.nan), np.full(npix, np.nan), np.full(npix, 7, np.uint32)
        total = 0
        for i in range(n):
            nelem = shard_tiles(dw, dh, i, n) * 128
            mine = owner == i
            feat = _compact(drows, npix, slot, mine, nelem)
            out_s, out_m, out_n = np.empty((nelem, 3)), np.empty(nelem), np.empty(nelem, np.uint32)
            reused = C.c_uint64(99)
            L.hostemu_reproject_part(C.byref(dc), dw, dh, i, n, _p(feat), nelem, float(RAYS), C.byref(scc), sw, sh, _p(src[0]),
                                     _p(src[1]), sc.ctypes.data_as(capi.c_u32_p), _p(src[2]), _p(src[3]), _p(src[4]), C.byref(pc),
                                     _p(out_s), _p(out_m), out_n.ctypes.data_as(capi.c_u32_p), C.byref(reused))
            assert reused.value == int((out_n > 0).sum())
            total += reused.value
            ragged = np.ones(nelem, bool)
            ragged[slot[mine]] = False
            assert (out_s[ragged] == 0).all() and (out_m[ragged] == 0).all() and (out_n[ragged] == 0).all()
            if nelem == 0:
                assert not mine.any() and reused.value == 0
            got_s[mine], got_m[mine], got_n[mine] = out_s[slot[mine]], out_m[slot[mine]], out_n[slot[mine]]
        assert total == want_reused, n
        assert got_s.reshape(dh, dw, 3).tobytes() == want_s.tobytes(), n
        assert got_m.reshape(dh, dw).tobytes() == want_m.tobytes(), n
        assert np.array_equal(got_n.reshape(dh, dw), want_n), n
    if dsize == (20, 10):
        assert shard_tiles(dw, dh, 4, 5) == 0 and shard_tiles(dw, dh, 7, 8) == 0


def test_reproject_shard_errors_before_any_device_work():
    L = capi.lib()
    a, b = C.c_void_p(1), C.c_void_p(2)
    good = api.Reproject().to_c()
    assert L.rptb_buffer_reproject_shard(None, b, C.byref(good), None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_reproject_shard(a, None, C.byref(good), None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_reproject_shard(a, b, None, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_reproject_shard(a, a, C.byref(good), None) == capi.ERR_BAD_ARG
    assert b"same buffer" in L.rptb_last_error()
    for prm in (api.Reproject(depth_tol=-0.1), api.Reproject(normal_cos=1.5), api.Reproject(max_history=1)):
        c = prm.to_c()
        assert L.rptb_buffer_reproject_shard(a, b, C.byref(c), None) == capi.ERR_BAD_ARG


def test_frame_arguments_are_those_of_render_frames():
    from rpt_b200.distributed import render_frames_distributed

    cfg = scenes.sphere_scene()
    r = api.Renderer(cfg.scene, cfg.camera).num_samples(6)
    for kw in (dict(entries=4), dict(entries=0), dict(entries=1, denoise=api.Denoise())):
        with pytest.raises(ValueError):
            next(r.render_frames([cfg.camera], **kw))
        with pytest.raises(ValueError):
            next(render_frames_distributed(r, [cfg.camera], **kw))
    assert r.camera is cfg.camera
