"""The cross-filtered denoiser with a smoothed selection map on the GPU (rptb_buffer_denoise_cross): the colour, k* and
M^ against numpy (tests/cross_ref.py) on the buffer's read-backs within 1e-12, on sphere, Cornell and teapot in f32 and
f64 at 64x48, 97x61 and 1920x1080; every pixel whose 5x5 neighbourhood chose level 0 against sums / counts and every
one that chose a level k against the same pixel of a call with more passes, bit for bit; every output a convex blend of
its pixel's levels; the same on buffers filled by adaptive and error-guided calls and on a reprojected buffer with
halves; replicas on a repeated device against one part; Renderer.render(cross=True); and the device-side refusals."""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, distributed, scenes
from tests import cross_ref as xref
from tests import util
from tests.test_reproject import orbit

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
D = api.Denoise()
MAKE = {"sphere": scenes.sphere_scene, "cornell": scenes.cornell_scene, "teapot": scenes.teapot_scene}


def _renderer(cfg, w, h, mb=3, prec=F64, seed=5, device=0, cam=None):
    return api.Renderer(cfg.scene, cam or cfg.camera).width(w).height(h).max_bounces(mb).seed(seed).precision(prec).device(device)


def _fill(r, buf, entries=4, spp=2):
    r.sample_features(8, buf)
    for _ in range(entries):
        r.sample(spp, buf, want_stats=False)


def _state(buf):
    h, w = buf.height, buf.width
    sums, m2, counts = buf.pixel_stats()
    nrm, z, albedo, _ = buf.features()
    return (sums.reshape(h, w, 3), m2.reshape(h, w), buf.half_sums().reshape(h, w, 3), counts.reshape(h, w), nrm, z, albedo)


def _close(got, want, rel=1e-12):
    assert np.array_equal(np.isnan(got), np.isnan(want))
    fin = np.isfinite(want)
    scale = np.max(np.abs(want[fin]), initial=0.0)
    assert np.max(np.abs(got[fin] - want[fin]), initial=0.0) <= rel * scale


def _check(buf, d=D):
    """denoise_cross(d) against numpy, the uniform-neighbourhood and convex-blend properties, and cross_image against
    the colour's bytes.  Returns (rgb, level, mse)."""
    rgb, level, mse = buf.denoise_cross(d)
    assert level.max() <= d.iterations
    state = _state(buf)
    lv = xref.levels(*state, d)
    wlevel = xref.argmin([M for _, _, M in lv])
    near = xref.ties(lv)
    assert np.array_equal(level[~near], wlevel[~near]), np.argwhere((level != wlevel) & ~near)[:8]
    # the blend over the device's own k*, everywhere; over numpy's where no neighbour's k* differs
    wrgb, wM = xref.blend(lv, level)
    _close(rgb, wrgb)
    _close(mse, wM)
    same = ~xref.dilate(level != wlevel)
    wrgb2, wM2 = xref.blend(lv, wlevel)
    _close(np.where(same[..., None], rgb, 0.0), np.where(same[..., None], wrgb2, 0.0))
    _close(np.where(same, mse, 0.0), np.where(same, wM2, 0.0))
    # level 0 bit for bit where the whole neighbourhood chose it
    sums, _, _, counts = state[:4]
    at = ~xref.dilate(level != 0)
    assert np.array_equal(rgb[at], (sums / counts.astype(np.float64)[..., None])[at], equal_nan=True)
    # convex: between the least and the greatest of the levels the pixel blends (numpy's levels, 1e-12 apart)
    used = np.stack([xref.beta(level, k)[0] > 0.0 for k in range(d.iterations + 1)])
    O = np.stack([o for o, _, _ in lv])
    lo = np.where(used[..., None], O, np.inf).min(0)
    hi = np.where(used[..., None], O, -np.inf).max(0)
    tol = 1e-11 * np.max(np.abs(O[np.isfinite(O)]))
    assert (rgb >= lo - tol).all() and (rgb <= hi + tol).all()
    return rgb, level, mse


def _level(d, k):
    return api.Denoise(iterations=k, sigma_normal=d.sigma_normal, sigma_depth=d.sigma_depth, sigma_luminance=d.sigma_luminance,
                       albedo_eps=d.albedo_eps)


def _check_levels_agree(buf, d=D):
    """A pixel whose 5x5 neighbourhood chose level k is O_k, which does not depend on the pass count beyond k: it is the
    same bits in a call with d.iterations passes as in one with k passes, where that call also chose k there."""
    rgb, level, _ = buf.denoise_cross(d)
    for k in range(1, d.iterations):
        rgb_k, level_k, _ = buf.denoise_cross(_level(d, k))
        at = ~xref.dilate(level != k) & ~xref.dilate(level_k != k)
        assert np.array_equal(rgb[at], rgb_k[at], equal_nan=True), k


@pytest.mark.parametrize("name", ["sphere", "cornell", "teapot"])
@pytest.mark.parametrize("prec", [F32, F64])
@pytest.mark.parametrize("w,h", [(64, 48), (97, 61)])
def test_matches_numpy(name, prec, w, h):
    cfg = MAKE[name]()
    r = _renderer(cfg, w, h, mb=0 if name == "teapot" else 3, prec=prec)
    with r.device_buffer(halves=True) as buf:
        _fill(r, buf)
        _, level, mse = _check(buf)
        assert np.isfinite(mse).all()
        assert (level > 0).any()
        _check(buf, api.Denoise(iterations=2))
        _check(buf, api.Denoise(iterations=3, sigma_luminance=1e9))
        _check_levels_agree(buf)
    r.close()


def test_matches_numpy_at_1080p():
    cfg = scenes.cornell_scene()
    r = _renderer(cfg, 1920, 1080, prec=F32)
    with r.device_buffer(halves=True) as buf:
        _fill(r, buf, entries=2, spp=1)
        _, level, _ = _check(buf, api.Denoise(iterations=2))
        assert (level == 0).any() and (level > 0).any()
    r.close()


def test_adaptive_and_error_guided_buffers():
    cfg = scenes.cornell_scene()
    r = _renderer(cfg, 96, 64, prec=F32)
    with r.device_buffer(halves=True) as buf:
        _fill(r, buf, entries=2)
        r.sample(2, buf, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 2))
        for _ in range(3):
            r.sample(2, buf, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 3, guide=D, estimate="halves"))
        counts = buf.counts()
        assert counts.min() < counts.max() and (counts % 2 == 1).any()  # adaptive in effect, odd counts among them
        _check(buf)
        _check_levels_agree(buf)
    r.close()


def test_reprojected_buffer():
    center = (0.0, 0.5, 0.0)
    a = api.Camera.look_at(api.vec3(0.3, 0.6, 4.5), np.asarray(center), api.vec3(0.0, 1.0, 0.0), 0.7)
    b = orbit(a, center, 0.07, lift=0.05)
    cfg = scenes.sphere_scene()
    w, h = 64, 48
    ra = _renderer(cfg, w, h, mb=2, cam=a)
    rb = _renderer(cfg, w, h, mb=2, cam=b)
    rb._next_sample = 100
    with ra.device_buffer(halves=True) as src, rb.device_buffer(halves=True) as dst:
        _fill(ra, src)
        rb.sample_features(8, dst)
        assert dst.reproject_from(src) > 0
        for _ in range(2):  # every pixel to 2 entries at least: the filter needs them
            rb.sample(2, dst, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 3))
        _check(dst)
    ra.close()
    rb.close()


@pytest.mark.parametrize("parts", [2, 3, 8])
def test_replicas_are_one_part(parts, monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")  # replicas on a repeated device 0
    cfg = scenes.cornell_scene()
    got = []
    for dev in (0, [0] * parts):
        r = _renderer(cfg, 80, 64, prec=F32, device=dev)
        with r.device_buffer(halves=True) as buf:
            _fill(r, buf)
            r.sample(2, buf, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 2))
            got.append(buf.denoise_cross(D) + (buf.cross_image(D),))
        r.close()
    for x, y in zip(*got):
        assert np.array_equal(x, y, equal_nan=True)


def test_render_cross():
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 48, 32, prec=F32).num_samples(8)
    img = r.render(denoise=D, entries=4, feature_samples=8, cross=True)
    assert img.shape == (32, 48, 3) and img.dtype == np.uint8
    # the same calls into a buffer of one's own give the same bytes, and they are the colour's film resolve: the
    # bytes of a plain buffer holding the blended colour as its one entry
    r2 = _renderer(cfg, 48, 32, prec=F32).num_samples(8)
    with r2.device_buffer(halves=True) as buf:
        for _ in range(4):
            r2.sample(2, buf, want_stats=False)
        r2.sample_features(8, buf)
        assert np.array_equal(img, buf.cross_image(D))
        rgb, _, _ = buf.denoise_cross(D)
    with r2.device_buffer() as one:
        one.add_samples(rgb.reshape(-1, 3))
        assert np.array_equal(img, one.image())
    r.close()
    r2.close()


def test_refusals():
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 32, 16, prec=F32)
    plain, halves = r.device_buffer(), r.device_buffer(halves=True)
    for b in (plain, halves):
        _fill(r, b, entries=3)
    with pytest.raises(capi.RptbError, match="halves") as e:
        plain.denoise_cross(D)
    assert "status %d" % capi.ERR_BAD_ARG in str(e.value)
    with pytest.raises(capi.RptbError, match="iterations") as e:
        halves.denoise_cross(api.Denoise(iterations=0))
    assert "status %d" % capi.ERR_BAD_ARG in str(e.value)
    sb = distributed.ShardBuffer(r.device_scene(), 32, 16, rank=0, world=2, halves=True)
    rgb = np.empty((16, 32, 3))
    d = D.to_c()
    assert capi.lib().rptb_buffer_denoise_cross(sb.handle, C.byref(d), rgb.ctypes.data_as(capi.c_double_p), None, None,
                                                None) == capi.ERR_UNSUPPORTED
    sb.close()
    nf = r.device_buffer(halves=True)  # entries, no features
    for _ in range(2):
        r.sample(2, nf, want_stats=False)
    with pytest.raises(capi.RptbError, match="features"):
        nf.denoise_cross(D)
    one = r.device_buffer(halves=True)  # features, one entry
    r.sample_features(4, one)
    r.sample(2, one, want_stats=False)
    with pytest.raises(capi.RptbError, match="fewer than 2"):
        one.denoise_cross(D)
    for b in (plain, halves, nf, one):
        b.close()
    r.close()
