"""The choice of each pixel's number of filter passes on the GPU (rptb_buffer_denoise_select): every output pixel
against rptb_buffer_denoise(iterations = its level), bit for bit, on sphere, Cornell and teapot in f32 and f64 at 128x96,
97x61 and 1920x1080, and the bytes against denoised_image's; the same on buffers filled by adaptive and error-guided
calls and on a reprojected buffer with halves; replicas on a repeated device against one part; m and the levels against
numpy (tests/select_ref.py) on the buffer's read-backs; Renderer.render(select=True); and the device-side refusals."""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, distributed, scenes
from tests import select_ref as sref
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


def _level(d, k):
    return api.Denoise(iterations=k, sigma_normal=d.sigma_normal, sigma_depth=d.sigma_depth, sigma_luminance=d.sigma_luminance,
                       albedo_eps=d.albedo_eps)


def _check_levels(buf, d=D):
    """Every pixel of denoise_select(d) is denoise(iterations = its level) there, bit for bit, and at level 0 sums / counts;
    selected_image is each level's denoised_image there.  Returns (rgb, level, mse)."""
    rgb, level, mse = buf.denoise_select(d)
    img = buf.selected_image(d)
    assert level.max() <= d.iterations
    sums, _, counts = buf.pixel_stats()
    raw = (sums / counts.astype(np.float64)[:, None]).reshape(rgb.shape)
    for k in range(d.iterations + 1):
        at = level == k
        if not at.any():
            continue
        want = buf.denoise(_level(d, k))
        assert np.array_equal(rgb[at], want[at], equal_nan=True), k
        assert np.array_equal(img[at], buf.denoised_image(_level(d, k))[at]), k
        if k == 0:
            assert np.array_equal(rgb[at], raw[at], equal_nan=True)
    return rgb, level, mse


@pytest.mark.parametrize("name", ["sphere", "cornell", "teapot"])
@pytest.mark.parametrize("prec", [F32, F64])
@pytest.mark.parametrize("w,h", [(128, 96), (97, 61)])
def test_every_pixel_is_its_levels_denoise(name, prec, w, h):
    cfg = MAKE[name]()
    r = _renderer(cfg, w, h, mb=0 if name == "teapot" else 3, prec=prec)
    with r.device_buffer(halves=True) as buf:
        _fill(r, buf)
        _, level, mse = _check_levels(buf)
        assert np.isfinite(mse).all()
        assert (level > 0).any()
        _check_levels(buf, api.Denoise(iterations=2))
    r.close()


def test_every_pixel_is_its_levels_denoise_at_1080p():
    cfg = scenes.cornell_scene()
    r = _renderer(cfg, 1920, 1080, prec=F32)
    with r.device_buffer(halves=True) as buf:
        _fill(r, buf, entries=2, spp=1)
        _, level, _ = _check_levels(buf)
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
        assert counts.min() < counts.max()  # the calls were adaptive in effect
        _check_levels(buf)
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
        _check_levels(dst)
    ra.close()
    rb.close()


@pytest.mark.parametrize("parts", [2, 3])
def test_replicas_are_one_part(parts, monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")  # replicas on a repeated device 0
    cfg = scenes.cornell_scene()
    got = []
    for dev in (0, [0] * parts):
        r = _renderer(cfg, 80, 64, prec=F32, device=dev)
        with r.device_buffer(halves=True) as buf:
            _fill(r, buf)
            r.sample(2, buf, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 2))
            got.append(buf.denoise_select(D) + (buf.selected_image(D),))
        r.close()
    for x, y in zip(*got):
        assert np.array_equal(x, y, equal_nan=True)


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


@pytest.mark.parametrize("name,prec", [("sphere", F32), ("cornell", F64), ("teapot", F32)])
def test_matches_numpy(name, prec):
    cfg = MAKE[name]()
    r = _renderer(cfg, 64, 48, mb=0 if name == "teapot" else 3, prec=prec)
    with r.device_buffer(halves=True) as buf:
        _fill(r, buf)
        r.sample(2, buf, want_stats=False, adaptive=api.Adaptive(0.1, 1e-3, 2))
        for d in (D, api.Denoise(iterations=1), api.Denoise(iterations=3, sigma_luminance=1e9)):
            state = _state(buf)
            rgb, level, mse = buf.denoise_select(d)
            wrgb, wlevel, wM = sref.select(*state, d)
            near = sref.ties(*state, d)
            assert np.array_equal(level[~near], wlevel[~near]), np.argwhere((level != wlevel) & ~near)[:8]
            same = level == wlevel
            _close(np.where(same, mse, 0.0), np.where(same, wM, 0.0))
            _close(np.where(same[..., None], rgb, 0.0), np.where(same[..., None], wrgb, 0.0))
    r.close()


def test_render_select():
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 48, 32, prec=F32).num_samples(8)
    img = r.render(denoise=D, entries=4, feature_samples=8, select=True)
    assert img.shape == (32, 48, 3) and img.dtype == np.uint8
    # the same calls into a buffer of one's own give the same bytes
    r2 = _renderer(cfg, 48, 32, prec=F32).num_samples(8)
    with r2.device_buffer(halves=True) as buf:
        for _ in range(4):
            r2.sample(2, buf, want_stats=False)
        r2.sample_features(8, buf)
        assert np.array_equal(img, buf.selected_image(D))
    r.close()
    r2.close()


def test_refusals():
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 32, 16, prec=F32)
    plain, halves = r.device_buffer(), r.device_buffer(halves=True)
    for b in (plain, halves):
        _fill(r, b, entries=3)
    with pytest.raises(capi.RptbError, match="halves") as e:
        plain.denoise_select(D)
    assert "status %d" % capi.ERR_BAD_ARG in str(e.value)
    with pytest.raises(capi.RptbError, match="iterations"):
        halves.denoise_select(api.Denoise(iterations=0))
    sb = distributed.ShardBuffer(r.device_scene(), 32, 16, rank=0, world=2, halves=True)
    rgb = np.empty((16, 32, 3))
    d = D.to_c()
    assert capi.lib().rptb_buffer_denoise_select(sb.handle, C.byref(d), rgb.ctypes.data_as(capi.c_double_p), None, None,
                                                 None) == capi.ERR_UNSUPPORTED
    sb.close()
    nf = r.device_buffer(halves=True)  # entries, no features
    for _ in range(2):
        r.sample(2, nf, want_stats=False)
    with pytest.raises(capi.RptbError, match="features"):
        nf.denoise_select(D)
    one = r.device_buffer(halves=True)  # features, one entry
    r.sample_features(4, one)
    r.sample(2, one, want_stats=False)
    with pytest.raises(capi.RptbError, match="fewer than 2"):
        one.denoise_select(D)
    for b in (plain, halves, nf, one):
        b.close()
    r.close()
