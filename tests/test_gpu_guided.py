"""Adaptive sampling guided by the denoiser on the GPU (rptb_sample_into_guided, rptb_buffer_denoise_variance): the
variance read-back against numpy; each call's decisions replayed in numpy on the state read before it; active pixels
getting their plain entry; iterations 0 as plain adaptive sampling; the early calls that skip the filter; guided calls
after a reprojection; the same bits for every replica count; one call at 1920x1080; the loops that take a guided
criterion; and every refusal."""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, distributed, scenes
from tests import guided_ref as gref
from tests import util

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
GUIDE = api.Denoise(iterations=4)
CENTER = {"sphere": (0.0, -0.25, 0.0), "cornell": (278.0, 273.0, 280.0)}
MAKE = {"sphere": scenes.sphere_scene, "cornell": scenes.cornell_scene}


def _moved(cfg, name, offset):
    """The scene's camera moved by `offset`, looking at the scene's centre."""
    eye = np.asarray(cfg.camera.eye, dtype=np.float64) + np.asarray(offset)
    return api.Camera.look_at(api.vec3(*eye), np.asarray(CENTER[name]), api.vec3(0.0, 1.0, 0.0), cfg.camera.fov)


def _renderer(cfg, w, h, mb=3, prec=F32, seed=5, device=0, camera=None):
    return (api.Renderer(cfg.scene, camera or cfg.camera).width(w).height(h).max_bounces(mb).seed(seed).precision(prec)
            .device(device))


def _guided(r, n, buf, crit, want_stats=True):
    """One guided call through the C ABI: (pixels that got the entry, stats dict)."""
    ds, p, cam, c, g = r.device_scene(), r.params(n, r._next_sample), r.camera.to_c(), crit.to_c(), crit.guide.to_c()
    active, st = C.c_uint64(0), capi.Stats()
    capi.check(capi.lib().rptb_sample_into_guided(ds.handle, C.byref(cam), C.byref(p), C.byref(c), C.byref(g), buf.handle,
                                                  C.byref(active), C.byref(st) if want_stats else None), "rptb_sample_into_guided")
    r._next_sample += n
    return int(active.value), st.as_dict()


def _plain_entry(r, n, first_sample):
    """rptb_render_samples of the same call: the entry every pixel would get, row-major (npix, 3)."""
    out = np.empty((r._width * r._height, 3))
    p, cam = r.params(n, first_sample), r.camera.to_c()
    capi.check(capi.lib().rptb_render_samples(r.device_scene().handle, C.byref(cam), C.byref(p), out.ctypes.data_as(capi.c_double_p),
                                              None), "rptb_render_samples")
    return out


def _numpy_decision(buf, crit):
    """The numpy decision on the buffer's state as it is now: (active (npix,), borderline (npix,), c', v')."""
    h, w = buf.height, buf.width
    sums, m2, counts = buf.pixel_stats()
    nrm, z, albedo, _ = buf.features()
    c, v = gref.filtered(sums.reshape(h, w, 3), m2.reshape(h, w), counts.reshape(h, w), nrm, z, albedo, crit.guide)
    counts = counts.reshape(h, w)
    return (gref.active(counts, c, v, crit).reshape(-1), gref.borderline(counts, c, v, crit).reshape(-1), c, v)


def _replay(r, buf, crit, spp, prec):
    """One guided call checked against the numpy decision on the state read before it.  Returns the active count."""
    s0, m0, c0 = buf.pixel_stats()
    want, near, _, _ = _numpy_decision(buf, crit)
    assert near.sum() <= max(2, len(want) // 1000), near.sum()
    first = r._next_sample
    active, _ = _guided(r, spp, buf, crit)
    s1, m1, c1 = buf.pixel_stats()
    took = c1 != c0
    assert np.array_equal(c1[took], c0[took] + 1)
    assert active == int(took.sum())
    assert not np.any((took != want) & ~near), np.flatnonzero((took != want) & ~near)[:8]
    # a pixel that took no entry keeps its bits; one that did took exactly its plain-render entry
    assert np.array_equal(s1[~took], s0[~took]) and np.array_equal(m1[~took], m0[~took])
    entry = _plain_entry(r, spp, first)
    if prec == F64:
        assert np.array_equal(s1[took], s0[took] + entry[took])
    else:
        np.testing.assert_allclose(s1[took], s0[took] + entry[took], rtol=1e-6, atol=1e-6)
    return active


# ---- the variance read-back ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["sphere", "cornell"])
def test_denoised_variance_matches_numpy(gpu_ok, name):
    cfg = MAKE[name]()
    w, h = 100, 60
    r = _renderer(cfg, w, h)
    buf = r.device_buffer()
    for _ in range(6):
        r.sample(2, buf, want_stats=False)
    r.sample_features(16, buf)
    sums, m2, counts = buf.pixel_stats()
    nrm, z, albedo, _ = buf.features()
    for d in (api.Denoise(iterations=0), api.Denoise(iterations=1), api.Denoise(), api.Denoise(iterations=7, sigma_normal=32)):
        got = buf.denoised_variance(d)
        if d.iterations == 0:  # each pixel's variance of the mean, bit for bit
            dn = counts.astype(np.float64)
            assert np.array_equal(got.ravel(), m2 / (((dn - 1.0) * dn) * 3.0))
            continue
        c, v = gref.filtered(sums.reshape(h, w, 3), m2.reshape(h, w), counts.reshape(h, w), nrm, z, albedo, d)
        assert np.isfinite(v).all()
        np.testing.assert_allclose(got, v, rtol=1e-12, atol=0.0)
        np.testing.assert_allclose(buf.denoise(d), c, rtol=1e-12, atol=1e-300)
    # the decision taken on the GPU's own c' and v' is the decision the guide takes, with no borderline allowance:
    # the guide's c' is denoise()'s output and its v' denoised_variance()'s, bit for bit
    crit = api.Adaptive(0.05, 1e-3, 3, guide=GUIDE)
    want = gref.active(counts.reshape(h, w), buf.denoise(GUIDE), buf.denoised_variance(GUIDE), crit).ravel()
    c0 = buf.counts().ravel()
    active, _ = _guided(r, 1, buf, crit)
    assert np.array_equal(buf.counts().ravel() - c0, want.astype(np.uint32))
    assert active == want.sum() and 0 < active < w * h
    buf.close()
    r.close()


# ---- decisions ---------------------------------------------------------------------------------------------------------
REPLAY = {  # name: (config, w, h, max_bounces, precision, spp per call, criterion)
    "sphere": (scenes.sphere_scene, 64, 40, 2, F32, 2, api.Adaptive(0.05, 1e-3, 3, guide=GUIDE)),
    "cornell": (scenes.cornell_scene, 48, 48, 3, F32, 2, api.Adaptive(0.05, 2e-3, 3, guide=GUIDE)),
    "sphere_f64": (scenes.sphere_scene, 40, 24, 2, F64, 2, api.Adaptive(0.03, 1e-3, 2, guide=api.Denoise(iterations=3))),
    "cornell_f64": (scenes.cornell_scene, 37, 29, 3, F64, 1, api.Adaptive(0.08, 1e-3, 4, guide=api.Denoise())),
}


@pytest.mark.parametrize("name", sorted(REPLAY))
def test_decisions_replay_in_numpy(gpu_ok, name):
    make, w, h, mb, prec, spp, crit = REPLAY[name]
    r = _renderer(make(), w, h, mb, prec)
    buf = r.device_buffer()
    r.sample_features(16, buf)
    for _ in range(crit.min_entries):
        _guided(r, spp, buf, crit)
    actives = [_replay(r, buf, crit, spp, prec) for _ in range(6)]
    assert any(0 < a < w * h for a in actives), actives
    buf.close()
    r.close()


def test_zero_iterations_is_plain_adaptive(gpu_ok):
    cfg = scenes.cornell_scene()
    w, h = 53, 37
    crit = api.Adaptive(0.06, 1e-3, 3)
    guided = api.Adaptive(0.06, 1e-3, 3, guide=api.Denoise(iterations=0))
    ra, rg = _renderer(cfg, w, h), _renderer(cfg, w, h)
    ba, bg = ra.device_buffer(), rg.device_buffer()  # no features: iterations 0 needs none
    actives = []
    for _ in range(8):
        a = ra.sample(2, ba, adaptive=crit)
        g, st = _guided(rg, 2, bg, guided)
        assert a == g and st["launches"] == ra.last_stats["launches"]
        actives.append(a)
    assert any(0 < a < w * h for a in actives)
    for x, y in zip(ba.pixel_stats(), bg.pixel_stats()):
        assert np.array_equal(x, y)
    for x in (ba, bg, ra, rg):
        x.close()


def test_early_calls_skip_the_filter(gpu_ok):
    cfg = scenes.sphere_scene()
    w, h = 64, 40
    crit = api.Adaptive(0.05, 1e-3, 4, guide=api.Denoise(iterations=5))
    plain = api.Adaptive(0.05, 1e-3, 4)
    rg, rp = _renderer(cfg, w, h), _renderer(cfg, w, h)
    bg, bp = rg.device_buffer(), rp.device_buffer()
    rg.sample_features(8, bg)
    for k in range(crit.min_entries):  # no pixel can hold min_entries yet: every pixel renders, no filter kernel runs
        active, st = _guided(rg, 2, bg, crit)
        rp.sample(2, bp, adaptive=plain)
        assert active == w * h
        assert st["launches"] == rp.last_stats["launches"], k
    assert (bg.counts() == crit.min_entries).all()
    for x, y in zip(bg.pixel_stats(), bp.pixel_stats()):
        assert np.array_equal(x, y)
    # the next call runs the filter: gather (1 part), resolve, demodulate, 5 passes and the mark kernel, and no plain mark
    _, st = _guided(rg, 2, bg, crit)
    rp.sample(2, bp, adaptive=plain)
    assert st["launches"] == rp.last_stats["launches"] - 1 + 1 + 1 + 1 + 5 + 1
    for x in (bg, bp, rg, rp):
        x.close()


@pytest.mark.parametrize("history", [False, True], ids=["reproject", "history_test"])
def test_guided_calls_after_a_reprojection(gpu_ok, history):
    cfg = scenes.cornell_scene()
    w, h = 64, 48
    cam2 = _moved(cfg, "cornell", (60.0, 0.0, 0.0))
    crit = api.Adaptive(0.05, 2e-3, 3, guide=GUIDE)
    r = _renderer(cfg, w, h)
    src = r.device_buffer()
    for _ in range(6):
        r.sample(2, src, want_stats=False)
    r.sample_features(8, src)
    r.camera = cam2
    dst = r.device_buffer()
    r.sample_features(8, dst)
    if history:
        for _ in range(2):
            r.sample(2, dst, want_stats=False)
        dst.merge_history_from(src, api.Reproject(), api.HistoryTest())
    else:
        dst.reproject_from(src, api.Reproject())
    c = dst.counts().ravel()
    if not history:
        assert (c <= 1).any() and (c >= 3).any()
    low = c < crit.min_entries
    want, _, _, v = _numpy_decision(dst, crit)
    assert want[low].all() and np.isnan(v.ravel()[c <= 1]).all()
    before = dst.counts().ravel()
    _replay(r, dst, crit, 2, F32)
    assert (dst.counts().ravel()[low] == before[low] + 1).all()  # the 0- and 1-entry pixels render first
    for _ in range(3):
        _replay(r, dst, crit, 2, F32)
    for x in (src, dst, r):
        x.close()


def test_replicas_give_the_same_bits(gpu_ok, monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")
    cfg = scenes.cornell_scene()
    w, h = 203, 117
    crit = api.Adaptive(0.1, 2e-3, 2, guide=api.Denoise(iterations=3))
    ref = None
    for devices in util.replica_lists(gpu_ok):
        r = _renderer(cfg, w, h, device=devices)
        buf = r.device_buffer()
        r.sample_features(8, buf)
        actives = [_guided(r, 2, buf, crit, want_stats=False)[0] for _ in range(5)]
        got = buf.pixel_stats() + (actives,)
        if ref is None:
            ref = got
            assert 0 < actives[-1] < w * h
        else:
            for a, b in zip(got[:3], ref[:3]):
                assert np.array_equal(a, b), devices
            assert got[3] == ref[3], devices
        buf.close()
        r.close()


def test_one_call_at_1080p(gpu_ok):
    cfg = scenes.sphere_scene()
    crit = api.Adaptive(0.05, 1e-3, 2, guide=api.Denoise(iterations=2))
    r = _renderer(cfg, 1920, 1080, mb=1)
    buf = r.device_buffer()
    r.sample_features(2, buf)
    for _ in range(2):
        _guided(r, 1, buf, crit, want_stats=False)
    active = _replay(r, buf, crit, 1, F32)
    assert 0 < active < 1920 * 1080
    buf.close()
    r.close()


# ---- the loops -----------------------------------------------------------------------------------------------------------
def test_iterative_render_with_a_guided_criterion_ends(gpu_ok):
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 64, 40).num_samples(400)
    buf = r.device_buffer()
    seen = []
    r.iterative_render(2, lambda i, b: seen.append(i), buffer=buf, adaptive=api.Adaptive(0.2, 1e-2, 2, guide=GUIDE), feature_samples=8)
    assert buf.feature_rays == 8  # the feature pass came first
    assert seen and seen[-1] < 400  # converged: the last batch rendered nothing
    assert buf.counts().min() >= 2 and buf.counts().max() <= len(seen)
    buf.close()
    r.close()


def test_render_frames_is_the_hand_replay(gpu_ok):
    cfg = scenes.cornell_scene()
    w, h = 48, 40
    cams = [cfg.camera, _moved(cfg, "cornell", (40.0, 0.0, 0.0))]
    crit, d = api.Adaptive(0.05, 2e-3, 3, guide=GUIDE), api.Denoise()
    ra = _renderer(cfg, w, h).num_samples(8)
    frames = list(ra.render_frames(cams, entries=4, feature_samples=8, adaptive=crit, denoise=d))
    rb = _renderer(cfg, w, h).num_samples(8)
    prev, want = None, []
    for cam in cams:
        rb.camera = cam
        buf = rb.device_buffer()
        rb.sample_features(8, buf)
        if prev is not None:
            buf.reproject_from(prev, api.Reproject())
            prev.close()
        for _ in range(4):
            _guided(rb, 2, buf, crit, want_stats=False)
        want.append(buf.denoised_image(d))
        prev = buf
    prev.close()
    for a, b in zip(frames, want):
        assert np.array_equal(a, b)
    ra.close()
    rb.close()


# ---- refusals ------------------------------------------------------------------------------------------------------------
def _refused(fn, code, text):
    with pytest.raises(capi.RptbError) as e:
        fn()
    assert f"status {code}:" in str(e.value) and text in str(e.value), str(e.value)


def test_refusals(gpu_ok):
    cfg = scenes.sphere_scene()
    w, h = 32, 24
    crit = api.Adaptive(0.05, 1e-3, 2, guide=GUIDE)
    other = _moved(cfg, "sphere", (0.3, 0.0, 0.0))
    r = _renderer(cfg, w, h)
    L = capi.lib()

    def call(buf, c=crit):
        return _guided(r, 1, buf, c, want_stats=False)

    # no features (iterations > 0); iterations 0 needs none
    b = r.device_buffer()
    _refused(lambda: call(b), capi.ERR_BAD_ARG, "no features")
    call(b, api.Adaptive(0.05, 1e-3, 2, guide=api.Denoise(iterations=0)))
    b.close()
    # features through another camera
    b = r.device_buffer()
    r.camera = other
    r.sample_features(4, b)
    r.camera = cfg.camera
    _refused(lambda: call(b), capi.ERR_BAD_ARG, "features were made through another camera")
    b.close()
    # features through several cameras
    b = r.device_buffer()
    r.sample_features(4, b)
    r.camera = other
    r.sample_features(4, b)
    r.camera = cfg.camera
    _refused(lambda: call(b), capi.ERR_BAD_ARG, "features have no single camera")
    b.close()
    # entries through another camera, through several, from the host
    for how in ("other", "mixed", "host"):
        b = r.device_buffer()
        r.sample_features(4, b)
        if how == "host":
            b.add_samples(np.ones((w * h, 3)))
        else:
            r.camera = other
            r.sample(1, b, want_stats=False)
            r.camera = cfg.camera
            if how == "mixed":
                r.sample(1, b, want_stats=False)
        _refused(lambda: call(b), capi.ERR_BAD_ARG, "another camera" if how == "other" else "no single camera")
        b.close()
    # the wavefront engine; a shard buffer
    b = r.device_buffer()
    r.sample_features(4, b)
    r.engine(capi.ENGINE_WAVEFRONT)
    _refused(lambda: call(b), capi.ERR_UNSUPPORTED, "wavefront")
    r.engine(capi.ENGINE_AUTO)
    call(b)  # the same buffer is fine with the megakernel
    with pytest.raises(capi.RptbError, match="fewer than 2 entries|no samples"):
        b.denoised_variance(GUIDE)  # one entry: refused as denoise() is
    b.close()
    s = distributed.ShardBuffer(r.device_scene(), w, h, rank=0, world=2)
    r.sample_features(4, s)
    _refused(lambda: r.sample(1, s, adaptive=crit), capi.ERR_UNSUPPORTED, "shard buffer")
    with pytest.raises(capi.RptbError, match="shard buffer"):
        s.denoised_variance(GUIDE)
    s.close()
    assert L.rptb_buffer_denoise_variance(None, None, None) == capi.ERR_BAD_ARG
    r.close()
