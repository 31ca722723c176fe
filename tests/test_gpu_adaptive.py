"""Adaptive sampling on the device Buffer (rptb_sample_into_adaptive) on the GPU: an active pixel gets exactly the entry
the plain render gives it, an inactive one nothing; the decisions replay in numpy; a buffer with mixed counts is the
reference's Buffer with per-pixel entry lists; and the bits do not depend on the device count."""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import util

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64


def _renderer(cfg, w, h, mb, prec=F32, radius=1, seed=5, accel=capi.ACCEL_AUTO, device=0):
    return (api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).seed(seed).precision(prec)
            .filter(api.Filter.Box(radius)).accel(accel).device(device))


def _adaptive(r, n, buf, crit, want_stats=True):
    """One adaptive call through the C ABI: (pixels that got the entry, stats dict)."""
    ds, p, cam, c = r.device_scene(), r.params(n, r._next_sample), r.camera.to_c(), crit.to_c()
    active, st = C.c_uint64(0), capi.Stats()
    capi.check(capi.lib().rptb_sample_into_adaptive(ds.handle, C.byref(cam), C.byref(p), C.byref(c), buf.handle, C.byref(active),
                                                    C.byref(st) if want_stats else None), "rptb_sample_into_adaptive")
    r._next_sample += n
    return int(active.value), st.as_dict()


def _plain_entry(r, n, first_sample):
    """rptb_render_samples of the same call: the entry every pixel would get, row-major (npix, 3)."""
    out = np.empty((r._width * r._height, 3))
    p, cam = r.params(n, first_sample), r.camera.to_c()
    capi.check(capi.lib().rptb_render_samples(r.device_scene().handle, C.byref(cam), C.byref(p), out.ctypes.data_as(capi.c_double_p),
                                              None), "rptb_render_samples")
    return out


@pytest.mark.parametrize("name,make,w,h,mb,prec", [
    ("sphere_f64", scenes.sphere_scene, 48, 32, 2, F64),
    ("cornell_f64", scenes.cornell_scene, 37, 29, 3, F64),
    ("sphere_f32", scenes.sphere_scene, 64, 40, 2, F32),
    ("cornell_f32", scenes.cornell_scene, 48, 48, 3, F32),
])
def test_always_active_is_the_plain_render(gpu_ok, name, make, w, h, mb, prec):
    cfg = make()
    ra, rp = _renderer(cfg, w, h, mb, prec), _renderer(cfg, w, h, mb, prec)
    da, dp = ra.device_buffer(), rp.device_buffer()
    crit = api.Adaptive(0.0, 0.0, 100)  # min_entries above the number of calls: every pixel stays active
    for n in (4, 3, 1, 2):
        active, sa = _adaptive(ra, n, da, crit)
        rp.sample(n, dp)
        assert active == w * h
        assert sa["segments"] == rp.last_stats["segments"] if prec == F64 else sa["segments"] > 0
    (sa_, ma, ca), (sp_, mp, cp) = da.pixel_stats(), dp.pixel_stats()
    assert (ca == 4).all() and (cp == 4).all()
    if prec == F64:
        assert np.array_equal(sa_, sp_) and np.array_equal(ma, mp)
        np.testing.assert_array_equal(da.image(), dp.image())
        assert da.variance() == dp.variance()
    else:
        np.testing.assert_allclose(sa_, sp_, rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(da.variance(), dp.variance(), rtol=1e-5)
        print(f"{name}: f32 adaptive sums bit-identical to the plain render: {np.array_equal(sa_, sp_)}")
    for x in (da, dp, ra, rp):
        x.close()


REPLAY = {  # name: (config, w, h, max_bounces, precision, renderer settings, spp per call)
    "sphere": (scenes.sphere_scene, 64, 40, 2, F32, {}, 2),
    "cornell": (scenes.cornell_scene, 48, 48, 3, F32, {}, 2),
    "glass": (lambda: scenes.glass_scene(256, 128), 64, 40, 4, F32, {}, 2),
    "teapot_bvh": (scenes.teapot_scene, 64, 40, 1, F32, {"accel": capi.ACCEL_BVH}, 2),
    "sphere_f64": (scenes.sphere_scene, 40, 24, 2, F64, {}, 2),
    "glass_f64_deep": (lambda: scenes.glass_scene(64, 32), 32, 24, 20, F64, {}, 1),   # max_bounces > 16: MAXD = 64
}


@pytest.mark.parametrize("name", sorted(REPLAY))
def test_decisions_replay_in_numpy(gpu_ok, name):
    make, w, h, mb, prec, extra, spp = REPLAY[name]
    cfg = make()
    r = _renderer(cfg, w, h, mb, prec, **extra)
    buf = r.device_buffer()
    crit = api.Adaptive(0.08, 2e-3, 3)
    _adaptive(r, spp, buf, crit)
    seen_partial = False
    for _ in range(7):
        s0, m0, c0 = buf.pixel_stats()
        mask = crit.active(c0, s0, m0)
        first = r._next_sample
        active, _ = _adaptive(r, spp, buf, crit)
        entry = _plain_entry(r, spp, first)
        s1, m1, c1 = buf.pixel_stats()
        assert active == int(mask.sum())
        assert np.array_equal(c1, c0 + mask)                                   # +1 on the mask, nowhere else
        assert np.array_equal(s1[~mask], s0[~mask]) and np.array_equal(m1[~mask], m0[~mask])
        if prec == F64:
            assert np.array_equal(s1[mask], s0[mask] + entry[mask])           # that call's plain entry, to the bit
        else:
            np.testing.assert_allclose(s1[mask], s0[mask] + entry[mask], rtol=1e-6, atol=1e-6)
        x = entry                                                              # the entry the buffer took
        n = c1.astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            welford = m0 + ((x - s0 / (n - 1)[:, None]) * (x - s1 / n[:, None])).sum(1)
        if prec == F64:
            np.testing.assert_allclose(m1[mask], welford[mask], rtol=1e-12, atol=1e-300)
        else:  # (the f32 entry of the list-scheduled kernel may round apart from the plain kernel's)
            np.testing.assert_allclose(m1[mask], welford[mask], rtol=1e-4, atol=1e-9)
        seen_partial = seen_partial or 0 < active < w * h
    assert seen_partial, "the criterion never split the image"
    buf.close()
    r.close()


def _reference_buffer(entries, takes, w, h, radius):
    """src/buffer.rs with per-pixel entry lists: entries (ncalls, npix, 3), takes (ncalls, npix) bool ->
    (image bytes (h, w, 3), variance)."""
    sums = np.zeros((h * w, 3))
    for e, t in zip(entries, takes):  # each pixel's entries summed in order, as Vec<Color>::iter().sum
        sums[t] = sums[t] + e[t]
    counts = takes.sum(0).astype(np.float64)
    S, N = sums.reshape(h, w, 3), counts.reshape(h, w)
    acc, cnt = np.zeros((h, w, 3)), np.zeros((h, w))
    for di in range(-radius, radius + 1):          # x outer, y inner: get_filtered_color's order
        for dj in range(-radius, radius + 1):
            ys, xs = slice(max(0, -dj), min(h, h - dj)), slice(max(0, -di), min(w, w - di))
            yd, xd = slice(max(0, dj), min(h, h + dj)), slice(max(0, di), min(w, w + di))
            acc[ys, xs] += S[yd, xd]
            cnt[ys, xs] += N[yd, xd]
    c = np.clip(acc / cnt[..., None], 0.0, 1.0)
    img = (np.power(c, 1.0 / 2.2) * 255.0).astype(np.uint8)
    mean = sums / counts[:, None]
    ss = np.zeros(h * w)
    for e, t in zip(entries, takes):
        d = np.where(t[:, None], e - mean, 0.0)
        ss += (d * d).sum(1)
    return img, float(np.mean(ss / (counts - 1.0)))


@pytest.mark.parametrize("radius", [0, 3])
def test_mixed_counts_are_the_reference_buffer(gpu_ok, radius):
    cfg = scenes.sphere_scene()
    w, h, spp = 203, 117, 2
    r = _renderer(cfg, w, h, 2, F64, radius=radius)
    buf = r.device_buffer()
    crit = api.Adaptive(0.1, 2e-3, 2)
    entries, takes = [], []
    for calls in range(1, 7):
        s0, m0, c0 = buf.pixel_stats()
        first = r._next_sample
        _adaptive(r, spp, buf, crit, want_stats=False)
        c1 = buf.counts().reshape(-1)
        assert c1.min() >= min(calls, 2)  # what rptb_buffer_denoise's "fewer than 2 entries" check relies on
        takes.append(c1 > c0)
        entries.append(_plain_entry(r, spp, first))
    counts = buf.counts().reshape(-1)
    assert counts.min() < counts.max()
    img, var = _reference_buffer(np.array(entries), np.array(takes), w, h, radius)
    got = buf.image()
    assert (np.abs(got.astype(int) - img.astype(int)) <= 1).all() and (got == img).mean() > 0.999
    np.testing.assert_allclose(buf.variance(), var, rtol=1e-12)
    assert buf.sums().shape == (w * h, 3) and buf.entries == counts.max()
    # a plain call, and a host entry, add to every pixel on top of its own count
    first = r._next_sample
    r.sample(spp, buf, want_stats=False)
    entries.append(_plain_entry(r, spp, first))
    takes.append(np.ones(w * h, bool))
    host = np.random.default_rng(3).uniform(0, 1, (w * h, 3))
    buf.add_samples(host)
    entries.append(host)
    takes.append(np.ones(w * h, bool))
    assert np.array_equal(buf.counts().reshape(-1), counts + 2)
    img, var = _reference_buffer(np.array(entries), np.array(takes), w, h, radius)
    got = buf.image()
    assert (np.abs(got.astype(int) - img.astype(int)) <= 1).all() and (got == img).mean() > 0.999
    np.testing.assert_allclose(buf.variance(), var, rtol=1e-12)
    buf.close()
    r.close()


def test_convergence_ends(gpu_ok):
    cfg = scenes.sphere_scene()
    w, h = 96, 54
    r = _renderer(cfg, w, h, 2)
    buf = r.device_buffer()
    crit = api.Adaptive(0.0, 0.0, 3)  # only a pixel whose entries all agree stops
    for _ in range(5):
        _adaptive(r, 2, buf, crit)
    s, m2, counts = buf.pixel_stats()
    background = (s == 0).all(1)  # the black sky: every sample 0
    assert background.sum() > 40
    assert (counts[background] == 3).all()
    assert (counts[~background & (m2 > 0)] == 5).all()
    # nothing active: no work, no change
    done = api.Adaptive(0.0, 1e9, 2)
    active, st = _adaptive(r, 2, buf, done)
    assert active == 0 and st["segments"] == 0
    s2, m22, c2 = buf.pixel_stats()
    assert np.array_equal(s2, s) and np.array_equal(m22, m2) and np.array_equal(c2, counts)
    buf.close()
    # Python: iterative_render stops after the first batch that rendered nothing
    r2 = _renderer(cfg, w, h, 2).num_samples(100)
    buf2 = r2.device_buffer()
    calls = []
    r2.iterative_render(1, lambda it, b: calls.append((it, b.entries)), buffer=buf2, adaptive=api.Adaptive(0.0, 1e9, 2))
    assert calls == [(1, 1), (2, 2)]
    assert (buf2.counts() == 2).all() and r2._next_sample == 3
    buf2.close()
    r.close()
    r2.close()


def test_any_device_count_gives_the_same_bits(gpu_ok, monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")
    cfg = scenes.cornell_scene()
    w, h = 203, 117
    crit = api.Adaptive(0.1, 2e-3, 2)
    ref = None
    for devices in util.replica_lists(gpu_ok):
        r = _renderer(cfg, w, h, 3, device=devices)
        buf = r.device_buffer()
        actives = [_adaptive(r, 2, buf, crit, want_stats=False)[0] for _ in range(5)]
        got = buf.pixel_stats() + (buf.image(), buf.variance(), actives)
        if ref is None:
            ref = got
            assert 0 < actives[-1] < w * h
        else:
            for a, b in zip(got[:4], ref[:4]):
                assert np.array_equal(a, b), devices
            assert got[4] == ref[4] and got[5] == ref[5], devices
        buf.close()
        r.close()
