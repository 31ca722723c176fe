"""The denoised image's error from two half buffers on the GPU (rptb_buffer_create_halves, rptb_buffer_half_sums,
rptb_buffer_denoise_error, rptb_sample_into_guided_error): the HALF plane against numpy's odd-entry sums over plain,
adaptive, guided and host entries; a buffer with halves against a plain one, bit for bit, for every existing read-back,
on 1 part and 2-4 replicas on a repeated device, at 128x128 and 1920x1080; E against numpy; the guided-error decisions
replayed in numpy; every refusal; and E's calibration against the variance of c' over seeds, beside v''s."""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import guided_ref as gref
from tests import halves_ref as href
from tests import util

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
GUIDE = api.Denoise(iterations=4)
MAKE = {"sphere": scenes.sphere_scene, "cornell": scenes.cornell_scene}


def _renderer(cfg, w, h, mb=3, prec=F64, seed=5, device=0):
    return api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).seed(seed).precision(prec).device(device)


def _plain_entry(r, n, first_sample):
    """rptb_render_samples of the same call: the entry every pixel would get, row-major (npix, 3)."""
    out = np.empty((r._width * r._height, 3))
    p, cam = r.params(n, first_sample), r.camera.to_c()
    capi.check(capi.lib().rptb_render_samples(r.device_scene().handle, C.byref(cam), C.byref(p), out.ctypes.data_as(capi.c_double_p),
                                              None), "rptb_render_samples")
    return out


def _state(buf):
    """(sums, m2, half, counts, nrm, z, albedo) row-major, as halves_ref takes them."""
    h, w = buf.height, buf.width
    sums, m2, counts = buf.pixel_stats()
    nrm, z, albedo, _ = buf.features()
    return (sums.reshape(h, w, 3), m2.reshape(h, w), buf.half_sums().reshape(h, w, 3), counts.reshape(h, w), nrm, z, albedo)


def _calls(r, buf, rng_host, crit_plain, crit_filter, crit_error, spp=2):
    """A sequence of every kind of entry, each yielding (the render every pixel would get, kind) before it runs: 2 plain,
    adaptive, guided on v', guided on E (twice), plain, and a host entry last (the guided calls refuse a buffer with one)."""
    kinds = ["plain", "plain", "adaptive", "filter", "error", "error", "plain", "host"]
    for kind in kinds:
        first = r._next_sample
        if kind == "host":
            x = rng_host.uniform(0, 1, (r._width * r._height, 3))
            yield x, kind
            buf.add_samples(x)
            continue
        x = _plain_entry(r, spp, first)
        yield x, kind
        crit = {"plain": None, "adaptive": crit_plain, "filter": crit_filter, "error": crit_error}[kind]
        r.sample(spp, buf, want_stats=False, adaptive=crit)


def _run(r, buf, record=None):
    crit_plain = api.Adaptive(0.05, 1e-3, 2)
    crit_filter = api.Adaptive(0.02, 1e-3, 3, guide=GUIDE)
    crit_error = api.Adaptive(0.05, 1e-3, 3, guide=GUIDE, estimate="halves")
    r.sample_features(8, buf)
    for x, kind in _calls(r, buf, np.random.default_rng(1), crit_plain, crit_filter, crit_error):
        if record is not None:
            record.append((x, buf.counts().reshape(-1).copy()))


@pytest.mark.parametrize("name", ["sphere", "cornell"])
def test_half_plane_is_the_odd_entry_sums(name):
    cfg = MAKE[name]()
    r = _renderer(cfg, 48, 32)
    with r.device_buffer(halves=True) as buf:
        rec = []
        _run(r, buf, rec)
        counts_after = buf.counts().reshape(-1)
        entries = []
        for k, (x, before) in enumerate(rec):
            after = rec[k + 1][1] if k + 1 < len(rec) else counts_after
            took = after != before
            assert np.array_equal(after[took], before[took] + 1)
            entries.append((x, took))
        assert any(not t.all() for _, t in entries)  # some calls were adaptive in effect
        assert np.array_equal(buf.half_sums(), href.odd_sums(entries))
    r.close()


def _readbacks(r, buf):
    """Every existing read-back of a buffer, and the guided decisions of one more call of each kind."""
    out = {"sums": buf.sums(), "stats": buf.pixel_stats(), "image": buf.image(), "variance": buf.variance(), "features": buf.features(),
           "denoise": buf.denoise(GUIDE), "v": buf.denoised_variance(GUIDE), "denoise0": buf.denoise(api.Denoise(iterations=0))}
    out["active_filter"] = r.sample(2, buf, want_stats=False, adaptive=api.Adaptive(0.02, 1e-3, 3, guide=GUIDE))
    out["active_plain"] = r.sample(2, buf, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 3))
    out["after"] = buf.pixel_stats()
    # a host entry last: the guided calls refuse a buffer holding one
    buf.add_samples(np.random.default_rng(2).uniform(0, 1, (buf.width * buf.height, 3)))
    out["after_host"] = (buf.pixel_stats(), buf.image(), buf.variance(), buf.denoise(GUIDE))
    return out


def _same(a, b):
    if isinstance(a, dict):
        return all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


@pytest.mark.parametrize("w,h,parts", [(128, 128, 1), (128, 128, 2), (128, 128, 3), (128, 128, 4), (1920, 1080, 1), (1920, 1080, 2)])
def test_halves_buffer_is_a_plain_buffer_bit_for_bit(w, h, parts, monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")  # replicas on a repeated device 0
    cfg = scenes.cornell_scene()
    dev = [0] * parts if parts > 1 else 0
    got = {}
    for halves in (False, True):
        r = _renderer(cfg, w, h, prec=F32, device=dev)
        buf = r.device_buffer(halves=halves)
        r.sample_features(4, buf)
        for _ in range(3):
            r.sample(2, buf, want_stats=False)
        r.sample(2, buf, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 2))
        got[halves] = _readbacks(r, buf)
        if halves:
            got["half"] = buf.half_sums()
        buf.close()
        r.close()
    assert _same(got[False], got[True])
    if parts > 1:  # the HALF plane too is the same bits for any replica count
        r = _renderer(cfg, w, h, prec=F32, device=0)
        buf = r.device_buffer(halves=True)
        r.sample_features(4, buf)
        for _ in range(3):
            r.sample(2, buf, want_stats=False)
        r.sample(2, buf, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 2))
        _readbacks(r, buf)
        assert np.array_equal(buf.half_sums(), got["half"])
        buf.close()
        r.close()


def _close(got, want, rel=1e-12):
    assert np.array_equal(np.isnan(got), np.isnan(want))
    fin = np.isfinite(want)
    scale = np.max(np.abs(want[fin]), initial=0.0)
    assert np.max(np.abs(got[fin] - want[fin]), initial=0.0) <= rel * scale


@pytest.mark.parametrize("name,prec", [("sphere", F32), ("cornell", F64)])
def test_denoised_error_matches_numpy(name, prec):
    cfg = MAKE[name]()
    r = _renderer(cfg, 64, 48, prec=prec)
    with r.device_buffer(halves=True) as buf:
        r.sample_features(8, buf)
        for _ in range(5):
            r.sample(2, buf, want_stats=False)
        r.sample(2, buf, want_stats=False, adaptive=api.Adaptive(0.1, 1e-3, 2))
        for d in (GUIDE, api.Denoise(iterations=1), api.Denoise()):
            c, v, E = href.error(*_state(buf), d)
            _close(buf.denoised_error(d), E)
            _close(buf.denoise(d), c)
            assert np.isfinite(E).all()
    r.close()


@pytest.mark.parametrize("name", ["sphere", "cornell"])
def test_guided_error_decisions_replayed_in_numpy(name):
    cfg = MAKE[name]()
    r = _renderer(cfg, 64, 48, prec=F64)
    crit = api.Adaptive(0.05, 1e-3, 3, guide=GUIDE, estimate="halves")
    with r.device_buffer(halves=True) as buf:
        r.sample_features(8, buf)
        near_total, calls, skipped = 0, 0, 0
        for _ in range(10):
            st = _state(buf)
            counts = st[3]
            if buf.entries >= crit.min_entries:
                c, _, E = href.error(*st, GUIDE)
                want, near = href.active(counts, c, E, crit).reshape(-1), href.borderline(counts, c, E, crit).reshape(-1)
            else:
                want, near = np.ones(counts.size, bool), np.zeros(counts.size, bool)
            first = r._next_sample
            active = r.sample(2, buf, want_stats=False, adaptive=crit)
            s1, _, c1 = buf.pixel_stats()
            took = c1 != counts.reshape(-1)
            assert active == int(took.sum())
            assert not np.any((took != want) & ~near), np.flatnonzero((took != want) & ~near)[:8]
            near_total += int(near.sum())
            entry = _plain_entry(r, 2, first)
            assert np.array_equal(s1[took], st[0].reshape(-1, 3)[took] + entry[took])
            calls += 1
            skipped += int((~took).sum())
        assert near_total <= max(2, calls * counts.size // 1000), near_total
        assert skipped > 0  # the criterion stopped some pixels
    r.close()


def test_refusals():
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 32, 16, prec=F32)
    L = capi.lib()
    plain, halves = r.device_buffer(), r.device_buffer(halves=True)
    for b in (plain, halves):
        r.sample_features(4, b)
        for _ in range(3):
            r.sample(2, b, want_stats=False)
    err = api.Adaptive(0.05, 1e-3, 2, guide=GUIDE, estimate="halves")
    # a buffer without halves
    with pytest.raises(capi.RptbError, match="halves"):
        plain.half_sums()
    with pytest.raises(capi.RptbError, match="halves"):
        plain.denoised_error(GUIDE)
    with pytest.raises(capi.RptbError, match="halves"):
        r.sample(2, plain, want_stats=False, adaptive=err)
    # iterations 0
    with pytest.raises(capi.RptbError, match="iterations"):
        halves.denoised_error(api.Denoise(iterations=0))
    with pytest.raises(capi.RptbError, match="iterations"):
        r.sample(2, halves, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 2, guide=api.Denoise(iterations=0), estimate="halves"))
    # the wavefront engine
    ds, cam, c, g = r.device_scene(), r.camera.to_c(), err.to_c(), GUIDE.to_c()
    p = r.params(2, r._next_sample)
    p.engine = capi.ENGINE_WAVEFRONT
    assert L.rptb_sample_into_guided_error(ds.handle, C.byref(cam), C.byref(p), C.byref(c), C.byref(g), halves.handle, None,
                                           None) == capi.ERR_UNSUPPORTED
    # a shard buffer
    from rpt_b200 import distributed
    sb = distributed.ShardBuffer(r.device_scene(), 32, 16, rank=0, world=2)
    p = r.params(2, r._next_sample, 0, 2)
    assert L.rptb_sample_into_guided_error(ds.handle, C.byref(cam), C.byref(p), C.byref(c), C.byref(g), sb.handle, None,
                                           None) == capi.ERR_UNSUPPORTED
    sb.close()
    # history has no halves: a halves dst is refused, a halves src is fine
    dst = r.device_buffer(halves=True)
    r.sample_features(4, dst)
    with pytest.raises(capi.RptbError, match="halves") as e:
        dst.reproject_from(plain)
    assert "status %d" % capi.ERR_UNSUPPORTED in str(e.value)
    for _ in range(2):
        r.sample(2, dst, want_stats=False)
    with pytest.raises(capi.RptbError, match="halves"):
        dst.merge_history_from(plain)
    fresh = r.device_buffer()
    r.sample_features(4, fresh)
    assert fresh.reproject_from(halves) > 0
    # the same refusals as denoise(): no features, fewer than 2 entries
    nf = r.device_buffer(halves=True)
    r.sample(2, nf, want_stats=False)
    with pytest.raises(capi.RptbError):
        nf.denoised_error(GUIDE)
    r.sample_features(4, nf)
    with pytest.raises(capi.RptbError, match="fewer than 2"):
        nf.denoised_error(GUIDE)
    for b in (plain, halves, dst, fresh, nf):
        b.close()
    r.close()


def test_iterative_render_makes_a_halves_buffer():
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 32, 24, prec=F32).num_samples(16)
    seen = []
    r.iterative_render(2, lambda i, b: seen.append((i, b.halves, int(b.counts().sum()))),
                       adaptive=api.Adaptive(0.05, 1e-3, 3, guide=GUIDE, estimate="halves"))
    assert seen and all(h for _, h, _ in seen)
    with pytest.raises(TypeError):  # the filter estimate still needs a buffer given
        r.iterative_render(2, lambda i, b: None, adaptive=api.Adaptive(guide=GUIDE))
    r.close()


def _calibration(name, d, fixed_features, seeds=16, w=128, h=128):
    """median over pixels of (variance of c' over the seeds) / (mean of E) and / (mean of v'), for filter parameters d.
    Each seed renders 8 entries of 2 spp and 16 feature rays; fixed_features: the feature rays of one seed for all."""
    cfg = MAKE[name]()
    cs, Es, vs = [], [], []
    for k in range(seeds):
        r = _renderer(cfg, w, h, prec=F32, seed=1000 + k)
        with r.device_buffer(halves=True) as b:
            if fixed_features:
                rf = _renderer(cfg, w, h, prec=F32, seed=999)
                rf.sample_features(16, b)
                rf.close()
            for _ in range(8):
                r.sample(2, b, want_stats=False)
            if not fixed_features:
                r.sample_features(16, b)
            cs.append(b.denoise(d))
            Es.append(b.denoised_error(d))
            vs.append(b.denoised_variance(d))
        r.close()
    emp = np.var(np.stack(cs), axis=0, ddof=1).mean(-1)
    Ebar, vbar = np.mean(Es, 0), np.mean(vs, 0)
    ok = np.isfinite(emp) & (Ebar > 0) & (vbar > 0) & np.isfinite(Ebar) & np.isfinite(vbar)
    return float(np.median(emp[ok] / Ebar[ok])), float(np.median(emp[ok] / vbar[ok]))


@pytest.mark.parametrize("name", ["sphere", "cornell"])
def test_calibration(name):
    """E is unbiased for the variance of c' under weights that do not depend on the entries: with the features of one seed
    for every seed and the luminance edge-stop off (sigma_luminance 1e9), the median ratio of the variance of c' over
    the seeds to E lies in [1/3, 3].  In the section 3.0f protocol (each seed its own features, Denoise()) the weights
    follow each seed's features and noise, which E, computed under that seed's weights, does not see: E is then reported
    beside v' and must be closer to the empirical variance than v' (DESIGN.md section 6g)."""
    rE, rv = _calibration(name, api.Denoise(sigma_luminance=1e9), True)
    dE, dv = _calibration(name, api.Denoise(), False)
    print(f"\n{name} fixed weights: median(var c' / E) = {rE:.3f}, median(var c' / v') = {rv:.3f}; "
          f"Denoise(), own features: median(var c' / E) = {dE:.3f}, median(var c' / v') = {dv:.3f}")
    assert 1.0 / 3.0 <= rE <= 3.0, rE
    assert abs(np.log(rE)) < abs(np.log(rv)), (rE, rv)
    assert abs(np.log(dE)) < abs(np.log(dv)), (dE, dv)
