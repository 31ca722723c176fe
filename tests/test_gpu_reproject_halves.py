"""Reprojected history with halves on the GPU (rptb_buffer_reproject, _merge and their shard forms into buffers with
halves): the kernels against numpy (tests/reproject_halves_ref.py) on the pre-call state; a dst with halves against a
plain dst given the same calls, bit for bit; the error-guided call after a reprojection, replayed in numpy; replicas of
2-8 parts on a repeated device against one part; shards of 1-8 reprojected or merged from a gathered whole buffer with
halves and then driven by error-guided calls with deltas, against the whole-buffer sequence after every call; and every
refusal, by code and text."""
import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from rpt_b200.distributed import ShardBuffer
from tests import halves_ref as href
from tests import reproject_halves_ref as hr
from tests import util
from tests.test_gpu_halves_shard import _deltas, _full, _import, _same_state
from tests.test_reproject import orbit

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
CENTER = (0.0, 0.5, 0.0)  # above the sphere: the upper part of the view sees the environment
GUIDE = api.Denoise()
CRIT_E = api.Adaptive(0.05, 1e-3, 3, guide=GUIDE, estimate="halves")
PRM = api.Reproject()
GAMMA = api.HistoryTest().gamma
MODES = ["reproject", "merge"]


def _cameras(angle=0.07):
    a = api.Camera.look_at(api.vec3(0.3, 0.6, 4.5), np.asarray(CENTER), api.vec3(0.0, 1.0, 0.0), 0.7)
    return a, orbit(a, CENTER, angle, lift=0.05)


def _renderer(cam, w, h, prec=F64, device=0):
    cfg = scenes.sphere_scene()
    return api.Renderer(cfg.scene, cam).width(w).height(h).max_bounces(2).seed(5).precision(prec).device(device)


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


def _source(r, cam, w, h, ds, halves=True):
    """A whole buffer through `cam` at w x h: three plain entries (one adaptive, so counts differ) and 16 feature rays."""
    own = (r.camera, r._width, r._height)
    r.camera, r._width, r._height = cam, w, h
    r._next_sample = 0
    src = api.DeviceBuffer(ds, w, h, halves=halves)
    for k in range(4):
        r.sample(2, src, want_stats=False, adaptive=api.Adaptive(0.1, 1e-3, 2) if k == 3 else None)
    r.sample_features(16, src)
    r.camera, r._width, r._height = own
    return src


def _prepare(r, buf, mode):
    """dst's 16 feature rays through the renderer's camera, and for a merge two fresh entries from sample 100 on."""
    r.sample_features(16, buf)
    if mode == "merge":
        r._next_sample = 100
        for _ in range(2):
            r.sample(2, buf, want_stats=False)


def _carry(buf, src, mode):
    if mode == "merge":
        return buf.merge_history_from(src, PRM, api.HistoryTest(GAMMA))
    return buf.reproject_from(src, PRM)


def _state(buf):
    h, w = buf.height, buf.width
    s, m, c = buf.pixel_stats()
    return s.reshape(h, w, 3), m.reshape(h, w), c.reshape(h, w), buf.half_sums().reshape(h, w, 3)


def _want(src, dst, scam, dcam, mode):
    ss, sm, sc, sh = _state(src)
    sN, sz, _, sf = src.features()
    dN, dz, _, df = dst.features()
    if mode == "merge":
        return hr.reproject_merge(dcam, dN, dz, df, scam, ss, sm, sc, sh, sN, sz, sf, PRM, GAMMA, *_state(dst))[:4]
    return hr.reproject(dcam, dN, dz, df, scam, ss, sm, sc, sh, sN, sz, sf, PRM)


def _close(got, want, rel=1e-12):
    fin = np.isfinite(want)
    assert np.array_equal(fin, np.isfinite(got))
    assert np.max(np.abs(got[fin] - want[fin]), initial=0.0) <= rel * np.max(np.abs(want[fin]), initial=1e-300)


def _check(buf, want):
    s, m, c, h = _state(buf)
    assert np.array_equal(c, want[2])
    for g, w in ((s, want[0]), (m, want[1]), (h, want[3])):
        _close(g, w)


def _reads(r, buf):
    """Every read-back of a carried buffer once two adaptive entries have given every pixel two or more entries."""
    r._next_sample = 200
    for _ in range(2):
        r.sample(2, buf, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 2))
    return [*buf.pixel_stats(), buf.image(), np.float64(buf.variance()), buf.denoise(GUIDE)]


@pytest.mark.parametrize("prec", [F32, F64])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("dsize,ssize", [((64, 48), (64, 48)), ((61, 37), (50, 44))])
def test_matches_numpy_and_the_plain_dst(gpu_ok, dsize, ssize, mode, prec):
    (w, h), (sw, sh) = dsize, ssize
    a, b = _cameras()
    r = _renderer(b, w, h, prec)
    ds = r.device_scene()
    src = _source(r, a, sw, sh, ds)
    got = {}
    for halves in (True, False):
        dst = api.DeviceBuffer(ds, w, h, halves=halves)
        _prepare(r, dst, mode)
        want = _want(src, dst, a, b, mode) if halves else None
        counts = _carry(dst, src, mode)
        if halves:
            _check(dst, want)
            assert (want[2] % 2 == 1).any() and (want[2] % 2 == 0).any()
            if mode == "reproject":
                assert counts == int((want[2] > 0).sum()) and 0 < counts < w * h
        got[halves] = (counts, dst.pixel_stats(), _reads(r, dst))
        dst.close()
    assert got[True][0] == got[False][0]
    for x, y in zip(got[True][1] + tuple(got[True][2]), got[False][1] + tuple(got[False][2])):
        assert _bits(x) == _bits(y)
    src.close()
    r.close()


@pytest.mark.parametrize("mode", MODES)
def test_error_guided_call_after_the_carry(gpu_ok, mode):
    """An estimate="halves" guided call on a carried buffer renders every pixel with 0 or 1 entries, and its decisions
    replay in numpy from the buffer's state (E from halves_ref)."""
    w, h = 64, 48
    a, b = _cameras()
    r = _renderer(b, w, h, F64)
    ds = r.device_scene()
    src = _source(r, a, w, h, ds)
    buf = api.DeviceBuffer(ds, w, h, halves=True)
    _prepare(r, buf, mode)
    _carry(buf, src, mode)
    r._next_sample = 300
    skipped = 0
    for k in range(4):
        s0, m0, c0, h0 = _state(buf)
        nrm, z, albedo, _ = buf.features()
        c, _, E = href.error(s0, m0, h0, c0, nrm, z, albedo, GUIDE)
        want, near = href.active(c0, c, E, CRIT_E).reshape(-1), href.borderline(c0, c, E, CRIT_E).reshape(-1)
        active = r.sample(2, buf, want_stats=False, adaptive=CRIT_E)
        took = buf.counts().reshape(-1) != c0.reshape(-1)
        assert active == int(took.sum())
        assert took[c0.reshape(-1) <= 1].all()
        if k == 0 and mode == "reproject":
            assert (c0 <= 1).any()
        assert not np.any((took != want) & ~near), np.flatnonzero((took != want) & ~near)[:8]
        assert int(near.sum()) <= 2
        skipped += int((~took).sum())
    assert skipped > 0  # E stopped some pixels
    for x in (src, buf):
        x.close()
    r.close()


@pytest.mark.parametrize("parts", [2, 3, 5, 8])
def test_replicas_are_one_part(gpu_ok, parts, monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")  # replicas on a repeated device 0
    w, h = 97, 61
    a, b = _cameras()
    got = {}
    for dev in (0, [0] * parts):
        r = _renderer(b, w, h, F32, device=dev)
        ds = r.device_scene()
        src = _source(r, a, w, h, ds)
        out = []
        for mode in MODES:
            dst = api.DeviceBuffer(ds, w, h, halves=True)
            _prepare(r, dst, mode)
            out.append(_carry(dst, src, mode))
            out += [*dst.pixel_stats(), dst.half_sums()]
            r._next_sample = 200
            for _ in range(2):  # every pixel then holds 2 or more entries
                r.sample(2, dst, want_stats=False, adaptive=CRIT_E)
            out += [*dst.pixel_stats(), dst.half_sums(), dst.denoised_error(GUIDE)]
            dst.close()
        got[isinstance(dev, list)] = out
        src.close()
        r.close()
    assert len(got[True]) == len(got[False])
    for x, y in zip(got[True], got[False]):
        assert _bits(np.asarray(x)) == _bits(np.asarray(y))


def _shard_sequence(r, ds, src, w, h, n, mode, calls):
    """The whole-buffer sequence and n shards given the same carry from `src`, then `calls` E-guided calls: the shards
    decide over a gathered whole buffer kept current by deltas, and after every call it equals the whole buffer."""
    whole = api.DeviceBuffer(ds, w, h, halves=True)
    shards = [ShardBuffer(ds, w, h, rank=i, world=n, halves=True) for i in range(n)]
    for buf in [whole] + shards:
        _prepare(r, buf, mode)
    want = _carry(whole, src, mode)
    got = [_carry(s, src, mode) for s in shards]
    if mode == "merge":
        assert tuple(map(sum, zip(*got))) == want
    else:
        assert sum(got) == want
    synced = _full(shards, ds, w, h)
    _same_state(synced, whole)
    for k in range(calls):
        r._next_sample = 300 + 2 * k
        total = r.sample(2, whole, want_stats=False, adaptive=CRIT_E)
        actives = []
        for s in shards:
            r._next_sample = 300 + 2 * k
            actives.append(r.sample(2, s, want_stats=False, adaptive=CRIT_E, guide_buffer=synced))
        assert sum(actives) == total, (k, actives, total)
        cap = max(actives)
        gathered, pixels = _deltas(shards, cap)
        assert pixels == actives
        assert _import(synced, gathered, n, cap) == capi.OK, capi.lib().rptb_last_error()
        _same_state(synced, whole)
    for buf in [whole, synced] + shards:
        buf.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("dsize,ssize", [((128, 96), (128, 96)), ((97, 61), (80, 70)), ((20, 10), (24, 14))])
def test_shards_follow_the_whole_buffer(gpu_ok, dsize, ssize, mode):
    (w, h), (sw, sh) = dsize, ssize
    a, b = _cameras()
    r = _renderer(b, w, h, F32)
    ds = r.device_scene()
    src = _source(r, a, sw, sh, ds)
    for n in range(1, 9):  # 20x10 is 4 tiles: shards 4.. of 5 to 8 own none
        _shard_sequence(r, ds, src, w, h, n, mode, calls=3)
    src.close()
    r.close()


@pytest.mark.parametrize("mode", MODES)
def test_shards_at_1080p(gpu_ok, mode):
    w, h = 1920, 1080
    a, b = _cameras()
    r = _renderer(b, w, h, F32)
    ds = r.device_scene()
    src = _source(r, a, w, h, ds)
    _shard_sequence(r, ds, src, w, h, 3, mode, calls=2)
    src.close()
    r.close()


def _refused(fn, code, text):
    with pytest.raises(capi.RptbError) as e:
        fn()
    assert f"status {code}:" in str(e.value) and text in str(e.value), str(e.value)


def test_refusals(gpu_ok):
    w, h = 40, 24
    a, b = _cameras()
    r = _renderer(b, w, h, F32)
    ds = r.device_scene()
    BAD, UNSUP = capi.ERR_BAD_ARG, capi.ERR_UNSUPPORTED
    plain_src, halves_src = _source(r, a, w, h, ds, halves=False), _source(r, a, w, h, ds)
    # a dst with halves from a plain src: whole and shard, reprojection and merge
    for mode in MODES:
        for make in (lambda: api.DeviceBuffer(ds, w, h, halves=True), lambda: ShardBuffer(ds, w, h, rank=1, world=3, halves=True)):
            dst = make()
            _prepare(r, dst, mode)
            _refused(lambda: _carry(dst, plain_src, mode), UNSUP, "halves")
            _carry(dst, halves_src, mode)  # the same dst takes a src with halves
            dst.close()
    # a plain dst takes a src with halves and gives a plain one's bits
    got = []
    for src in (plain_src, halves_src):
        dst = api.DeviceBuffer(ds, w, h)
        _prepare(r, dst, "reproject")
        got.append((_carry(dst, src, "reproject"), dst.pixel_stats()))
        dst.close()
    assert got[0][0] == got[1][0] and all(_bits(x) == _bits(y) for x, y in zip(got[0][1], got[1][1]))
    # kept refusals: a shard src, a whole dst through the shard entry, a dst holding entries, an open aperture
    shard_src = ShardBuffer(ds, w, h, rank=0, world=2, halves=True)
    r.sample(2, shard_src, want_stats=False)
    r.sample_features(4, shard_src)
    dst = api.DeviceBuffer(ds, w, h, halves=True)
    _prepare(r, dst, "reproject")
    _refused(lambda: dst.reproject_from(shard_src), UNSUP, "shard buffer")
    _refused(lambda: ShardBuffer.reproject_from(dst, halves_src), BAD, "not a shard buffer")
    dst.reproject_from(halves_src)
    _refused(lambda: dst.reproject_from(halves_src), BAD, "already holds entries")
    _refused(lambda: dst.merge_history_from(halves_src), BAD, "already reprojected")
    ap = api.DeviceBuffer(ds, w, h, halves=True)
    r.camera = api.Camera(b.eye, b.direction, b.up, b.fov).focus(np.asarray(CENTER), 0.05)
    r.sample_features(4, ap)
    _refused(lambda: ap.reproject_from(halves_src), UNSUP, "aperture")
    r.camera = b
    for x in (plain_src, halves_src, shard_src, dst, ap):
        x.close()
    r.close()
