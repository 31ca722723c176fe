"""The device Buffer's multi-part paths on one GPU.  Under RPTB_ALLOW_REPEATED_DEVICES=1 a device listed n times is a
scene of n replicas and a whole buffer of n parts, each part with its own stream, event, scratch and tile deal (i, n) --
what a part on a distinct GPU has.  So one GPU runs what only a buffer of two or more parts runs: the copies between the
parts and the staging (copy_planes), the i > 0 branches of buffer_gather and buffer_write_back, the part loop of
buffer_order_behind, the per-replica stream and event handoffs of sample / add_samples / add_features and their
out_active summed over parts, reprojection between multi-part buffers, and shard imports into one.

Every result is compared bit for bit with the same calls on a one-replica buffer unless a reference is named:
  a. one life cycle of calls with no host read in between, then every read, then a reprojection;
  b. parts that own no tile (fewer tiles than replicas);
  c. host entries against exact sums and an exact two-pass M2 (fractions), the oracle's image and variance;
  d. shard blocks imported into a multi-part buffer, with and without features, and sampled on afterwards;
  e. a multi-part buffer outliving its scene, and giving its device memory back;
  f. the switch itself.
With two or more GPUs every case also runs on a list that alternates devices 0 and 1, so the same buffer copies both
within a device and across devices.  On one H100 80GB HBM3 at a 700 W power limit the whole file ran in 20 s."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from rpt_b200.distributed import ShardBuffer
from tests import util
from tests.test_reproject import orbit

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
PREC = [pytest.param(F32, id="f32"), pytest.param(F64, id="f64")]
CRIT = api.Adaptive(0.1, 2e-3, 2)
DENOISE = (api.Denoise(), api.Denoise(iterations=3, sigma_normal=32, sigma_luminance=2.0))
MAKE = {"sphere": scenes.sphere_scene, "cornell": scenes.cornell_scene}
CENTER = {"sphere": (0.0, -0.25, 0.0), "cornell": (278.0, 273.0, 280.0)}
EPS = float(np.finfo(np.float64).eps)


@pytest.fixture(autouse=True)
def _repeated_devices(monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")


def _lists(gpu_ok, k):
    """k replicas on device 0; with two GPUs also k replicas alternating between devices 0 and 1."""
    return [[0] * k] + ([[i % 2 for i in range(k)]] if gpu_ok >= 2 else [])


def _renderer(cfg, w, h, prec, devices, mb=3, cam=None, seed=11):
    return (api.Renderer(cfg.scene, cam or cfg.camera).width(w).height(h).max_bounces(mb).seed(seed).precision(prec)
            .device(devices))


def _adaptive(r, buf, n, out_active=True):
    """One adaptive call through the C ABI and nothing read after it (Renderer.sample reads the buffer's counts): the
    pixels that got the entry, or None without out_active, and then nothing waits for the call."""
    ds, p, cam, c = r.device_scene(), r.params(n, r._next_sample), r.camera.to_c(), CRIT.to_c()
    active = C.c_uint64(0)
    capi.check(capi.lib().rptb_sample_into_adaptive(ds.handle, C.byref(cam), C.byref(p), C.byref(c), buf.handle,
                                                    C.byref(active) if out_active else None, None), "rptb_sample_into_adaptive")
    r._next_sample += n
    return int(active.value) if out_active else None


def _script(r, buf, spp, host_entry, out_active, feature_stats=False):
    """A plain sample, the seeded host entry (when asked), a plain sample, three adaptive calls and a feature pass,
    enqueued back to back with nothing read.  Returns the adaptive calls' active counts and the feature pass's rays."""
    r.sample(spp, buf, want_stats=False)
    if host_entry:
        buf.add_samples(np.random.default_rng(7).uniform(0.0, 1.5, (buf.width * buf.height, 3)))
    r.sample(spp, buf, want_stats=False)
    active = [_adaptive(r, buf, spp, out_active) for _ in range(3)]
    r.sample_features(2, buf, want_stats=feature_stats)
    return active, (r.last_stats["rays"] if feature_stats else None)


def _state(buf):
    """The pixel state a buffer gives back: image first (the first gather), variance twice, the per-pixel planes."""
    out = {"image": buf.image(), "variance": buf.variance(), "variance again": buf.variance()}
    out["sums"], out["m2"], out["counts"] = buf.pixel_stats()
    return out


def _reads(buf):
    """_state, the resolved features and both denoisings."""
    out = _state(buf)
    out.update(zip(("normal", "depth", "albedo", "hit fraction"), buf.features()))
    for i, d in enumerate(DENOISE):
        out[f"denoise {i}"] = buf.denoise(d)
    return out


def _same(got, want, where):
    assert got.keys() == want.keys(), where
    for k in want:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        assert g.dtype == w.dtype and g.shape == w.shape and g.tobytes() == w.tobytes(), (where, k)


def _variance_is_fixed(out):
    # the variance reduction has a fixed order: the same bits on every read
    assert np.asarray(out["variance"]).tobytes() == np.asarray(out["variance again"]).tobytes()


# ---- a. one life cycle ---------------------------------------------------------------------------------------------
def _life(name, w, h, prec, devices, radii):
    """Buffer B: the script without a host entry, each adaptive call asking for its active count (a host entry would
    leave B no single camera to reproject from).  Buffer A: the script with the host entry and no out_active, so nothing
    waits until A is read.  C gets features through an orbited camera.  Then A is read while B's and C's work may still
    run, C is reprojected from B, B is read, and C is read, sampled adaptively twice and denoised."""
    cfg = MAKE[name]()
    cam = api.Camera.look_at(cfg.camera.eye, np.asarray(CENTER[name]), api.vec3(0.0, 1.0, 0.0), cfg.camera.fov)
    r = _renderer(cfg, w, h, prec, devices, cam=cam)
    ds = r.device_scene()
    a, b, c = (api.DeviceBuffer(ds, w, h, api.Filter.Box(rad)) for rad in radii)
    out = {}
    out["B active"], _ = _script(r, b, 2, host_entry=False, out_active=True)
    _script(r, a, 2, host_entry=True, out_active=False)
    r.camera = orbit(cam, CENTER[name], -0.05)
    r.sample_features(2, c)
    out.update({"A " + k: v for k, v in _reads(a).items()})
    out["C reused"] = c.reproject_from(b)
    out.update({"B " + k: v for k, v in _reads(b).items()})
    out.update({"C reprojected " + k: v for k, v in zip(("sums", "m2", "counts"), c.pixel_stats())})
    out["C active"] = [_adaptive(r, c, 2) for _ in range(2)]
    out.update({"C " + k: v for k, v in _reads(c).items()})
    for buf in (a, b, c):
        buf.close()
    r.close()
    return out


LIFE = [("cornell", 203, 117, F32, 3, (0, 1, 3)), ("cornell", 203, 117, F64, 5, (3, 0, 1)),
        ("sphere", 97, 61, F32, 8, (1, 3, 0)), ("sphere", 97, 61, F64, 2, (3, 1, 0))]


@pytest.mark.parametrize("name,w,h,prec,k,radii", LIFE, ids=[f"{c[0]}-{'f32' if c[3] == F32 else 'f64'}-{c[4]}" for c in LIFE])
def test_life_cycle_without_host_reads(gpu_ok, name, w, h, prec, k, radii):
    want = _life(name, w, h, prec, [0], radii)
    for buf in ("A", "B", "C"):
        _variance_is_fixed({key[2:]: v for key, v in want.items() if key.startswith(buf + " variance")})
    assert 0 < want["B active"][-1] < w * h and 0 < want["C reused"] < w * h
    for devices in _lists(gpu_ok, k):
        _same(_life(name, w, h, prec, devices, radii), want, devices)


# ---- b. parts that own no tile -------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PREC)
@pytest.mark.parametrize("w,h,k", [(1, 1, 3), (16, 8, 3), (17, 9, 5), (33, 8, 8)], ids=["1x1-3", "16x8-3", "17x9-5", "33x8-8"])
def test_parts_that_own_no_tile(gpu_ok, w, h, k, prec):
    assert ((w + 15) // 16) * ((h + 7) // 8) < k  # some part owns no tile

    def run(devices):
        r = _renderer(scenes.cornell_scene(), w, h, prec, devices)
        buf = r.device_buffer()
        out = {}
        out["active"], out["rays"] = _script(r, buf, 2, host_entry=True, out_active=True, feature_stats=True)
        out.update(_reads(buf))
        buf.close()
        r.close()
        return out

    want = run([0])
    assert want["rays"] == w * h * 2
    _variance_is_fixed(want)
    for devices in _lists(gpu_ok, k):
        _same(run(devices), want, devices)


# ---- c. host entries against an independent reference -------------------------------------------------------------
def _entries(kind, n, npix, seed):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.uniform(0.0, 2.0, (n, npix, 3))
    if kind == "signed":
        return rng.normal(0.0, 1.0, (n, npix, 3))
    return 1e6 + rng.normal(0.0, 1e-3, (n, npix, 3))  # M2 is ill-conditioned: |mean| / sigma ~ 1e9


def _exact(e):
    """Exactly (fractions), then rounded: per pixel and channel the mean and the two-pass sum of squared deviations, and
    per pixel that sum over the channels."""
    fr = np.frompyfunc(Fraction, 1, 1)(e)
    mean = fr.sum(axis=0) / e.shape[0]
    dev = fr - mean
    m2c = (dev * dev).sum(axis=0)
    return mean.astype(np.float64), m2c.astype(np.float64), m2c.sum(axis=1).astype(np.float64)


@pytest.mark.parametrize("kind", ["uniform", "signed", "offset"])
@pytest.mark.parametrize("w,h,k,n", [(70, 41, 3, 2), (70, 41, 3, 11), (17, 9, 5, 3), (17, 9, 5, 200)],
                         ids=["70x41-3-n2", "70x41-3-n11", "17x9-5-n3", "17x9-5-n200"])
def test_host_entries_match_an_exact_reference(orc, gpu_ok, kind, w, h, k, n):
    """add_samples alone, through the gather of a multi-part buffer.  The sums are added in entry order, so they are
    np.sum(entries, axis=0) bit for bit.  M2 is Welford's update M2 += sum_c (x_c - S_old,c / (n-1)) (x_c - S_new,c / n)
    on the running sums S.  Bound on its error, per channel: S_k, a sum of k entries, is off by at most (k-1) eps
    sum_i |x_i| <= k (k-1) eps (|mean| + sigma) to first order, so the mean it gives by at most k eps (|mean| + sigma);
    each update multiplies two deviations of size ~sigma, one of them shifted by that much, and rounds the product and
    the sum (~eps M2_k).  Summed over k <= n updates the error is at most ~n^2 eps sigma (|mean| + sigma) + n eps M2,
    and M2 ~ (n-1) sigma^2, so the relative error is O(n eps (1 + |mean| / sigma)).  The test allows
    64 n eps (1 + |mean| / sigma) relative -- in absolute terms 64 n eps (M2 + |mean| sqrt((n-1) M2)), which needs no
    division by sigma -- summed over the channels, a margin of ~30 over the first-order bound.  The exact M2 is the
    two-pass sum in fractions.  The printout gives the worst error / bound seen.  The variance is checked against the
    oracle's two passes at rtol 1e-12 where the entries are well conditioned; on 1e6 + N(0, 1e-3) the Welford M2 is
    only as good as the bound above, which then bounds the variance too."""
    npix = w * h
    e = _entries(kind, n, npix, seed=1000 * n + w)
    ds1 = api.DeviceScene(scenes.sphere_scene().scene, [0])
    ref = api.DeviceBuffer(ds1, w, h, api.Filter.Box(1))
    for x in e:
        ref.add_samples(x)
    want_state = ref.pixel_stats() + (ref.image(),)
    mean, m2c, m2 = _exact(e)
    bound = 64 * n * EPS * (m2c + np.abs(mean) * np.sqrt((n - 1) * m2c)).sum(axis=1)
    worst = 0.0
    for devices in _lists(gpu_ok, k):
        ds = api.DeviceScene(scenes.sphere_scene().scene, devices)
        dev = api.DeviceBuffer(ds, w, h, api.Filter.Box(1))
        for x in e:
            dev.add_samples(x)
        sums, got_m2, counts = dev.pixel_stats()
        assert np.array_equal(sums, np.sum(e, axis=0)), devices
        assert (counts == n).all(), devices
        err = np.abs(got_m2 - m2)
        assert (err <= bound).all(), (devices, float(np.max(err / np.where(bound > 0, bound, 1.0))))
        worst = max(worst, float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), 0.0))))
        img = dev.image()
        for g, want in zip((sums, got_m2, counts, img), want_state):
            assert g.tobytes() == want.tobytes(), devices  # and the one-replica buffer's, bit for bit
        oimg = orc.film_resolve(np.sum(e, axis=0), n, w, h, 1)
        assert (np.abs(img.astype(int) - oimg.astype(int)) <= 1).all(), devices
        assert (img == oimg).mean() > 0.999, devices
        var, ovar = dev.variance(), orc.variance(e)
        if kind == "offset":
            assert abs(var - ovar) <= np.mean(bound / (n - 1)) + 1e-12 * abs(ovar), (devices, var, ovar)
        else:
            np.testing.assert_allclose(var, ovar, rtol=1e-12)
        dev.close()
        ds.close()
    print(f"{kind} {w}x{h} n={n}: worst M2 error / bound {worst:.3g}")
    ref.close()
    ds1.close()


# ---- d. shard blocks imported into a multi-part buffer -------------------------------------------------------------
def _shard_calls(r, buf):
    r._next_sample = 0
    for _ in range(2):
        r.sample(2, buf, want_stats=False)
    r.sample_features(4, buf)
    for _ in range(3):
        r.sample(2, buf, want_stats=False, adaptive=CRIT)


def _blocks(shards, with_features):
    """torch.cat of every shard's exchange block: what the all-gather of ShardBuffer.gather gives."""
    import torch

    out = [torch.empty(s.block_bytes(with_features), dtype=torch.uint8, device="cuda:0") for s in shards]
    for s, o in zip(shards, out):
        s.export(o, with_features)
    g = torch.cat(out)
    torch.cuda.synchronize()
    return g


def _import(dst, gathered, n, with_features, feature_rays):
    capi.check(capi.lib().rptb_buffer_import_shards(dst.handle, C.c_void_p(gathered.data_ptr()), n, 1 if with_features else 0),
               "rptb_buffer_import_shards")
    dst.feature_rays = feature_rays if with_features else 0


@pytest.mark.parametrize("prec", PREC)
@pytest.mark.parametrize("n", [1, 2, 3, 5])
def test_shards_import_into_a_multi_part_buffer(gpu_ok, n, prec):
    """Shards of a one-replica scene, imported into a buffer on [0, 0, 0] and into one on [0]: with features (every part
    allocates its feature planes), then without (every part frees them), then a fresh feature pass and more entries.
    Each step's state, features and denoisings agree."""
    w, h = 97, 61
    cfg = scenes.sphere_scene()
    one = _renderer(cfg, w, h, prec, [0], mb=2)
    shards = [ShardBuffer(one.device_scene(), w, h, rank=i, world=n) for i in range(n)]
    for s in shards:
        _shard_calls(one, s)
    blocks = {wf: _blocks(shards, wf) for wf in (True, False)}

    def run(devices):
        r = _renderer(cfg, w, h, prec, devices, mb=2)
        dst = r.device_buffer()
        out = {}
        _import(dst, blocks[True], n, True, shards[0].feature_rays)
        out.update({"with " + k: v for k, v in _reads(dst).items()})
        _import(dst, blocks[False], n, False, shards[0].feature_rays)
        out.update({"without " + k: v for k, v in _state(dst).items()})
        with pytest.raises(capi.RptbError, match="no features"):
            dst.features()
        r.sample_features(4, dst)  # from nothing, as on a buffer that never had features
        out.update({"fresh " + k: v for k, v in _reads(dst).items()})
        r._next_sample = 100
        r.sample(2, dst, want_stats=False)
        out["active"] = [_adaptive(r, dst, 2) for _ in range(2)]
        out.update({"sampled " + k: v for k, v in _reads(dst).items()})
        dst.close()
        r.close()
        return out

    want = run([0])
    assert np.array_equal(want["fresh normal"], want["with normal"])  # the fresh pass is the shards' own
    for devices in _lists(gpu_ok, 3):
        _same(run(devices), want, devices)
    for s in shards:
        s.close()
    one.close()


# ---- e. lifetime and memory ----------------------------------------------------------------------------------------
def test_a_multi_part_buffer_outlives_its_scene(gpu_ok):
    cfg = scenes.sphere_scene()
    outs = []
    for devices in [[0]] + _lists(gpu_ok, 3):
        r = _renderer(cfg, 48, 32, F32, devices, mb=2)
        buf = r.device_buffer()
        r.sample(4, buf, want_stats=False)
        r.sample(4, buf, want_stats=False)  # still running when the scene goes
        r.close()
        outs.append((devices, _state(buf)))
        buf.close()
    for devices, got in outs[1:]:
        _same(got, outs[0][1], devices)


def test_multi_part_buffers_give_their_device_memory_back(gpu_ok):
    """21 buffers of 1920x1080 on three replicas keep less than 32 MB of device memory between them, read as
    test_gpu_device_buffer.py::test_buffers_give_their_device_memory_back reads it: after every buffer, the check on the
    20 smallest of 21 steps."""
    torch = pytest.importorskip("torch")
    r = _renderer(scenes.sphere_scene(), 1920, 1080, F32, [0, 0, 0], mb=0)
    warm = r.device_buffer()
    r.sample(1, warm, want_stats=False)
    warm.image()
    warm.close()  # the replicas' own scratch for this size now exists
    torch.cuda.synchronize()
    free = [torch.cuda.mem_get_info(0)[0]]
    for _ in range(21):
        b = r.device_buffer()
        r.sample(1, b, want_stats=False)
        b.image()
        b.close()
        free.append(torch.cuda.mem_get_info(0)[0])
    steps = -np.diff(np.array(free, dtype=np.int64))
    kept = int(np.sort(steps)[:-1].sum())
    assert kept <= (32 << 20), (kept / 2**20, (steps / 2**20).tolist())
    r.close()


# ---- f. the switch -------------------------------------------------------------------------------------------------
def test_the_repeated_device_switch(gpu_ok, monkeypatch):
    """Read on every rptb_scene_create_multi: without it (or with anything but 1) a repeated device is refused; with it
    each listing is a replica, and what a multi-replica scene refuses it refuses."""
    import torch

    lib = capi.lib()
    flat = api.FlatScene(scenes.sphere_scene().scene)
    two = (C.c_int * 2)(0, 0)
    h = C.c_void_p()
    for value in (None, "0", ""):
        if value is None:
            monkeypatch.delenv(util.REPEATED_DEVICES)
        else:
            monkeypatch.setenv(util.REPEATED_DEVICES, value)
        assert lib.rptb_scene_create_multi(C.byref(flat.desc), two, 2, C.byref(h)) == capi.ERR_BAD_ARG and not h
        assert "listed twice" in lib.rptb_last_error().decode()
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")
    with api.DeviceScene(flat, [0, 0]) as ds:
        assert ds.device_count() == 2
        hd = C.c_void_p()
        assert lib.rptb_buffer_create_shard(ds.handle, 32, 16, 0, 0, 2, C.byref(hd)) == capi.ERR_UNSUPPORTED and not hd
        r = _renderer(scenes.sphere_scene(), 32, 16, F32, [0, 0], mb=1)
        t = torch.empty(32 * 16 * 3, dtype=torch.float32, device="cuda:0")
        cam, p = r.camera.to_c(), r.params(1)
        assert lib.rptb_render_samples_device(ds.handle, C.byref(cam), C.byref(p), C.c_void_p(t.data_ptr()), None, None) == capi.ERR_UNSUPPORTED
    monkeypatch.delenv(util.REPEATED_DEVICES)
    assert lib.rptb_scene_create_multi(C.byref(flat.desc), two, 2, C.byref(h)) == capi.ERR_BAD_ARG and not h
