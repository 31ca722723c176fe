"""Reprojection on the GPU: the kernel against its numpy restatement on the buffers' own state, the identity camera, the
same bits for every device count, what a reprojected buffer's image / variance / denoise / adaptive calls do, every
error of rptb_buffer_reproject, and the quality it buys on a short orbit of the sphere and of Cornell."""
import ctypes as C
import math

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import reproject_ref as ref
from tests import util
from tests.test_reproject import orbit

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
CENTER = {"sphere": (0.0, -0.25, 0.0), "cornell": (278.0, 273.0, 280.0)}
MAKE = {"sphere": scenes.sphere_scene, "cornell": scenes.cornell_scene}


def _setup(name):
    cfg = MAKE[name]()
    cam = api.Camera.look_at(cfg.camera.eye, np.asarray(CENTER[name]), api.vec3(0.0, 1.0, 0.0), cfg.camera.fov)
    return cfg, cam


def _renderer(cfg, cam, w, h, mb=3, prec=F32, seed=5, device=0):
    return api.Renderer(cfg.scene, cam).width(w).height(h).max_bounces(mb).seed(seed).precision(prec).device(device)


def _src(r, entries, spp, fspp, adaptive=None):
    buf = r.device_buffer()
    for _ in range(entries):
        r.sample(spp, buf, want_stats=False, adaptive=adaptive)
    r.sample_features(fspp, buf)
    return buf


def _dst(r, cam, w, h, fspp):
    r.camera = cam
    r.width(w).height(h)
    buf = r.device_buffer()
    r.sample_features(fspp, buf)
    return buf


def _want(src, dst, scam, dcam, prm):
    sums, m2, counts = src.pixel_stats()
    sN, sz, _, sf = src.features()
    dN, dz, _, df = dst.features()
    h, w = sz.shape
    return ref.reproject(dcam, dN, dz, df, scam, sums.reshape(h, w, 3), m2.reshape(h, w), counts.reshape(h, w), sN, sz, sf, prm)


def _check(got, want):
    (gs, gm, gc), (ws, wm, wc) = got, want
    h, w = wc.shape
    assert np.array_equal(gc.reshape(h, w), wc)
    assert np.max(np.abs(gs.reshape(h, w, 3) - ws)) <= 1e-12 * np.abs(ws).max()
    assert np.max(np.abs(gm.reshape(h, w) - wm)) <= 1e-12 * np.abs(wm).max()


@pytest.mark.parametrize("prec,adaptive,dsize", [(F32, False, (61, 47)), (F64, False, (50, 40)), (F32, True, (45, 52)),
                                                 (F64, True, (61, 47))], ids=["f32-uniform", "f64-uniform-resized", "f32-adaptive-resized",
                                                                              "f64-adaptive"])
def test_kernel_matches_numpy_on_the_buffer_state(gpu_ok, prec, adaptive, dsize):
    cfg, scam = _setup("cornell")
    dcam = orbit(scam, CENTER["cornell"], 0.04, lift=5.0)
    w, h = 61, 47
    r = _renderer(cfg, scam, w, h, prec=prec)
    src = _src(r, 5, 2, 4, adaptive=api.Adaptive(0.05, 1e-3, 3) if adaptive else None)
    if adaptive:
        c = src.counts()
        assert c.min() >= 3 and c.max() > c.min()
    dst = _dst(r, dcam, *dsize, 4)
    prm = api.Reproject()
    want = _want(src, dst, scam, dcam, prm)
    reused = dst.reproject_from(src, prm)
    _check(dst.pixel_stats(), want)
    assert reused == int((want[2] > 0).sum()) and reused > 0.5 * want[2].size
    assert dst.entries == int(want[2].max())
    # other parameters, into a fresh buffer
    prm2 = api.Reproject(depth_tol=0.01, normal_cos=0.99, max_history=3)
    dst2 = _dst(r, dcam, *dsize, 4)
    dst2.reproject_from(src, prm2)
    _check(dst2.pixel_stats(), _want(src, dst2, scam, dcam, prm2))


def test_identity_keeps_the_mean(gpu_ok):
    cfg, cam = _setup("sphere")
    w, h, n = 48, 36, 4
    r = _renderer(cfg, cam, w, h)
    src = _src(r, n, 2, 4)
    dst = _dst(r, cam, w, h, 4)
    assert all(np.array_equal(a, b) for a, b in zip(src.features(), dst.features()))
    for mh in (32, 3):
        d = _dst(r, cam, w, h, 4)
        assert d.reproject_from(src, api.Reproject(max_history=mh)) == w * h
        sums, m2, counts = d.pixel_stats()
        assert (counts == min(n, mh)).all()
        s0, m0, _ = src.pixel_stats()
        mean = s0 / n
        assert np.max(np.abs(sums / counts[:, None] - mean)) <= 1e-12 * np.abs(mean).max()
        assert np.max(np.abs(m2 / (counts - 1.0) - m0 / (n - 1.0))) <= 1e-12 * (m0 / (n - 1.0)).max()


def test_same_bits_for_every_device_count(gpu_ok, monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")
    cfg, scam = _setup("cornell")
    dcam = orbit(scam, CENTER["cornell"], -0.05)
    lists = util.replica_lists(gpu_ok)
    outs = []
    for devices in lists:
        r = _renderer(cfg, scam, 53, 37, device=devices)
        src = _src(r, 3, 2, 3)
        dst = _dst(r, dcam, 47, 41, 3)
        reused = dst.reproject_from(src)
        outs.append((reused,) + dst.pixel_stats())
        for b in (src, dst):
            b.close()
        r.close()
    for devices, o in zip(lists[1:], outs[1:]):
        assert o[0] == outs[0][0] and all(np.array_equal(x, y) for x, y in zip(o[1:], outs[0][1:])), devices


def test_a_reprojected_buffer_renders_its_holes_first(gpu_ok):
    cfg, scam = _setup("sphere")
    w, h = 48, 36
    dcam = orbit(scam, CENTER["sphere"], 0.3, lift=0.5)
    r = _renderer(cfg, scam, w, h)
    src = _src(r, 3, 2, 4)
    dst = _dst(r, dcam, w, h, 4)
    dst.reproject_from(src)
    counts = dst.counts()
    holes = counts == 0
    assert holes.any() and (~holes).any()
    with pytest.raises(capi.RptbError, match="no samples"):
        dst.image()
    with pytest.raises(capi.RptbError, match="status -1.*no samples"):
        dst.denoise()
    assert math.isnan(dst.variance())
    # the entry a plain render of the same samples gives
    plain_r = _renderer(cfg, dcam, w, h)
    plain_r._next_sample = r._next_sample
    plain = plain_r.device_buffer()
    plain_r.sample(2, plain, want_stats=False)
    crit = api.Adaptive(0.05, 1e-3, 2)
    before = dst.pixel_stats()
    active = r.sample(2, dst, adaptive=crit)
    assert active >= int(holes.sum())
    sums, _, after = dst.pixel_stats()
    want = plain.sums()
    assert (after[holes.ravel()] == 1).all()
    assert np.array_equal(sums[holes.ravel()], want[holes.ravel()])
    kept = ~holes.ravel() & (after == before[2])
    assert np.array_equal(sums[kept], before[0][kept])
    assert dst.image().shape == (h, w, 3)
    assert math.isnan(dst.variance())
    with pytest.raises(capi.RptbError, match="status -1.*fewer than 2"):
        dst.denoise()
    r.sample(2, dst, adaptive=crit)
    assert dst.counts().min() >= 2
    assert np.isfinite(dst.variance()) and np.isfinite(dst.denoise()).all()


def _rc(dst, src, prm=None):
    c = (prm or api.Reproject()).to_c()
    return capi.lib().rptb_buffer_reproject(dst.handle, src.handle, C.byref(c), None), capi.lib().rptb_last_error().decode()


def test_errors(gpu_ok, monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")
    cfg, cam = _setup("sphere")
    other = orbit(cam, CENTER["sphere"], 0.1)
    w, h = 16, 12
    r = _renderer(cfg, cam, w, h)
    good = _src(r, 2, 1, 1)
    fresh = _dst(r, other, w, h, 1)
    bare = r.device_buffer()  # no features, no entries
    assert _rc(fresh, fresh)[0] == capi.ERR_BAD_ARG
    assert _rc(bare, good) == (capi.ERR_BAD_ARG, "dst holds no features (rptb_buffer_add_features)")
    assert _rc(good, good)[0] == capi.ERR_BAD_ARG
    full = _src(r, 1, 1, 1)
    rc = _rc(full, good)
    assert rc[0] == capi.ERR_BAD_ARG and "already holds entries" in rc[1]
    r.camera = cam
    nofeat = r.device_buffer()
    r.sample(1, nofeat, want_stats=False)
    assert _rc(fresh, nofeat) == (capi.ERR_BAD_ARG, "src holds no features (rptb_buffer_add_features)")
    noent = r.device_buffer()
    r.sample_features(1, noent)
    assert _rc(fresh, noent) == (capi.ERR_BAD_ARG, "src holds no entries")

    def src_with(entry_cams, feat_cams, host=False):
        b = r.device_buffer()
        for c in entry_cams:
            r.camera = c
            r.sample(1, b, want_stats=False)
        if host:
            b.add_samples(np.zeros((w * h, 3)))
        for c in feat_cams:
            r.camera = c
            r.sample_features(1, b)
        r.camera = cam
        return b

    for b, what in ((src_with([cam, other], [cam]), "entries have no single camera: mixed"),
                    (src_with([cam], [cam, other]), "features have no single camera: mixed"),
                    (src_with([cam], [cam], host=True), "entries have no single camera: unknown"),
                    (src_with([other], [cam]), "different cameras")):
        rc = _rc(fresh, b)
        assert rc[0] == capi.ERR_BAD_ARG and what in rc[1], rc
    mixed_dst = src_with([], [other, cam])
    rc = _rc(mixed_dst, good)
    assert rc[0] == capi.ERR_BAD_ARG and "dst's features have no single camera: mixed" in rc[1]
    # the same camera again is one camera
    assert _rc(src_with([], [other, other]), src_with([cam, cam], [cam, cam]))[0] == capi.OK
    # an open aperture on either side
    focused = api.Camera(cam.eye, cam.direction, cam.up, cam.fov).focus(np.asarray(CENTER["sphere"]), 0.05)
    rc = _rc(fresh, src_with([focused], [focused]))
    assert rc[0] == capi.ERR_UNSUPPORTED and "aperture" in rc[1]
    rc = _rc(src_with([], [focused]), good)
    assert rc[0] == capi.ERR_UNSUPPORTED and "aperture" in rc[1]
    # buffers of scenes with other device lists: two replicas on one device against one, and another GPU
    for devices in [[0, 0]] + ([[1]] if gpu_ok >= 2 else []):
        r1 = _renderer(cfg, other, w, h, device=devices)
        on1 = r1.device_buffer()
        r1.sample_features(1, on1)
        rc = _rc(on1, good)
        assert rc[0] == capi.ERR_BAD_ARG and "device lists" in rc[1], devices
        r1.camera = cam
        src1 = _src(r1, 2, 1, 1)
        rc = _rc(fresh, src1)
        assert rc[0] == capi.ERR_BAD_ARG and "device lists" in rc[1], devices
        for b in (on1, src1):
            b.close()
        r1.close()
    # and nothing it refused touched dst
    assert fresh.reproject_from(good) > 0


# Floors on MSE(fresh) / MSE(reprojected) over frames 1.. of a six-frame orbit with the default Reproject(), each about
# 15 % below the ratio measured on an H100 80GB HBM3 (700 W): the renders are seeded, so the ratios move only if the
# kernels' rounding does.  Measured: sphere 4.80, Cornell 3.37.
QUALITY = {"sphere": 4.1, "cornell": 2.9}


@pytest.mark.parametrize("name", sorted(QUALITY))
def test_reprojection_beats_fresh_frames_on_an_orbit(gpu_ok, name):
    cfg, cam = _setup(name)
    w, h, frames, step = 96, 72, 6, 0.03
    cams = [orbit(cam, CENTER[name], step * i) for i in range(frames)]
    truth = []
    rr = _renderer(cfg, cam, w, h, mb=4, seed=999)
    for c in cams:
        rr.camera = c
        b = rr.device_buffer()
        for _ in range(8):
            rr.sample(64, b, want_stats=False)
        truth.append(b.image().astype(np.float64) / 255.0)
        b.close()

    def mse(reproject):
        r = _renderer(cfg, cam, w, h, mb=4, seed=1).num_samples(8)
        imgs = list(r.render_frames(cams, entries=4, feature_samples=8, reproject=reproject))
        return [float(np.mean((im / 255.0 - t) ** 2)) for im, t in zip(imgs, truth)]

    fresh, rep = mse(None), mse(api.Reproject())
    assert fresh[0] == rep[0]
    ratio = sum(fresh[1:]) / sum(rep[1:])
    print(name, "mse fresh", fresh, "reprojected", rep, "ratio", ratio)
    assert all(b < a for a, b in zip(fresh[2:], rep[2:]))
    assert ratio >= QUALITY[name]


def test_render_frames_adaptive_and_denoised(gpu_ok):
    cfg, cam = _setup("sphere")
    cams = [orbit(cam, CENTER["sphere"], 0.05 * i) for i in range(3)]
    r = _renderer(cfg, cam, 32, 24).num_samples(8)
    out = list(r.render_frames(cams, entries=4, feature_samples=2, adaptive=api.Adaptive(0.05, 1e-3, 2), denoise=api.Denoise()))
    assert len(out) == 3 and all(o.shape == (24, 32, 3) and o.dtype == np.uint8 for o in out)
    assert r.camera is cam
    with pytest.raises(ValueError):
        next(r.render_frames(cams, entries=3))
