"""The denoiser on the GPU: the feature pass against closest-hit queries, the filter against its numpy restatement on the
buffer's own state, the bytes path, the identity, device-count independence, and the quality it buys on Cornell, the
sphere and the BVH teapot against a high-spp reference."""

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import denoise_ref as ref
from tests import util

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64


def _renderer(cfg, w, h, mb, prec=F32, seed=5, device=0):
    return api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).seed(seed).precision(prec).device(device)


# f32 floors: the host emulation's (tests/test_denoise.py FEATURE_SCENES), where they are justified by what it measures
@pytest.mark.parametrize("name,make,w,h,spp,floor", [("sphere", scenes.sphere_scene, 33, 21, 3, 0.97),
                                                     ("cornell", scenes.cornell_scene, 29, 23, 3, 0.97),
                                                     ("teapot", scenes.teapot_scene, 24, 18, 2, 0.95)])
def test_f64_features_are_the_closest_hit_sums(gpu_ok, name, make, w, h, spp, floor):
    cfg = make()
    r = _renderer(cfg, w, h, 2, F64, seed=9)
    buf = r.device_buffer()
    r.sample_features(spp, buf, want_stats=True)
    assert r.last_stats["rays"] == w * h * spp
    rays = ref.camera_rays(cfg.camera.to_c(), w, h, spp, 9)
    t, obj, nrm = r.device_scene().closest_hit(rays.reshape(-1, 6), precision=F64)
    sn, sa, hits, sz = ref.feature_sums(rays, t, obj, nrm, ref.object_colors(api.FlatScene(cfg.scene)))
    N, z, a, f = ref.features_resolve(hits, sn, sz, sa, float(spp))
    gN, gz, ga, gf = buf.features()
    assert np.array_equal(gN.reshape(-1, 3), N) and np.array_equal(gz.ravel(), z)
    assert np.array_equal(ga.reshape(-1, 3), a) and np.array_equal(gf.ravel(), f)
    # the f32 pass: the host-emulation floors
    r32 = _renderer(cfg, w, h, 2, F32, seed=9)
    b32 = r32.device_buffer()
    r32.sample_features(spp, b32)
    _, z32, _, f32 = b32.features()
    same = f32.ravel() == f
    with np.errstate(invalid="ignore"):
        close = np.where(np.isfinite(z), np.abs(z32.ravel() - z) <= 1e-4 * np.abs(z), True)
    print(name, "f32 features agreeing", (same & close).mean())
    assert (same & close).mean() >= floor


def _buffer(cfg, w, h, mb, entries, spp, fspp, adaptive=None, device=0, seed=5):
    r = _renderer(cfg, w, h, mb, seed=seed, device=device)
    buf = r.device_buffer()
    for _ in range(entries):
        r.sample(spp, buf, want_stats=False, adaptive=adaptive)
    r.sample_features(fspp, buf)
    return r, buf


@pytest.mark.parametrize("adaptive", [None, api.Adaptive(0.05, 1e-3, 3)], ids=["uniform", "adaptive"])
def test_filter_matches_numpy_on_the_buffer_state(gpu_ok, adaptive):
    cfg = scenes.cornell_scene()
    w, h = 61, 47
    r, buf = _buffer(cfg, w, h, 4, 6, 2, 4, adaptive=adaptive)
    sums, m2, counts = buf.pixel_stats()
    N, z, a, _ = buf.features()
    if adaptive is not None:
        assert counts.min() >= 3 and counts.max() > counts.min()
    for d in (api.Denoise(), api.Denoise(iterations=3, sigma_normal=32, sigma_luminance=2.0)):
        got = buf.denoise(d)
        want = ref.denoise(sums.reshape(h, w, 3), m2.reshape(h, w), counts.reshape(h, w), N, z, a, d)
        assert np.isfinite(got).all()
        assert np.max(np.abs(got - want)) <= 1e-12 * np.abs(want).max()
        img = buf.denoised_image(d)
        bytes_ = np.array([api.color_bytes(c) for c in got.reshape(-1, 3)], np.uint8).reshape(h, w, 3)
        assert np.array_equal(img, bytes_)


def test_zero_iterations_is_image_at_radius_zero(gpu_ok):
    cfg = scenes.sphere_scene()
    r, buf = _buffer(cfg, 40, 30, 2, 3, 2, 1)
    assert np.array_equal(buf.denoised_image(api.Denoise(iterations=0)), buf.image())


def test_errors(gpu_ok):
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 16, 8, 1)
    buf = r.device_buffer()
    with pytest.raises(capi.RptbError, match="no samples"):
        buf.denoise()
    r.sample(1, buf, want_stats=False)
    with pytest.raises(capi.RptbError, match="fewer than 2"):
        buf.denoise()
    r.sample(1, buf, want_stats=False)
    with pytest.raises(capi.RptbError, match="no features"):
        buf.denoise()
    with pytest.raises(capi.RptbError, match="no features"):
        buf.features()
    r.sample_features(1, buf)
    assert np.isfinite(buf.denoise()).all()
    # one adaptive entry is one entry in every pixel, too few
    ad = r.device_buffer()
    r.sample(1, ad, want_stats=False, adaptive=api.Adaptive(0.0, 0.0, 2))
    r.sample_features(1, ad)
    with pytest.raises(capi.RptbError, match="fewer than 2"):
        ad.denoise()


def test_same_bits_for_every_device_count(gpu_ok, monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")
    cfg = scenes.cornell_scene()
    lists = util.replica_lists(gpu_ok)
    outs = []
    for devices in lists:
        r, buf = _buffer(cfg, 53, 37, 3, 3, 2, 3, device=devices)
        outs.append((buf.features(), buf.denoise()))
        buf.close()
        r.close()
    for devices, (f, d) in zip(lists[1:], outs[1:]):
        assert all(np.array_equal(x, y) for x, y in zip(f, outs[0][0])) and np.array_equal(d, outs[0][1]), devices


def _edge_band(N, z):
    """Pixels whose 4-neighbours differ in depth by > 5 % or in normal by dot < 0.9."""
    band = np.zeros(z.shape, bool)
    for dy, dx in ((0, 1), (1, 0)):
        a, b = (slice(0, z.shape[0] - dy), slice(0, z.shape[1] - dx)), (slice(dy, None), slice(dx, None))
        with np.errstate(invalid="ignore"):
            dz = ~(np.abs(z[a] - z[b]) <= 0.05 * np.minimum(z[a], z[b]))
        dn = (N[a] * N[b]).sum(-1) < 0.9
        e = dz | dn
        band[a] |= e
        band[b] |= e
    return band


def _box(mean, radius):
    H, W, _ = mean.shape
    out = np.zeros_like(mean)
    cnt = np.zeros((H, W, 1))
    for dy in range(-radius, radius + 1):
        for dx in range(-radius, radius + 1):
            ok = ref._inside(H, W, dx, dy)[..., None]
            out += np.where(ok, ref._shift(mean, dx, dy, 0.0), 0.0)
            cnt += ok
    return out / cnt


# Floors on raw MSE / denoised MSE, each below the ratio measured on an H100 80GB HBM3 (700 W): the renders are seeded,
# so the ratios move only if the kernels' rounding does, and the margins (15-25 % on the image, about 7 % on the edge
# bands, whose measured gains are the smaller ones) cover that.  Measured: cornell image 4.89, edge band 1.70; sphere
# 6.77, 1.18; teapot 2.78, 1.23.
QUALITY = {  # name: (config factory, max_bounces, floor over the image, floor on the edge band)
    "cornell": (scenes.cornell_scene, 6, 4.0, 1.55),
    "sphere": (scenes.sphere_scene, 4, 5.5, 1.1),
    "teapot": (scenes.teapot_scene, 4, 2.3, 1.15),
}


@pytest.mark.parametrize("name", sorted(QUALITY))
def test_denoised_beats_raw_and_box_against_a_reference(gpu_ok, name):
    mk, mb, floor, edge_floor = QUALITY[name]
    cfg = mk()
    w = h = 128
    rr = _renderer(cfg, w, h, mb, seed=1234)
    refbuf = rr.device_buffer()
    for _ in range(8):
        rr.sample(128, refbuf, want_stats=False)
    truth = refbuf.sums().reshape(h, w, 3) / 8.0
    _, buf = _buffer(cfg, w, h, mb, 8, 2, 16)
    sums, _, counts = buf.pixel_stats()
    raw = sums.reshape(h, w, 3) / counts.reshape(h, w, 1)
    den = buf.denoise()
    N, z, _, _ = buf.features()
    band = _edge_band(N, z)

    def mse(x, m=None):
        e = (np.clip(x, 0, 1) - np.clip(truth, 0, 1)) ** 2
        return float(e[m].mean() if m is not None else e.mean())

    m = {"raw": mse(raw), "box1": mse(_box(raw, 1)), "box2": mse(_box(raw, 2)), "denoised": mse(den)}
    e = {"raw": mse(raw, band), "box1": mse(_box(raw, 1), band), "box2": mse(_box(raw, 2), band), "denoised": mse(den, band)}
    print(name, "mse", m, "edge", e, "band", int(band.sum()))
    assert band.sum() > 0
    assert m["denoised"] < min(m["box1"], m["box2"]) and m["raw"] / m["denoised"] >= floor, m
    assert e["denoised"] < min(e["raw"], e["box1"], e["box2"]) and e["raw"] / e["denoised"] >= edge_floor, e


def test_render_with_denoise(gpu_ok):
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 32, 24, 2).num_samples(8)
    img = r.render(denoise=api.Denoise(), entries=4, feature_samples=2)
    assert img.shape == (24, 32, 3) and img.dtype == np.uint8
    assert r.render().shape == (24, 32, 3)
