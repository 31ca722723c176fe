"""The denoiser without a GPU: the C ABI's struct and argument checks, properties of the numpy restatement
(tests/denoise_ref.py), and the device code in host emulation -- the filter's per-pixel functions (denoise.h) against
numpy, and the first-hit feature pass (features.cuh) against sums built from the oracle's closest hits."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import denoise_ref as ref
from tests.hostemu import emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dp = capi.c_double_p
_lib = None


def _emu():
    """tests/hostemu/_build/libhostemu_denoise.so: the host emulation of hostemu.cu plus the feature pass and denoise.h."""
    global _lib
    if _lib is not None:
        return _lib
    emu.lib()  # `make hostemu` builds every emulation library
    L = C.CDLL(os.path.join(ROOT, "tests", "hostemu", "_build", "libhostemu_denoise.so"))
    L.hostemu_scene_create.restype = C.c_void_p
    L.hostemu_scene_create.argtypes = [C.POINTER(capi.SceneDesc), C.c_char_p, C.c_size_t]
    L.hostemu_scene_destroy.argtypes = [C.c_void_p]
    L.hostemu_features.argtypes = [C.c_void_p, C.POINTER(capi.Camera), C.POINTER(capi.RenderParams), dp]
    L.hostemu_features_resolve.restype = None
    L.hostemu_features_resolve.argtypes = [dp, C.c_uint64, C.c_double, dp, dp, dp, dp]
    L.hostemu_demodulate.restype = None
    L.hostemu_demodulate.argtypes = [dp, dp, capi.c_u32_p, C.c_uint64, dp, C.c_double, dp, dp]
    L.hostemu_denoise_pass.restype = None
    L.hostemu_denoise_pass.argtypes = [dp, dp, dp, dp, dp, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(capi.Denoise), dp, dp]
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(dp)


def emu_denoise(sums, m2, counts, nrm, z, albedo, d):
    """The device's sequence of kernels, each through the host-compiled denoise.h."""
    H, W = z.shape
    n = H * W
    counts = np.ascontiguousarray(counts, np.uint32)
    if d.iterations == 0:
        return sums / counts[..., None]
    i, v = np.empty((H, W, 3)), np.empty((H, W))
    _emu().hostemu_demodulate(_p(np.ascontiguousarray(sums)), _p(np.ascontiguousarray(m2)), counts.ctypes.data_as(capi.c_u32_p), n,
                              _p(np.ascontiguousarray(albedo)), d.albedo_eps, _p(i), _p(v))
    c = d.to_c()
    for k in range(d.iterations):
        i2, v2 = np.empty_like(i), np.empty_like(v)
        _emu().hostemu_denoise_pass(_p(i), _p(v), _p(np.ascontiguousarray(nrm)), _p(np.ascontiguousarray(z)), _p(np.ascontiguousarray(albedo)), W, H,
                                    1 << k, C.byref(c),
                                    _p(i2), _p(v2))
        i, v = i2, v2
    return i * (albedo + d.albedo_eps)


def random_state(rng, H, W, counted=False, holes=True):
    """A random buffer state: per-pixel sums, M2, counts, and resolved features with misses, zero normals and NaNs."""
    counts = rng.integers(2, 9, (H, W)).astype(np.uint32) if counted else np.full((H, W), 6, np.uint32)
    mean = rng.uniform(0, 1, (H, W, 3)) * rng.choice([0.1, 1.0, 5.0], (H, W, 1))
    sums = mean * counts[..., None]
    m2 = rng.uniform(0, 0.5, (H, W)) * (counts - 1)
    nrm = rng.normal(size=(H, W, 3))
    nrm /= np.linalg.norm(nrm, axis=-1, keepdims=True)
    nrm[: H // 2] = nrm[0, 0]                        # a flat region the weights let through
    z = rng.uniform(1, 3, (H, W))
    albedo = rng.uniform(0, 1, (H, W, 3))
    if holes and H * W > 4:
        miss = rng.random((H, W)) < 0.1
        nrm[miss], z[miss], albedo[miss] = 0.0, np.inf, 1.0
        sums[rng.random((H, W)) < 0.02] = np.nan
        m2[rng.random((H, W)) < 0.02] = np.nan
    return sums, m2, counts, nrm, z, albedo


# ---- the C ABI -------------------------------------------------------------------------------------------------
def test_denoise_struct_size_matches_header(tmp_path):
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include "rpt_b200.h"\nint main(void){printf("%zu\\n", sizeof(rptb_denoise));return 0;}\n')
    exe = tmp_path / "s"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    assert int(subprocess.check_output([str(exe)]).decode()) == C.sizeof(capi.Denoise) == 32


def test_denoise_errors_before_any_device_work():
    L = capi.lib()
    bad = [capi.Denoise(13, 128, 1.0, 4.0, 1e-3), capi.Denoise(5, 128, -1.0, 4.0, 1e-3), capi.Denoise(5, 128, 1.0, float("nan"), 1e-3),
           capi.Denoise(5, 128, 1.0, 4.0, float("inf")), capi.Denoise(5, 128, 1.0, 4.0, -1e-9), capi.Denoise(5, 128, 1.0, 4.0, 0.0),
           capi.Denoise(5, 128, 1.0, 4.0, -0.0), capi.Denoise(5, 128, 1.0, 4.0, float("nan"))]
    for d in bad:  # checked before the buffer is looked at
        assert L.rptb_buffer_denoise(C.c_void_p(1), C.byref(d), None, None) == capi.ERR_BAD_ARG
        assert b"iterations" in L.rptb_last_error() or b"finite" in L.rptb_last_error()
        assert L.rptb_buffer_denoise_variance(C.c_void_p(1), C.byref(d), _p(np.empty(1))) == capi.ERR_BAD_ARG
    # albedo_eps 0 divides a black albedo's pixel by 0 (a NaN colour for a raw mean of 0): refused, as every value <= 0
    for eps in (0.0, -0.0):
        assert L.rptb_buffer_denoise(C.c_void_p(1), C.byref(capi.Denoise(5, 128, 1.0, 4.0, eps)), None, None) == capi.ERR_BAD_ARG
        assert b"albedo_eps" in L.rptb_last_error() and b"> 0" in L.rptb_last_error()
    tiny = capi.Denoise(5, 128, 1.0, 4.0, 5e-324)  # the least positive double passes the argument check: the buffer is next
    assert L.rptb_buffer_denoise(None, C.byref(tiny), None, None) == capi.ERR_BAD_ARG
    assert b"null" in L.rptb_last_error()
    good = api.Denoise().to_c()
    assert L.rptb_buffer_denoise(None, C.byref(good), None, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise(C.c_void_p(1), None, None, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_features(None, None, None, None, None) == capi.ERR_BAD_ARG
    cam, p = capi.Camera(), capi.RenderParams()
    p.width, p.height, p.iterations, p.shard_count = 8, 8, 1, 1
    assert L.rptb_buffer_add_features(None, C.byref(cam), C.byref(p), None, None) == capi.ERR_BAD_ARG


def test_render_rejects_unequal_entries():
    cfg = scenes.sphere_scene()
    r = api.Renderer(cfg.scene, cfg.camera).width(8).height(8).num_samples(10)
    with pytest.raises(ValueError):
        r.render(denoise=api.Denoise(), entries=4)
    with pytest.raises(ValueError):
        r.render(denoise=api.Denoise(), entries=1)


# ---- properties of the restatement -------------------------------------------------------------------------------
def test_zero_iterations_is_the_mean():
    sums, m2, counts, nrm, z, albedo = random_state(np.random.default_rng(1), 13, 17, counted=True)
    out = ref.denoise(sums, m2, counts, nrm, z, albedo, api.Denoise(iterations=0))
    assert np.array_equal(out, sums / counts[..., None], equal_nan=True)


def test_constant_image_with_uniform_features_is_a_fixed_point():
    H, W = 24, 19
    albedo = np.full((H, W, 3), 0.5)
    d = api.Denoise()
    i0 = np.array([0.3, 0.6, 0.9])
    mean = i0 * (albedo + d.albedo_eps)
    counts = np.full((H, W), 8, np.uint32)
    nrm = np.zeros((H, W, 3))
    nrm[..., 2] = 1.0
    out = ref.denoise(mean * 8, np.full((H, W), 0.1), counts, nrm, np.full((H, W), 2.0), albedo, d)
    np.testing.assert_allclose(out, mean, rtol=1e-14, atol=0)


def test_normal_and_kernel_weights_are_symmetric():
    rng = np.random.default_rng(3)
    a, b = rng.normal(size=(1000, 3)), rng.normal(size=(1000, 3))
    a /= np.linalg.norm(a, axis=1, keepdims=True)
    b /= np.linalg.norm(b, axis=1, keepdims=True)

    def wn(p, q):
        c = (p[:, 0] * q[:, 0] + p[:, 1] * q[:, 1]) + p[:, 2] * q[:, 2]
        return ref.powu(np.where(c > 0, c, 0.0), 128)

    assert np.array_equal(wn(a, b), wn(b, a))
    K = np.outer(ref.K5, ref.K5)
    assert np.array_equal(K, K.T) and np.array_equal(K, K[::-1, ::-1]) and np.isclose(K.sum(), 1.0)


def test_nan_pixel_stays_local():
    rng = np.random.default_rng(4)
    sums, m2, counts, nrm, z, albedo = random_state(rng, 20, 20, holes=False)
    sums[7, 9] = np.nan
    out = ref.denoise(sums, m2, counts, nrm, z, albedo, api.Denoise())
    bad = ~np.isfinite(out).all(-1)
    assert bad[7, 9] and bad.sum() == 1


def test_output_variance_never_exceeds_input_on_uniform_features():
    rng = np.random.default_rng(5)
    H, W = 32, 24
    counts = np.full((H, W), 4, np.uint32)
    sums = rng.uniform(0, 1, (H, W, 3)) * 4
    m2 = rng.uniform(0, 1, (H, W))
    nrm = np.zeros((H, W, 3))
    nrm[..., 1] = 1.0
    z, albedo = np.full((H, W), 3.0), np.full((H, W, 3), 0.7)
    d = api.Denoise()
    _, v0 = ref.demodulate(sums, m2, counts, albedo, d.albedo_eps)
    for it in range(1, 6):
        _, v = ref.denoise(sums, m2, counts, nrm, z, albedo, api.Denoise(iterations=it), return_variance=True)
        assert v.max() <= v0.max() and v.mean() < v0.mean()


# ---- host emulation: the filter ------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W,counted,it", [(1, 1, False, 5), (1, 23, False, 5), (29, 37, False, 5), (29, 37, True, 5),
                                            (16, 16, True, 12), (8, 40, False, 0), (37, 29, True, 3)])
def test_filter_matches_numpy(H, W, counted, it):
    state = random_state(np.random.default_rng(H * 100 + W + it), H, W, counted=counted)
    d = api.Denoise(iterations=it, sigma_normal=128 if it != 3 else 7, sigma_depth=1.0 if it != 3 else 0.25)
    got = emu_denoise(*state, d)
    want = ref.denoise(*state, d)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    scale = np.nanmax(np.abs(want)) if np.isfinite(want).any() else 1.0
    fin = np.isfinite(want)
    assert np.array_equal(got[~fin], want[~fin], equal_nan=True)
    assert np.max(np.abs(got[fin] - want[fin]), initial=0.0) <= 1e-12 * scale


def test_features_resolve_matches_numpy():
    rng = np.random.default_rng(9)
    n, rays = 500, 6.0
    hits = rng.integers(0, 7, n).astype(float)
    sn = rng.normal(size=(n, 3)) * hits[:, None]
    sz, sa = rng.uniform(1, 5, n) * hits, rng.uniform(0, 1, (n, 3)) * hits[:, None]
    sums = np.concatenate([sn.ravel(), sa.ravel(), hits, sz])
    N, z, a, f = np.empty((n, 3)), np.empty(n), np.empty((n, 3)), np.empty(n)
    _emu().hostemu_features_resolve(_p(sums), n, rays, _p(N), _p(z), _p(a), _p(f))
    wN, wz, wa, wf = ref.features_resolve(hits, sn, sz, sa, rays)
    for g, w in ((N, wN), (z, wz), (a, wa), (f, wf)):
        assert np.array_equal(g, w)
    assert np.isinf(z[hits == 0]).all() and (N[hits == 0] == 0).all()


# ---- host emulation: the feature pass ------------------------------------------------------------------------------
def _glass_focus():
    cfg = scenes.glass_scene(64, 32)
    cfg.camera = cfg.camera.focus(api.vec3(0.0, 0.0, 0.0), 0.05)
    return cfg


FEATURE_SCENES = {  # name: (config factory, w, h, samples, f32 floor on the fraction of pixels whose hits and depth agree)
    "sphere": (scenes.sphere_scene, 21, 13, 3, 0.97),
    "cornell": (scenes.cornell_scene, 19, 17, 3, 0.97),
    "glass_aperture": (_glass_focus, 17, 11, 3, 0.97),
    "teapot": (scenes.teapot_scene, 18, 14, 2, 0.95),
    "fractal_spheres": (lambda: scenes.fractal_spheres_scene(3), 16, 12, 2, 0.95),
}


def emu_features(scene, cfg, w, h, spp, precision, seed=7):
    p = api.Renderer(cfg.scene, cfg.camera).width(w).height(h).seed(seed).precision(precision).params(spp)
    out = np.empty(w * h * 8)
    cam = cfg.camera.to_c()
    feat = _emu().hostemu_features(scene, C.byref(cam), C.byref(p), _p(out))
    assert feat >= 0
    n = w * h
    return out[: 3 * n].reshape(n, 3), out[3 * n: 6 * n].reshape(n, 3), out[6 * n: 7 * n], out[7 * n:]


@pytest.mark.parametrize("name", sorted(FEATURE_SCENES))
def test_feature_pass_matches_oracle_hits(orc, name):
    mk, w, h, spp, floor = FEATURE_SCENES[name]
    cfg = mk()
    flat = api.FlatScene(cfg.scene)
    handle = C.c_void_p(_emu().hostemu_scene_create(C.byref(flat.desc), C.create_string_buffer(512), 512))
    try:
        rays = ref.camera_rays(cfg.camera.to_c(), w, h, spp, 7)
        t, obj, nrm, _ = orc.OracleScene(flat).closest_hit(rays.reshape(-1, 6))
        want = ref.feature_sums(rays, t, obj, nrm, ref.object_colors(flat))
        got = emu_features(handle, cfg, w, h, spp, capi.PRECISION_F64)
        for g, wnt in zip(got, want):
            assert np.array_equal(g, wnt)
        assert want[2].sum() > 0
        # f32: the same rays in float; silhouettes may flip, elsewhere the depth agrees closely
        sn, sa, hits, sz = emu_features(handle, cfg, w, h, spp, capi.PRECISION_F32)
        same = hits == want[2]
        with np.errstate(invalid="ignore", divide="ignore"):
            close = np.where(hits > 0, np.abs(sz - want[3]) <= 1e-4 * np.abs(want[3]), True)
        print(name, "f32 features agreeing", (same & close).mean())
        assert (same & close).mean() >= floor, (same.mean(), (same & close).mean())
    finally:
        _emu().hostemu_scene_destroy(handle)
