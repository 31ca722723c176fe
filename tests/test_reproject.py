"""Reprojection without a GPU: the C ABI's struct and argument checks, the per-pixel functions of reproject.h in host
emulation against their numpy restatement (tests/reproject_ref.py) bit for bit, on synthetic states and on features the
emulated feature pass renders, and the properties the restatement must have: the identity camera, a pure rotation of
an environment view, pixels with no valid tap, and the history cap."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import denoise_ref
from tests import reproject_ref as ref
from tests.hostemu import emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dp = capi.c_double_p
_lib = None


def _emu():
    """tests/hostemu/_build/libhostemu_reproject.so: the feature pass and reproject.h compiled for the host."""
    global _lib
    if _lib is not None:
        return _lib
    emu.lib()  # `make hostemu` builds every emulation library
    L = C.CDLL(os.path.join(ROOT, "tests", "hostemu", "_build", "libhostemu_reproject.so"))
    L.hostemu_scene_create.restype = C.c_void_p
    L.hostemu_scene_create.argtypes = [C.POINTER(capi.SceneDesc), C.c_char_p, C.c_size_t]
    L.hostemu_scene_destroy.argtypes = [C.c_void_p]
    L.hostemu_features.argtypes = [C.c_void_p, C.POINTER(capi.Camera), C.POINTER(capi.RenderParams), dp]
    cam = C.POINTER(capi.Camera)
    L.hostemu_reproject.restype = None
    L.hostemu_reproject.argtypes = [cam, C.c_uint32, C.c_uint32, dp, dp, dp, cam, C.c_uint32, C.c_uint32, dp, dp, capi.c_u32_p, dp,
                                    dp, dp, C.POINTER(capi.Reproject), dp, dp, capi.c_u32_p]
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(dp)


def emu_reproject(dcam, dnrm, dz, df, scam, ssums, sm2, scounts, snrm, sz, sf, prm):
    dh, dw = dz.shape
    sh, sw = sz.shape
    c = [np.ascontiguousarray(a, np.float64) for a in (dnrm, dz, df, ssums, sm2, snrm, sz, sf)]
    sc = np.ascontiguousarray(scounts, np.uint32)
    out_s, out_m, out_n = np.empty((dh, dw, 3)), np.empty((dh, dw)), np.empty((dh, dw), np.uint32)
    dc, scc, pc = _c(dcam), _c(scam), prm.to_c()
    _emu().hostemu_reproject(C.byref(dc), dw, dh, _p(c[0]), _p(c[1]), _p(c[2]), C.byref(scc), sw, sh, _p(c[3]), _p(c[4]),
                             sc.ctypes.data_as(capi.c_u32_p), _p(c[5]), _p(c[6]), _p(c[7]), C.byref(pc), _p(out_s), _p(out_m),
                             out_n.ctypes.data_as(capi.c_u32_p))
    return out_s, out_m, out_n


def _c(cam):
    return cam.to_c() if hasattr(cam, "to_c") else cam


def orbit(cam, center, angle, lift=0.0):
    """`cam` turned by `angle` about the vertical axis through `center` (and raised by `lift`), still looking at it."""
    c = np.asarray(center, np.float64)
    d = cam.eye - c
    ca, sa = math.cos(angle), math.sin(angle)
    eye = c + np.array([ca * d[0] + sa * d[2], d[1] + lift, -sa * d[0] + ca * d[2]])
    return api.Camera.look_at(eye, c, api.vec3(0.0, 1.0, 0.0), cam.fov)


def random_features(rng, H, W, env_frac=0.2):
    nrm = rng.normal(size=(H, W, 3))
    nrm /= np.linalg.norm(nrm, axis=-1, keepdims=True)
    z = rng.uniform(2.0, 8.0, (H, W))
    f = rng.choice([0.25, 0.5, 1.0], (H, W))
    env = rng.random((H, W)) < env_frac
    nrm[env], z[env], f[env] = 0.0, np.inf, 0.0
    return nrm, z, f


def random_stats(rng, H, W, lo=2, hi=9):
    counts = rng.integers(lo, hi, (H, W)).astype(np.uint32)
    mean = rng.uniform(0.1, 1.0, (H, W, 3))
    return mean * counts[..., None], rng.uniform(0, 0.5, (H, W)) * (counts - 1.0), counts


def assert_same(got, want):
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and np.array_equal(g, w), np.nanmax(np.abs(g.astype(float) - w.astype(float)))


# ---- the C ABI -------------------------------------------------------------------------------------------------
def test_reproject_struct_size_matches_header(tmp_path):
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include "rpt_b200.h"\nint main(void){printf("%zu\\n", sizeof(rptb_reproject));return 0;}\n')
    exe = tmp_path / "s"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    assert int(subprocess.check_output([str(exe)]).decode()) == C.sizeof(capi.Reproject) == 24


def test_reproject_errors_before_any_device_work():
    L = capi.lib()
    a, b = C.c_void_p(1), C.c_void_p(2)
    good = api.Reproject().to_c()
    assert L.rptb_buffer_reproject(None, b, C.byref(good), None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_reproject(a, None, C.byref(good), None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_reproject(a, b, None, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_reproject(a, a, C.byref(good), None) == capi.ERR_BAD_ARG
    assert b"same buffer" in L.rptb_last_error()
    bad = [api.Reproject(depth_tol=-0.1), api.Reproject(depth_tol=float("inf")), api.Reproject(depth_tol=float("nan")),
           api.Reproject(normal_cos=1.5), api.Reproject(normal_cos=-1.01), api.Reproject(normal_cos=float("nan")),
           api.Reproject(max_history=1), api.Reproject(max_history=0)]
    for prm in bad:  # checked before the buffers are looked at
        c = prm.to_c()
        assert L.rptb_buffer_reproject(a, b, C.byref(c), None) == capi.ERR_BAD_ARG
        msg = L.rptb_last_error()
        assert b"depth_tol" in msg or b"normal_cos" in msg or b"max_history" in msg


# ---- host emulation against numpy -----------------------------------------------------------------------------------
@pytest.mark.parametrize("dsize,ssize,angle,seed", [((23, 17), (23, 17), 0.05, 1), ((31, 20), (19, 27), -0.08, 2),
                                                     ((1, 1), (9, 7), 0.0, 3), ((40, 9), (40, 9), 0.4, 4)])
def test_emulation_matches_numpy_on_synthetic_states(dsize, ssize, angle, seed):
    rng = np.random.default_rng(seed)
    (dw, dh), (sw, sh) = dsize, ssize
    scam = api.Camera.look_at(api.vec3(1.0, 2.0, 6.0), api.vec3(0.0, 0.0, 0.0), api.vec3(0.0, 1.0, 0.0), 0.8)
    dcam = orbit(scam, (0.0, 0.0, 0.0), angle, lift=0.1)
    dN, dz, df = random_features(rng, dh, dw)
    sN, sz, sf = random_features(rng, sh, sw)
    sums, m2, counts = random_stats(rng, sh, sw, lo=0)
    sums[rng.random((sh, sw)) < 0.05] = np.nan
    m2[rng.random((sh, sw)) < 0.05] = np.inf
    for prm in (api.Reproject(), api.Reproject(depth_tol=0.5, normal_cos=-1.0, max_history=4), api.Reproject(0.0, 1.0, 2)):
        want = ref.reproject(dcam, dN, dz, df, scam, sums, m2, counts, sN, sz, sf, prm)
        got = emu_reproject(dcam, dN, dz, df, scam, sums, m2, counts, sN, sz, sf, prm)
        assert_same(got, want)


def _emu_scene_features(flat, cam, w, h, spp, precision):
    handle = C.c_void_p(_emu().hostemu_scene_create(C.byref(flat.desc), C.create_string_buffer(512), 512))
    try:
        p = api.Renderer(api.Scene(), cam).width(w).height(h).seed(3).precision(precision).params(spp)
        out = np.empty(w * h * 8)
        assert _emu().hostemu_features(handle, C.byref(cam.to_c()), C.byref(p), _p(out)) >= 0
    finally:
        _emu().hostemu_scene_destroy(handle)
    n = w * h
    N, z, _, f = denoise_ref.features_resolve(out[6 * n: 7 * n], out[: 3 * n].reshape(n, 3), out[7 * n:], out[3 * n: 6 * n].reshape(n, 3),
                                              float(spp))
    return N.reshape(h, w, 3), z.reshape(h, w), f.reshape(h, w)


@pytest.mark.parametrize("name,precision", [("sphere", capi.PRECISION_F64), ("cornell", capi.PRECISION_F32)])
def test_emulation_matches_numpy_on_rendered_features(name, precision):
    cfg = {"sphere": scenes.sphere_scene, "cornell": scenes.cornell_scene}[name]()
    center = {"sphere": (0.0, -0.25, 0.0), "cornell": (278.0, 273.0, 280.0)}[name]
    flat = api.FlatScene(cfg.scene)
    scam = api.Camera.look_at(cfg.camera.eye, np.asarray(center), api.vec3(0.0, 1.0, 0.0), cfg.camera.fov)
    dcam = orbit(scam, center, 0.06)
    sw, sh, dw, dh = 36, 28, 33, 29
    sN, sz, sf = _emu_scene_features(flat, scam, sw, sh, 3, precision)
    dN, dz, df = _emu_scene_features(flat, dcam, dw, dh, 3, precision)
    assert (sf > 0).mean() > 0.3 and (df > 0).mean() > 0.3
    sums, m2, counts = random_stats(np.random.default_rng(5), sh, sw)
    prm = api.Reproject()
    want = ref.reproject(dcam, dN, dz, df, scam, sums, m2, counts, sN, sz, sf, prm)
    got = emu_reproject(dcam, dN, dz, df, scam, sums, m2, counts, sN, sz, sf, prm)
    assert_same(got, want)
    print(name, "reused", (want[2] > 0).mean())
    assert (want[2] > 0).mean() > 0.5


# ---- properties ---------------------------------------------------------------------------------------------------
def _cam():
    return api.Camera.look_at(api.vec3(0.5, 1.5, 7.0), api.vec3(0.0, 0.0, 0.0), api.vec3(0.0, 1.0, 0.0), 0.9)


def test_identity_camera_keeps_the_mean():
    rng = np.random.default_rng(11)
    H, W, n = 21, 26, 6
    N, z, f = random_features(rng, H, W)
    sums, m2, counts = random_stats(rng, H, W, n, n + 1)
    cam = _cam()
    for mh in (32, 4):
        prm = api.Reproject(max_history=mh)
        s, m, c = ref.reproject(cam, N, z, f, cam, sums, m2, counts, N, z, f, prm)
        assert_same(emu_reproject(cam, N, z, f, cam, sums, m2, counts, N, z, f, prm), (s, m, c))
        assert (c == min(n, mh)).all()
        mean = sums / n
        assert np.max(np.abs(s / c[..., None] - mean)) <= 1e-12 * np.abs(mean).max()


def test_pure_rotation_resamples_the_environment_bilinearly():
    from scipy.ndimage import map_coordinates
    rng = np.random.default_rng(12)
    H, W, n = 30, 40, 5
    scam = _cam()
    dcam = api.Camera.look_at(scam.eye, api.vec3(0.6, -0.3, 0.2), api.vec3(0.0, 1.0, 0.0), 0.9)
    sums, m2, counts = random_stats(rng, H, W, n, n + 1)
    zero3, env = np.zeros((H, W, 3)), np.zeros((H, W))
    dz = rng.uniform(1.0, 50.0, (H, W))  # an environment pixel is placed by its direction, whatever its depth says
    prm = api.Reproject()
    s, m, c = ref.reproject(dcam, zero3, dz, env, scam, sums, m2, counts, zero3, np.full((H, W), np.inf), env, prm)
    assert_same(emu_reproject(dcam, zero3, dz, env, scam, sums, m2, counts, zero3, np.full((H, W), np.inf), env, prm), (s, m, c))
    # the same projection through the orthonormal frame of a look_at camera, and scipy's bilinear resample
    eye, D, U, R, dc, dim = ref.view(dcam, W, H)
    _, sD, sU, sR, sdc, sdim = ref.view(scam, W, H)
    xs, ys = np.meshgrid(np.arange(W), np.arange(H))
    xn, yn = (2 * xs + 1 - W) / dim, (2 * (H - ys) - 1 - H) / dim
    r = dc * D + xn[..., None] * R + yn[..., None] * U
    px = (sdc * (r @ sR) / (r @ sD) * sdim + W - 1) / 2
    py = (H - 1 - sdc * (r @ sU) / (r @ sD) * sdim) / 2
    inner = (px >= 0) & (px <= W - 1.001) & (py >= 0) & (py <= H - 1.001)
    assert inner.mean() > 0.5
    mean = sums / n
    want = np.stack([map_coordinates(mean[..., k], [py, px], order=1) for k in range(3)], -1)
    assert (c[inner] == n).all()
    assert np.max(np.abs(s[inner] / n - want[inner])) <= 1e-9
    # translating the eye moves no environment pixel
    moved = api.Camera(dcam.eye + np.array([3.0, -1.0, 2.0]), dcam.direction, dcam.up, dcam.fov)
    assert_same(ref.reproject(moved, zero3, dz, env, scam, sums, m2, counts, zero3, np.full((H, W), np.inf), env, prm), (s, m, c))


def test_no_valid_tap_gives_no_history():
    rng = np.random.default_rng(13)
    H, W = 17, 23
    N, z, f = random_features(rng, H, W, env_frac=0.0)
    sums, m2, counts = random_stats(rng, H, W)
    cam = _cam()
    behind = api.Camera(cam.eye, -cam.direction, cam.up, cam.fov)
    prm = api.Reproject()
    cases = {
        "behind the source camera": (behind, sums, m2, counts, N, z, f),
        "depth": (cam, sums, m2, counts, N, z * 1.5, f),
        "normal": (cam, sums, m2, counts, -N, z, f),
        "one entry": (cam, sums / counts[..., None], m2 * 0, np.ones((H, W), np.uint32), N, z, f),
        "environment seen from a surface": (cam, sums, m2, counts, np.zeros_like(N), np.full((H, W), np.inf), np.zeros((H, W))),
    }
    for what, (scam, s_, m_, c_, sN, sz, sf) in cases.items():
        want = ref.reproject(cam, N, z, f, scam, s_, m_, c_, sN, sz, sf, prm)
        assert_same(emu_reproject(cam, N, z, f, scam, s_, m_, c_, sN, sz, sf, prm), want)
        s, m, c = want
        assert (c == 0).all() and (s == 0).all() and (m == 0).all(), what


def test_history_cap_keeps_the_per_entry_variance():
    rng = np.random.default_rng(14)
    H, W, n = 19, 24, 8
    N, z, f = random_features(rng, H, W)
    sums, m2, counts = random_stats(rng, H, W, n, n + 1)
    cam = _cam()
    prm = api.Reproject(max_history=3)
    s, m, c = ref.reproject(cam, N, z, f, cam, sums, m2, counts, N, z, f, prm)
    assert (c == 3).all()
    s2 = m2 / (n - 1)
    assert np.max(np.abs(m / (c - 1.0) - s2)) <= 1e-12 * s2.max()
    assert np.max(np.abs(s / 3.0 - sums / n)) <= 1e-12 * (sums / n).max()
