"""The denoised image's error from two half buffers without a GPU: halves.h's per-pixel functions in host emulation against
their numpy restatement (tests/halves_ref.py) on random states with n = 0, 1, 2, 3 ..., NaN neighbours, image borders and
infinite depths; the passes' colour and variance against the plain filter's, bit for bit; the estimate's statistics on
synthetic i.i.d. entries; the criterion; api.Adaptive(estimate=...); and the C ABI's layout, signatures and refusals before
any device work, including those of the frame and distributed loops."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, distributed, scenes
from tests import denoise_ref as dr
from tests import halves_ref as href
from tests.hostemu import emu
from tests.test_guided import edge_state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dp, u32p = capi.c_double_p, capi.c_u32_p
_lib = None


def _emu():
    """tests/hostemu/_build/libhostemu_halves.so: halves.h compiled for the host."""
    global _lib
    if _lib is not None:
        return _lib
    emu.lib()  # `make hostemu` builds every emulation library
    L = C.CDLL(os.path.join(ROOT, "tests", "hostemu", "_build", "libhostemu_halves.so"))
    L.hostemu_halves_demodulate.restype = None
    L.hostemu_halves_demodulate.argtypes = [dp, dp, dp, u32p, C.c_uint64, dp, C.c_double, dp, dp, dp]
    L.hostemu_halves_pass.restype = None
    L.hostemu_halves_pass.argtypes = [dp, dp, dp, dp, dp, dp, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(capi.Denoise), dp, dp, dp]
    L.hostemu_halves_plain_pass.restype = None
    L.hostemu_halves_plain_pass.argtypes = [dp, dp, dp, dp, dp, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(capi.Denoise), dp, dp]
    L.hostemu_halves_error.restype = None
    L.hostemu_halves_error.argtypes = [dp, dp, C.c_uint32, C.c_uint32, C.c_double, dp]
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(dp)


def halves_state(seed, H, W):
    """edge_state (counts 0..9, NaN and inf sums, zero variance, misses with inf depth) plus a HALF plane: a share of the
    sums for pixels with n >= 2, zero for n < 2 (no odd entry yet), NaN where the sums are."""
    sums, m2, counts, nrm, z, albedo = edge_state(seed, H, W)
    rng = np.random.default_rng(seed + 1)
    nb = (counts >> 1).astype(np.float64)[..., None]
    with np.errstate(invalid="ignore"):
        half = np.where(nb > 0, sums * (nb / np.maximum(counts, 1)[..., None]) * rng.uniform(0.8, 1.2, sums.shape), 0.0)
    return sums, m2, np.ascontiguousarray(half), counts, nrm, z, albedo


def emu_error(sums, m2, half, counts, nrm, z, albedo, d):
    """The device's kernels through the host-compiled halves.h: (i', v', U', E), and the plain passes' (i', v')."""
    H, W = z.shape
    L, c = _emu(), d.to_c()
    i, v, u = np.empty((H, W, 3)), np.empty((H, W)), np.empty((H, W, 3))
    L.hostemu_halves_demodulate(_p(np.ascontiguousarray(sums)), _p(np.ascontiguousarray(m2)), _p(half), counts.ctypes.data_as(u32p), H * W,
                                _p(albedo), d.albedo_eps, _p(i), _p(v), _p(u))
    pi, pv = i.copy(), v.copy()
    for k in range(d.iterations):
        i2, v2, u2 = np.empty_like(i), np.empty_like(v), np.empty_like(u)
        L.hostemu_halves_pass(_p(i), _p(v), _p(u), _p(nrm), _p(z), _p(albedo), W, H, 1 << k, C.byref(c), _p(i2), _p(v2), _p(u2))
        pi2, pv2 = np.empty_like(i), np.empty_like(v)
        L.hostemu_halves_plain_pass(_p(pi), _p(pv), _p(nrm), _p(z), _p(albedo), W, H, 1 << k, C.byref(c), _p(pi2), _p(pv2))
        i, v, u, pi, pv = i2, v2, u2, pi2, pv2
    E = np.empty((H, W))
    L.hostemu_halves_error(_p(u), _p(albedo), W, H, d.albedo_eps, _p(E))
    return i, v, u, E, pi, pv


def _agree(got, want):
    """Equal where not finite; within 1e-12 of the largest value elsewhere (exp's last bit in the weights)."""
    assert np.array_equal(np.isnan(got), np.isnan(want))
    fin = np.isfinite(want)
    assert np.array_equal(got[~fin], want[~fin], equal_nan=True)
    scale = np.nanmax(np.abs(want[fin])) if fin.any() else 1.0
    assert np.max(np.abs(got[fin] - want[fin]), initial=0.0) <= 1e-12 * scale


STATES = [(1, 1, 1), (7, 9, 5), (29, 37, 5), (37, 29, 3), (24, 48, 1), (45, 61, 5), (16, 16, 12)]


@pytest.mark.parametrize("H,W,it", STATES)
def test_estimate_matches_numpy(H, W, it):
    state = halves_state(H * 1000 + W + it, H, W)
    sums, m2, half, counts, nrm, z, albedo = state
    d = api.Denoise(iterations=it)
    i, v, u, E, pi, pv = emu_error(*state, d)
    # the passes carry colour and variance bit for bit as the plain filter does
    assert np.array_equal(i, pi, equal_nan=True) and np.array_equal(v, pv, equal_nan=True)
    # u has no exp in it: bit for bit
    want_u = href.u_plane(sums, half, counts, albedo, d.albedo_eps)
    got_u = np.empty((H, W, 3))
    ii, vv = np.empty((H, W, 3)), np.empty((H, W))
    _emu().hostemu_halves_demodulate(_p(np.ascontiguousarray(sums)), _p(np.ascontiguousarray(m2)), _p(half), counts.ctypes.data_as(u32p),
                                     H * W, _p(albedo), d.albedo_eps, _p(ii), _p(vv), _p(got_u))
    assert np.array_equal(got_u, want_u, equal_nan=True)
    assert np.isnan(want_u[counts <= 1]).all()
    # the whole estimate against numpy
    c, wv, wE = href.error(sums, m2, half, counts, nrm, z, albedo, d)
    _agree(i * (albedo + d.albedo_eps), c)
    _agree(v, wv)
    _agree(E, wE)
    # numpy's own passes give denoise_ref's colour and variance exactly
    wi, wvv = dr.demodulate(sums, m2, counts, albedo, d.albedo_eps)
    hi, hv = wi, wvv
    for k in range(it):
        wi, wvv = dr.atrous_pass(wi, wvv, nrm, z, albedo, 1 << k, d)
        hi, hv, _ = href.atrous_pass(hi, hv, want_u, nrm, z, albedo, 1 << k, d)
    assert np.array_equal(wi, hi, equal_nan=True) and np.array_equal(wvv, hv, equal_nan=True)
    if H * W > 100:
        assert np.isfinite(E).mean() > 0.5


def test_u_is_unbiased_for_iid_entries():
    """E[u^2] = Var(S / n) per channel for i.i.d. entries, whatever the count (odd counts included)."""
    rng = np.random.default_rng(3)
    trials, sigma = 200000, 0.7
    for n in (2, 3, 4, 5, 8, 9):
        x = rng.normal(1.0, sigma, (trials, n, 3))
        odd = np.arange(n) % 2 == 1
        S, half = x.sum(1), x[:, odd].sum(1)
        u = href.u_plane(S, half, np.full(trials, n, np.uint32), np.full((trials, 3), 1.0), 0.0)
        ratio = np.mean(u * u) / (sigma * sigma / n)
        assert abs(ratio - 1.0) < 0.02, (n, ratio)


def test_estimate_matches_the_variance_of_a_fixed_filter():
    """With flat features (weights that do not depend on the noise), E over many seeds averages to the empirical variance of
    c' -- correlations between the passes included -- while v' falls short of it."""
    H, W, n, seeds, sigma = 24, 24, 8, 300, 0.3
    d = api.Denoise(iterations=3, sigma_luminance=1e9)
    nrm = np.zeros((H, W, 3))
    nrm[..., 2] = 1.0
    z, albedo = np.full((H, W), 2.0), np.full((H, W, 3), 0.5)
    counts = np.full((H, W), n, np.uint32)
    rng = np.random.default_rng(11)
    cs, Es, vs = [], [], []
    for _ in range(seeds):
        x = rng.normal(0.5, sigma, (n, H, W, 3))
        sums, half = x.sum(0), x[1::2].sum(0)
        m2 = ((x - x.mean(0)) ** 2).sum((0, 3))
        c, v, E = href.error(sums, m2, half, counts, nrm, z, albedo, d)
        cs.append(c[6:-6, 6:-6])
        Es.append(E[6:-6, 6:-6])
        vs.append(v[6:-6, 6:-6])
    emp = np.var(np.stack(cs), axis=0, ddof=1).mean(-1)
    rE, rv = np.median(emp / np.mean(Es, 0)), np.median(emp / np.mean(vs, 0))
    assert 0.9 < rE < 1.1, rE
    assert rv > 2.0, rv


def test_criterion_is_guided_active_on_E():
    counts = np.array([[1, 4, 4, 4]], np.uint32)
    c = np.array([[[1.0, 1, 1], [1.0, 1, 1], [1.0, 1, 1], [1.0, 1, 1]]])
    E = np.array([[0.0, 1e-6, 1e-2, np.nan]])
    crit = api.Adaptive(rel_tol=0.02, abs_tol=0.0, min_entries=2, guide=api.Denoise(), estimate="halves")
    assert href.active(counts, c, E, crit).tolist() == [[True, False, True, True]]


def test_odd_sums_rule():
    xs = [np.full((3, 3), float(k + 1)) for k in range(5)]
    took = [np.array([True, True, True]), np.array([True, False, True]), np.array([True, True, False]),
            np.array([True, True, True]), np.array([False, True, True])]
    half = href.odd_sums(list(zip(xs, took)))
    # pixel 0 takes entries 1..4 at counts 0..3: odd counts 1, 3 -> 2 + 4; pixel 1 takes 1, 3, 4, 5 -> counts 1, 3 -> 3 + 5;
    # pixel 2 takes 1, 2, 4, 5 -> counts 1, 3 -> 2 + 5
    assert half[:, 0].tolist() == [6.0, 8.0, 7.0]


# ---- api.Adaptive ----------------------------------------------------------------------------------------------------
def test_adaptive_estimate_argument():
    assert api.Adaptive().estimate == "filter"
    assert api.Adaptive(guide=api.Denoise()).estimate == "filter"
    a = api.Adaptive(0.05, 1e-3, 5, api.Denoise(), "halves")
    assert a.estimate == "halves" and bytes(a.to_c()) == bytes(api.Adaptive(0.05, 1e-3, 5).to_c())
    with pytest.raises(ValueError):
        api.Adaptive(estimate="halves")  # no guide: no denoised value to estimate
    with pytest.raises(ValueError):
        api.Adaptive(guide=api.Denoise(), estimate="v")


# ---- the C ABI -------------------------------------------------------------------------------------------------------
def test_abi_signatures_match_header():
    text = open(os.path.join(ROOT, "include", "rpt_b200.h")).read()
    want = {
        "rptb_buffer_create_halves": "int rptb_buffer_create_halves(rptb_scene* scene, uint32_t width, uint32_t height, uint32_t box_radius, rptb_buffer** out);",
        "rptb_buffer_half_sums": "int rptb_buffer_half_sums(rptb_buffer* buffer, double* out);",
        "rptb_buffer_denoise_error": "int rptb_buffer_denoise_error(rptb_buffer* buffer, const rptb_denoise* params, double* out);",
    }
    flat = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", text, flags=re.S))
    for name, decl in want.items():
        assert decl in flat, name
    m = re.search(r"int rptb_sample_into_guided_error\(([^;]*)\);", flat)
    assert m and len(m.group(1).split(",")) == 8
    syms = {name: (res, args) for name, res, args in capi.SYMBOLS}
    assert syms["rptb_buffer_create_halves"][1] == syms["rptb_buffer_create"][1]
    assert syms["rptb_sample_into_guided_error"][1] == syms["rptb_sample_into_guided"][1]
    assert len(syms["rptb_buffer_half_sums"][1]) == 2 and len(syms["rptb_buffer_denoise_error"][1]) == 3
    for name in want:
        assert hasattr(capi.lib(), name)
    assert hasattr(capi.lib(), "rptb_sample_into_guided_error")


def test_errors_before_any_device_work():
    L = capi.lib()
    cam, p = capi.Camera(), capi.RenderParams()
    p.width, p.height, p.iterations, p.shard_count = 8, 8, 1, 1
    good_c, good_d = api.Adaptive().to_c(), api.Denoise().to_c()
    fake = C.c_void_p(1)  # never looked at: the arguments are refused first
    out = C.c_void_p()
    assert L.rptb_buffer_create_halves(None, 8, 8, 0, C.byref(out)) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_create_halves(fake, 0, 8, 0, C.byref(out)) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_create_halves(fake, 8, 8, 0, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_half_sums(None, _p(np.empty(3))) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_half_sums(fake, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_error(None, C.byref(good_d), _p(np.empty(1))) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_error(fake, None, _p(np.empty(1))) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_error(fake, C.byref(good_d), None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_error(fake, C.byref(capi.Denoise(13, 128, 1.0, 4.0, 1e-3)), _p(np.empty(1))) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_error(fake, C.byref(capi.Denoise(0, 128, 1.0, 4.0, 1e-3)), _p(np.empty(1))) == capi.ERR_BAD_ARG
    for eps in (0.0, -1e-9, float("nan")):  # albedo_eps must be finite and > 0
        assert L.rptb_buffer_denoise_error(fake, C.byref(capi.Denoise(5, 128, 1.0, 4.0, eps)), _p(np.empty(1))) == capi.ERR_BAD_ARG
        assert b"albedo_eps" in L.rptb_last_error()

    def call(crit, guide, scene=fake, buf=fake):
        return L.rptb_sample_into_guided_error(scene, C.byref(cam), C.byref(p), crit, guide, buf, None, None)

    assert call(C.byref(capi.Adaptive(0.02, 1e-3, 1, 0)), C.byref(good_d)) == capi.ERR_BAD_ARG
    assert call(None, C.byref(good_d)) == capi.ERR_BAD_ARG
    assert call(C.byref(good_c), None) == capi.ERR_BAD_ARG
    assert call(C.byref(good_c), C.byref(capi.Denoise(13, 128, 1.0, 4.0, 1e-3))) == capi.ERR_BAD_ARG
    assert call(C.byref(good_c), C.byref(capi.Denoise(0, 128, 1.0, 4.0, 1e-3))) == capi.ERR_BAD_ARG
    assert b"iterations" in L.rptb_last_error()
    assert call(C.byref(good_c), C.byref(capi.Denoise(4, 128, 1.0, 4.0, 0.0))) == capi.ERR_BAD_ARG
    assert b"albedo_eps" in L.rptb_last_error()
    assert call(C.byref(good_c), C.byref(good_d), scene=None) == capi.ERR_BAD_ARG
    assert call(C.byref(good_c), C.byref(good_d), buf=None) == capi.ERR_BAD_ARG


def test_loops_refuse_the_halves_estimate_before_device_work():
    cfg = scenes.sphere_scene()
    r = api.Renderer(cfg.scene, cfg.camera).width(8).height(8).num_samples(4)
    a = api.Adaptive(guide=api.Denoise(), estimate="halves")
    with pytest.raises(ValueError, match="halves"):
        next(r.render_frames([cfg.camera], entries=2, adaptive=a))
    with pytest.raises(ValueError, match="halves"):
        distributed.render_iterative_distributed(r, 1, lambda i, b: None, adaptive=a)
    with pytest.raises(ValueError, match="halves"):
        next(distributed.render_frames_distributed(r, [cfg.camera], entries=2, adaptive=a))
    assert r._dev_scene is None  # nothing reached the device
