"""The cross-filtered denoiser with a smoothed selection map without a GPU (rptb_buffer_denoise_cross): cross.h's
per-pixel functions in host emulation against their numpy restatement (tests/cross_ref.py) on edge-case states (counts
0..9, odd ones included, NaN and inf sums, image borders, infinite depths, pixels left with one finite tap); every pixel
whose 5x5 neighbourhood chose one level against that level's output, bit for bit, and every output as a convex blend of
its pixel's levels; the estimate's statistics on synthetic entries under fixed weights, for even and odd counts, against
the empirical error of every level; and the C ABI's signature and refusals before any device work, including
Renderer.render(cross=True)'s."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import cross_ref as xref
from tests.hostemu import emu
from tests.test_halves import _agree, _emu as _halves_emu, halves_state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dp, u32p, u8p = capi.c_double_p, capi.c_u32_p, capi.c_u8_p
_lib = None


def _emu():
    """tests/hostemu/_build/libhostemu_cross.so: cross.h compiled for the host."""
    global _lib
    if _lib is not None:
        return _lib
    emu.lib()  # `make hostemu` builds every emulation library
    L = C.CDLL(os.path.join(ROOT, "tests", "hostemu", "_build", "libhostemu_cross.so"))
    L.hostemu_cross_demodulate.restype = None
    L.hostemu_cross_demodulate.argtypes = [dp, dp, dp, u32p, C.c_uint64, dp, C.c_double, dp, dp, dp, dp]
    L.hostemu_cross_m.restype = None
    L.hostemu_cross_m.argtypes = [dp, dp, dp, dp, dp, dp, u32p, dp, C.c_uint64, C.c_double, dp]
    L.hostemu_cross_level.restype = None
    L.hostemu_cross_level.argtypes = [dp, C.c_uint32, C.c_uint32, C.c_uint32, dp, u8p]
    L.hostemu_cross_blend.restype = None
    L.hostemu_cross_blend.argtypes = [u8p, dp, dp, dp, dp, u32p, dp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, dp, dp]
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(dp)


def emu_cross(sums, m2, half, counts, nrm, z, albedo, d):
    """cross.cu's sequence through the host-compiled halves.h and cross.h, both sweeps: (rgb, level, M^, [m_k], [O_k]).
    O_k is the blend kernel's own value of level k: its step at k over a level plane that is k everywhere."""
    H, W = z.shape
    Lh, Lx, c = _halves_emu(), _emu(), d.to_c()
    eps = d.albedo_eps
    sums, m2 = np.ascontiguousarray(sums), np.ascontiguousarray(m2)
    cp = counts.ctypes.data_as(u32p)
    iA0, vA0, iB0, vB0 = np.empty((H, W, 3)), np.empty((H, W)), np.empty((H, W, 3)), np.empty((H, W))
    Lx.hostemu_cross_demodulate(_p(sums), _p(m2), _p(half), cp, H * W, _p(albedo), eps, _p(iA0), _p(vA0), _p(iB0), _p(vB0))
    level, M, m = np.empty((H, W), np.uint8), np.empty((H, W)), np.empty((H, W))
    rgb, ms, Os = np.empty((H, W, 3)), [], []

    def chains():
        """Yields (k, X_A, X_B) for k = 0 .. d.iterations: both chains' passes, as cross.cu launches them."""
        gA, vA, XB, gB, vB, XA = iA0, vA0, iB0, iB0, vB0, iA0
        yield 0, XA, XB
        for k in range(d.iterations):
            out = [np.empty_like(a) for a in (gA, vA, XB, gB, vB, XA)]
            Lh.hostemu_halves_pass(_p(gA), _p(vA), _p(XB), _p(nrm), _p(z), _p(albedo), W, H, 1 << k, C.byref(c), _p(out[0]), _p(out[1]),
                                   _p(out[2]))
            Lh.hostemu_halves_pass(_p(gB), _p(vB), _p(XA), _p(nrm), _p(z), _p(albedo), W, H, 1 << k, C.byref(c), _p(out[3]), _p(out[4]),
                                   _p(out[5]))
            gA, vA, XB, gB, vB, XA = out
            yield k + 1, XA, XB

    for k, XA, XB in chains():
        Lx.hostemu_cross_m(_p(XA), _p(XB), _p(iA0), _p(iB0), _p(vA0), _p(vB0), cp, _p(albedo), H * W, eps, _p(m))
        Lx.hostemu_cross_level(_p(m), W, H, k, _p(M), level.ctypes.data_as(u8p))
        ms.append(m.copy())
        O, junk, only = np.empty((H, W, 3)), np.empty((H, W)), np.full((H, W), k, np.uint8)
        Lx.hostemu_cross_blend(only.ctypes.data_as(u8p), _p(m), _p(XA), _p(XB), _p(sums), cp, _p(albedo), W, H, k, eps, _p(O), _p(junk))
        Os.append(O)
    for k, XA, XB in chains():
        Lx.hostemu_cross_m(_p(XA), _p(XB), _p(iA0), _p(iB0), _p(vA0), _p(vB0), cp, _p(albedo), H * W, eps, _p(m))
        Lx.hostemu_cross_blend(level.ctypes.data_as(u8p), _p(m), _p(XA), _p(XB), _p(sums), cp, _p(albedo), W, H, k, eps, _p(rgb), _p(M))
    return rgb, level, M, ms, Os


STATES = [(1, 1, 1), (7, 9, 3), (29, 37, 5), (37, 29, 3), (24, 48, 1), (45, 61, 5), (16, 16, 12), (40, 33, 12)]


def _state(H, W, it):
    return halves_state(H * 1000 + W + 7 * it + 1, H, W)


@pytest.mark.parametrize("H,W,it", STATES)
def test_cross_matches_numpy(H, W, it):
    state = _state(H, W, it)
    d = api.Denoise(iterations=it)
    rgb, level, M, ms, Os = emu_cross(*state, d)
    lv = xref.levels(*state, d)
    for k, (wO, wm, _) in enumerate(lv):
        _agree(ms[k], wm)
        _agree(Os[k], wO)
    wlevel = xref.argmin([wM for _, _, wM in lv])
    near = xref.ties(lv)
    assert np.array_equal(level[~near], wlevel[~near]), np.argwhere((level != wlevel) & ~near)[:8]
    # the blend restated over the emulation's own k*, and over numpy's where no neighbour's k* differs
    wrgb, wM = xref.blend(lv, level)
    _agree(rgb, wrgb)
    _agree(M, wM)
    same = ~xref.dilate(level != wlevel)
    wrgb2, wM2 = xref.blend(lv, wlevel)
    _agree(np.where(same[..., None], rgb, 0.0), np.where(same[..., None], wrgb2, 0.0))
    _agree(np.where(same, M, 0.0), np.where(same, wM2, 0.0))
    if H * W > 100:
        assert (level > 0).any() and np.isfinite(M).mean() > 0.5


def _uniform(level, k):
    """Pixels whose 5x5 in-image neighbourhood chose k throughout."""
    return ~xref.dilate(level != k)


@pytest.mark.parametrize("H,W,it", STATES)
def test_uniform_neighbourhood_is_its_level_and_every_output_a_convex_blend(H, W, it):
    state = _state(H, W, it)
    d = api.Denoise(iterations=it)
    rgb, level, _, _, Os = emu_cross(*state, d)
    for k in range(it + 1):
        at = _uniform(level, k)
        assert np.array_equal(rgb[at], Os[k][at], equal_nan=True), k
    # convex: between the least and the greatest of the levels the pixel blends, per channel
    used = np.stack([xref.beta(level, k)[0] > 0.0 for k in range(it + 1)])
    O = np.stack(Os)
    with np.errstate(invalid="ignore"):
        lo = np.where(used[..., None], O, np.inf).min(0)
        hi = np.where(used[..., None], O, -np.inf).max(0)
    ok = np.isfinite(lo) & np.isfinite(hi) & np.isfinite(rgb)
    tol = 1e-12 * np.maximum(np.abs(lo), np.abs(hi))
    assert (rgb[ok] >= lo[ok] - tol[ok]).all() and (rgb[ok] <= hi[ok] + tol[ok]).all()
    # a pixel with a NaN among the levels it blends is NaN, and only then
    bad = (used[..., None] & ~np.isfinite(O)).any(0)
    assert np.array_equal(~np.isfinite(rgb), bad)


def test_halves_demodulate_to_the_plain_mean():
    """n_A i_A + n_B i_B is n i: the halves add up to the plain demodulation, up to rounding."""
    sums, m2, half, counts, nrm, z, albedo = halves_state(5, 12, 14)
    eps = api.Denoise().albedo_eps
    iA, vA, iB, vB = xref.demodulate(sums, m2, half, counts, albedo, eps)
    n = counts.astype(np.float64)
    nb = np.floor(n / 2)
    with np.errstate(invalid="ignore", divide="ignore"):
        got = ((n - nb)[..., None] * iA + nb[..., None] * iB) / n[..., None]
        want = (sums / n[..., None]) / (albedo + eps)
        vwant = sums[..., 0] * 0 + m2 / ((n - 1) * n * 3)
    ok = (nb > 0) & np.isfinite(want).all(-1)
    assert np.allclose(got[ok], want[ok], rtol=1e-12, atol=1e-300)
    assert np.isnan(iA[nb == 0]).all() and np.isnan(vB[nb == 0]).all()
    fin = ok & np.isfinite(vwant)
    assert np.allclose(vA[fin] * (n - nb)[fin], vwant[fin] * n[fin], rtol=1e-12)
    assert np.allclose(vB[fin] * nb[fin], vwant[fin] * n[fin], rtol=1e-12)


# ---- statistics under fixed weights ----------------------------------------------------------------------------------
H_S, W_S, SEEDS = 32, 32, 300


def _truth():
    """(H, W, 3) radiance: a step (0.2 | 0.8 at the middle column) with a fine checker (+-0.1)."""
    y, x = np.mgrid[0:H_S, 0:W_S]
    t = np.where(x < W_S // 2, 0.2, 0.8) + 0.1 * np.where((x + y) % 2 == 0, 1.0, -1.0)
    return np.repeat(t[..., None], 3, -1) * np.array([1.0, 0.9, 0.8])


def _synthetic(n, sigma, d, seed=11):
    """Over SEEDS seeds of n Gaussian entries about the truth, flat features and albedo 0.5: per level k the mean of m_k
    and the empirical MSE of O_k (channel mean)."""
    truth = _truth()
    nrm = np.zeros((H_S, W_S, 3))
    nrm[..., 2] = 1.0
    z, albedo = np.full((H_S, W_S), 2.0), np.full((H_S, W_S, 3), 0.5)
    counts = np.full((H_S, W_S), n, np.uint32)
    rng = np.random.default_rng(seed)
    L = d.iterations + 1
    msum, esum = np.zeros((L, H_S, W_S)), np.zeros((L, H_S, W_S))
    for _ in range(SEEDS):
        x = truth + rng.normal(0.0, sigma, (n, H_S, W_S, 3))
        sums, half = x.sum(0), x[1::2].sum(0)
        m2 = ((x - x.mean(0)) ** 2).sum((0, 3))
        for k, (O, m, _) in enumerate(xref.levels(sums, m2, half, counts, nrm, z, albedo, d)):
            msum[k] += m
            esum[k] += ((O - truth) ** 2).mean(-1)
    return msum / SEEDS, esum / SEEDS


IN = (slice(6, -6), slice(6, -6))


@pytest.mark.parametrize("n", [8, 7])
def test_estimate_matches_the_error_of_every_level(n):
    """With weights that do not depend on the entries, m_k averaged over seeds is the MSE of level k, bias included, for
    even and odd counts: a step and a fine checker give the filtered levels a bias that grows with k."""
    d = api.Denoise(iterations=3, sigma_luminance=1e9)
    mbar, emp = _synthetic(n, 0.3, d)
    for k in range(d.iterations + 1):
        ratio = np.median(mbar[k][IN] / emp[k][IN])
        assert 0.9 < ratio < 1.1, (n, k, ratio)
    # the bias is real: every filtered level averages the checker away, so its error exceeds the checker's squared
    # amplitude (0.1^2 times the channels' mean squared scale, 0.00817)
    for k in range(1, d.iterations + 1):
        assert np.median(emp[k][IN]) > 0.0081, (n, k)


# ---- the C ABI -------------------------------------------------------------------------------------------------------
def test_abi_signature_matches_header():
    text = open(os.path.join(ROOT, "include", "rpt_b200.h")).read()
    flat = re.sub(r"\s+([,)])", r"\1", re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", text, flags=re.S)))
    assert ("int rptb_buffer_denoise_cross(rptb_buffer* buffer, const rptb_denoise* params, double* out_rgb, uint8_t* out_rgb8, "
            "uint8_t* out_level, double* out_mse);") in flat
    syms = {name: (res, args) for name, res, args in capi.SYMBOLS}
    assert syms["rptb_buffer_denoise_cross"] == syms["rptb_buffer_denoise_select"]
    assert hasattr(capi.lib(), "rptb_buffer_denoise_cross")
    hpp = open(os.path.join(ROOT, "include", "rpt.hpp")).read()
    assert "denoise_cross(const rptb_denoise& d)" in hpp


def test_errors_before_any_device_work():
    L = capi.lib()
    good = api.Denoise().to_c()
    fake = C.c_void_p(1)  # never looked at: the arguments are refused first
    assert L.rptb_buffer_denoise_cross(None, C.byref(good), None, None, None, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_cross(fake, None, None, None, None, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_cross(fake, C.byref(capi.Denoise(13, 128, 1.0, 4.0, 1e-3)), None, None, None, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_cross(fake, C.byref(capi.Denoise(0, 128, 1.0, 4.0, 1e-3)), None, None, None, None) == capi.ERR_BAD_ARG
    assert b"iterations" in L.rptb_last_error()
    for eps in (0.0, -1e-9, float("inf")):  # albedo_eps must be finite and > 0
        assert L.rptb_buffer_denoise_cross(fake, C.byref(capi.Denoise(5, 128, 1.0, 4.0, eps)), None, None, None, None) == capi.ERR_BAD_ARG
        assert b"albedo_eps" in L.rptb_last_error()


@pytest.mark.parametrize("kw,match", [({"cross": True}, "denoise"), ({"cross": True, "select": True, "denoise": api.Denoise()}, "one of")])
def test_render_cross_refusals_before_device_work(kw, match):
    cfg = scenes.sphere_scene()
    r = api.Renderer(cfg.scene, cfg.camera).width(8).height(8).num_samples(4)
    with pytest.raises(ValueError, match=match):
        r.render(**kw)
    assert r._dev_scene is None  # nothing reached the device
