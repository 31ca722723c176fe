"""The choice of each pixel's number of filter passes without a GPU (rptb_buffer_denoise_select): select.h's per-pixel
functions in host emulation against their numpy restatement (tests/select_ref.py) on edge-case states (counts 0..9, NaN
and inf sums, image borders, infinite depths); every selected pixel against its level's plain filter output, bit for bit;
the estimate's statistics on synthetic entries under fixed weights, against the empirical error of every level; and the
C ABI's signature and refusals before any device work, including Renderer.render(select=True)'s."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import select_ref as sref
from tests.hostemu import emu
from tests.test_halves import _agree, _emu as _halves_emu, halves_state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dp, u32p, u8p = capi.c_double_p, capi.c_u32_p, capi.c_u8_p
_lib = None


def _emu():
    """tests/hostemu/_build/libhostemu_select.so: select.h compiled for the host."""
    global _lib
    if _lib is not None:
        return _lib
    emu.lib()  # `make hostemu` builds every emulation library
    L = C.CDLL(os.path.join(ROOT, "tests", "hostemu", "_build", "libhostemu_select.so"))
    L.hostemu_select_m.restype = None
    L.hostemu_select_m.argtypes = [dp, dp, dp, dp, dp, C.c_uint64, C.c_double, dp]
    L.hostemu_select_level.restype = None
    L.hostemu_select_level.argtypes = [dp, dp, dp, dp, u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, dp, dp, u8p]
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(dp)


def emu_select(sums, m2, half, counts, nrm, z, albedo, d):
    """select.cu's sequence through the host-compiled halves.h and select.h: (rgb, level, M, [m_k], [plain c'_k]), the last
    the plain filter's remodulated output after k passes (k >= 1) from hostemu_halves_plain_pass."""
    H, W = z.shape
    Lh, Ls, c = _halves_emu(), _emu(), d.to_c()
    eps = d.albedo_eps
    sums, m2 = np.ascontiguousarray(sums), np.ascontiguousarray(m2)
    i0, v0, u0 = np.empty((H, W, 3)), np.empty((H, W)), np.empty((H, W, 3))
    Lh.hostemu_halves_demodulate(_p(sums), _p(m2), _p(half), counts.ctypes.data_as(u32p), H * W, _p(albedo), eps, _p(i0), _p(v0), _p(u0))
    rgb, M, level, m = np.empty((H, W, 3)), np.empty((H, W)), np.empty((H, W), np.uint8), np.empty((H, W))
    Ls.hostemu_select_m(_p(i0), _p(u0), _p(i0), _p(u0), _p(albedo), H * W, eps, _p(m))
    Ls.hostemu_select_level(_p(m), _p(i0), _p(albedo), _p(sums), counts.ctypes.data_as(u32p), W, H, 0, eps, _p(rgb), _p(M),
                            level.ctypes.data_as(u8p))
    ms, plain = [m.copy()], [None]
    i, v, u, pi, pv = i0, v0, u0, i0.copy(), v0.copy()
    for k in range(d.iterations):
        i2, v2, u2 = np.empty_like(i), np.empty_like(v), np.empty_like(u)
        Lh.hostemu_halves_pass(_p(i), _p(v), _p(u), _p(nrm), _p(z), _p(albedo), W, H, 1 << k, C.byref(c), _p(i2), _p(v2), _p(u2))
        pi2, pv2 = np.empty_like(pi), np.empty_like(pv)
        Lh.hostemu_halves_plain_pass(_p(pi), _p(pv), _p(nrm), _p(z), _p(albedo), W, H, 1 << k, C.byref(c), _p(pi2), _p(pv2))
        i, v, u, pi, pv = i2, v2, u2, pi2, pv2
        Ls.hostemu_select_m(_p(i), _p(u), _p(i0), _p(u0), _p(albedo), H * W, eps, _p(m))
        Ls.hostemu_select_level(_p(m), _p(i), _p(albedo), _p(sums), counts.ctypes.data_as(u32p), W, H, k + 1, eps, _p(rgb), _p(M),
                                level.ctypes.data_as(u8p))
        ms.append(m.copy())
        with np.errstate(invalid="ignore", over="ignore"):
            plain.append(pi * (albedo + eps))
    return rgb, level, M, ms, plain


STATES = [(1, 1, 1), (7, 9, 3), (29, 37, 5), (37, 29, 3), (24, 48, 1), (45, 61, 5), (16, 16, 12), (40, 33, 12)]


@pytest.mark.parametrize("H,W,it", STATES)
def test_selection_matches_numpy(H, W, it):
    state = halves_state(H * 1000 + W + 7 * it, H, W)
    d = api.Denoise(iterations=it)
    rgb, level, M, ms, _ = emu_select(*state, d)
    lv = sref.levels(*state, d)
    for k, (_, wm, _) in enumerate(lv):
        _agree(ms[k], wm)
    wrgb, wlevel, wM = sref.select(*state, d)
    near = sref.ties(*state, d)
    assert np.array_equal(level[~near], wlevel[~near]), np.argwhere((level != wlevel) & ~near)[:8]
    same = level == wlevel
    _agree(np.where(same, M, 0.0), np.where(same, wM, 0.0))
    _agree(np.where(same[..., None], rgb, 0.0), np.where(same[..., None], wrgb, 0.0))
    if H * W > 100:
        assert (level > 0).any() and np.isfinite(M).mean() > 0.5


@pytest.mark.parametrize("H,W,it", STATES)
def test_every_pixel_is_its_levels_plain_output(H, W, it):
    sums, m2, half, counts, nrm, z, albedo = state = halves_state(H * 1000 + W + 7 * it, H, W)
    rgb, level, _, _, plain = emu_select(*state, api.Denoise(iterations=it))
    with np.errstate(invalid="ignore", divide="ignore"):
        raw = sums / counts.astype(np.float64)[..., None]
    for k in range(it + 1):
        at = level == k
        want = raw if k == 0 else plain[k]
        assert np.array_equal(rgb[at], want[at], equal_nan=True), k


def test_level_zero_estimate_is_the_raw_variance():
    """m_0 = u_0^2 remodulated: 2x - x is exact, so level 0 needs no rule of its own."""
    sums, m2, half, counts, nrm, z, albedo = halves_state(5, 12, 14)
    d = api.Denoise(iterations=1)
    u0 = sref.href.u_plane(sums, half, counts, albedo, d.albedo_eps)
    _, _, _, ms, _ = emu_select(sums, m2, half, counts, nrm, z, albedo, d)
    with np.errstate(invalid="ignore"):
        r = (u0 * u0 * (albedo + d.albedo_eps)) * (albedo + d.albedo_eps)
        want = ((r[..., 0] + r[..., 1]) + r[..., 2]) / 3.0
    assert np.array_equal(ms[0], want, equal_nan=True)


# ---- statistics under fixed weights ----------------------------------------------------------------------------------
H_S, W_S, N_S, SEEDS = 32, 32, 8, 300


def _truth(kind):
    """(H, W, 3) radiance: "detail" a step (0.2 | 0.8 at the middle column) with a fine checker (+-0.1), "flat" 0.5."""
    if kind == "flat":
        return np.full((H_S, W_S, 3), 0.5)
    y, x = np.mgrid[0:H_S, 0:W_S]
    t = np.where(x < W_S // 2, 0.2, 0.8) + 0.1 * np.where((x + y) % 2 == 0, 1.0, -1.0)
    return np.repeat(t[..., None], 3, -1) * np.array([1.0, 0.9, 0.8])


def _synthetic(kind, sigma, d, seed=11):
    """Over SEEDS seeds of N_S Gaussian entries about the truth, flat features and albedo 0.5: per level k the mean of
    m_k and the empirical MSE of c_k (channel mean), and the selection's level and MSE."""
    truth = _truth(kind)
    nrm = np.zeros((H_S, W_S, 3))
    nrm[..., 2] = 1.0
    z, albedo = np.full((H_S, W_S), 2.0), np.full((H_S, W_S, 3), 0.5)
    counts = np.full((H_S, W_S), N_S, np.uint32)
    rng = np.random.default_rng(seed)
    L = d.iterations + 1
    msum, esum = np.zeros((L, H_S, W_S)), np.zeros((L, H_S, W_S))
    sel_err, levels = np.zeros((H_S, W_S)), []
    for _ in range(SEEDS):
        x = truth + rng.normal(0.0, sigma, (N_S, H_S, W_S, 3))
        sums, half = x.sum(0), x[1::2].sum(0)
        m2 = ((x - x.mean(0)) ** 2).sum((0, 3))
        state = (sums, m2, half, counts, nrm, z, albedo)
        for k, (c, m, _) in enumerate(sref.levels(*state, d)):
            msum[k] += m
            esum[k] += ((c - truth) ** 2).mean(-1)
        rgb, level, _ = sref.select(*state, d)
        sel_err += ((rgb - truth) ** 2).mean(-1)
        levels.append(level)
    return msum / SEEDS, esum / SEEDS, sel_err / SEEDS, np.stack(levels)


IN = (slice(6, -6), slice(6, -6))


def test_estimate_matches_the_error_of_every_level():
    """With weights that do not depend on the entries, m_k averaged over seeds is the MSE of level k, bias included: a
    step and a fine checker give the filtered levels a bias that grows with k."""
    d = api.Denoise(iterations=3, sigma_luminance=1e9)
    mbar, emp, _, _ = _synthetic("detail", 0.3, d)
    for k in range(d.iterations + 1):
        ratio = np.median(mbar[k][IN] / emp[k][IN])
        assert 0.9 < ratio < 1.1, (k, ratio)
    # the bias is real: the deepest level is worse than raw at the checker
    assert np.median(emp[-1][IN]) > np.median(emp[0][IN])


def test_flat_truth_selects_filtered_levels():
    d = api.Denoise(iterations=3, sigma_luminance=1e9)
    _, emp, sel, levels = _synthetic("flat", 0.3, d)
    assert (levels[:, 6:-6, 6:-6] >= 1).mean() > 0.9
    assert sel[IN].mean() < 0.5 * emp[0][IN].mean(), (sel[IN].mean(), emp[0][IN].mean())


def test_converged_detail_keeps_the_raw_mean():
    """A fine checker with tiny noise: every filtered level is all bias, so most pixels keep level 0 and the output does
    not lose to the raw mean."""
    d = api.Denoise(iterations=3, sigma_luminance=1e9)
    _, emp, sel, levels = _synthetic("detail", 1e-3, d)
    assert (levels[:, 6:-6, 6:-6] == 0).mean() > 0.9
    assert sel[IN].mean() <= emp[0][IN].mean(), (sel[IN].mean(), emp[0][IN].mean())


# ---- the C ABI -------------------------------------------------------------------------------------------------------
def test_abi_signature_matches_header():
    text = open(os.path.join(ROOT, "include", "rpt_b200.h")).read()
    flat = re.sub(r"\s+([,)])", r"\1", re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", text, flags=re.S)))
    assert ("int rptb_buffer_denoise_select(rptb_buffer* buffer, const rptb_denoise* params, double* out_rgb, uint8_t* out_rgb8, "
            "uint8_t* out_level, double* out_mse);") in flat
    syms = {name: (res, args) for name, res, args in capi.SYMBOLS}
    assert syms["rptb_buffer_denoise_select"][1][:4] == syms["rptb_buffer_denoise"][1]
    assert len(syms["rptb_buffer_denoise_select"][1]) == 6
    assert hasattr(capi.lib(), "rptb_buffer_denoise_select")
    hpp = open(os.path.join(ROOT, "include", "rpt.hpp")).read()
    assert "denoise_select(const rptb_denoise& d)" in hpp


def test_errors_before_any_device_work():
    L = capi.lib()
    good = api.Denoise().to_c()
    fake = C.c_void_p(1)  # never looked at: the arguments are refused first
    assert L.rptb_buffer_denoise_select(None, C.byref(good), None, None, None, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_select(fake, None, None, None, None, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_select(fake, C.byref(capi.Denoise(13, 128, 1.0, 4.0, 1e-3)), None, None, None, None) == capi.ERR_BAD_ARG
    assert L.rptb_buffer_denoise_select(fake, C.byref(capi.Denoise(0, 128, 1.0, 4.0, 1e-3)), None, None, None, None) == capi.ERR_BAD_ARG
    assert b"iterations" in L.rptb_last_error()
    for eps in (0.0, -1e-9, float("inf")):  # albedo_eps must be finite and > 0
        assert L.rptb_buffer_denoise_select(fake, C.byref(capi.Denoise(5, 128, 1.0, 4.0, eps)), None, None, None, None) == capi.ERR_BAD_ARG
        assert b"albedo_eps" in L.rptb_last_error()


def test_render_select_needs_denoise_before_device_work():
    cfg = scenes.sphere_scene()
    r = api.Renderer(cfg.scene, cfg.camera).width(8).height(8).num_samples(4)
    with pytest.raises(ValueError, match="denoise"):
        r.render(select=True)
    assert r._dev_scene is None  # nothing reached the device
