"""The history halves of a reprojection and a merge without a GPU: reproject_pixel_halves, reproject_slot_halves,
reproject_merge_halves and reproject_merge_slot_halves (reproject.h) in host emulation against their numpy restatement
(tests/reproject_halves_ref.py) bit for bit -- on synthetic states (odd and even counts, capped and uncapped histories,
one-tap histories, environment pixels) and per element of every shard's compact tiles for 1 to 8 shards (ragged tiles
and shards with no tile included) -- with sums, M2 and counts that are the plain functions' bits.  Then the properties
the halves must have: the parity rule of the merge on constant entries, and the calibration of the error estimate's u
on Gaussian entries of known sigma, after a reprojection and after accepted merges."""
import ctypes as C
import math

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api
from rpt_b200.distributed import gather_permutation, shard_tiles
from tests import halves_ref as href
from tests import reproject_halves_ref as hr
from tests import reproject_merge_ref as mref
from tests.test_reproject import _cam, _p, emu_reproject, orbit, random_features, random_stats
from tests.test_reproject_merge import emu_merge
from tests.test_shard_reproject import RAYS, SIZES, _cameras, _compact, _feature_sums, _lib, _resolve

dp, u32p = capi.c_double_p, capi.c_u32_p
u64 = C.POINTER(C.c_uint64)


def _halves_lib():
    L = _lib()
    cam, prm = C.POINTER(capi.Camera), C.POINTER(capi.Reproject)
    L.hostemu_reproject_halves.restype = None
    L.hostemu_reproject_halves.argtypes = [cam, C.c_uint32, C.c_uint32, dp, dp, dp, cam, C.c_uint32, C.c_uint32, dp, dp, u32p, dp, dp, dp,
                                           dp, prm, dp, dp, u32p, dp]
    L.hostemu_reproject_halves_part.restype = None
    L.hostemu_reproject_halves_part.argtypes = [cam, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, dp, C.c_uint64, C.c_double, cam,
                                                C.c_uint32, C.c_uint32, dp, dp, u32p, dp, dp, dp, dp, prm, dp, dp, u32p, dp, u64]
    L.hostemu_merge_halves_pixels.restype = None
    L.hostemu_merge_halves_pixels.argtypes = [dp, dp, u32p, dp, C.c_uint64, C.c_double, dp, dp, u32p, dp, C.POINTER(C.c_int32)]
    L.hostemu_reproject_merge_halves_part.restype = None
    L.hostemu_reproject_merge_halves_part.argtypes = [cam, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, dp, C.c_uint64, C.c_double,
                                                      cam, C.c_uint32, C.c_uint32, dp, dp, u32p, dp, dp, dp, dp, prm, C.c_double, dp, dp,
                                                      u32p, dp, u64, u64]
    return L


def _u32(a):
    return a.ctypes.data_as(u32p)


def _f64(*arrays):
    return [np.ascontiguousarray(a, np.float64) for a in arrays]


def _same(got, want):
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.tobytes() == w.tobytes(), np.nanmax(np.abs(g.astype(float) - w.astype(float)))


def random_half(rng, sums, counts):
    """A HALF plane for states of random_stats: the odd entries' share of the sums, with noise of its own."""
    nb = (np.asarray(counts, np.uint32) >> 1).astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = np.where(counts[..., None] > 0, sums / counts[..., None].astype(np.float64), 0.0)
    return (mean + rng.normal(0.0, 0.1, sums.shape)) * nb[..., None]


def emu_reproject_halves(dcam, dnrm, dz, df, scam, ssums, sm2, scounts, shalf, snrm, sz, sf, prm):
    dh, dw = dz.shape
    sh, sw = sz.shape
    c = _f64(dnrm, dz, df, ssums, sm2, shalf, snrm, sz, sf)
    sc = np.ascontiguousarray(scounts, np.uint32)
    out_s, out_m, out_n, out_h = np.empty((dh, dw, 3)), np.empty((dh, dw)), np.empty((dh, dw), np.uint32), np.empty((dh, dw, 3))
    dc, scc, pc = dcam.to_c(), scam.to_c(), prm.to_c()
    _halves_lib().hostemu_reproject_halves(C.byref(dc), dw, dh, _p(c[0]), _p(c[1]), _p(c[2]), C.byref(scc), sw, sh, _p(c[3]), _p(c[4]),
                                           _u32(sc), _p(c[5]), _p(c[6]), _p(c[7]), _p(c[8]), C.byref(pc), _p(out_s), _p(out_m),
                                           _u32(out_n), _p(out_h))
    return out_s, out_m, out_n, out_h


def emu_merge_halves(hs, hm, hn, hh, gamma, fs, fm, fn, fh):
    s, m, n, h = np.array(fs, np.float64), np.array(fm, np.float64), np.array(fn, np.uint32), np.array(fh, np.float64)
    verdict = np.empty(len(n), np.int32)
    hs, hm, hh = _f64(hs, hm, hh)
    hn = np.ascontiguousarray(hn, np.uint32)
    _halves_lib().hostemu_merge_halves_pixels(_p(hs), _p(hm), _u32(hn), _p(hh), len(n), gamma, _p(s), _p(m), _u32(n), _p(h),
                                              verdict.ctypes.data_as(C.POINTER(C.c_int32)))
    return s, m, n, h, verdict


PRMS = [api.Reproject(), api.Reproject(depth_tol=0.5, normal_cos=-1.0, max_history=3), api.Reproject(0.02, 0.9, 64)]


@pytest.mark.parametrize("dsize,ssize,angle,seed", [((23, 17), (23, 17), 0.05, 1), ((31, 20), (19, 27), -0.08, 2),
                                                     ((1, 1), (9, 7), 0.0, 3), ((40, 9), (40, 9), 0.4, 4)])
def test_emulation_matches_numpy_on_synthetic_states(dsize, ssize, angle, seed):
    rng = np.random.default_rng(seed)
    (dw, dh), (sw, sh) = dsize, ssize
    scam = api.Camera.look_at(api.vec3(1.0, 2.0, 6.0), api.vec3(0.0, 0.0, 0.0), api.vec3(0.0, 1.0, 0.0), 0.8)
    dcam = orbit(scam, (0.0, 0.0, 0.0), angle, lift=0.1)
    dN, dz, df = random_features(rng, dh, dw)
    sN, sz, sf = random_features(rng, sh, sw)
    sums, m2, counts = random_stats(rng, sh, sw, lo=0, hi=12)
    half = random_half(rng, sums, counts)
    sums[rng.random((sh, sw)) < 0.05] = np.nan
    m2[rng.random((sh, sw)) < 0.05] = np.inf
    for prm in PRMS:
        want = hr.reproject(dcam, dN, dz, df, scam, sums, m2, counts, half, sN, sz, sf, prm)
        got = emu_reproject_halves(dcam, dN, dz, df, scam, sums, m2, counts, half, sN, sz, sf, prm)
        _same(got, want)
        _same(got[:3], emu_reproject(dcam, dN, dz, df, scam, sums, m2, counts, sN, sz, sf, prm))  # the plain bits
        assert (got[3][got[2] == 0] == 0).all()  # no history: HALF 0


def test_one_tap_histories_and_the_environment():
    """The identity camera (one tap a pixel, or nearly) over surface and environment pixels, capped and uncapped, with odd
    and even counts: numpy's bits, and every pixel keeps history."""
    rng = np.random.default_rng(21)
    H, W = 21, 26
    N, z, f = random_features(rng, H, W, env_frac=0.3)
    cam = _cam()
    for lo, hi in ((2, 3), (3, 4), (2, 20)):
        sums, m2, counts = random_stats(rng, H, W, lo, hi)
        half = random_half(rng, sums, counts)
        for mh in (2, 3, 8, 64):
            prm = api.Reproject(max_history=mh)
            want = hr.reproject(cam, N, z, f, cam, sums, m2, counts, half, N, z, f, prm)
            _same(emu_reproject_halves(cam, N, z, f, cam, sums, m2, counts, half, N, z, f, prm), want)
            assert (want[2] > 0).all() and ((f == 0) & (want[2] > 0)).any()
            assert (want[2] == np.minimum(counts, mh)).mean() > 0.5  # most pixels take their own pixel's history


def _shard_setup(dsize, ssize, seed):
    (dw, dh), (sw, sh) = dsize, ssize
    scam, dcam = _cameras()
    drows = _feature_sums(dcam, dw, dh)
    dN, dz, df = _resolve(drows, dw, dh)
    sN, sz, sf = _resolve(_feature_sums(scam, sw, sh), sw, sh)
    rng = np.random.default_rng(seed)
    ssums, sm2, scounts = random_stats(rng, sh, sw, lo=2, hi=14)
    shalf = random_half(rng, ssums, scounts)
    return rng, scam, dcam, drows, (dN, dz, df), (ssums, sm2, scounts, shalf, sN, sz, sf)


def _deal(dw, dh, count):
    perm = gather_permutation(dw, dh, count)
    slots = shard_tiles(dw, dh, 0, count) * 128
    return perm // slots, perm % slots


@pytest.mark.parametrize("dsize,ssize", SIZES)
def test_shards_reproject_halves_like_numpy(dsize, ssize):
    (dw, dh), (sw, sh) = dsize, ssize
    L = _halves_lib()
    rng, scam, dcam, drows, (dN, dz, df), src = _shard_setup(dsize, ssize, dw)
    ssums, sm2, scounts, shalf, sN, sz, sf = src
    c = _f64(ssums, sm2, shalf, sN, sz, sf)
    sc = np.ascontiguousarray(scounts, np.uint32)
    npix = dw * dh
    for prm in (api.Reproject(), api.Reproject(max_history=5)):
        want = hr.reproject(dcam, dN, dz, df, scam, ssums, sm2, scounts, shalf, sN, sz, sf, prm)
        assert (want[2] % 2 == 1).any() and (want[2] % 2 == 0).any() and (want[2] == 0).any()
        dc, scc, pc = dcam.to_c(), scam.to_c(), prm.to_c()
        for count in range(1, 9):
            owner, slot = _deal(dw, dh, count)
            got = [np.full((npix, 3), np.nan), np.full(npix, np.nan), np.full(npix, 7, np.uint32), np.full((npix, 3), np.nan)]
            total = 0
            for i in range(count):
                nelem = shard_tiles(dw, dh, i, count) * 128
                mine = owner == i
                feat = _compact(drows, npix, slot, mine, nelem)
                out = [np.empty((nelem, 3)), np.empty(nelem), np.empty(nelem, np.uint32), np.empty((nelem, 3))]
                plain = [np.empty((nelem, 3)), np.empty(nelem), np.empty(nelem, np.uint32)]
                r, rp = C.c_uint64(99), C.c_uint64(99)
                L.hostemu_reproject_halves_part(C.byref(dc), dw, dh, i, count, _p(feat), nelem, float(RAYS), C.byref(scc), sw, sh, _p(c[0]),
                                                _p(c[1]), _u32(sc), _p(c[2]), _p(c[3]), _p(c[4]), _p(c[5]), C.byref(pc), _p(out[0]),
                                                _p(out[1]), _u32(out[2]), _p(out[3]), C.byref(r))
                L.hostemu_reproject_part(C.byref(dc), dw, dh, i, count, _p(feat), nelem, float(RAYS), C.byref(scc), sw, sh, _p(c[0]),
                                         _p(c[1]), _u32(sc), _p(c[3]), _p(c[4]), _p(c[5]), C.byref(pc), _p(plain[0]), _p(plain[1]),
                                         _u32(plain[2]), C.byref(rp))
                _same(out[:3], plain)
                assert r.value == rp.value
                total += r.value
                ragged = np.ones(nelem, bool)
                ragged[slot[mine]] = False
                assert (out[3][ragged] == 0).all() and (out[2][ragged] == 0).all()
                if nelem == 0:
                    assert not mine.any() and r.value == 0
                for g, o in zip(got, out):
                    g[mine] = o[slot[mine]]
            assert total == int((want[2] > 0).sum()), count
            _same((got[0].reshape(dh, dw, 3), got[1].reshape(dh, dw), got[2].reshape(dh, dw), got[3].reshape(dh, dw, 3)), want)
    if dsize == (20, 10):
        assert shard_tiles(dw, dh, 4, 5) == 0 and shard_tiles(dw, dh, 7, 8) == 0


@pytest.mark.parametrize("dsize,ssize", SIZES)
def test_shards_merge_halves_like_numpy(dsize, ssize):
    (dw, dh), (sw, sh) = dsize, ssize
    L = _halves_lib()
    rng, scam, dcam, drows, (dN, dz, df), src = _shard_setup(dsize, ssize, dw + 1)
    ssums, sm2, scounts, shalf, sN, sz, sf = src
    prm = api.Reproject()
    hist = hr.reproject(dcam, dN, dz, df, scam, ssums, sm2, scounts, shalf, sN, sz, sf, prm)
    fs, fm, fn = random_stats(rng, dh, dw, lo=1, hi=9)
    with np.errstate(invalid="ignore", divide="ignore"):
        hmu = np.where(hist[2][..., None] > 0, hist[0] / hist[2][..., None].astype(np.float64), 0.5)
    near = rng.random((dh, dw)) < 0.5
    fs = np.where(near[..., None], (hmu + rng.normal(0, 0.02, (dh, dw, 3))) * fn[..., None], fs)
    fh = random_half(rng, fs, fn)
    c = _f64(ssums, sm2, shalf, sN, sz, sf)
    sc = np.ascontiguousarray(scounts, np.uint32)
    dc, scc, pc = dcam.to_c(), scam.to_c(), prm.to_c()
    npix = dw * dh
    for gamma in (3.0, 0.0, math.inf):
        want = hr.reproject_merge(dcam, dN, dz, df, scam, ssums, sm2, scounts, shalf, sN, sz, sf, prm, gamma, fs, fm, fn, fh)
        plain = mref.reproject_merge(dcam, dN, dz, df, scam, ssums, sm2, scounts, sN, sz, sf, prm, gamma, fs, fm, fn)
        _same(want[:3] + (want[4],), plain[:3] + (plain[3],))
        acc = want[4] == mref.REUSED
        if gamma != 0.0:
            assert (acc & (fn % 2 == 1)).any() and (acc & (fn % 2 == 0)).any()
        assert want[3][~acc].tobytes() == fh[~acc].tobytes()
        for count in range(1, 9):
            owner, slot = _deal(dw, dh, count)
            got = [np.full((npix, 3), np.nan), np.full(npix, np.nan), np.full(npix, 7, np.uint32), np.full((npix, 3), np.nan)]
            tr = tj = 0
            for i in range(count):
                nelem = shard_tiles(dw, dh, i, count) * 128
                mine = owner == i
                feat = _compact(drows, npix, slot, mine, nelem)
                # the fresh state in element order; past a ragged edge a marker the merge must leave alone
                es, em, en, eh = np.full((nelem, 3), -5.0), np.full(nelem, -6.0), np.full(nelem, 3, np.uint32), np.full((nelem, 3), -7.0)
                es[slot[mine]], em[slot[mine]], en[slot[mine]] = fs.reshape(-1, 3)[mine], fm.reshape(-1)[mine], fn.reshape(-1)[mine]
                eh[slot[mine]] = fh.reshape(-1, 3)[mine]
                r, j = C.c_uint64(99), C.c_uint64(99)
                L.hostemu_reproject_merge_halves_part(C.byref(dc), dw, dh, i, count, _p(feat), nelem, float(RAYS), C.byref(scc), sw, sh,
                                                      _p(c[0]), _p(c[1]), _u32(sc), _p(c[2]), _p(c[3]), _p(c[4]), _p(c[5]), C.byref(pc),
                                                      gamma, _p(es), _p(em), _u32(en), _p(eh), C.byref(r), C.byref(j))
                ragged = np.ones(nelem, bool)
                ragged[slot[mine]] = False
                assert (es[ragged] == -5.0).all() and (em[ragged] == -6.0).all() and (en[ragged] == 3).all() and (eh[ragged] == -7.0).all()
                if nelem == 0:
                    assert not mine.any() and r.value == 0 and j.value == 0
                tr += r.value
                tj += j.value
                for g, o in zip(got, (es, em, en, eh)):
                    g[mine] = o[slot[mine]]
            assert (tr, tj) == (int(acc.sum()), int((want[4] == mref.REJECTED).sum())), count
            _same((got[0].reshape(dh, dw, 3), got[1].reshape(dh, dw), got[2].reshape(dh, dw), got[3].reshape(dh, dw, 3)), want[:4])


def test_merge_halves_matches_numpy_and_the_plain_merge_on_synthetic_states():
    rng = np.random.default_rng(31)
    n = 20000
    fn = rng.integers(0, 12, n).astype(np.uint32)
    hn = np.where(rng.random(n) < 0.15, 0, rng.integers(2, 12, n)).astype(np.uint32)
    fmu, hmu = rng.uniform(0, 2, (n, 3)), rng.uniform(0, 2, (n, 3))
    hmu = np.where((rng.random(n) < 0.5)[:, None], fmu, hmu)
    fs, hs = fmu * fn[:, None], hmu * hn[:, None]
    fm, hm = rng.uniform(0, 0.3, n) * np.maximum(fn - 1.0, 0), rng.uniform(0, 0.3, n) * np.maximum(hn - 1.0, 0)
    fh, hh = random_half(rng, fs, fn), random_half(rng, hs, hn)
    for gamma in (0.0, 1.0, 3.0, math.inf):
        got = emu_merge_halves(hs, hm, hn, hh, gamma, fs, fm, fn, fh)
        _same(got, hr.merge(hs, hm, hn, hh, gamma, fs, fm, fn, fh))
        _same(got[:3] + (got[4],), emu_merge(hs, hm, hn, gamma, fs, fm, fn))


def _u(sums, half, counts):
    """halves_u before the albedo (albedo 0, eps_a 1)."""
    z = np.zeros(sums.shape)
    return href.u_plane(sums, half, counts, z, 1.0)


def test_parity_rule_gives_u_zero_on_constant_entries():
    """Taps and fresh entries all c = 0.5: after a reprojection and a merge at gamma = inf, u is exactly 0 for every parity
    of n_f and n_h.  Without the swap (always adding the history's B half) a pixel with n_f and n_h both odd gets u != 0."""
    c = 0.5
    H, W = 9, 12
    rng = np.random.default_rng(41)
    N, z, f = random_features(rng, H, W, env_frac=0.3)
    cam = _cam()
    prm = api.Reproject(max_history=8)
    for nq in (2, 3, 4, 5, 7, 9, 12):  # odd and even histories below max_history, and capped ones
        counts = np.full((H, W), nq, np.uint32)
        sums = np.full((H, W, 3), c * nq)
        half = np.full((H, W, 3), c * (nq // 2))
        hs, hm, hn, hh = emu_reproject_halves(cam, N, z, f, cam, sums, np.zeros((H, W)), counts, half, N, z, f, prm)
        exact = (hn > 0) & (hs == hn[..., None] * c).all(-1)  # taps whose weights sum to 1 exactly
        assert exact.mean() > 0.5
        hs, hm, hn, hh = hs[exact], hm[exact], hn[exact], hh[exact]
        assert (_u(hs, hh, hn) == 0).all()
        for nf in (2, 3, 4, 5):
            k = len(hn)
            fs, fh = np.full((k, 3), c * nf), np.full((k, 3), c * (nf // 2))
            s, m, n, h, v = emu_merge_halves(hs, hm, hn, hh, math.inf, fs, np.zeros(k), np.full(k, nf, np.uint32), fh)
            assert (v == mref.REUSED).all()
            assert (_u(s, h, n) == 0).all(), (nq, nf)
            naive = fh + hh  # the history's B half whatever n_f's parity
            u_naive = _u(s, naive, n)
            if nf % 2 == 1 and int(hn[0]) % 2 == 1:
                assert (u_naive != 0).all(), (nq, nf)
            else:
                assert (u_naive == 0).all(), (nq, nf)


def _gaussian_state(rng, H, W, sigma, m, lo, hi):
    """States of entries N(m, sigma^2) with counts lo..hi-1: sums, M2, counts and HALF drawn from their exact laws."""
    counts = rng.integers(lo, hi, (H, W)).astype(np.uint32)
    nb = (counts >> 1).astype(np.float64)
    na = counts.astype(np.float64) - nb
    SA = na[..., None] * m + rng.normal(size=(H, W, 3)) * (sigma * np.sqrt(na))[..., None]
    SB = nb[..., None] * m + rng.normal(size=(H, W, 3)) * (sigma * np.sqrt(nb))[..., None]
    m2 = sigma * sigma * rng.chisquare(counts - 1.0)
    return SA + SB, m2, counts, SB


def test_calibration_of_u_after_reprojection_and_merge():
    """Entries N(m, sigma^2), counts 2..64, an environment view turned so that pixels take up to four taps: the mean of
    u^2 n_h / sigma^2 over the reprojected pixels lies within 3 % of 1, and so does u^2 n / sigma^2 after accepted merges
    (gamma = inf) with fresh entries of the same law."""
    rng = np.random.default_rng(51)
    H, W, sigma = 300, 400, 0.3
    scam = _cam()
    dcam = api.Camera.look_at(scam.eye, api.vec3(0.1, -0.05, 0.04), api.vec3(0.0, 1.0, 0.0), 0.9)
    zero3, env = np.zeros((H, W, 3)), np.zeros((H, W))
    zinf = np.full((H, W), np.inf)
    m = np.array([0.2, 0.5, 0.9])
    sums, m2, counts, half = _gaussian_state(rng, H, W, sigma, m, 2, 65)
    prm = api.Reproject(max_history=16)
    hs, hm, hn, hh = hr.reproject(dcam, zero3, zinf, env, scam, sums, m2, counts, half, zero3, zinf, env, prm)
    got = hn > 0
    assert got.sum() >= 100000
    assert (hn[got] < 16).any() and (hn[got] == 16).any()  # uncapped and capped histories
    u = _u(hs, hh, hn)[got]
    ratio = float(np.mean(u * u * hn[got][:, None] / sigma**2))
    print(f"\nreprojected: mean u^2 n_h / sigma^2 = {ratio:.4f} over {int(got.sum())} pixels")
    assert abs(ratio - 1.0) < 0.03, ratio
    # fresh entries of the same law, merged at gamma = inf
    fs, fm, fn, fh = _gaussian_state(rng, H, W, sigma, m, 2, 17)
    s, _, n, h, v = hr.merge(hs, hm, hn, hh, math.inf, fs, fm, fn, fh)
    acc = v == mref.REUSED
    assert acc.sum() >= 100000
    u = _u(s, h, n)[acc]
    ratio = float(np.mean(u * u * n[acc][:, None] / sigma**2))
    print(f"merged: mean u^2 n / sigma^2 = {ratio:.4f} over {int(acc.sum())} pixels")
    assert abs(ratio - 1.0) < 0.03, ratio
