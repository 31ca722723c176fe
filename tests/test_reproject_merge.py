"""The history test of rptb_buffer_reproject_merge without a GPU: reproject_merge and reproject_merge_slot
(reproject.h) in host emulation against their numpy restatement (tests/reproject_merge_ref.py) bit for bit -- on
synthetic states, on the whole image with features the emulated feature pass renders, and per element of every shard's
compact tiles for 1, 2, 3, 5 and 8 shards (ragged tiles and shards with no tile included) -- and the properties the
test must have: gamma = inf accepts every history, gamma = 0 rejects exactly the histories whose mean differs, a
rejected pixel keeps its bits, accepted sums are the two groups' sums, and the merged M2 is the exact two-group M2 to
within a bound derived from the operations.  Also the new entry points' argument checks and render_frames' refusals."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from rpt_b200.distributed import gather_permutation, render_frames_distributed, shard_tiles
from tests import reproject_merge_ref as mref
from tests.test_reproject import _p, emu_reproject, random_stats
from tests.test_shard_reproject import RAYS, SIZES, _cameras, _compact, _feature_sums, _lib, _resolve

dp, u32p = capi.c_double_p, capi.c_u32_p
EPS = np.finfo(np.float64).eps
GAMMAS = [0.0, 1.0, 3.0, math.inf]


def _merge_lib():
    L = _lib()
    cam, u64 = C.POINTER(capi.Camera), C.POINTER(C.c_uint64)
    L.hostemu_merge_pixels.restype = None
    L.hostemu_merge_pixels.argtypes = [dp, dp, u32p, C.c_uint64, C.c_double, dp, dp, u32p, C.POINTER(C.c_int32)]
    L.hostemu_reproject_merge.restype = None
    L.hostemu_reproject_merge.argtypes = [cam, C.c_uint32, C.c_uint32, dp, dp, dp, cam, C.c_uint32, C.c_uint32, dp, dp, u32p, dp, dp, dp,
                                          C.POINTER(capi.Reproject), C.c_double, dp, dp, u32p, u64, u64]
    L.hostemu_reproject_merge_part.restype = None
    L.hostemu_reproject_merge_part.argtypes = [cam, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, dp, C.c_uint64, C.c_double, cam,
                                               C.c_uint32, C.c_uint32, dp, dp, u32p, dp, dp, dp, C.POINTER(capi.Reproject), C.c_double,
                                               dp, dp, u32p, u64, u64]
    return L


def _u32(a):
    return a.ctypes.data_as(u32p)


def synthetic(rng, n):
    """Fresh and history states of n pixels: counts 0..9 on both sides (so some pixels have no history or fewer than 2
    fresh entries), means that sometimes agree exactly, nearly or not at all, and a few pixels of zero variance."""
    fn = rng.integers(0, 10, n).astype(np.uint32)
    hn = np.where(rng.random(n) < 0.15, 0, rng.integers(2, 10, n)).astype(np.uint32)
    fmu = rng.uniform(0.0, 2.0, (n, 3))
    kind = rng.integers(0, 3, n)
    hmu = np.where((kind == 0)[:, None], fmu, np.where((kind == 1)[:, None], fmu + rng.normal(0, 0.05, (n, 3)), rng.uniform(0, 2, (n, 3))))
    fm = rng.uniform(0.0, 0.3, n) * np.maximum(fn.astype(np.float64) - 1.0, 0.0)
    hm = rng.uniform(0.0, 0.3, n) * np.maximum(hn.astype(np.float64) - 1.0, 0.0)
    fm[rng.random(n) < 0.05] = 0.0
    hm[rng.random(n) < 0.05] = 0.0
    return hmu * hn[:, None], hm, hn, fmu * fn[:, None], fm, fn


def emu_merge(hs, hm, hn, gamma, fs, fm, fn):
    s, m, n = np.ascontiguousarray(fs, np.float64).copy(), np.ascontiguousarray(fm, np.float64).copy(), np.array(fn, np.uint32)
    verdict = np.empty(len(n), np.int32)
    hs, hm, hn = np.ascontiguousarray(hs, np.float64), np.ascontiguousarray(hm, np.float64), np.ascontiguousarray(hn, np.uint32)
    _merge_lib().hostemu_merge_pixels(_p(hs), _p(hm), _u32(hn), len(n), gamma, _p(s), _p(m), _u32(n),
                                      verdict.ctypes.data_as(C.POINTER(C.c_int32)))
    return s, m, n, verdict


def _same(got, want):
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.tobytes() == w.tobytes(), np.nanmax(np.abs(g.astype(float) - w.astype(float)))


@pytest.mark.parametrize("gamma", GAMMAS)
def test_merge_matches_numpy_on_synthetic_states(gamma):
    state = synthetic(np.random.default_rng(11), 20000)
    got = emu_merge(*state[:3], gamma, *state[3:])
    want = mref.merge(*state[:3], gamma, *state[3:])
    _same(got, want)
    v = want[3]
    assert (v == mref.NONE).any() and (v == mref.REUSED).any()
    assert (v == mref.REJECTED).any() == (gamma < math.inf)


def test_the_properties_of_the_test():
    hs, hm, hn, fs, fm, fn = synthetic(np.random.default_rng(12), 20000)
    tested = (hn > 0) & (fn >= 2)
    # gamma = inf accepts every history, even one of zero variance on both sides
    s, m, n, v = emu_merge(hs, hm, hn, math.inf, fs, fm, fn)
    assert np.array_equal(v == mref.REUSED, tested) and (v[~tested] == mref.NONE).all()
    assert ((fm == 0) & (hm == 0) & tested & (v == mref.REUSED)).any()
    # gamma = 0 rejects exactly where the means differ
    with np.errstate(invalid="ignore", divide="ignore"):
        d = hs / hn[:, None].astype(np.float64) - fs / fn[:, None].astype(np.float64)
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    for gamma in GAMMAS:
        s, m, n, v = emu_merge(hs, hm, hn, gamma, fs, fm, fn)
        if gamma == 0.0:
            assert np.array_equal(v == mref.REJECTED, tested & (d2 > 0)) and ((v == mref.REUSED) == (tested & (d2 == 0))).all()
        keep = v != mref.REUSED  # rejected and untested pixels keep their bits
        assert s[keep].tobytes() == fs[keep].tobytes() and m[keep].tobytes() == fm[keep].tobytes() and np.array_equal(n[keep], fn[keep])
        acc = v == mref.REUSED
        assert (s[acc] + 0.0).tobytes() == (fs[acc] + hs[acc]).tobytes()
        assert np.array_equal(n[acc], fn[acc] + hn[acc])
    # a larger gamma rejects a subset
    rej = [emu_merge(hs, hm, hn, g, fs, fm, fn)[3] == mref.REJECTED for g in GAMMAS]
    for a, b in zip(rej, rej[1:]):
        assert (b <= a).all()


def test_merged_m2_is_the_exact_two_group_m2():
    """The merged M2 against (M2_f + M2_h) + |mu_h - mu_f|^2 n_f n_h / n in fractions, from the same double inputs.
    Bound, first order in eps per operation: each delta_c = S_h/n_h - S_f/n_f carries at most eps (|mu_h| + |mu_f| +
    |delta_c|) of error, so d2 carries at most 2 eps sum_c |delta_c| (|mu_h| + |mu_f| + |delta_c|) + 2 eps d2; the
    weight n_f n_h / n three roundings, the products and the two sums one each.  Hence
        |M2 - M2_exact| <= 8 eps ((M2_f + M2_h) + w (d2 + sum_c |delta_c| (|mu_h| + |mu_f|))),  w = n_f n_h / n,
    with a margin of ~2 over those coefficients.  The printout gives the worst error / bound seen."""
    hs, hm, hn, fs, fm, fn = synthetic(np.random.default_rng(13), 3000)
    s, m, n, v = emu_merge(hs, hm, hn, math.inf, fs, fm, fn)
    worst = 0.0
    for p in np.flatnonzero(v == mref.REUSED):
        nf, nh = int(fn[p]), int(hn[p])
        mf = [Fraction(float(x)) / nf for x in fs[p]]
        mh = [Fraction(float(x)) / nh for x in hs[p]]
        w = Fraction(nf * nh, nf + nh)
        exact = Fraction(float(fm[p])) + Fraction(float(hm[p])) + w * sum((a - b) ** 2 for a, b in zip(mh, mf))
        dl = [float(a - b) for a, b in zip(mh, mf)]
        d2 = sum(x * x for x in dl)
        scale = sum(abs(x) * (abs(float(a)) + abs(float(b))) for x, a, b in zip(dl, mh, mf))
        bound = 8 * EPS * ((float(fm[p]) + float(hm[p])) + float(w) * (d2 + scale))
        err = abs(float(Fraction(float(m[p])) - exact))
        assert err <= bound, (p, err, bound)
        if bound > 0:
            worst = max(worst, err / bound)
    print(f"worst merged M2 error / bound {worst:.3g}")


def _fresh(rng, shape, hist_sums, hist_counts):
    """Fresh states for the destination: half the pixels near the history's mean (so they pass), half elsewhere."""
    fs, fm, fn = random_stats(rng, *shape)
    with np.errstate(invalid="ignore", divide="ignore"):
        hmu = np.where(hist_counts[..., None] > 0, hist_sums / hist_counts[..., None].astype(np.float64), 0.5)
    near = rng.random(shape) < 0.5
    fs = np.where(near[..., None], (hmu + rng.normal(0, 0.02, shape + (3,))) * fn[..., None], fs)
    fn[rng.random(shape) < 0.05] = 1  # a pixel an adaptive call would not have left at one entry: no test
    return fs, fm, fn


@pytest.mark.parametrize("dsize,ssize", SIZES)
def test_whole_and_shards_merge_like_numpy(dsize, ssize):
    (dw, dh), (sw, sh) = dsize, ssize
    scam, dcam = _cameras()
    L = _merge_lib()
    drows = _feature_sums(dcam, dw, dh)
    dN, dz, df = _resolve(drows, dw, dh)
    sN, sz, sf = _resolve(_feature_sums(scam, sw, sh), sw, sh)
    rng = np.random.default_rng(dw + 1)
    ssums, sm2, scounts = random_stats(rng, sh, sw)
    prm = api.Reproject()
    hist = emu_reproject(dcam, dN, dz, df, scam, ssums, sm2, scounts, sN, sz, sf, prm)
    plain_reused = int((hist[2] > 0).sum())
    fs, fm, fn = _fresh(rng, (dh, dw), hist[0], hist[2])
    src = [np.ascontiguousarray(a, np.float64) for a in (ssums, sm2, sN, sz, sf)]
    sc = np.ascontiguousarray(scounts, np.uint32)
    dc, scc, pc = dcam.to_c(), scam.to_c(), prm.to_c()
    dplanes = [np.ascontiguousarray(a, np.float64) for a in (dN, dz, df)]
    npix = dw * dh
    for gamma in (3.0, 0.0, math.inf):
        want = mref.reproject_merge(dcam, dN, dz, df, scam, ssums, sm2, scounts, sN, sz, sf, prm, gamma, fs, fm, fn)
        want_reused, want_rejected = int((want[3] == mref.REUSED).sum()), int((want[3] == mref.REJECTED).sum())
        # the identity: every pixel the plain reprojection gives history is tested, unless it has < 2 fresh entries
        assert want_reused + want_rejected == plain_reused - int(((hist[2] > 0) & (fn < 2)).sum())
        if gamma == 3.0:
            assert want_reused > 0 and want_rejected > 0
        # whole, row-major
        s, m, n = fs.copy(), fm.copy(), fn.copy()
        r, j = C.c_uint64(99), C.c_uint64(99)
        L.hostemu_reproject_merge(C.byref(dc), dw, dh, _p(dplanes[0]), _p(dplanes[1]), _p(dplanes[2]), C.byref(scc), sw, sh, _p(src[0]),
                                  _p(src[1]), _u32(sc), _p(src[2]), _p(src[3]), _p(src[4]), C.byref(pc), gamma, _p(s), _p(m), _u32(n),
                                  C.byref(r), C.byref(j))
        _same((s, m, n), want[:3])
        assert (r.value, j.value) == (want_reused, want_rejected)
        # per element of every shard's compact tiles
        for count in (1, 2, 3, 5, 8):
            perm = gather_permutation(dw, dh, count)
            slots = shard_tiles(dw, dh, 0, count) * 128
            owner, slot = perm // slots, perm % slots
            got_s, got_m, got_n = np.full((npix, 3), np.nan), np.full(npix, np.nan), np.full(npix, 7, np.uint32)
            total_r = total_j = 0
            for i in range(count):
                nelem = shard_tiles(dw, dh, i, count) * 128
                mine = owner == i
                feat = _compact(drows, npix, slot, mine, nelem)
                # the fresh state in element order; past a ragged edge a marker the merge must leave alone
                es, em, en = np.full((nelem, 3), -5.0), np.full(nelem, -6.0), np.full(nelem, 3, np.uint32)
                es[slot[mine]], em[slot[mine]], en[slot[mine]] = fs.reshape(-1, 3)[mine], fm.reshape(-1)[mine], fn.reshape(-1)[mine]
                L.hostemu_reproject_merge_part(C.byref(dc), dw, dh, i, count, _p(feat), nelem, float(RAYS), C.byref(scc), sw, sh,
                                               _p(src[0]), _p(src[1]), _u32(sc), _p(src[2]), _p(src[3]), _p(src[4]), C.byref(pc), gamma,
                                               _p(es), _p(em), _u32(en), C.byref(r), C.byref(j))
                ragged = np.ones(nelem, bool)
                ragged[slot[mine]] = False
                assert (es[ragged] == -5.0).all() and (em[ragged] == -6.0).all() and (en[ragged] == 3).all()
                if nelem == 0:
                    assert not mine.any() and r.value == 0 and j.value == 0
                total_r += r.value
                total_j += j.value
                got_s[mine], got_m[mine], got_n[mine] = es[slot[mine]], em[slot[mine]], en[slot[mine]]
            assert (total_r, total_j) == (want_reused, want_rejected), count
            _same((got_s.reshape(dh, dw, 3), got_m.reshape(dh, dw), got_n.reshape(dh, dw)), want[:3])
    if dsize == (20, 10):
        assert shard_tiles(dw, dh, 4, 5) == 0 and shard_tiles(dw, dh, 7, 8) == 0


def test_merge_errors_before_any_device_work():
    L = capi.lib()
    a, b = C.c_void_p(1), C.c_void_p(2)
    good = api.Reproject().to_c()
    for fn in (L.rptb_buffer_reproject_merge, L.rptb_buffer_reproject_merge_shard):
        assert fn(None, b, C.byref(good), 3.0, None, None) == capi.ERR_BAD_ARG
        assert fn(a, None, C.byref(good), 3.0, None, None) == capi.ERR_BAD_ARG
        assert fn(a, b, None, 3.0, None, None) == capi.ERR_BAD_ARG
        assert fn(a, a, C.byref(good), 3.0, None, None) == capi.ERR_BAD_ARG
        assert b"same buffer" in L.rptb_last_error()
        for prm in (api.Reproject(depth_tol=-0.1), api.Reproject(normal_cos=1.5), api.Reproject(max_history=1)):
            c = prm.to_c()
            assert fn(a, b, C.byref(c), 3.0, None, None) == capi.ERR_BAD_ARG
        for gamma in (math.nan, -1.0, -math.inf):
            assert fn(a, b, C.byref(good), gamma, None, None) == capi.ERR_BAD_ARG
            assert b"gamma" in L.rptb_last_error()


def test_render_frames_refuses_a_history_test_it_cannot_run():
    cfg = scenes.sphere_scene()
    r = api.Renderer(cfg.scene, cfg.camera).num_samples(8)
    bad = [dict(entries=4, history_test=api.HistoryTest(fresh_entries=1)),
           dict(entries=2, history_test=api.HistoryTest(fresh_entries=4)),
           dict(entries=4, reproject=None, history_test=api.HistoryTest())]
    for kw in bad:
        with pytest.raises(ValueError):
            next(r.render_frames([cfg.camera], **kw))
        with pytest.raises(ValueError):
            next(render_frames_distributed(r, [cfg.camera], **kw))
    assert r.camera is cfg.camera
