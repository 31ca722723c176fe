"""Every list-scheduled render variant on the GPU (-m gpu): adaptive sampling's render_list_kernel and
resolve_chunks_list_kernel against the tile schedule and the oracle, under masks the test chooses.

An adaptive call renders the pixels its criterion leaves active, and that criterion is a pure function of the pixel's
entries.  So a fresh DeviceBuffer given two host entries, (1, 1, 1) then (-1, -1, -1) on the pixels of a mask and 0
then 0 elsewhere, holds S = 0, M2 = 6, n = 2 on the mask (err^2 = 6 / (1 * 2 * 3) = 1) and zeros off it; under
Adaptive(0, 0.5, 2) exactly the mask is active (1 > 0.25, 0 <= 0.25), and after one call a masked pixel's sum is
0 + x = x, the entry it took, to the bit (test_adaptive.py::test_programmed_state_is_the_mask pins the state).  That
drives the list schedule -- the mark kernel, the select, the list kernel, the chunk resolve and the masked accumulate --
over any mask through the public C ABI alone:

  * the matrix (pathwise.LIST_MATRIX: every pathwise case in f32, f64 on one case per f64 variant, the counting
    variants): one sample at a time under a random mask M and under its complement.  The entries of M and ~M equal
    the plain render's (rptb_render_samples) -- bit for bit in f64 and in f32 -- and, stacked, are compared with the
    oracle path by path like test_gpu_paths.py; the counters of M and ~M add up to the plain render's;
  * mask edges: no pixel, every pixel, the last pixel, the ragged tiles only, a checkerboard of 8x4 warp blocks and
    every other tile, at 1x1, 7x3, 16x8, 17x9 and 203x117;
  * sample chunks: 130 and 2100 samples in one call (3 and 32 chunks, one group per chunk), f32 and f64;
  * with two or more GPUs, the same bits on every device list.

On one H100 80GB HBM3 at a 700 W power limit every f32 list entry came out bit-identical to the plain render's entry
(both schedules inline the same render_thread), so f32 is held to equality like f64, and the counters to exact sums.
The pathwise agreement and bias are those test_gpu_paths.py measures for the tile schedule, path for path.  The
printout gives, per case, the list variant, the fraction bit-identical to the plain render and the pathwise line.
The whole file ran in 6.3 s there (oracle included).
"""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api
from tests import pathwise as pw
from tests.hostemu import emu

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
CRIT = api.Adaptive(0.0, 0.5, 2)
COUNTERS = ("segments", "rays", "node_visits", "tri_tests", "object_tests", "bvh_node_visits", "bvh_tri_tests", "mesh_hits",
            "env_lookups")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


class Target:
    """A pathwise case on the GPU: its renderer (seed 1, as pathwise.oracle_paths), the device scene made under the
    case's switches, and the scene features the launchers dispatch on."""

    def __init__(self, case, scene, cam, precision, w=None, h=None, device=0):
        self.w, self.h = w or case.w, h or case.h
        self.r = pw.renderer(case, scene, cam, 1, precision).width(self.w).height(self.h).accel(case.accel).device(device)
        with pw.scene_env(case.env):
            self.ds = self.r.device_scene()
            e = emu.EmuScene(api.FlatScene(scene, accel=case.accel))
            self.features = e.features
            e.close()
        self.cam = cam.to_c()

    def close(self):
        self.r.close()

    def params(self, n, first, stats):
        p = self.r.params(n, first, collect_stats=stats)
        p.engine = capi.ENGINE_MEGAKERNEL
        return p

    def plain(self, n, first, stats):
        """rptb_render_samples: (every pixel's entry, row-major (npix, 3); stats dict)."""
        out, st = np.empty((self.w * self.h, 3)), capi.Stats()
        capi.check(capi.lib().rptb_render_samples(self.ds.handle, C.byref(self.cam), C.byref(self.params(n, first, stats)),
                                                  out.ctypes.data_as(capi.c_double_p), C.byref(st)), "rptb_render_samples")
        return out, st.as_dict()

    def programmed(self, on):
        """A fresh DeviceBuffer whose active pixels under CRIT are exactly `on` (npix bools); (buffer, pixel_stats)."""
        buf = self.r.device_buffer()
        buf.add_samples(np.repeat(np.where(on, 1.0, 0.0)[:, None], 3, axis=1))
        buf.add_samples(np.repeat(np.where(on, -1.0, 0.0)[:, None], 3, axis=1))
        s0, m0, c0 = buf.pixel_stats()
        assert np.array_equal(CRIT.active(c0, s0, m0), on)
        return buf, (s0, m0, c0)

    def masked(self, mask, n, first, stats):
        """One adaptive call (n samples from `first`) on a buffer programmed with `mask`: (the entry each masked pixel
        took, NaN elsewhere; stats dict).  Checks that nothing else changed."""
        on = np.asarray(mask, bool).reshape(-1)
        buf, (s0, m0, c0) = self.programmed(on)
        active, st = C.c_uint64(0), capi.Stats()
        crit = CRIT.to_c()
        capi.check(capi.lib().rptb_sample_into_adaptive(self.ds.handle, C.byref(self.cam), C.byref(self.params(n, first, stats)),
                                                        C.byref(crit), buf.handle, C.byref(active), C.byref(st)),
                   "rptb_sample_into_adaptive")
        s1, m1, c1 = buf.pixel_stats()
        buf.close()
        assert active.value == on.sum()
        assert np.array_equal(c1, c0 + on)                                      # +1 on the mask, nowhere else
        assert np.array_equal(_bits(s1[~on]), _bits(s0[~on])) and np.array_equal(_bits(m1[~on]), _bits(m0[~on]))
        x = s1[on]                                                              # 0 + x: the entry, to the bit
        welford = m0[on] + ((x - s0[on] / 2.0) * (x - x / 3.0)).sum(1)
        np.testing.assert_allclose(m1[on], welford, rtol=1e-12, atol=1e-300)
        entry = np.full_like(s1, np.nan)
        entry[on] = x
        return entry, st.as_dict()


def _counters_add_up(sa, sb, sp, exact, where):
    for k in COUNTERS:
        got, want = sa[k] + sb[k], sp[k]
        if exact:
            assert got == want, (where, k, sa[k], sb[k], want)
        else:  # the wavefront test's bound
            assert abs(got - want) <= 1e-4 * max(want, 1), (where, k, sa[k], sb[k], want)


_ORACLE = {}


def _oracle(orc, name, scene, cam):
    if name not in _ORACLE:
        _ORACLE[name] = pw.oracle_paths(orc, pw.CASES[name], scene, cam)
    return _ORACLE[name]


def _prec(p):
    return "f64" if p == F64 else "f32"


@pytest.mark.parametrize("name,precision,stats", pw.LIST_MATRIX,
                         ids=["%s-%s-s%d" % (n, _prec(p), s) for n, p, s in pw.LIST_MATRIX])
def test_list_variant_is_the_plain_render_and_the_oracle(orc, gpu_ok, name, precision, stats):
    c = pw.CASES[name]
    scene, cam = c.make()
    t = Target(c, scene, cam, precision)
    (vstats, feat, maxd), compiled = emu.pick_render_list(t.features, stats, precision, c.max_bounces)
    assert compiled and vstats == (stats != 0)
    on = pw.list_mask(c.w, c.h, 7).reshape(-1)
    got, want, seg = [], [], 0
    try:
        for s in range(c.spp):
            plain, sp = t.plain(1, s, stats)
            a, sa = t.masked(on.reshape(c.h, c.w), 1, s, stats)
            b, sb = t.masked(~on.reshape(c.h, c.w), 1, s, stats)
            entry = np.where(on[:, None], a, b)
            _counters_add_up(sa, sb, sp, precision == F64 or np.array_equal(entry, plain), (name, s))
            got.append(entry)
            want.append(plain)
            seg += sa["segments"] + sb["segments"]
    finally:
        t.close()
    got, want = np.concatenate(got), np.concatenate(want)
    same = float((_bits(got) == _bits(want)).all(1).mean())
    line = "%-20s %s stats %d  list FEAT %3d MAXD %2d  bit-identical to plain %.6f" % (name, _prec(precision), stats, feat, maxd, same)
    if precision == F32:
        f64, seg64 = _oracle(orc, name, scene, cam)
        st = pw.compare(got, f64, seg, seg64)
        line += "  |  " + st.line(name, feat)
    print(line)
    assert np.isfinite(got).all()
    assert np.array_equal(_bits(got), _bits(want)), line
    if precision == F32:
        assert st.rel.size >= pw.MIN_PATHS
        assert st.agree >= c.gpu_floor, line
        assert abs(st.bias) <= c.bias, line
        assert st.seg32 <= st.seg64, line


EDGE_CASES = ("cornell", "teapot_kd", "fractal_teapots_bvh")   # F_FLAT, F_TREE, F_EVERY | F_BVH
SIZES = ((1, 1), (7, 3), (16, 8), (17, 9), (203, 117))


@pytest.mark.parametrize("w,h", SIZES, ids=["%dx%d" % s for s in SIZES])
@pytest.mark.parametrize("name", EDGE_CASES)
def test_mask_edges(gpu_ok, name, w, h):
    c = pw.CASES[name]
    scene, cam = c.make()
    t = Target(c, scene, cam, F32, w, h)
    try:
        plain, sp = t.plain(2, 3, 0)
        for mname, m in pw.edge_masks(w, h).items():
            on = m.reshape(-1)
            entry, st = t.masked(m, 2, 3, 0)
            where = (name, w, h, mname)
            assert np.array_equal(_bits(entry[on]), _bits(plain[on])), where
            if not on.any():
                assert st["segments"] == 0 and st["rays"] == 0, where
            else:
                assert 0 < st["segments"] <= sp["segments"], where
            if mname == "all":
                _counters_add_up(st, dict.fromkeys(COUNTERS, 0), sp, True, where)
    finally:
        t.close()


@pytest.mark.parametrize("n", [130, 2100])
@pytest.mark.parametrize("precision", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["cornell", "fractal_spheres"])
def test_sample_chunks(gpu_ok, name, precision, n):
    """130 samples: 3 chunks of 64; 2100: 32 of 66 -- on a 37x23 image (9 tiles) every chunk is a group of its own, so
    render_list_kernel runs a grid of 9 x nchunks and resolve_chunks_list_kernel adds the chunk sums of the listed
    pixels."""
    c = pw.CASES[name]
    scene, cam = c.make()
    w, h = 37, 23
    t = Target(c, scene, cam, precision, w, h)
    m = pw.list_mask(w, h, 11)
    on = m.reshape(-1)
    try:
        plain, sp = t.plain(n, 5, 0)
        entry, st = t.masked(m, n, 5, 0)
        entry_c, st_c = t.masked(~m, n, 5, 0)
    finally:
        t.close()
    got = np.where(on[:, None], entry, entry_c)
    assert np.isfinite(got).all()
    assert np.array_equal(_bits(got), _bits(plain))
    _counters_add_up(st, st_c, sp, True, (name, n))


def test_every_device_list_gives_the_same_bits(gpu_ok):
    if gpu_ok < 2:
        pytest.skip("one GPU visible")
    c = pw.CASES["fractal_teapots_bvh"]
    scene, cam = c.make()
    w, h = 203, 117
    m = pw.list_mask(w, h, 13)
    ref = None
    for devices in ([0], [1], [0, 1], list(range(min(gpu_ok, 8)))):
        t = Target(c, scene, cam, F32, w, h, device=devices)
        try:
            entry, st = t.masked(m, 2, 1, 1)
        finally:
            t.close()
        got = (_bits(np.nan_to_num(entry)), tuple(st[k] for k in COUNTERS))
        if ref is None:
            ref = got
        else:
            assert np.array_equal(got[0], ref[0]) and got[1] == ref[1], devices
