"""Adaptive sampling without a GPU: the convergence criterion, the C ABI's argument checks, and the list-scheduled
megakernel body (render_list_kernel) in host emulation against the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import pathwise as pw
from tests.hostemu import emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F_FLAT, F_LIST, F_EVERY = 128, 256, 55


def _emu():
    """tests/hostemu/_build/libhostemu_list.so: the host emulation of hostemu.cu plus the list schedule and the criterion."""
    return emu.list_lib()


class ListEmuScene:
    """A scene of the list-schedule emulation library (the flattened arrays, as emu.EmuScene holds them)."""

    def __init__(self, flat):
        self.flat = flat
        err = C.create_string_buffer(512)
        self.handle = C.c_void_p(_emu().hostemu_scene_create(C.byref(flat.desc), err, 512))
        if not self.handle:
            raise ValueError(err.value.decode())

    def render(self, camera, params, ext_bvh=False):
        """The tile-scheduled megakernel body, as emu.EmuScene.render: ((w*h, 3), stats dict, FEAT)."""
        out = np.empty((params.width * params.height, 3))
        st = capi.Stats()
        cam = camera.to_c()
        feat = _emu().hostemu_render(self.handle, C.byref(cam), C.byref(params), 1 if ext_bvh else 0, out.ctypes.data_as(capi.c_double_p),
                                     C.byref(st))
        return out, st.as_dict(), int(feat)

    def render_list(self, camera, params, mask, ext_bvh=False):
        """The list-scheduled body over the pixels `mask` (w*h bools) sets: ((w*h, 3), NaN off the mask; stats dict; FEAT)."""
        out = np.empty((params.width * params.height, 3))
        st = capi.Stats()
        cam = camera.to_c()
        m = np.ascontiguousarray(mask, np.uint8).reshape(-1)
        feat = _emu().hostemu_render_list(self.handle, C.byref(cam), C.byref(params), 1 if ext_bvh else 0,
                                          m.ctypes.data_as(C.POINTER(C.c_uint8)), out.ctypes.data_as(capi.c_double_p), C.byref(st))
        return out, st.as_dict(), int(feat)

    @property
    def features(self) -> int:
        return int(_emu().hostemu_scene_features(self.handle))

    def __del__(self):
        if getattr(self, "handle", None):
            _emu().hostemu_scene_destroy(self.handle)
            self.handle = C.c_void_p()


def emu_active(counts, sums, m2, crit: api.Adaptive) -> np.ndarray:
    counts = np.ascontiguousarray(counts, np.uint32)
    sums = np.ascontiguousarray(sums, np.float64).reshape(-1, 3)
    m2 = np.ascontiguousarray(m2, np.float64)
    out = np.empty(counts.shape[0], np.uint8)
    c = crit.to_c()
    _emu().hostemu_adaptive_active(counts.ctypes.data_as(capi.c_u32_p), sums.ctypes.data_as(capi.c_double_p),
                                   m2.ctypes.data_as(capi.c_double_p), counts.shape[0], C.byref(c),
                                   out.ctypes.data_as(C.POINTER(C.c_uint8)))
    return out.astype(bool)


def _cases(rng, n):
    counts = rng.integers(0, 40, n).astype(np.uint32)
    mean = rng.choice([0.0, 1e-4, 0.05, 0.5, 3.0, 1e3], n)[:, None] * rng.uniform(0.5, 1.5, (n, 3))
    sums = mean * counts[:, None]
    # M2 near the decision boundary of the default criterion, and far from it
    m2 = rng.uniform(0, 2, n) * (0.02 * mean.mean(1) + 1e-3) ** 2 * np.maximum(counts.astype(float) - 1, 0) * counts * 3
    edge_counts = np.array([0, 1, 2, 3, 4, 4, 4, 4, 5, 6, 7, 8, 9, 4_000_000_000], np.uint32)
    edge_sums = np.array([[0, 0, 0], [1, 1, 1], [0, 0, 0], [0, 0, 0], [np.nan, 0, 0], [1e300, 1e300, 1e300],
                          [-1, -2, -3], [0, 0, 0], [1, 1, 1], [np.inf, 0, 0], [1e-300, 0, 0], [2, 2, 2], [5, 5, 5], [4e9, 4e9, 4e9]])
    edge_m2 = np.array([0, 0, 0, 0, 0, 1e300, 0.5, np.nan, 0.0, 0.0, 1e-310, np.inf, 1e-5, 1.0])
    return (np.concatenate([counts, edge_counts]), np.concatenate([sums, edge_sums]), np.concatenate([m2, edge_m2]))


@pytest.mark.parametrize("crit", [api.Adaptive(), api.Adaptive(0.0, 0.0, 2), api.Adaptive(0.1, 0.0, 3), api.Adaptive(0.0, 0.05, 9),
                                  api.Adaptive(1e-3, 1e-6, 2)], ids=["default", "zero", "rel", "abs", "tight"])
def test_criterion_matches_numpy_restatement(crit):
    counts, sums, m2 = _cases(np.random.default_rng(7), 20000)
    got = emu_active(counts, sums, m2, crit)
    want = crit.active(counts, sums, m2)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]
    assert got.any() and not got.all()
    # the documented corners
    assert got[counts < crit.min_entries].all()                      # too few entries
    nan = np.isnan(m2) | np.isnan(sums).any(1)
    assert got[nan & (counts >= 2)].all()                             # a NaN statistic keeps the pixel active


def test_zero_variance_pixel_stops_at_min_entries():
    crit = api.Adaptive(0.0, 0.0, 5)
    counts = np.arange(0, 9, dtype=np.uint32)
    sums = np.repeat(counts[:, None].astype(float) * 0.25, 3, axis=1)
    active = emu_active(counts, sums, np.zeros(9), crit)
    assert list(active) == [True] * 5 + [False] * 4


def test_adaptive_struct_size_matches_header(tmp_path):
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include "rpt_b200.h"\nint main(void){printf("%zu\\n", sizeof(rptb_adaptive));return 0;}\n')
    exe = tmp_path / "s"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    assert int(subprocess.check_output([str(exe)]).decode()) == C.sizeof(capi.Adaptive) == 24


def test_error_statuses_before_any_device_work():
    L = capi.lib()
    cam, p = capi.Camera(), capi.RenderParams()
    p.width, p.height, p.iterations, p.shard_count = 8, 8, 1, 1
    active = C.c_uint64(7)
    for crit in (capi.Adaptive(0.1, 0.0, 1, 0), capi.Adaptive(-0.1, 0.0, 4, 0), capi.Adaptive(0.1, float("nan"), 4, 0),
                 capi.Adaptive(float("inf"), 0.0, 4, 0), capi.Adaptive(0.1, -1e-9, 4, 0)):
        assert L.rptb_sample_into_adaptive(None, C.byref(cam), C.byref(p), C.byref(crit), None, C.byref(active), None) == capi.ERR_BAD_ARG
        assert b"min_entries" in L.rptb_last_error() or b"tolerances" in L.rptb_last_error()
    good = capi.Adaptive(0.1, 0.0, 4, 0)
    assert L.rptb_sample_into_adaptive(None, C.byref(cam), C.byref(p), None, None, None, None) == capi.ERR_BAD_ARG
    assert L.rptb_sample_into_adaptive(None, C.byref(cam), C.byref(p), C.byref(good), None, None, None) == capi.ERR_BAD_ARG
    assert active.value == 7
    assert L.rptb_buffer_pixel_stats(None, None, None, None) == capi.ERR_BAD_ARG


def _params(cfg, w, h, spp, mb, precision, seed=3):
    return api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).seed(seed).precision(precision).params(spp)


LIST_RENDERS = {  # name: (config factory, w, h, spp, max_bounces, FEAT of the f32 list variant)
    "sphere": (scenes.sphere_scene, 45, 27, 8, 2, F_FLAT | 8 | F_LIST),
    "cornell": (scenes.cornell_scene, 32, 29, 8, 6, F_FLAT | F_LIST),
    "fractal_spheres": (lambda: scenes.fractal_spheres_scene(3), 40, 24, 4, 2, F_EVERY | F_LIST),
    "cornell_chunks": (scenes.cornell_scene, 19, 11, 130, 3, F_FLAT | F_LIST),   # nchunks > 1: resolve walks the list
}


@pytest.mark.parametrize("name", sorted(LIST_RENDERS))
def test_list_schedule_is_the_plain_render_on_the_mask(orc, name):
    mk, w, h, spp, mb, want_feat = LIST_RENDERS[name]
    cfg = mk()
    flat = api.FlatScene(cfg.scene)
    e, o = ListEmuScene(flat), orc.OracleScene(flat)
    rng = np.random.default_rng(11)
    mask = (rng.random(w * h) < 0.3).astype(np.uint8)
    mask[: w * 4] = 0                                    # whole warp blocks without a pixel
    mask[-w:] = 1                                        # the ragged last row of tiles
    cam = cfg.camera.to_c()
    on = mask.astype(bool)

    def render_list(precision):
        out = np.empty((w * h, 3))
        st = capi.Stats()
        p = _params(cfg, w, h, spp, mb, precision)
        feat = _emu().hostemu_render_list(e.handle, C.byref(cam), C.byref(p), 0, mask.ctypes.data_as(C.POINTER(C.c_uint8)),
                                          out.ctypes.data_as(capi.c_double_p), C.byref(st))
        return out, st.as_dict(), feat

    ref, _ = o.render(cfg.camera, _params(cfg, w, h, spp, mb, capi.PRECISION_F32))
    g64, s64, f64 = render_list(capi.PRECISION_F64)
    plain64, _, _ = e.render(cfg.camera, _params(cfg, w, h, spp, mb, capi.PRECISION_F64))
    assert f64 & F_LIST
    assert np.array_equal(g64[on], plain64[on])          # the masked pixels: the tile schedule's bits,
    if spp <= 64:
        assert np.array_equal(g64[on], ref[on])          # which are the oracle's
    else:                                                # (chunk sums: as test_megakernel_body_is_trace_ray allows)
        np.testing.assert_allclose(g64[on], ref[on], rtol=1e-12, atol=0)
    assert np.isnan(g64[~on]).all()                      # and nothing written anywhere else
    # the f32 product variant through the list, against the same variant through the tile schedule
    g32, s32, f32 = render_list(capi.PRECISION_F32)
    plain32, sp32, fp32 = e.render(cfg.camera, _params(cfg, w, h, spp, mb, capi.PRECISION_F32))
    assert f32 == want_feat and fp32 == want_feat & ~F_LIST
    assert np.array_equal(g32[on], plain32[on]) and np.isnan(g32[~on]).all()
    assert 0 < s32["segments"] < sp32["segments"]


COUNTERS = ("segments", "rays", "node_visits", "tri_tests", "object_tests", "bvh_node_visits", "bvh_tri_tests", "mesh_hits",
            "env_lookups")


@pytest.mark.parametrize("name", sorted(pw.CASES))
def test_list_matrix_is_the_plain_render_on_the_mask(name):
    """Every case of the pathwise matrix, 2 spp, f32 and f64: through the list schedule, each mask of
    pathwise.edge_masks and a random one (pathwise.list_mask) gets exactly the plain render's pixels and nothing else,
    and the counters of a mask and its complement add up to the plain render's, without counters and with both kinds."""
    c = pw.CASES[name]
    scene, cam = c.make()
    with pw.scene_env(c.env):
        e = ListEmuScene(api.FlatScene(scene, accel=c.accel))
    ext_bvh = (e.features & pw.F_BVH) != 0  # as test_hostemu_paths: the library sends F_BVH with F_EXT
    masks = {"random": pw.list_mask(c.w, c.h, 5), **pw.edge_masks(c.w, c.h)}
    for precision in (capi.PRECISION_F32, capi.PRECISION_F64):
        for stats in (0, 1, 2):
            r = pw.renderer(c, scene, cam, 1, precision)
            p = r.params(2, 0, collect_stats=stats)
            plain, pst, pfeat = e.render(cam, p, ext_bvh)
            assert pfeat >= 0 and not pfeat & F_LIST
            if precision == capi.PRECISION_F32 and stats == 0:
                assert pfeat == c.feat
            for mname, m in masks.items():
                if stats and mname != "random":
                    continue
                on = m.reshape(-1)
                (g, st, feat), (gc, stc, featc) = (e.render_list(cam, p, on, ext_bvh), e.render_list(cam, p, ~on, ext_bvh))
                where = (name, precision, stats, mname)
                assert feat == featc == pfeat | F_LIST, where
                assert np.array_equal(g[on], plain[on]) and np.isnan(g[~on]).all(), where
                assert np.array_equal(gc[~on], plain[~on]) and np.isnan(gc[on]).all(), where
                for k in COUNTERS:
                    assert st[k] + stc[k] == pst[k], where + (k, st[k], stc[k], pst[k])
                if mname == "none":
                    assert st["segments"] == 0 and st["rays"] == 0, where
            if stats:
                assert pst["node_visits"] > 0 or pst["object_tests"] > 0 or pst["bvh_node_visits"] > 0, (name, precision, stats)


def test_programmed_state_is_the_mask():
    """The state test_gpu_list_matrix.py programs through rptb_buffer_add_samples: entries (1, 1, 1) then (-1, -1, -1)
    leave S = 0, M2 = 6, n = 2 (err^2 = 6 / (1 * 2 * 3) = 1), entries 0 then 0 leave everything 0; under
    Adaptive(0, 0.5, 2) the first is active (1 > 0.25) and the second not, on the device criterion and in numpy."""
    crit = api.Adaptive(0.0, 0.5, 2)
    counts = np.array([2, 2], np.uint32)
    sums = np.zeros((2, 3))
    m2 = np.array([6.0, 0.0])
    assert list(emu_active(counts, sums, m2, crit)) == [True, False]
    assert list(crit.active(counts, sums, m2)) == [True, False]
    # Welford over the two entries, as the buffer adds them
    for x1, x2, want in (((1.0,) * 3, (-1.0,) * 3, 6.0), ((0.0,) * 3, (0.0,) * 3, 0.0)):
        a, b = np.array(x1), np.array(x2)
        mean1 = a / 1.0
        assert float((((b - mean1) * (b - (a + b) / 2.0))).sum()) == want
