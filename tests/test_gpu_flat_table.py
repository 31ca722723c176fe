"""The packed primitive table (F_FLAT, scene_dev.cuh) against the scan over scene.objects it replaces, on the GPU.

Scenes made only of spheres, planes, cubes and one-leaf meshes are traced through the table; RPTB_NO_FLAT (read when
a scene is created) keeps the old scan.  Both must give the same closest hit bit for bit, and the same images: the table
changes the loads and the dispatch, and shares the plane test of coplanar triangles, never the arithmetic of a primitive.
The F_FLAT render kernels are compared with variant 0, F_FLAT | F_SMALL with F_SMALL.  tests/test_hostemu_flat.py makes
the same comparisons in the host emulation, and checks the table's layout."""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import util
from tests.hostemu import emu
from tests.test_hostemu_flat import (ADVERSARIAL, CONFIGS, F_FLAT, TABLE_SCENES, camera_for, flat_switch, named_scene, probe_rays,
                                     rays_for, table_scene)
from tests.test_hostemu_fuzz import random_scene

pytestmark = pytest.mark.gpu


def closest_hits(scene, rays, flat_on):
    with flat_switch(flat_on):
        with api.DeviceScene(scene) as ds:
            return ds.closest_hit(rays)


def assert_flat_ok(scene):
    """the scene is one the library traces through the table (the host emulation flattens it the same way)"""
    e = emu.EmuScene(api.FlatScene(scene))
    assert e.flat_table()[1] and e.features & F_FLAT
    return e


def assert_same_hits(scene, rays, rng):
    assert_flat_ok(scene)
    t0, o0, n0 = closest_hits(scene, rays, False)
    # and rays that start exactly on the surfaces just hit, leaving in random directions
    hit = o0 >= 0
    p = rays[hit, :3] + t0[hit, None] * rays[hit, 3:]
    rays = np.concatenate([rays, np.concatenate([p, util.random_unit(rng, int(hit.sum()))], axis=1)])
    t0, o0, n0 = closest_hits(scene, rays, False)
    t1, o1, n1 = closest_hits(scene, rays, True)
    np.testing.assert_array_equal(o1, o0)
    np.testing.assert_array_equal(t1, t0)
    np.testing.assert_array_equal(n1, n0)
    return o0


def probe_same_hits(scene, center, radius, seed):
    rng = np.random.default_rng(seed)
    o = assert_same_hits(scene, probe_rays(rng, center, radius, 100_000), rng)
    assert (o >= 0).mean() > 0.05


@pytest.mark.parametrize("name", ["sphere", "cornell", "glass"])
def test_configs_same_hits(gpu_ok, name):
    cfg = {"sphere": scenes.sphere_scene, "cornell": scenes.cornell_scene, "glass": lambda: scenes.glass_scene(64, 32)}[name]()
    center, radius = {"sphere": ((0.0, 0.0, 0.0), 4.0), "cornell": ((278.0, 274.0, 280.0), 290.0), "glass": ((0.0, 0.0, 0.0), 3.0)}[name]
    probe_same_hits(cfg.scene, center, radius, 7)


@pytest.mark.parametrize("seed", range(8))
def test_fuzz_scenes_same_hits(gpu_ok, seed):
    # the seeded scenes of test_hostemu_fuzz without kd-trees of meshes or of shapes, or monomials: they take the table
    scene, _ = random_scene(100 + seed, table_only=True)
    probe_same_hits(scene, (0.0, 0.0, 0.0), 5.0, seed)


@pytest.mark.parametrize("seed", range(6))
def test_table_scenes_same_hits(gpu_ok, seed):
    probe_same_hits(table_scene(300 + seed), (0.0, 0.0, 0.0), 5.0, seed)


@pytest.mark.parametrize("name", ADVERSARIAL)
def test_adversarial_scenes_same_hits(gpu_ok, orc, name):
    """runs, layers, duplicates, ties and parallel rays: the table's hits are the scan's bit for bit, and the oracle's
    within test_gpu_parity's f32 tolerances"""
    scene, rays, rng = rays_for(name, 40_000)
    o = assert_same_hits(scene, rays, rng)
    if name != "empty":
        assert (o >= 0).mean() > 0.05
    probe = rays[:20_000]                                   # from outside and from inside, in random directions
    t0, o0, n0, _ = orc.OracleScene(api.FlatScene(scene)).closest_hit(probe)
    t1, o1, n1 = closest_hits(scene, probe, True)
    with np.errstate(invalid="ignore"):
        tie = (o1 >= 0) & (o0 >= 0) & (np.abs(t1 - t0) <= 1e-5 * np.abs(t0))   # coincident surfaces of two objects
    assert ((o1 == o0) | tie).mean() > 0.999
    hit = (o1 == o0) & (o0 >= 0)
    if hit.any():
        rel = np.abs(t1[hit] - t0[hit]) / np.abs(t0[hit])
        assert np.median(rel) <= 2e-7 and np.quantile(rel, 0.99) <= 1e-5 and np.quantile(rel, 0.999) <= 1e-3
        assert np.quantile(np.abs(n1[hit] - n0[hit]).max(1), 0.99) < 1e-3


# ---------------------------------------------------------------- renders -----------------------------------------------
def render(scene, camera, w, h, spp, mb, flat_on, **kw):
    """rptb_render_samples of a scene created with RPTB_NO_FLAT unset (flat_on) or set -> (image, stats)"""
    p = api.Renderer(scene, camera).width(w).height(h).max_bounces(mb).seed(3).params(spp, **kw)
    colors = np.empty((w * h, 3), np.float64)
    stats = capi.Stats()
    cam = camera.to_c()
    with flat_switch(flat_on):
        with api.DeviceScene(scene) as ds:
            capi.check(capi.lib().rptb_render_samples(ds.handle, C.byref(cam), C.byref(p), colors.ctypes.data_as(capi.c_double_p),
                                                      C.byref(stats)), "rptb_render_samples")
    return colors, stats.as_dict()


def render_pair(scene, camera, w, h, spp, mb, **kw):
    e = assert_flat_ok(scene)
    (_, feat, _), _ = emu.pick_variant(emu.ENGINE_RENDER, e.features, 0, capi.PRECISION_F32, mb)
    assert feat & F_FLAT                                      # the f32 megakernel walks the table for this scene
    a, sa = render(scene, camera, w, h, spp, mb, True, **kw)
    b, sb = render(scene, camera, w, h, spp, mb, False, **kw)
    # (NaN pixels, where the reference's own arithmetic makes them -- the oracle renders multirun_xf with the same ones --
    # must sit at the same places: assert_array_equal compares them as equal only there)
    np.testing.assert_array_equal(a, b)
    assert (sa["segments"], sa["rays"]) == (sb["segments"], sb["rays"])
    return a, sa


@pytest.mark.parametrize("name", TABLE_SCENES)
def test_table_render_is_the_scan_render(gpu_ok, name):
    if name in CONFIGS:
        cfg = CONFIGS[name][0]()
        scene, camera = cfg.scene, cfg.camera
    else:
        scene, center, radius = named_scene(name)
        camera = camera_for(center, radius)
    _, st = render_pair(scene, camera, 64, 48, 16, 6)
    assert st["segments"] >= 64 * 48 * 16


def test_table_render_with_chunks_and_shards(gpu_ok):
    cfg = scenes.cornell_scene()
    full, _ = render_pair(cfg.scene, cfg.camera, 40, 24, 150, 4)                    # 3 chunks of 64
    parts = [render_pair(cfg.scene, cfg.camera, 40, 24, 150, 4, shard_index=i, shard_count=3)[0] for i in range(3)]
    np.testing.assert_array_equal(parts[0] + parts[1] + parts[2], full)
