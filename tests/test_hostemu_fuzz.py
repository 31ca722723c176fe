"""Seeded random scenes through the host emulation of the device code (tests/hostemu) against the oracle.

Every scene mixes the shape kinds the boundary knows (sphere, cube, plane, mesh, monomial surface, kd-tree of
shapes), random non-uniform transforms, and ray families chosen to hit the awkward cases: axis-aligned
directions (exactly zero components), origins on surfaces, grazing rays.  Real = double must reproduce the oracle
bit for bit (closest hits, any-hit shadow queries, whole images through the emulated megakernel); Real = float
must stay inside the f32 tolerances, through the kd-trees and through the BVH."""
import numpy as np
import pytest

from rpt_b200 import api, scenes
from rpt_b200 import _capi as capi
from tests import util
from tests.hostemu import emu


def random_xf(rng, shape, big=False):
    s = rng.uniform(0.3, 1.6, 3) * (3.0 if big else 1.0)
    axis = util.random_unit(rng, 1)[0]
    return shape.scale(api.vec3(*s)).rotate(rng.uniform(0, 6.28), axis).translate(api.vec3(*rng.uniform(-3, 3, 3)))


def soup(rng, n, spread=1.0):
    c = rng.uniform(-spread, spread, (n, 1, 3))
    v = c + rng.normal(0, 0.15, (n, 3, 3))
    return np.stack([api.Triangle.from_vertices(*t) for t in v])


def random_scene(seed, table_only=False):
    """table_only: only what the packed primitive table holds (spheres, cubes, one-leaf meshes, planes; no kd-tree of a
    mesh or of shapes, no monomial) and no transparent material, so that the f32 megakernel walks the table too.  The
    default scenes are those of the seeds before the option existed."""
    rng = np.random.default_rng(seed)
    scene = api.Scene()
    mats = [api.Material.diffuse(api.hex_color(0x8090A0)), api.Material.specular(api.hex_color(0xC04020), 0.3),
            api.Material.metallic_(api.hex_color(0xE0E0E0), 0.2), api.Material.clear(1.5, 0.05),
            api.Material.light(api.hex_color(0xFFFFFF), 2.0)]
    mesh_big = api.Mesh(soup(rng, 400))            # a real kd-tree / BVH
    mesh_small = api.Mesh(soup(rng, 6, 0.5))       # one leaf
    makers = [lambda: api.sphere(), lambda: api.cube(), lambda: mesh_big, lambda: mesh_small,
              lambda: api.monomial_surface(rng.uniform(0.5, 2.5), 4.0)]
    if table_only:
        makers = [lambda: api.sphere(), lambda: api.cube(), lambda: mesh_small, lambda: api.Mesh(soup(rng, 3, 0.4))]
        mats = mats[:3] + mats[4:]
    for _ in range(rng.integers(3, 7)):
        shape = makers[rng.integers(0, len(makers))]()
        shape = random_xf(rng, shape) if rng.random() < 0.8 else shape
        scene.add(api.Object(shape).material(mats[rng.integers(0, len(mats))]))
    if rng.random() < 0.7 and not table_only:      # a kd-tree over 20-40 transformed shapes
        kids = [random_xf(rng, makers[rng.integers(0, len(makers))]()) for _ in range(rng.integers(20, 40))]
        group = api.KdTree(kids)
        scene.add(api.Object(group if rng.random() < 0.5 else random_xf(rng, group)).material(mats[rng.integers(0, 3)]))
    if rng.random() < 0.6:
        scene.add(api.Object(api.plane(api.vec3(0.0, 1.0, 0.0), -4.0)).material(mats[0]))
    scene.add(api.Light.Point(api.vec3(30.0, 30.0, 30.0), api.vec3(*rng.uniform(-5, 5, 3))))
    scene.add(api.Light.Directional(api.vec3(0.5, 0.5, 0.5), [api.vec3(0.0, -1.0, 0.0), api.vec3(1.0, 0.0, 0.0),
                                                              api.vec3(0.3, -0.8, 0.1)][rng.integers(0, 3)]))
    if rng.random() < 0.5:
        scene.add(api.Light.Ambient(api.vec3(0.03, 0.03, 0.03)))
    if rng.random() < 0.5:
        scene.add(api.Light.Object(api.Object(random_xf(rng, api.sphere())).material(api.Material.light(api.vec3(1, 1, 1), 20.0))))
    scene.environment = api.Environment.Color(api.vec3(0.1, 0.12, 0.2))
    return scene, rng


def ray_families(rng, osc, n=6000, lift=1e-9):
    """random rays into the scene; axis-aligned rays; rays restarted on the surfaces the first family hit, `lift`
    above them (1e-9: meaningful in f64 only -- the reference restarts ON the surface with t_min = 1e-12; the f32
    path offsets its own continuation rays by ~2e-6 |x|, so f32 is probed with rays lifted by 2e-4)"""
    o = util.random_unit(rng, n) * rng.uniform(6, 10, (n, 1))
    d = util.normalize(rng.uniform(-3, 3, (n, 3)) - o)
    fam = [np.concatenate([o, d], axis=1)]
    axes = np.eye(3)[rng.integers(0, 3, n)] * rng.choice([-1.0, 1.0], (n, 1))
    oa = rng.uniform(-3.5, 3.5, (n, 3)) - 9.0 * axes
    fam.append(np.concatenate([oa, axes], axis=1))
    two = np.zeros((n, 3))                                   # one zero component
    k = rng.integers(0, 3, n)
    v = util.normalize(rng.normal(size=(n, 3)))
    v[np.arange(n), k] = 0.0
    two = util.normalize(v)
    fam.append(np.concatenate([rng.uniform(-3.5, 3.5, (n, 3)) - 9.0 * two, two], axis=1))
    t, obj, nrm, _ = osc.closest_hit(fam[0])
    hit = obj >= 0
    p = fam[0][hit, :3] + t[hit, None] * fam[0][hit, 3:]
    d2 = util.normalize(nrm[hit] + 0.7 * util.random_unit(rng, hit.sum()))   # leave the surface, often at a grazing angle
    fam.append(np.concatenate([p + lift * nrm[hit], d2], axis=1))
    return np.concatenate(fam)


@pytest.mark.parametrize("seed", range(8))
def test_random_scene_queries(orc, seed):
    scene, rng = random_scene(100 + seed)
    flat = api.FlatScene(scene, accel=capi.ACCEL_BVH)
    e, o = emu.EmuScene(flat), orc.OracleScene(flat)
    rays = ray_families(rng, o)
    t0, o0, n0, _ = o.closest_hit(rays)
    # f64: the oracle, bit for bit
    t1, o1, n1, _ = e.closest_hit(rays, precision=capi.PRECISION_F64)
    np.testing.assert_array_equal(o1, o0)
    np.testing.assert_array_equal(t1, t0)
    np.testing.assert_array_equal(n1, n0)
    occ64 = e.occluded(rays, np.inf, precision=capi.PRECISION_F64)
    np.testing.assert_array_equal(occ64 == 1, o0 >= 0)       # any-hit == "there is a closest hit"
    # f32 through the kd-trees and through the BVH
    rays = ray_families(np.random.default_rng(seed), o, lift=2e-4)
    t0, o0, n0, _ = o.closest_hit(rays)
    for use_bvh in (False, True):
        flat32 = flat if use_bvh else api.FlatScene(scene, accel=capi.ACCEL_KDTREE)
        e32 = e if use_bvh else emu.EmuScene(flat32)
        t2, o2, n2, _ = e32.closest_hit(rays, precision=capi.PRECISION_F32)
        with np.errstate(invalid="ignore"):
            tie = (o2 >= 0) & (o0 >= 0) & (np.abs(t2 - t0) <= 1e-4 * np.abs(t0))
        ok = (o2 == o0) | tie
        assert ok.mean() >= 0.995, (use_bvh, ok.mean())      # rays restarted ON a surface are decided by the last ulp
        # (a vertical ray through a MonomialSurface makes the reference's Newton step 0/0: its hit time is NaN in
        # the oracle, in the f64 gate and here alike -- compared above, excluded from the tolerance statistics)
        hit = (o2 == o0) & (o0 >= 0) & np.isfinite(t0) & np.isfinite(t2)
        rel = np.abs(t2[hit] - t0[hit]) / np.maximum(np.abs(t0[hit]), 1e-6)
        assert np.median(rel) <= 5e-7 and np.quantile(rel, 0.99) <= 1e-3, (use_bvh, np.quantile(rel, [0.5, 0.99]))
        occ = e32.occluded(rays, np.inf, precision=capi.PRECISION_F32, use_bvh=use_bvh)
        assert ((occ == 1) == (o0 >= 0)).mean() >= 0.995


@pytest.mark.parametrize("seed", range(8))
def test_random_scene_renders(orc, seed):
    scene, rng = random_scene(200 + seed)
    cam = api.Camera.look_at(api.vec3(*(util.random_unit(rng, 1)[0] * 11.0)), api.vec3(0.0, 0.0, 0.0), api.vec3(0.0, 1.0, 0.0), 0.9)
    flat = api.FlatScene(scene, accel=capi.ACCEL_BVH)
    e, o = emu.EmuScene(flat), orc.OracleScene(flat)
    r = api.Renderer(scene, cam).width(40).height(30).max_bounces(3).seed(seed)
    ref, st0 = o.render(cam, r.params(6))
    g64, s64, _ = e.render(cam, r.precision(capi.PRECISION_F64).params(6))
    np.testing.assert_allclose(g64, ref, rtol=1e-12, atol=0)
    assert (s64["segments"], s64["rays"]) == (st0["segments"], st0["rays"])
    ref2, _ = o.render(cam, api.Renderer(scene, cam).width(40).height(30).max_bounces(3).seed(seed + 50).params(6))
    cl = lambda a: np.clip(a, 0.0, 1.0)
    noise = util.rmse(cl(ref), cl(ref2))
    # The reference itself yields NaN pixels on some of these scenes (a ray parallel to a MonomialSurface's axis
    # makes its Newton step 0/0, monomial_surface.rs:53-61): the f64 gate reproduces them above (assert_allclose
    # treats NaN == NaN), the f32 path must be finite wherever the reference is.
    fin = np.isfinite(ref).all(axis=1) & np.isfinite(ref2).all(axis=1)
    assert fin.mean() > 0.95
    noise = util.rmse(cl(ref[fin]), cl(ref2[fin]))
    for ext_bvh in (False, True):
        g32, s32, _ = e.render(cam, r.precision(capi.PRECISION_F32).params(6), ext_bvh=ext_bvh)
        assert np.isfinite(g32[fin]).all()
        # same streams: the f32 image is the f64 image up to rounding, except where a path took another branch at a
        # threshold (one path in thousands; it moves ONE pixel by up to the full range, so those are counted, not averaged)
        dev = np.abs(cl(g32[fin]) - cl(ref[fin])).max(axis=1)
        off = dev > 2e-2
        assert off.mean() <= 0.005, (ext_bvh, off.sum())
        assert util.rmse(cl(g32[fin][~off]), cl(ref[fin][~off])) <= 0.25 * noise + 1e-4, (ext_bvh, util.rmse(cl(g32[fin][~off]), cl(ref[fin][~off])), noise)
