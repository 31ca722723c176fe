"""The device code checked against the oracle WITHOUT a GPU.

tests/hostemu compiles the functions the CUDA kernels inline (closest_hit, kd_intersect, bvh_intersect,
group_intersect, monomial_intersect, finalize_hit, shape_sample, illuminate -- rpt_b200/csrc/geometry.cuh,
shading.cuh) and render_thread, the whole body of the path-tracing megakernel (integrator.cuh), for the
host and runs them over the arrays rptb_scene_create would upload.  With Real = double every operation is
the oracle's, so hits, normals and traversal counters must agree exactly; with Real = float within the
f32 tolerances the GPU parity tests use.  This is test infrastructure (it cannot say anything about the
kernels' scheduling or fast-math); the `-m gpu` tests through the C ABI remain the gate."""
import math

import numpy as np
import pytest

from rpt_b200 import api, scenes
from rpt_b200 import _capi as capi
from tests import util
from tests.hostemu import emu
from tests.test_oracle_instancing import rays_into, small_scene

F_TREE, F_TRANSP, F_HDRI, F_SMALL, F_GROUP, F_MONO, F_FLAT = 1, 2, 4, 8, 16, 32, 128


def scene_rays(name):
    rng = np.random.default_rng(11)
    if name == "mixed":
        scene, kids = small_scene(monomials=True)
        scene.add(api.Light.Object(api.Object(api.monomial_surface(2.0, 4.0).scale(api.vec3(1.5, 1.0, 0.8))
                                              .translate(api.vec3(0.0, 7.0, 0.0))).material(api.Material.light(api.vec3(1, 0.9, 0.8), 30.0))))
        scene.add(api.Light.Object(api.Object(api.KdTree(kids[:7]).rotate_y(0.4).translate(api.vec3(0.0, 9.0, 0.0)))
                                   .material(api.Material.light(api.vec3(1, 1, 1), 10.0))))
        rays = np.concatenate([rays_into(rng, 30000), util.interior_rays([-4, -4, -4], [4, 7, 4], 15000, rng)])
        return scene, rays, F_TREE | F_GROUP | F_MONO
    cfg, want = {
        "cornell": (scenes.cornell_scene, F_FLAT),
        "teapot": (scenes.teapot_scene, F_TREE | F_SMALL),
        "glass": (lambda: scenes.glass_scene(64, 32), F_TRANSP | F_HDRI | F_SMALL | F_FLAT),   # (rendered by a scan variant)
        "fractal_spheres": (lambda: scenes.fractal_spheres_scene(4), F_GROUP),
        "fractal_teapots": (lambda: scenes.fractal_teapots_scene(3), F_GROUP | F_TREE),
        "monomial_glass": (lambda: scenes.monomial_glass_scene(64, 32), F_MONO | F_HDRI),
    }[name]
    cfg = cfg()
    rays = util.camera_rays(cfg.camera, 20000, rng, spread=0.4)
    return cfg.scene, rays, want


NAMES = ["cornell", "teapot", "glass", "fractal_spheres", "fractal_teapots", "monomial_glass", "mixed"]


@pytest.mark.parametrize("name", NAMES)
def test_device_closest_hit_f64_is_the_oracles(orc, name):
    scene, rays, want_features = scene_rays(name)
    flat = api.FlatScene(scene)
    e, o = emu.EmuScene(flat), orc.OracleScene(flat)
    assert e.features == want_features          # the kernel variant rptb_render_samples would pick
    t0, o0, n0, s0 = o.closest_hit(rays)
    t1, o1, n1, s1 = e.closest_hit(rays, precision=capi.PRECISION_F64)
    np.testing.assert_array_equal(o1, o0)
    np.testing.assert_array_equal(t1, t0)
    np.testing.assert_array_equal(n1, n0)
    assert s1["node_visits"] == s0["node_visits"] and s1["tri_tests"] == s0["tri_tests"]   # the same leaves, the same trees
    assert (o0 >= 0).mean() > 0.3


@pytest.mark.parametrize("name", NAMES)
def test_device_closest_hit_f32_within_tolerance(orc, name):
    scene, rays, _ = scene_rays(name)
    flat = api.FlatScene(scene)
    e, o = emu.EmuScene(flat), orc.OracleScene(flat)
    t0, o0, n0, _ = o.closest_hit(rays)
    t1, o1, n1, _ = e.closest_hit(rays, precision=capi.PRECISION_F32)
    same = o1 == o0
    assert same.mean() > 0.999
    hit = same & (o0 >= 0)
    rel = np.abs(t1[hit] - t0[hit]) / np.abs(t0[hit])
    assert np.median(rel) <= 2e-7 and np.quantile(rel, 0.99) <= 1e-5 and np.quantile(rel, 0.999) <= 1e-3
    assert np.quantile(np.abs(n1[hit] - n0[hit]).max(1), 0.99) < 1e-3


def test_device_light_sampling_of_monomial_and_group_lights(orc):
    """Light::illuminate over MonomialSurface::sample and KdTree::sample (uniform child, pdf / num), with the
    oracle's random stream: identical draws -> identical samples in f64."""
    scene, _, _ = scene_rays("mixed")
    flat = api.FlatScene(scene)
    e, o = emu.EmuScene(flat), orc.OracleScene(flat)
    pos = np.random.default_rng(2).uniform(-3, 3, (3000, 3))
    for light in (1, 2):
        a = o.illuminate(light, pos, seed=5)
        b = e.illuminate(light, pos, seed=5, precision=capi.PRECISION_F64)
        for x, y in zip(a, b):
            np.testing.assert_array_equal(y, x)
        assert np.isfinite(a[0]).all() and 0.3 < (a[0][:, 0] > 0).mean() < 0.9
        c = e.illuminate(light, pos, seed=5, precision=capi.PRECISION_F32)
        # f32 decides rejection loops / child picks on 32-bit words: almost always the same sample
        same = np.abs(c[2] - a[2]) < 1e-3 * a[2]
        assert same.mean() > 0.995
        scale = np.abs(a[0][same]).max(1) + 1e-30
        assert np.quantile(np.abs(c[0][same] - a[0][same]).max(1) / scale, 0.99) < 1e-3


def test_flattener_rejects_what_the_device_cannot_hold():
    tea = api.Mesh(scenes.teapot_triangles(), build=False)
    with pytest.raises(TypeError):
        api.KdTree([api.plane(api.vec3(0, 1, 0), 0.0)])
    with pytest.raises(TypeError):
        api.KdTree([api.KdTree([api.sphere()])])
    scene = api.Scene()
    scene.add(api.Object(api.KdTree([api.sphere(), tea.translate(api.vec3(1, 0, 0))])))
    flat = api.FlatScene(scene)
    flat.groups[0].children[0].kind = capi.SHAPE_PLANE
    with pytest.raises(ValueError, match="not Bounded"):
        emu.EmuScene(flat)
    flat.groups[0].children[0].kind = capi.SHAPE_GROUP
    with pytest.raises(ValueError, match="not supported"):
        emu.EmuScene(flat)
    flat.groups[0].children[0].kind = capi.SHAPE_SPHERE
    flat.groups[0].children[1].mesh = 7
    with pytest.raises(ValueError, match="mesh 7 out of range"):
        emu.EmuScene(flat)
    flat.groups[0].children[1].mesh = 0
    flat.objects[0].mesh = 3
    with pytest.raises(ValueError, match="group 3 out of range"):
        emu.EmuScene(flat)
    # the product boundary reports the same as a status + message, before it even looks for a device
    import ctypes as C
    h = C.c_void_p()
    rc = capi.lib().rptb_scene_create(C.byref(flat.desc), 0, C.byref(h))
    assert rc == -1 and b"group 3 out of range" in capi.lib().rptb_last_error() and not h


# ---------------------------------------------------------------- the f32 path's own BVH ----------------
def _bvh_pair(scene):
    return (emu.EmuScene(api.FlatScene(scene, accel=capi.ACCEL_BVH)), emu.EmuScene(api.FlatScene(scene, accel=capi.ACCEL_KDTREE)))


@pytest.mark.parametrize("name", ["teapot", "dragon_small", "pegasus"])
def test_bvh_finds_the_hits_of_the_reference_tree(orc, name):
    """rptb_accel BVH (bvhbuild.cpp + bvh_intersect): a different structure over the same triangles and the same
    triangle test -> the f32 hits are those of the kd-tree traversal, to the bit (ties on shared edges aside),
    for a fraction of the node visits and triangle tests."""
    cfg = scenes.teapot_scene() if name == "teapot" else scenes.dragon_knot_scene(330, 82) if name == "dragon_small" else scenes.dragon_scene(level=0)
    eb, ek = _bvh_pair(cfg.scene)
    assert (eb.features & 64) and not (ek.features & 64)
    chk = eb.bvh_check(0)
    ntris = len(cfg.scene.objects[0].shape.shape.triangles)
    assert chk["violations"] == 0 and chk["distinct"] == ntris and chk["max_leaf"] <= 4 and chk["depth"] < 94
    assert ek.bvh_check(0) is None
    rng = np.random.default_rng(5)
    rays = np.concatenate([util.camera_rays(cfg.camera, 30000, rng, spread=0.4), util.interior_rays([-2, -0.99, -2], [2, 1.5, 2], 15000, rng)])
    tb, ob, nb, sb = eb.closest_hit(rays, precision=capi.PRECISION_F32)
    tk, ok, nk, sk = ek.closest_hit(rays, precision=capi.PRECISION_F32)
    same = (tb == tk) & (ob == ok)
    assert same.mean() >= 0.9999
    assert np.abs(nb[same] - nk[same]).max() <= 1e-6
    assert sb["node_visits"] == 0 and sb["tri_tests"] == 0 and sk["bvh_node_visits"] == 0   # each structure has its own counters
    assert 0 < sb["bvh_node_visits"] < 0.5 * sk["node_visits"] and 0 < sb["bvh_tri_tests"] < 0.1 * sk["tri_tests"]
    # and against the oracle, the usual f32 tolerances
    t0, o0, n0, _ = orc.OracleScene(api.FlatScene(cfg.scene)).closest_hit(rays)
    agree = ob == o0
    assert agree.mean() > 0.9999
    hit = agree & (o0 >= 0)
    rel = np.abs(tb[hit] - t0[hit]) / np.abs(t0[hit])
    assert np.median(rel) <= 2e-7 and np.quantile(rel, 0.99) <= 1e-5 and np.quantile(rel, 0.999) <= 1e-4
    # f64 never uses it
    tb64, ob64, _, s64 = eb.closest_hit(rays, precision=capi.PRECISION_F64)
    np.testing.assert_array_equal(tb64, t0)
    assert s64["tri_tests"] == sk["tri_tests"] or s64["tri_tests"] > sb["bvh_tri_tests"]


def test_bvh_builder_on_awkward_meshes():
    rng = np.random.default_rng(8)

    def mesh_scene(tris):
        scene = api.Scene()
        scene.add(api.Object(api.Mesh(np.asarray(tris))))
        return scene

    def check(tris, nrays=4000):
        scene = mesh_scene(tris)
        eb, ek = _bvh_pair(scene)
        if not (ek.features & 1):          # the reference tree is one leaf: no BVH is built, the leaf is scanned
            assert eb.bvh_check(0) is None and not (eb.features & 64)
            return None
        chk = eb.bvh_check(0)
        assert chk["violations"] == 0 and chk["distinct"] == len(tris) and chk["max_leaf"] <= 4 and chk["depth"] < 94
        lo, hi = np.asarray(tris)[:, :9].reshape(-1, 3).min(0), np.asarray(tris)[:, :9].reshape(-1, 3).max(0)
        c, r = (lo + hi) / 2, np.linalg.norm(hi - lo) + 1e-3
        o = c + util.random_unit(rng, nrays) * r
        tgt = lo + rng.uniform(0, 1, (nrays, 3)) * (hi - lo)
        rays = np.concatenate([o, util.normalize(tgt - o)], axis=1)
        tb, ob, _, _ = eb.closest_hit(rays, precision=capi.PRECISION_F32)
        tk, ok, _, _ = ek.closest_hit(rays, precision=capi.PRECISION_F32)
        assert ((tb == tk) & (ob == ok)).mean() >= 0.999
        return chk

    # 64 copies of one triangle: the kd builder gives up (one leaf) -> no BVH
    assert check(np.tile(api.Triangle.from_vertices([0, 0, 0], [1, 0, 0], [0, 1, 0]), (64, 1))) is None
    # a 40 x 40 grid of quads (3 200 triangles, many coplanar, zero-thickness boxes)
    g = []
    for i in range(40):
        for j in range(40):
            a, b, c_, d = [i, 0, j], [i + 1, 0, j], [i + 1, 0, j + 1], [i, 0, j + 1]
            g += [api.Triangle.from_vertices(a, b, c_), api.Triangle.from_vertices(a, c_, d)]
    assert check(np.stack(g))["nodes"] > 500
    # sizes spanning six decades along one axis (SAH peels them off one by one -> a deep, thin tree)
    s = []
    for k in range(60):
        x = 1.5 ** k * 1e-3
        s.append(api.Triangle.from_vertices([x, 0, 0], [x * 1.4, 0, 0], [x, x * 0.4, x * 0.1]))
    chk = check(np.stack(s))
    assert chk is None or chk["depth"] <= 60
    # random soup
    c = rng.uniform(-1, 1, (5000, 1, 3))
    v = c + rng.normal(0, 0.03, (5000, 3, 3))
    assert check(np.stack([api.Triangle.from_vertices(*t) for t in v]))["nodes"] > 1000


def test_accel_field_is_validated():
    flat = api.FlatScene(scenes.teapot_scene().scene)
    flat.desc.accel = 7
    with pytest.raises(ValueError, match="bad accel"):
        emu.EmuScene(flat)


def test_bvh_under_a_kd_tree_of_shapes(orc):
    """rptb_closest_hit without counters on a scene that has both a kd-tree of shapes and BVH meshes runs
    closest_hit<F_EVERY | F_BVH>: the instances of examples/fractal_teapots are entered through the group's
    kd-tree and then traversed through the shared teapot's BVH.  Same hits as through its kd-tree."""
    cfg = scenes.fractal_teapots_scene(3)
    eb, ek = _bvh_pair(cfg.scene)
    assert (eb.features & (16 | 64)) == (16 | 64) and eb.bvh_check(0)["violations"] == 0
    rng = np.random.default_rng(12)
    rays = np.concatenate([util.camera_rays(cfg.camera, 30000, rng, spread=0.35), util.interior_rays([-2.5] * 3, [2.5] * 3, 15000, rng)])
    tb, ob, nb, sb = eb.closest_hit(rays, precision=capi.PRECISION_F32)
    tk, ok, nk, sk = ek.closest_hit(rays, precision=capi.PRECISION_F32)
    same = (tb == tk) & (ob == ok)
    assert same.mean() >= 0.9999 and np.abs(nb[same] - nk[same]).max() <= 1e-6
    assert 0 < sb["bvh_tri_tests"] < 0.2 * sk["tri_tests"]
    t0, o0, _, _ = orc.OracleScene(api.FlatScene(cfg.scene)).closest_hit(rays)
    assert (ob == o0).mean() > 0.9995


# ---------------------------------------------------------------- the megakernel, lane by lane ----------
# render_thread (integrator.cuh) is the whole body of the path-tracing megakernel; hostemu runs it for every
# thread of the grid with a single-lane warp policy.  The flattened recursion (slot schedule, per-level clamp
# stack, forward accumulation, path regeneration, sample chunks) must then BE the reference's trace_ray:
# with Real = double, on the same libm as the oracle, every pixel and every counter comes out equal.
RENDERS = {  # name: (config factory, w, h, spp, max_bounces, accel, FEAT of the f32 variant)
    "cornell": (scenes.cornell_scene, 32, 32, 8, 6, capi.ACCEL_AUTO, F_FLAT),
    "sphere": (scenes.sphere_scene, 48, 27, 8, 2, capi.ACCEL_AUTO, F_FLAT | F_SMALL),
    "teapot_kd": (scenes.teapot_scene, 48, 27, 4, 2, capi.ACCEL_KDTREE, F_TREE),
    "teapot_bvh": (scenes.teapot_scene, 48, 27, 4, 2, capi.ACCEL_BVH, F_TREE | 64),
    "glass": (lambda: scenes.glass_scene(64, 32), 48, 27, 8, 12, capi.ACCEL_AUTO, F_TRANSP | F_HDRI | F_SMALL),
    "fractal_teapots": (lambda: scenes.fractal_teapots_scene(3), 48, 36, 4, 1, capi.ACCEL_AUTO, 7 | F_GROUP | F_MONO),
    "monomial_glass": (lambda: scenes.monomial_glass_scene(64, 32), 48, 36, 8, 1, capi.ACCEL_AUTO, 7 | F_GROUP | F_MONO),
}


def _params(cfg, w, h, spp, mb, seed=1, precision=capi.PRECISION_F32, **kw):
    return api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).seed(seed).precision(precision).params(spp, **kw)


@pytest.mark.parametrize("name", sorted(RENDERS))
def test_megakernel_body_is_trace_ray(orc, name):
    mk, w, h, spp, mb, accel, want_feat = RENDERS[name]
    cfg = mk()
    flat = api.FlatScene(cfg.scene, accel=accel)
    e, o = emu.EmuScene(flat), orc.OracleScene(flat)
    ref, st0 = o.render(cfg.camera, _params(cfg, w, h, spp, mb))
    g64, s64, f64 = e.render(cfg.camera, _params(cfg, w, h, spp, mb, precision=capi.PRECISION_F64))
    np.testing.assert_allclose(g64, ref, rtol=1e-12, atol=0)          # (equal to the bit in practice)
    assert (s64["segments"], s64["rays"]) == (st0["segments"], st0["rays"])
    assert s64["env_lookups"] == st0["env_lookups"] and s64["mesh_hits"] == st0["mesh_hits"]
    # the f32 product variant the library would launch for this scene, same random streams
    ref2, _ = o.render(cfg.camera, _params(cfg, w, h, spp, mb, seed=2))
    cl = lambda a: np.clip(a, 0.0, 1.0)
    noise = util.rmse(cl(ref), cl(ref2))
    g32, s32, f32 = e.render(cfg.camera, _params(cfg, w, h, spp, mb))
    assert f32 == want_feat
    assert np.isfinite(g32).all()
    assert util.rmse(cl(g32), cl(ref)) <= 0.25 * noise
    assert abs(cl(g32).mean() - cl(ref).mean()) <= 5e-3 * cl(ref).mean()
    assert 0.85 * st0["segments"] <= s32["segments"] <= st0["segments"]   # zero-weight subtrees are not traced in f32


def test_megakernel_counting_variant_and_counters(orc):
    cfg = scenes.teapot_scene()
    flat = api.FlatScene(cfg.scene, accel=capi.ACCEL_BVH)
    e, o = emu.EmuScene(flat), orc.OracleScene(flat)
    ref, st0 = o.render(cfg.camera, _params(cfg, 48, 27, 4, 2))
    a, sa, fa = e.render(cfg.camera, _params(cfg, 48, 27, 4, 2, precision=capi.PRECISION_F64, collect_stats=1))
    np.testing.assert_allclose(a, ref, rtol=1e-12, atol=0)
    assert fa == 7 | F_GROUP | F_MONO                                    # counting passes run F_EVERY on the kd-trees
    assert sa["node_visits"] > 0 and sa["tri_tests"] > 0
    # shadow rays are any-hit queries on the device: never more traversal work than the reference's closest-hit
    assert sa["node_visits"] <= st0["node_visits"] and sa["tri_tests"] <= st0["tri_tests"]
    assert sa["object_tests"] == st0["object_tests"] or sa["object_tests"] <= st0["object_tests"]
    b, sb, fb = e.render(cfg.camera, _params(cfg, 48, 27, 4, 2, collect_stats=2))   # f32 counting pass over the kd-trees vs f32 BVH pass
    c, sc, fc = e.render(cfg.camera, _params(cfg, 48, 27, 4, 2))
    assert fb == 7 | F_GROUP | F_MONO and fc == F_TREE | 64
    assert sb["segments"] == sc["segments"] and np.abs(b - c).max() <= 1e-5 * max(1.0, np.abs(b).max())
    assert sb["node_visits"] > 0 and sb["bvh_node_visits"] == 0
    # collect_stats = 1 counts the structure the product path traverses: the BVH, and the image is the BVH image bit for bit
    d, sd, fd = e.render(cfg.camera, _params(cfg, 48, 27, 4, 2, collect_stats=1))
    assert fd == 7 | F_GROUP | F_MONO | 64 and sd["node_visits"] == 0
    assert 0 < sd["bvh_node_visits"] < sb["node_visits"] and 0 < sd["bvh_tri_tests"] < 0.2 * sb["tri_tests"]
    np.testing.assert_array_equal(d, c)


def test_megakernel_chunks_shards_and_sample_ranges(orc):
    """Sample chunks (iterations > 64: partial sums + resolve), pixel-tile shards and first_sample ranges are
    bookkeeping around the same per-pixel streams: sums of shards are the image, bit for bit, and the f64 image
    still equals the oracle's."""
    cfg = scenes.cornell_scene()
    flat = api.FlatScene(cfg.scene)
    e, o = emu.EmuScene(flat), orc.OracleScene(flat)
    w, h, spp, mb = 20, 12, 150, 3                                           # 3 chunks of 64, ragged tiles
    ref, _ = o.render(cfg.camera, _params(cfg, w, h, spp, mb))
    g64, _, _ = e.render(cfg.camera, _params(cfg, w, h, spp, mb, precision=capi.PRECISION_F64))
    np.testing.assert_allclose(g64, ref, rtol=1e-12, atol=0)
    full, _, _ = e.render(cfg.camera, _params(cfg, w, h, spp, mb))
    parts = [e.render(cfg.camera, _params(cfg, w, h, spp, mb, shard_index=i, shard_count=3))[0] for i in range(3)]
    np.testing.assert_array_equal(parts[0] + parts[1] + parts[2], full)
    for i in range(3):                                                       # a shard only writes its own tiles
        own = (np.arange(w * h) % w // 16 + (np.arange(w * h) // w // 8) * ((w + 15) // 16)) % 3 == i
        assert (parts[i][~own] == 0).all()
    a, _, _ = e.render(cfg.camera, _params(cfg, w, h, 40, mb, first_sample=0))
    b, _, _ = e.render(cfg.camera, _params(cfg, w, h, 40, mb, first_sample=40))
    ab, _, _ = e.render(cfg.camera, _params(cfg, w, h, 80, mb, first_sample=0))
    assert not np.array_equal(a, b)                                          # disjoint streams ...
    np.testing.assert_allclose((a + b) / 2, ab, rtol=2e-5, atol=1e-7)        # ... of the same per-sample values


def test_megakernel_corner_cases_equal_the_oracle(orc):
    """Corners of Renderer::sample the BASELINE scenes do not touch, each through the emulated megakernel in f64
    (exactly the oracle) and f32 (finite, within noise): thin-lens camera (aperture > 0), exposure value,
    a directional light, an emissive object seen directly, a scene with no lights, one with no objects, and
    max_bounces > 16 (the MAXD = 64 instantiation)."""
    def check(scene, camera, w, h, spp, mb, ev=0.0):
        flat = api.FlatScene(scene)
        e, o = emu.EmuScene(flat), orc.OracleScene(flat)
        r = api.Renderer(scene, camera).width(w).height(h).max_bounces(mb).seed(4).exposure_value(ev)
        ref, st0 = o.render(camera, r.params(spp))
        g64, s64, _ = e.render(camera, r.precision(capi.PRECISION_F64).params(spp))
        np.testing.assert_allclose(g64, ref, rtol=1e-12, atol=0)
        assert (s64["segments"], s64["rays"]) == (st0["segments"], st0["rays"])
        g32, s32, _ = e.render(camera, r.precision(capi.PRECISION_F32).params(spp))
        assert np.isfinite(g32).all()
        scale = max(1e-3, float(np.abs(ref).mean()))
        assert abs(g32.mean() - ref.mean()) <= 0.02 * scale + 1e-6
        return ref

    base = scenes.sphere_scene()
    cam = api.Camera.look_at(api.vec3(-2.5, 4.0, 6.5), api.vec3(0.0, -0.25, 0.0), api.vec3(0.0, 1.0, 0.0), math.pi / 4)
    a = check(base.scene, cam.focus(api.vec3(0.0, 0.0, 0.0), 0.15), 32, 18, 8, 2)           # depth of field
    b = check(base.scene, api.Camera.look_at(api.vec3(-2.5, 4.0, 6.5), api.vec3(0.0, -0.25, 0.0), api.vec3(0.0, 1.0, 0.0), math.pi / 4),
              32, 18, 8, 2, ev=1.5)                                                       # 2^1.5 brighter
    assert b.mean() > 2.0 * a.mean() * 0.8
    scene = api.Scene()                                                                     # directional + ambient, emissive sphere in view
    scene.add(api.Object(api.sphere()).material(api.Material.light(api.hex_color(0xFFAA33), 3.0)))
    scene.add(api.Object(api.plane(api.vec3(0.0, 1.0, 0.0), -1.0)).material(api.Material.diffuse(api.hex_color(0x8888FF))))
    scene.add(api.Light.Directional(api.vec3(0.8, 0.8, 0.8), api.vec3(0.3, -1.0, -0.2)))
    scene.add(api.Light.Ambient(api.vec3(0.05, 0.05, 0.05)))
    check(scene, cam, 32, 18, 8, 3)
    nolight = api.Scene()                                                                   # no lights: environment only
    nolight.environment = api.Environment.Color(api.vec3(0.2, 0.4, 0.8))
    nolight.add(api.Object(api.sphere()).material(api.Material.metallic_(api.hex_color(0xFFFFFF), 0.2)))
    check(nolight, api.Camera.default(), 24, 16, 8, 4)
    empty = api.Scene()                                                                     # nothing at all: every path escapes
    empty.environment = api.Environment.Color(api.vec3(0.1, 0.2, 0.3))
    img = check(empty, api.Camera.default(), 16, 8, 2, 2)
    np.testing.assert_allclose(img, np.tile([0.1, 0.2, 0.3], (16 * 8, 1)), rtol=1e-15)
    glass = scenes.glass_scene(32, 16)                                                      # 40 bounces: MAXD = 64 kernels
    check(glass.scene, glass.camera, 24, 14, 4, 40)


def test_megakernel_kd_tree_of_shapes_over_bvh_meshes(orc):
    """RPTB_EXT_BVH=1 (opt-in until it has run on a GPU): render_kernel<F_EVERY | F_BVH>, the instances of
    examples/fractal_teapots entered through the group's kd-tree and traversed through the shared teapot's BVH.
    Emulated: same image as through the kd-tree."""
    cfg = scenes.fractal_teapots_scene(3)
    e = emu.EmuScene(api.FlatScene(cfg.scene, accel=capi.ACCEL_BVH))
    p = _params(cfg, 48, 36, 4, 1)
    a, sa, fa = e.render(cfg.camera, p)
    b, sb, fb = e.render(cfg.camera, p, ext_bvh=True)
    assert fa == 7 | F_GROUP | F_MONO and fb == 7 | F_GROUP | F_MONO | 64
    assert (sa["segments"], sa["rays"]) == (sb["segments"], sb["rays"])
    assert np.abs(a - b).max() <= 1e-5 * max(1.0, np.abs(a).max())


@pytest.mark.parametrize("name", ["teapot", "fractal_teapots"])
def test_bvh_with_exactly_zero_direction_components(orc, name):
    """Axis-aligned rays (a Directional light along an axis, an orthogonal view): 1/d is infinite for the zero
    components.  A slab test written as b/d - o/d then produces NaN for ONE plane of a box the ray is inside of,
    and min/max over a single NaN shrink the interval -- the BVH lost about half of the occluders of
    examples/fractal_teapots' directional light (0, -0.65, -1) before slab_rcp.  Any-hit and closest-hit queries
    through the BVH must equal those through the kd-tree, and the f64 gate."""
    cfg = scenes.teapot_scene() if name == "teapot" else scenes.fractal_teapots_scene(3)
    flat = api.FlatScene(cfg.scene, accel=capi.ACCEL_BVH)
    e, o = emu.EmuScene(flat), orc.OracleScene(flat)
    rng = np.random.default_rng(6)
    n = 20000
    for axis_dir in ([0.0, 0.65, 1.0], [0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [-1.0, 0.0, 0.0], [0.3, 0.0, -1.0]):
        d = np.asarray(axis_dir) / np.linalg.norm(axis_dir)
        # origins on a plane behind the scene, perpendicular-ish to d
        u = rng.uniform(-2.5, 2.5, (n, 3))
        org = u - (u @ d)[:, None] * d - 6.0 * d
        rays = np.concatenate([org, np.tile(d, (n, 1))], axis=1)
        kd = e.occluded(rays, np.inf, use_bvh=False)
        bvh = e.occluded(rays, np.inf, use_bvh=True)
        gate = e.occluded(rays, np.inf, precision=capi.PRECISION_F64)
        assert (kd != bvh).mean() <= 2e-4 and (bvh != gate).mean() <= 5e-4, axis_dir   # silhouette-grazing rays only
        assert bvh.mean() > 0.01
        tb, ob, _, _ = e.closest_hit(rays, precision=capi.PRECISION_F32)
        t0, o0, _, _ = o.closest_hit(rays)
        assert (ob == o0).mean() >= 0.9995
        assert ((ob >= 0) == (bvh == 1)).mean() >= 0.9995                             # any-hit agrees with closest-hit


def test_bvh_over_a_handful_of_triangles_behind_a_split_kd_root(orc):
    """ADVICE r1: a caller-supplied kd-tree may split over four triangles or fewer; the default accel (BVH) must take
    such a mesh (the root becomes an inner node over two leaf halves) instead of failing scene creation."""
    from rpt_b200.api import Camera, Light, Material, Mesh, Object, Scene, hex_color, vec3

    for ntris in (1, 2, 3, 4):
        tris = []
        for k in range(ntris):
            x = 0.7 * k
            v = [[x, 0, 0], [x + 0.5, 0, 0.1 * k], [x, 0.6, 0]]
            n = [0, 0, 1]
            tris.append(np.array(v + [n, n, n], dtype=np.float64).reshape(-1))
        tris = np.array(tris)
        mesh = Mesh(tris)
        if ntris >= 2:   # force a split root: left leaf = first triangle(s), right leaf = the rest (an inclusive partition may repeat)
            nodes = (capi.KdNode * 3)()
            nodes[0].split, nodes[0].kind, nodes[0].left, nodes[0].right = 0.6, 0, 1, 2
            nodes[1].kind, nodes[1].first_ref, nodes[1].num_refs = 3, 0, 1
            nodes[2].kind, nodes[2].first_ref, nodes[2].num_refs = 3, 1, ntris - 1
            mesh.nodes, mesh.refs = nodes, np.arange(ntris, dtype=np.uint32)
        scene = Scene()
        scene.add(Object(mesh).material(Material.diffuse(hex_color(0xFFFFFF))))
        scene.add(Light.Point(vec3(5, 5, 5), vec3(0, 0, 3)))
        flat = api.FlatScene(scene, accel=capi.ACCEL_BVH)
        e = emu.EmuScene(flat)
        rng = np.random.default_rng(ntris)
        o = np.concatenate([rng.uniform(-0.5, 3.0, (4000, 2)), np.full((4000, 1), 2.0)], axis=1)
        rays = np.concatenate([o, np.tile([0.0, 0.0, -1.0], (4000, 1)) + rng.normal(0, 0.05, (4000, 3))], axis=1)
        tb, ob, _, sb = e.closest_hit(rays, precision=capi.PRECISION_F32)
        t0, o0, _, _ = orc.OracleScene(flat).closest_hit(rays)
        assert (ob == o0).mean() > 0.999 and (o0 >= 0).any()
        hit = (ob == o0) & (o0 >= 0)
        assert np.abs(tb[hit] - t0[hit]).max() < 1e-5
        if ntris >= 2:
            assert e.features & 64 and sb["bvh_node_visits"] > 0


@pytest.mark.parametrize("name", ["cornell", "teapot", "glass", "dragon", "sphere"])
def test_vertex_at_once_engine_is_the_slot_engine_bit_for_bit(orc, monkeypatch, name):
    """integrator_vx.cuh (RPTB_VX=1: all rays of a path vertex staged at once, BVH traversals compacted into a work list)
    performs, per path, exactly the slot engine's operations in exactly its order: same images to the last bit, same
    segment and ray counts -- run one lane at a time here; tests/test_gpu_vx.py compares real warps on the GPU.  On
    Cornell and the sphere scene the slot engine walks the packed primitive table, which the vertex-at-once engine does not
    have: its variant is the slot engine's without F_FLAT."""
    size = {"cornell": (48, 48, 70, 6), "teapot": (64, 36, 8, 0), "glass": (48, 27, 16, 12), "dragon": (64, 36, 8, 2), "sphere": (48, 27, 16, 2)}[name]
    w, h, spp, mb = size
    cfg = scenes.glass_scene(64, 32) if name == "glass" else (scenes.dragon_scene(level=0) if name == "dragon" else scenes.CONFIGS[name]())
    e = emu.EmuScene(api.FlatScene(cfg.scene, accel=capi.ACCEL_BVH))
    monkeypatch.setenv("RPTB_VX", "0")
    a, sa, fa = e.render(cfg.camera, _params(cfg, w, h, spp, mb))
    monkeypatch.setenv("RPTB_VX", "1")
    b, sb, fb = e.render(cfg.camera, _params(cfg, w, h, spp, mb))
    np.testing.assert_array_equal(a, b)
    assert sa["segments"] == sb["segments"] and sa["rays"] == sb["rays"] and fa & ~F_FLAT == fb
    assert bool(fa & F_FLAT) == (name in ("cornell", "sphere"))


@pytest.mark.parametrize("name", ["teapot", "pegasus", "knot", "tiny"])
def test_eight_wide_bvh_is_the_binary_bvh_collapsed(name):
    """bvhbuild.cpp, emit8: the Bvh8Node tree the lane groups traverse on the GPU (geometry.cuh, bvh8_group_trace) holds
    the binary tree's leaves under fewer, fatter nodes: a scalar walk of it finds, ray for ray, the binary tree's
    closest hit (same t; the same triangle unless two triangles tie exactly) and the same any-hit verdict, with a
    third of the node visits."""
    from rpt_b200.api import Material, Mesh, Object, Scene, hex_color
    if name == "teapot":
        tris = scenes.teapot_triangles()
    elif name == "pegasus":
        tris = scenes.pegasus_proxy(0)
    elif name == "knot":
        tris = scenes.knot_proxy(330, 82)
    else:
        tris = scenes.teapot_triangles()[:3]
    scene = Scene()
    scene.add(Object(Mesh(tris)).material(Material.diffuse(hex_color(0xFFFFFF))))
    e = emu.EmuScene(api.FlatScene(scene, accel=capi.ACCEL_BVH))
    v = tris[:, :9].reshape(-1, 3)
    lo, hi = v.min(0), v.max(0)
    rng = np.random.default_rng(3)
    n = 40000
    o = rng.uniform(lo - 0.5 * (hi - lo), hi + 0.5 * (hi - lo), (n, 3))
    tgt = rng.uniform(lo, hi, (n, 3))
    d = util.normalize(tgt - o) * rng.uniform(0.5, 2.0, (n, 1))   # un-normalised directions, like rays under a Transformed
    d[:50, 0] = 0.0                                                # axis-aligned components (slab_rcp)
    rays = np.concatenate([o, d], axis=1)
    if name == "tiny":
        # a mesh the kd builder leaves as one leaf never gets a BVH: nothing to compare
        assert e.bvh8_probe(0, rays) is None
        return
    t, tri, info = e.bvh8_probe(0, rays)
    assert (np.isfinite(t[:, 0]) == np.isfinite(t[:, 1])).all() and np.isfinite(t[:, 0]).mean() > 0.2
    hit = np.isfinite(t[:, 0])
    np.testing.assert_array_equal(t[hit, 0], t[hit, 1])
    assert (tri[hit, 0] == tri[hit, 1]).mean() > 0.999
    assert info["max_children"] == 8 and info["visits8"] < 0.6 * info["visits2"], info   # (the scalar walk is unordered: the lane groups go front to back)
    ta, tria, _ = e.bvh8_probe(0, rays, any_hit=True)
    assert (np.isfinite(ta[:, 0]) == np.isfinite(ta[:, 1])).all() and (np.isfinite(ta[:, 0]) == hit).all()
    # ... and the four-wide tree one lane per ray walks in the product (bvh4_intersect: ordered, with entry distances on
    # the stack): the same hits from fewer than 0.6 of the dependent node fetches and no more triangle tests
    t4, tri4, info4 = e.bvh4_probe(0, rays)
    assert (np.isfinite(t4[:, 1]) == hit).all()
    np.testing.assert_array_equal(t4[hit, 0], t4[hit, 1])
    assert (tri4[hit, 0] == tri4[hit, 1]).mean() > 0.999
    assert info4["visits4"] < 0.6 * info4["visits2"] and info4["tris4"] <= info4["tris2"], info4
    print(name, info4)
    ta4, _, _ = e.bvh4_probe(0, rays, any_hit=True)
    assert (np.isfinite(ta4[:, 1]) == hit).all()


@pytest.mark.parametrize("ensure_every", [0, 1, 3, 7])
def test_f32_generators_hand_out_the_high_halves_of_the_f64_draws(orc, ensure_every):
    """rng.cuh: a path's 64-bit draws are two Philox streams side by side (draw 4b + w = word w of block b, over word w of
    block b | 2^31), so that the f32 kernels -- which look at the high half only -- compute the first stream alone and use
    every word of a block.  Whatever the buffering (two-and-two, four, eight, the ring) and wherever ensure() falls, the f32
    generators hand out exactly the high halves of the f64 generator's draws, in order: that is what keeps every
    same-stream parity test of the f32 path meaningful.  The halves themselves are pinned against the oracle's raw Philox
    blocks (known-answer tested in test_oracle.py)."""
    seed, pixel, sample, n = 0x0123456789ABCDEF, 4242, (7 << 32) | 9, 101
    o64, o32 = emu.draws(seed, pixel, sample, n, ensure_every)
    hi = (o64 >> np.uint64(32)).astype(np.uint32)
    for k, name in enumerate(("pair", "four", "eight", "ring")):
        np.testing.assert_array_equal(o32[k], hi, err_msg=name)
    nb = (n + 3) // 4
    first = orc.philox(seed, pixel, sample, nb).reshape(-1)[:n]
    second = orc.philox(seed, pixel, sample, nb, first_block=0x80000000).reshape(-1)[:n]
    np.testing.assert_array_equal(hi, first)
    np.testing.assert_array_equal((o64 & np.uint64(0xFFFFFFFF)).astype(np.uint32), second)
