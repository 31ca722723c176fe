"""The packed primitive table (F_FLAT, scene_dev.cuh) in the host emulation, WITHOUT a GPU.

Scenes made only of spheres, planes, cubes and one-leaf meshes are traced through one record stream built by
build_flat_table (flatten.h) and walked by flat_closest_hit (geometry.cuh); RPTB_NO_FLAT, read when a scene is created,
keeps the scan over scene.objects.  The table changes the loads and the dispatch and shares the plane test of a run of
coplanar triangles, never the arithmetic of a primitive, so with the emulation's -ffp-contract=off both walks do the same
float operations: hits (t, object, normal, triangle, barycentrics), any-hit verdicts and whole f32 images must be equal to
the bit.  This checks the table's layout and the walk's control flow; tests/test_gpu_flat_table.py makes the same
comparisons with the compiled kernels.  Also here: the variant the launchers pick for every reachable feature set
(launch.h), the one dispatch the library and the emulation share."""
import contextlib
import os

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import util
from tests.hostemu import emu
from tests.test_hostemu_fuzz import random_scene, random_xf, soup

F_TREE, F_TRANSP, F_HDRI, F_SMALL, F_GROUP, F_MONO, F_BVH, F_FLAT = 1, 2, 4, 8, 16, 32, 64, 128
F_ALL, F_EXT = F_TREE | F_TRANSP | F_HDRI, F_GROUP | F_MONO
F_EVERY = F_ALL | F_EXT
FLAT_TF = 0x100


@contextlib.contextmanager
def flat_switch(on):
    """RPTB_NO_FLAT as a scene created inside the block sees it: unset (on) or set (off)."""
    saved = os.environ.pop("RPTB_NO_FLAT", None)
    try:
        if not on:
            os.environ["RPTB_NO_FLAT"] = "1"
        yield
    finally:
        os.environ.pop("RPTB_NO_FLAT", None)
        if saved is not None:
            os.environ["RPTB_NO_FLAT"] = saved


# ---------------------------------------------------------------- scenes ------------------------------------------------
MAT = api.Material.diffuse(api.hex_color(0x8090A0))


def quad(rng):
    """a random planar quad as a two-triangle fan: its triangles' planes are often, not always, bitwise equal in f32"""
    c = rng.uniform(-2, 2, 3)
    u = util.random_unit(rng, 1)[0]
    v = util.normalize(np.cross(u, util.random_unit(rng, 1)[0]))
    a, b = rng.uniform(0.3, 1.5, 2)
    return api.polygon([api.vec3(*(c - a * u - b * v)), api.vec3(*(c + a * u - b * v)), api.vec3(*(c + a * u + b * v)),
                        api.vec3(*(c - a * u + b * v))])


def table_scene(seed):
    """spheres, cubes, small triangle soups, quads and planes, most of them transformed"""
    rng = np.random.default_rng(seed)
    scene = api.Scene()
    makers = [api.sphere, api.cube, lambda: api.Mesh(soup(rng, 4, 0.5)), lambda: quad(rng)]
    for _ in range(rng.integers(3, 7)):
        shape = makers[rng.integers(0, len(makers))]()
        scene.add(api.Object(random_xf(rng, shape) if rng.random() < 0.6 else shape).material(MAT))
    scene.add(api.Object(api.plane(api.vec3(0.0, 1.0, 0.0), -4.0)).material(MAT))
    scene.add(api.Light.Point(api.vec3(30.0, 30.0, 30.0), api.vec3(0.0, 5.0, 0.0)))
    return scene


def leaf_mesh(tris):
    """a mesh under a caller-supplied kd-tree of one leaf: the device scans it in triangle order whatever its size"""
    mesh = api.Mesh(np.asarray(tris), build=False)
    nodes = (capi.KdNode * 1)()
    nodes[0].kind, nodes[0].first_ref, nodes[0].num_refs = 3, 0, len(mesh)
    mesh.nodes, mesh.refs = nodes, np.arange(len(mesh), dtype=np.uint32)
    return mesh


def tri(a, b, c, normals=None):
    t = api.Triangle.from_vertices(a, b, c)
    if normals is not None:
        t[9:] = np.asarray(normals, np.float64).reshape(-1)
    return t


def square(x0, z0, s, y=0.0):
    """two triangles of one square in the plane y, wound alike (their planes are bitwise equal)"""
    a, b, c, d = [x0, y, z0], [x0 + s, y, z0], [x0 + s, y, z0 + s], [x0, y, z0 + s]
    return [tri(a, b, c), tri(a, c, d)]


def adversarial_scene(name):
    """(scene, centre, radius) of scenes built to break a table walk that is only nearly right"""
    scene = api.Scene()
    rng = np.random.default_rng(sum(map(ord, name)))
    add = lambda shape: scene.add(api.Object(shape).material(MAT))
    if name == "grid":          # 128 coplanar triangles in one leaf: one long run, too big for the parameter-space tables
        # (at y = 1: in y = 0 the plane offsets would be +0 or -0 by the sign of x and z, and split the run)
        add(leaf_mesh([t for i in range(8) for j in range(8) for t in square(i - 4.0, j - 4.0, 1.0, 1.0)]))
        add(api.sphere().translate(api.vec3(0.5, 2.5, 0.0)))
    elif name == "layers":      # same normal, other offset, adjacent in triangle order; then A B A
        tris = square(-1.0, -1.0, 2.0, 0.0) + square(-1.0, -1.0, 2.0, 0.25) + square(-1.5, -1.5, 1.0, 0.5)
        tris += [tri([1.0, 0.0, 1.0], [2.0, 0.0, 1.0], [2.0, 0.0, 2.0]), tri([1.0, 0.75, 1.0], [2.0, 0.75, 1.0], [2.0, 0.75, 2.0]),
                 tri([1.0, 0.0, -2.0], [2.0, 0.0, -2.0], [2.0, 0.0, -1.0])]
        add(leaf_mesh(tris))
    elif name == "duplicates":  # a triangle, its exact copy, a copy wound the other way, and a quad twice over
        t = tri([-1.0, 0.0, -1.0], [1.0, 0.2, -1.0], [0.0, 0.4, 1.0])
        r = tri([-1.0, 0.0, -1.0], [0.0, 0.4, 1.0], [1.0, 0.2, -1.0])
        q = square(-0.5, -0.5, 1.0, -0.7)
        add(leaf_mesh([t, t.copy(), r] + q + q))
    elif name == "vnormals":    # coplanar runs whose vertex normals differ per triangle: the normal names the triangle
        tris = []
        for t in [t for i in range(3) for j in range(3) for t in square(i - 1.5, j - 1.5, 1.0, 0.3)]:
            t[9:] = util.normalize(np.array([0.0, 1.0, 0.0]) + 0.4 * rng.normal(size=(3, 3))).reshape(-1)
            tris.append(t)
        add(leaf_mesh(tris))
        add(random_xf(rng, leaf_mesh(tris)))
    elif name == "ties":        # equal t on two objects: the lower index wins
        shared = leaf_mesh(square(-1.0, -1.0, 2.0, 0.5))
        add(shared)
        add(shared)                                             # the same mesh twice: bitwise the same t
        add(api.plane(api.vec3(0.0, 1.0, 0.0), 0.5))            # coincides with the mesh's face
        add(leaf_mesh(square(-1.0, -1.0, 2.0, -0.5)))
        add(api.plane(api.vec3(0.0, 1.0, 0.0), -0.5))           # ... and after one
        add(api.sphere().translate(api.vec3(0.0, 2.0, 0.0)))
        add(api.sphere().translate(api.vec3(0.0, 2.0, 0.0)))     # two identical spheres
        add(api.cube().scale(api.vec3(0.5, 0.5, 0.5)).translate(api.vec3(1.5, 2.0, 0.0)))
        add(api.cube().scale(api.vec3(0.5, 0.5, 0.5)).translate(api.vec3(1.5, 2.0, 0.0)))
    elif name == "multirun_xf":  # a closed box of six runs under a non-uniform transform, and translated
        c = np.array([[x, y, z] for x in (-1.0, 1.0) for y in (-1.0, 1.0) for z in (-1.0, 1.0)])
        faces = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
        box = leaf_mesh([t for f in faces for t in (tri(c[f[0]], c[f[1]], c[f[2]]), tri(c[f[0]], c[f[2]], c[f[3]]))])
        add(box.scale(api.vec3(1.7, 0.45, 0.9)).rotate(0.7, util.normalize(np.array([1.0, 2.0, 0.5]))).translate(api.vec3(0.3, -0.2, 0.1)))
        add(box.translate(api.vec3(0.0, 0.0, -3.0)))
        add(api.cube().scale(api.vec3(0.8, 2.0, 0.5)).rotate_y(0.3).translate(api.vec3(2.5, 0.0, 0.0)))
    elif name == "planes":
        add(api.plane(api.vec3(0.0, 1.0, 0.0), -1.0))
        add(api.plane(api.vec3(1.0, 0.5, 0.0), 2.0))
        add(api.plane(api.vec3(0.0, 0.0, 1.0), 0.0).rotate_x(0.4).translate(api.vec3(0.0, 0.0, -2.0)))
    elif name != "empty":
        raise KeyError(name)
    scene.add(api.Light.Point(api.vec3(20.0, 20.0, 20.0), api.vec3(1.0, 6.0, 2.0)))
    scene.environment = api.Environment.Color(api.vec3(0.2, 0.3, 0.4))
    return scene, (0.0, 0.0, 0.0), 4.0


ADVERSARIAL = ["grid", "layers", "duplicates", "vnormals", "ties", "multirun_xf", "empty", "planes"]
CONFIGS = {"sphere": (scenes.sphere_scene, (0.0, 0.0, 0.0), 4.0), "cornell": (scenes.cornell_scene, (278.0, 274.0, 280.0), 290.0)}


def named_scene(name):
    """(scene, centre, radius) of every scene these tests walk through the table"""
    if name in CONFIGS:
        mk, c, r = CONFIGS[name]
        return mk().scene, c, r
    if name.startswith("table"):
        return table_scene(300 + int(name[5:])), (0.0, 0.0, 0.0), 5.0
    if name.startswith("fuzz"):
        return random_scene(100 + int(name[4:]), table_only=True)[0], (0.0, 0.0, 0.0), 5.0
    return adversarial_scene(name)


TABLE_SCENES = ["sphere", "cornell"] + ["table%d" % i for i in range(6)] + ADVERSARIAL + ["fuzz%d" % i for i in range(4)]


# ---------------------------------------------------------------- rays ---------------------------------------------------
def probe_rays(rng, center, radius, n):
    """from outside towards the scene; from inside in every direction; axis-aligned; one zero component"""
    m = n // 4
    c = np.asarray(center, np.float64)
    o1 = c + util.random_unit(rng, m) * radius * rng.uniform(1.2, 3.0, (m, 1))
    d1 = util.normalize(c + rng.uniform(-radius, radius, (m, 3)) - o1)
    o2 = c + rng.uniform(-radius, radius, (m, 3))
    d2 = util.random_unit(rng, m)
    o3 = c + rng.uniform(-radius, radius, (m, 3))
    d3 = np.eye(3)[rng.integers(0, 3, m)] * rng.choice([-1.0, 1.0], (m, 1))
    v = rng.normal(size=(n - 3 * m, 3))
    v[np.arange(n - 3 * m), rng.integers(0, 3, n - 3 * m)] = 0.0
    o4 = c + rng.uniform(-radius, radius, (n - 3 * m, 3))
    return np.concatenate([np.concatenate([o, d], axis=1) for o, d in ((o1, d1), (o2, d2), (o3, d3), (o4, util.normalize(v)))])


def world_triangles(scene):
    """(vertices (n, 3, 3), plane normals (n, 3)) of every mesh object's triangles in world space"""
    vs = []
    for ob in scene.objects:
        shape = ob.shape
        m = shape.matrix if isinstance(shape, api.Transformed) else np.eye(4)
        base = shape.shape if isinstance(shape, api.Transformed) else shape
        if isinstance(base, api.Mesh):
            v = base.triangles[:, :9].reshape(-1, 3)
            vs.append((np.concatenate([v, np.ones((len(v), 1))], axis=1) @ m.T)[:, :3].reshape(-1, 3, 3))
    if not vs:
        return np.zeros((0, 3, 3)), np.zeros((0, 3))
    v = np.concatenate(vs)
    return v, util.normalize(np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]))


def edge_and_parallel_rays(rng, scene, center, radius, n):
    """rays through exact shared vertices and edge points of the meshes, and rays parallel to their planes: in the
    plane (cosine exactly 0 where the plane is axis-aligned) and tilted out of it by |cos| < 1e-8"""
    v, nrm = world_triangles(scene)
    if len(v) == 0:
        return np.zeros((0, 6))
    k = rng.integers(0, len(v), n)
    w = rng.integers(0, 3, n)
    corner, other = v[k, w], v[k, (w + 1) % 3]
    target = np.where(rng.random((n, 1)) < 0.5, corner, 0.5 * (corner + other))   # a vertex, or an edge's midpoint
    o = target + util.random_unit(rng, n) * radius * rng.uniform(0.5, 2.0, (n, 1))
    through = np.concatenate([o, util.normalize(target - o)], axis=1)
    along = util.normalize(np.cross(nrm[k], util.random_unit(rng, n)))
    exact = np.abs(nrm[k]).max(axis=1) == 1.0                                       # axis-aligned plane: zero that component
    along[exact] *= (np.abs(nrm[k][exact]) != 1.0)
    along = util.normalize(along)
    tilt = along + nrm[k] * rng.choice([-3e-9, 0.0, 3e-9], (n, 1))
    start = target - along * radius * rng.uniform(0.2, 1.5, (n, 1)) + nrm[k] * rng.choice([0.0, 1e-7, -1e-7], (n, 1))
    return np.concatenate([through, np.concatenate([start, tilt], axis=1)])


def rays_for(name, n=6000):
    scene, center, radius = named_scene(name)
    rng = np.random.default_rng(sum(map(ord, name)) + 1)
    return scene, np.concatenate([probe_rays(rng, center, radius, n), edge_and_parallel_rays(rng, scene, center, radius, n // 2)]), rng


def emu_pair(scene, accel=capi.ACCEL_AUTO):
    """(through the table, through the scan) -- and the first must be what the library runs for the scene"""
    flat = api.FlatScene(scene, accel=accel)
    with flat_switch(True):
        a = emu.EmuScene(flat)
    with flat_switch(False):
        b = emu.EmuScene(flat)
    assert a.flat_table()[1] and a.features & F_FLAT                # the scene qualifies for the table ...
    assert not (b.features & F_FLAT) and (b.features | F_FLAT) == a.features   # ... and RPTB_NO_FLAT only turns it off
    return a, b


# ---------------------------------------------------------------- layout --------------------------------------------------
def decode(words):
    """the table as records: (tag, object, k, first, tf rows (3, 4) or None, payload words)"""
    f = words.view(np.float32)
    recs, p = [], 0
    while p < len(words):
        tag, obj, k, first = (int(x) for x in words[p])
        p += 1
        rows = None
        if tag & FLAT_TF:
            rows = words[p:p + 3]
            p += 3
        kind = tag & 0xFF
        n = 1 if kind == capi.SHAPE_PLANE else 1 + 2 * k if kind == capi.SHAPE_MESH else 0
        assert p + n <= len(words), "record runs past the end of the table"
        recs.append((tag, obj, k, first, rows, words[p:p + n]))
        p += n
    assert p == len(words)
    return recs


def check_layout(scene):
    flat = api.FlatScene(scene)
    with flat_switch(True):
        e = emu.EmuScene(flat)
    words, ok, inv, tri48 = e.flat_table()
    assert ok
    inv_bits, tri_bits = inv.view(np.uint32), tri48.view(np.uint32)
    mesh_base = np.concatenate([[0], np.cumsum([flat.meshes[i].ntris for i in range(flat.desc.nmeshes)])]).astype(int)
    recs = decode(words)
    r = 0
    for i in range(flat.desc.nobjects):
        ob = flat.objects[i]
        tf = FLAT_TF if ob.has_transform else 0
        ntris = flat.meshes[ob.mesh].ntris if ob.kind == capi.SHAPE_MESH else 1
        covered = 0
        while covered < ntris:                                      # an object's records are consecutive and in order
            tag, obj, k, first, rows, payload = recs[r]
            r += 1
            assert obj == i and tag == (ob.kind | tf), (i, tag, obj)
            if tf:                                                  # on every record of the object, every run included
                np.testing.assert_array_equal(rows, inv_bits[i])
            else:
                assert rows is None
            if ob.kind == capi.SHAPE_PLANE:
                want = np.array(list(ob.plane_normal) + [ob.plane_value], np.float32).view(np.uint32)
                np.testing.assert_array_equal(payload[0], want)
            if ob.kind != capi.SHAPE_MESH:
                assert k == 0 and first == 0
                covered = 1
                continue
            q = tri_bits[mesh_base[ob.mesh]:mesh_base[ob.mesh + 1]]
            assert first == covered and k >= 1 and first + k <= ntris  # the runs cover 0..ntris-1 contiguously
            np.testing.assert_array_equal(payload[0], q[first, 0])
            for j in range(k):                                      # one plane for the run, bit for bit ...
                np.testing.assert_array_equal(q[first + j, 0], q[first, 0])
                np.testing.assert_array_equal(payload[1 + 2 * j], q[first + j, 1])
                np.testing.assert_array_equal(payload[2 + 2 * j], q[first + j, 2])
            if first + k < ntris:                                   # ... and the run is maximal
                assert not np.array_equal(q[first + k, 0], q[first, 0])
            covered += k
    assert r == len(recs)                                           # nothing but the objects
    return words, recs


@pytest.mark.parametrize("name", TABLE_SCENES)
def test_table_layout(name):
    check_layout(named_scene(name)[0])


def test_table_sizes():
    words, recs = check_layout(scenes.cornell_scene().scene)
    # five one-run quads (header, q0, 2 x (q1, q2)) and two transformed cubes (header, 3 rows); the light's quad is no object
    assert len(words) == 38 and len(recs) == 7
    words, recs = check_layout(adversarial_scene("grid")[0])
    assert [r[2] for r in recs if r[0] & 0xFF == capi.SHAPE_MESH] == [128]      # one run of all 128 triangles
    _, recs = check_layout(adversarial_scene("layers")[0])
    assert [r[2] for r in recs] == [2, 2, 2, 1, 1, 1]                          # parallel layers and A B A stay apart
    _, recs = check_layout(adversarial_scene("duplicates")[0])
    assert [r[2] for r in recs] == [2, 1, 4]                                   # copies join a run, the reversed one does not
    _, recs = check_layout(adversarial_scene("multirun_xf")[0])
    assert [r[2] for r in recs if r[1] == 0] == [2] * 6 and all(r[0] & FLAT_TF for r in recs if r[1] == 0)
    words, recs = check_layout(adversarial_scene("empty")[0])
    assert len(words) == 0


# ---------------------------------------------------------------- hits -------------------------------------------------
def assert_same_detail(a, b, rays):
    ta, oa, na, xa, ba, _ = a.closest_hit_detail(rays, precision=capi.PRECISION_F32)
    tb, ob, nb, xb, bb, _ = b.closest_hit_detail(rays, precision=capi.PRECISION_F32)
    np.testing.assert_array_equal(oa, ob)
    np.testing.assert_array_equal(ta, tb)
    np.testing.assert_array_equal(na, nb)
    np.testing.assert_array_equal(xa, xb)
    np.testing.assert_array_equal(ba, bb)
    return tb, ob


@pytest.mark.parametrize("name", TABLE_SCENES)
def test_table_walk_is_the_scan(orc, name):
    scene, rays, rng = rays_for(name)
    a, b = emu_pair(scene)
    t, obj = assert_same_detail(a, b, rays)
    if name != "empty":
        assert (obj >= 0).mean() > 0.05
    # rays that start on the surfaces just hit, leaving in random directions
    hit = obj >= 0
    p = rays[hit, :3] + t[hit, None] * rays[hit, 3:]
    assert_same_detail(a, b, np.concatenate([p, util.random_unit(rng, int(hit.sum()))], axis=1))
    # and the f32 walk against the f64 oracle, with test_hostemu's f32 tolerances (the probe rays from outside and from
    # inside in random directions: no grazing or edge rays).  Coincident surfaces of two objects are a tie the last ulp
    # decides, as in test_hostemu_fuzz
    probe = rays[:3000]
    t0, o0, n0, _ = orc.OracleScene(api.FlatScene(scene)).closest_hit(probe)
    t1, o1, n1, _ = a.closest_hit(probe, precision=capi.PRECISION_F32)
    same = o1 == o0
    with np.errstate(invalid="ignore"):
        tie = (o1 >= 0) & (o0 >= 0) & (np.abs(t1 - t0) <= 1e-5 * np.abs(t0))
    assert (same | tie).mean() > 0.999
    hit = same & (o0 >= 0)
    if hit.any():
        rel = np.abs(t1[hit] - t0[hit]) / np.abs(t0[hit])
        assert np.median(rel) <= 2e-7 and np.quantile(rel, 0.99) <= 1e-5 and np.quantile(rel, 0.999) <= 1e-3
        assert np.quantile(np.abs(n1[hit] - n0[hit]).max(1), 0.99) < 1e-3


@pytest.mark.parametrize("name", TABLE_SCENES)
def test_table_any_hit_is_the_scan(name):
    scene, rays, _ = rays_for(name)
    a, b = emu_pair(scene)
    t, obj, _, _ = b.closest_hit(rays, precision=capi.PRECISION_F32)
    t32 = t.astype(np.float32)
    for tmax, want in ((np.inf, obj >= 0),                                       # anything on the ray
                       (t, np.zeros(len(t), bool)),                              # strictly before the closest hit: nothing
                       (np.nextafter(t32, np.float32(np.inf)).astype(np.float64), obj >= 0)):   # the closest hit itself
        occ_a = a.occluded(rays, tmax, precision=capi.PRECISION_F32)
        occ_b = b.occluded(rays, tmax, precision=capi.PRECISION_F32)
        np.testing.assert_array_equal(occ_a, occ_b)
        np.testing.assert_array_equal(occ_a == 1, want)


# ---------------------------------------------------------------- renders -----------------------------------------------
def camera_for(center, radius):
    c = np.asarray(center, np.float64)
    return api.Camera.look_at(api.vec3(*(c + radius * np.array([0.9, 1.1, 2.2]))), api.vec3(*c), api.vec3(0.0, 1.0, 0.0), 0.9)


def render_pair(scene, camera, w, h, spp, mb, **kw):
    a, b = emu_pair(scene)
    p = api.Renderer(scene, camera).width(w).height(h).max_bounces(mb).seed(3).params(spp, **kw)
    ga, sa, fa = a.render(camera, p)
    gb, sb, fb = b.render(camera, p)
    assert fa & F_FLAT and fb == fa & ~F_FLAT                     # the table's variant against the scan's
    np.testing.assert_array_equal(ga, gb)
    assert (sa["segments"], sa["rays"]) == (sb["segments"], sb["rays"])
    return ga, sa


@pytest.mark.parametrize("name", TABLE_SCENES)
def test_table_render_is_the_scan_render(name):
    if name in CONFIGS:
        cfg = CONFIGS[name][0]()
        scene, camera = cfg.scene, cfg.camera
    else:
        scene, center, radius = named_scene(name)
        camera = camera_for(center, radius)
    img, st = render_pair(scene, camera, 24, 16, 4, 4)
    assert st["segments"] >= 24 * 16 * 4


def test_table_render_with_chunks_and_shards():
    cfg = scenes.cornell_scene()
    full, _ = render_pair(cfg.scene, cfg.camera, 20, 12, 150, 3)                  # 3 chunks of 64
    parts = [render_pair(cfg.scene, cfg.camera, 20, 12, 150, 3, shard_index=i, shard_count=3)[0] for i in range(3)]
    np.testing.assert_array_equal(parts[0] + parts[1] + parts[2], full)


# ---------------------------------------------------------------- dispatch ----------------------------------------------
def reachable_features():
    """every feature set a scene can present to the launchers (kernel_features, flatten.h)"""
    out = []
    for f in range(256):
        if f & F_BVH and not f & F_TREE:                              # a BVH is built over real kd-trees only
            continue
        if f & F_FLAT and f & (F_TREE | F_EXT | F_BVH):               # the table holds no trees, groups or monomials
            continue
        if f & F_SMALL and f & F_EXT:
            continue
        out.append(f)
    return out


def test_every_reachable_feature_set_has_its_variant():
    n = 0
    for f in reachable_features():
        for stats in (0, 1, 2):
            for prec in (capi.PRECISION_F32, capi.PRECISION_F64):
                for mb in (6, 16, 17, 40):
                    for engine in (emu.ENGINE_RENDER, emu.ENGINE_VX, emu.ENGINE_CLOSEST_HIT):
                        if engine == emu.ENGINE_VX and prec == capi.PRECISION_F64:
                            continue                                   # the vertex-at-once engine is f32 only
                        (vs, feat, maxd), compiled = emu.pick_variant(engine, f, stats, prec, mb)
                        where = (f, stats, prec, mb, engine, feat)
                        assert compiled, where
                        assert vs == (stats != 0), where
                        # (a closest hit reads geometry only: of F_ALL, just F_TREE concerns it)
                        need = f & (F_TREE if engine == emu.ENGINE_CLOSEST_HIT else F_ALL)
                        assert feat & need == need, where
                        if f & F_EXT:
                            assert feat & F_EVERY == F_EVERY, where
                        for bit in (F_FLAT, F_SMALL, F_BVH):
                            assert not (feat & bit) or (f & bit), where
                        if stats or prec == capi.PRECISION_F64:
                            assert not feat & F_FLAT, where
                        if stats == 2 or prec == capi.PRECISION_F64:
                            assert not feat & F_BVH, where
                        if engine == emu.ENGINE_RENDER:                # the f64 gate's level stack holds the path
                            assert maxd >= (mb if prec == capi.PRECISION_F64 else 16), where
                        # a flat scene without counters is traced through the table
                        if (f & F_FLAT and not stats and prec == capi.PRECISION_F32 and engine != emu.ENGINE_VX
                                and (engine == emu.ENGINE_CLOSEST_HIT or not f & F_ALL)):
                            assert feat & F_FLAT, where
                        n += 1
    assert n > 1000
