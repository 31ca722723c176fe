"""Path-by-path comparison of the f32 render kernels with the oracle.

The f32 kernels and the oracle draw from the same Philox stream for each (seed, pixel, sample): the f32 generators hand
out the high halves of the f64 draws (rng.cuh, pinned in test_hostemu.py).  A render with iterations = 1 and
first_sample = s is therefore one path per pixel, the same path in both precisions, and S such renders stacked give
S * W * H paths that can be compared one by one.  Most of them agree to ~1e-6; a path differs by more only where f32
rounding flips a discrete decision (a hit, a lobe, a rejection step) and the two paths part ways.  That makes the
comparison several orders of magnitude sharper than image statistics (RMSE within Monte-Carlo noise): a bias of a
fraction of a percent in one rule of the f32 path moves the signed bias of the agreeing paths by far more than its
limit, and a wrong discrete rule moves the agreement fraction.

`CASES` is the scene matrix both tiers run (test_hostemu_paths.py on the host emulation, test_gpu_paths.py on the GPU).
It reaches every f32 variant pick_render returns for collect_stats = 0 and every rule only the f32 path has: the forward
clamp composite (A, W, C) with the clamp engaged deep in the path and a signed direct term, the `dead` / zero-weight /
shadow-`skip` shortcuts, offset_origin, the one-pass and the two-loop sample_f, the packed primitive table, the kd-trees,
the BVH and the kd-trees of shapes.
"""
from __future__ import annotations

import contextlib
import math
import os
from dataclasses import dataclass, field
from typing import Callable, Dict

import numpy as np

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes

F_TREE, F_TRANSP, F_HDRI, F_SMALL, F_GROUP, F_MONO, F_BVH, F_FLAT = 1, 2, 4, 8, 16, 32, 64, 128
F_ALL = F_TREE | F_TRANSP | F_HDRI
F_EVERY = F_ALL | F_GROUP | F_MONO

REL_TOL = 1e-3       # a path "agrees" when max_c |f32 - f64| <= REL_TOL * max(max_c |f64|, 1e-3)
MIN_PATHS = 16384    # the agreement fraction then has a binomial error of ~0.1 % or less

# Every f32 render_kernel variant pick_render (launch.h) returns for collect_stats = 0 (the product's variants).
F32_RENDER_VARIANTS = {
    F_FLAT, F_FLAT | F_SMALL, F_SMALL, 0, F_TREE, F_TREE | F_BVH, F_ALL | F_BVH, F_TRANSP | F_HDRI | F_SMALL,
    F_TRANSP | F_HDRI, F_ALL, F_EVERY, F_EVERY | F_BVH,
}


@dataclass
class Case:
    """One scene of the matrix.  `make` returns (scene, camera).  `env`: the scene-creation switches of flatten.h
    (RPTB_NO_FLAT, RPTB_NO_SMALL) that route a scene to the variant without the packed table / parameter-space tables.
    `floor` / `gpu_floor`: the least fraction of paths within REL_TOL on the host emulation / on the H100; `bias`: the largest |signed bias|
    of those paths.  Both are measured; the docstring of test_hostemu_paths.py lists the measurements."""
    make: Callable
    w: int
    h: int
    spp: int
    max_bounces: int
    accel: int
    feat: int                      # FEAT of the f32 render_kernel variant that serves the scene
    floor: float
    gpu_floor: float
    bias: float = 1e-5
    ev: float = 0.0
    env: Dict[str, str] = field(default_factory=dict)
    wavefront: bool = False        # also rendered through ENGINE_WAVEFRONT on the GPU (every case it serves: not F_GROUP / F_MONO)
    base: str = ""                 # PLACEMENTS: the case whose world geometry this one shares ("" = none)
    degrades: bool = False         # PLACEMENTS: f32 agreement below the base's by design, or the oracle's own image moves
    base_slack: float = 0.0        # PLACEMENTS: measured shortfall of the f32 agreement below the base's floor


@contextlib.contextmanager
def scene_env(env):
    """flatten.h reads its switches when a scene is created."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def renderer(case: Case, scene, camera, seed: int, precision: int, engine: int = capi.ENGINE_AUTO) -> api.Renderer:
    return (api.Renderer(scene, camera).width(case.w).height(case.h).max_bounces(case.max_bounces).seed(seed)
            .precision(precision).exposure_value(case.ev).engine(engine))


def stack_paths(render: Callable[[int], tuple], spp: int):
    """render(s) -> (image (W*H, 3), stats) of the 1-sample render with first_sample = s.  Returns the paths of
    s = 0..spp-1 stacked into (spp*W*H, 3) and the summed trace_ray invocations."""
    imgs, segments = [], 0
    for s in range(spp):
        img, st = render(s)
        imgs.append(np.asarray(img, dtype=np.float64))
        segments += int(st["segments"])
    return np.concatenate(imgs), segments


def oracle_paths(orc, case: Case, scene, camera, seed: int = 1):
    osc = orc.OracleScene(api.FlatScene(scene))
    r = renderer(case, scene, camera, seed, capi.PRECISION_F64)
    try:
        return stack_paths(lambda s: osc.render(camera, r.params(1, s)), case.spp)
    finally:
        osc.close()


@dataclass
class PathStats:
    rel: np.ndarray         # per path: max_c |f32 - f64| / max(max_c |f64|, 1e-3)
    agree: float            # fraction of paths with rel <= REL_TOL
    tail: float             # fraction with rel > 0.1
    bias: float             # sum(f32 - f64) / sum(|f64|) over the agreeing paths
    seg32: int
    seg64: int

    def line(self, name, feat) -> str:
        return "%-18s FEAT %3d  paths %6d  agree %.5f  >1e-1 %.5f  bias %+.2e  segments %d / %d" % (
            name, feat, self.rel.size, self.agree, self.tail, self.bias, self.seg32, self.seg64)


def compare(f32: np.ndarray, f64: np.ndarray, seg32: int = 0, seg64: int = 0) -> PathStats:
    assert f32.shape == f64.shape
    scale = np.maximum(np.abs(f64).max(axis=1), 1e-3)
    with np.errstate(invalid="ignore"):
        rel = np.abs(f32 - f64).max(axis=1) / scale
    rel = np.where(np.isfinite(rel), rel, np.inf)
    ok = rel <= REL_TOL
    den = np.abs(f64[ok]).sum()
    bias = float((f32[ok] - f64[ok]).sum() / den) if den > 0 else 0.0
    return PathStats(rel, float(ok.mean()), float((rel > 0.1).mean()), bias, seg32, seg64)


# ------------------------------------------------------------------------------------------------ scenes ----------
def _cfg(factory):
    def make():
        cfg = factory()
        return cfg.scene, cfg.camera
    return make


def _clamp():
    """A near-mirror floor and a polished ball under a 4e4 point light (test_oracle's "clamp" scene): the per-level
    min(., 100) engages at the camera hit and again deeper, where the light's glint comes back through two or three
    mirror bounces."""
    from tests.test_oracle import _analytic_scene
    scene, cam, _, _ = _analytic_scene("clamp")
    return scene, cam


def _clamp_glass():
    """A tinted transmissive ball (signed direct term: a light behind the surface contributes f I (wi . n) < 0, and
    the shadow ray is traced although the cosine is negative) lit by a bright sphere light above a near-mirror floor:
    the clamp engages at depth >= 2 on paths whose A carries negative terms."""
    scene = api.Scene()
    scene.add(api.Object(api.sphere()).material(api.Material.transparent_(api.vec3(0.9, 0.6, 0.4), 1.4, 0.4)))
    scene.add(api.Object(api.plane(api.vec3(0, 1, 0), -1.0)).material(api.Material.specular(api.hex_color(0xDDDDDD), 0.05)))
    scene.add(api.Light.Object(api.Object(api.sphere().scale(api.vec3(0.4, 0.4, 0.4)).translate(api.vec3(0.8, 1.6, -2.5)))
                               .material(api.Material.light(api.vec3(1, 1, 1), 3000.0))))
    # a frosted pane to the side, lit from behind: a closed transmissive ball shadows its own back-lit side, a thin
    # pane does not, so here the negative direct terms reach the film
    pane = api.polygon([api.vec3(-2.6, -1.0, -1.2), api.vec3(-1.05, -1.0, -1.2), api.vec3(-1.05, 1.8, -1.2), api.vec3(-2.6, 1.8, -1.2)])
    scene.add(api.Object(pane).material(api.Material.transparent_(api.vec3(0.7, 0.9, 0.8), 1.5, 0.5)))
    scene.environment = api.Environment.Color(api.vec3(0.3, 0.35, 0.4))
    return scene, api.Camera.look_at(api.vec3(0, 1.2, 5), api.vec3(0, -0.2, 0), api.vec3(0, 1, 0), 0.9)


def _lights():
    """Every analytic and object light kind with a leading and a trailing ambient light, seen through a thin lens."""
    scene = api.Scene()
    scene.add(api.Light.Ambient(api.vec3(0.02, 0.02, 0.03)))
    scene.add(api.Object(api.plane(api.vec3(0, 1, 0), -1.0)).material(api.Material.diffuse(api.hex_color(0xAAAAAA))))
    scene.add(api.Object(api.sphere()).material(api.Material.specular(api.hex_color(0x3366CC), 0.2)))
    scene.add(api.Object(api.cube().scale(api.vec3(0.6, 0.8, 0.6)).rotate_y(0.5).translate(api.vec3(2.0, -0.2, -0.5)))
              .material(api.Material.metallic_(api.hex_color(0xD4AF37), 0.3)))
    scene.add(api.Light.Directional(api.vec3(0.8, 0.75, 0.7), api.vec3(-0.3, -1.0, -0.2)))
    scene.add(api.Light.Point(api.vec3(20, 10, 10), api.vec3(-3, 4, 2)))
    scene.add(api.Light.Object(api.Object(api.sphere().scale(api.vec3(0.3, 0.3, 0.3)).translate(api.vec3(-2, 2.5, 1)))
                               .material(api.Material.light(api.vec3(1, 0.9, 0.8), 20.0))))
    scene.add(api.Light.Object(api.Object(api.cube().scale(api.vec3(1.0, 0.2, 2.0)).rotate_z(0.4).translate(api.vec3(-3, 3, 0)))
                               .material(api.Material.light(api.vec3(1, 0.9, 0.8), 8.0))))
    fan = api.polygon([api.vec3(0, 0, 0), api.vec3(1, 0, 0), api.vec3(1.5, 0, 1), api.vec3(0.5, 0, 1.8), api.vec3(-0.5, 0, 1)])
    scene.add(api.Light.Object(api.Object(fan.rotate_x(math.pi).scale(api.vec3(1.5, 1.0, 1.5)).translate(api.vec3(2, 4, -1)))
                               .material(api.Material.light(api.vec3(0.8, 0.9, 1.0), 12.0))))
    scene.add(api.Light.Ambient(api.vec3(0.0, 0.01, 0.0)))
    cam = api.Camera.look_at(api.vec3(0, 2, 7), api.vec3(0, 0, 0), api.vec3(0, 1, 0), 0.7).focus(api.vec3(0, 0, 0), 0.15)
    return scene, cam


def smooth_sphere_mesh(nu: int = 12, nv: int = 6) -> np.ndarray:
    """A coarse UV sphere whose triangles carry the exact sphere normals at their corners, wound one way and the other
    in turn, as scanned meshes often are.  The face normal ng (from the winding) then points out of half the faces and
    into the other half, while the shading normal n always points out and differs from the face's by up to ~15
    degrees: the f32 path must decide `dead` (an opaque surface seen from behind) by n, as the bsdf does."""
    th = np.linspace(0.0, math.pi, nv + 1)
    ph = np.linspace(0.0, 2.0 * math.pi, nu + 1)
    p = np.stack([np.sin(th)[:, None] * np.cos(ph)[None, :], np.cos(th)[:, None] * np.ones_like(ph)[None, :],
                  np.sin(th)[:, None] * np.sin(ph)[None, :]], axis=-1)
    tris = []
    for i in range(nv):
        for j in range(nu):
            a, b, c, d = p[i, j], p[i + 1, j], p[i + 1, j + 1], p[i, j + 1]
            for t in ((a, c, b), (a, d, c)):
                if np.linalg.norm(np.cross(t[1] - t[0], t[2] - t[0])) < 1e-9:
                    continue
                if len(tris) % 2:
                    t = (t[0], t[2], t[1])
                tris.append(np.concatenate([t[0], t[1], t[2], t[0], t[1], t[2]]))
    return np.asarray(tris)


def _smooth(transparent_ball: bool):
    def make():
        scene = api.Scene()
        mesh = api.Mesh(smooth_sphere_mesh())
        for k, x in enumerate((-1.3, 0.0, 1.3)):
            scene.add(api.Object(mesh.scale(api.vec3(0.6, 0.6, 0.6)).translate(api.vec3(x, 0.0, 0.3 * k)))
                      .material(api.Material.specular(api.hex_color(0xCC8844), 0.3)))
        scene.add(api.Object(api.plane(api.vec3(0, 1, 0), -0.6)).material(api.Material.diffuse(api.hex_color(0x999999))))
        if transparent_ball:
            scene.add(api.Object(api.sphere().scale(api.vec3(0.4, 0.4, 0.4)).translate(api.vec3(0.6, -0.2, 1.4)))
                      .material(api.Material.clear(1.5, 0.05)))
            scene.environment = api.Environment.Hdri(scenes.synthetic_hdri(32, 16))
        scene.add(api.Light.Point(api.vec3(30, 30, 30), api.vec3(-2, 5, 4)))
        return scene, api.Camera.look_at(api.vec3(0, 0.8, 4.5), api.vec3(0, 0, 0.3), api.vec3(0, 1, 0), 0.8)
    return make


def _glass_lit():
    """The glass spheres of examples/glass.rs over a floor, under an HDRI and a point light, 40 bounces: long paths
    through the dielectric (the f32 path has no depth limit; the f64 gate takes its MAXD = 64 instantiation)."""
    cfg = scenes.glass_scene(32, 16)
    scene = cfg.scene
    scene.add(api.Object(api.plane(api.vec3(0, 1, 0), -1.0)).material(api.Material.specular(api.hex_color(0xAAAAAA), 0.3)))
    scene.add(api.Light.Point(api.vec3(20, 20, 20), api.vec3(0, 5, 3)))
    return scene, cfg.camera


K, B, A = capi.ACCEL_KDTREE, capi.ACCEL_BVH, capi.ACCEL_AUTO
NO_FLAT, NO_SMALL = {"RPTB_NO_FLAT": "1"}, {"RPTB_NO_SMALL": "1"}

CASES: Dict[str, Case] = {
    # name: Case(scene, width, height, spp, max_bounces, accel, FEAT, floor, gpu_floor, ...)
    # the product's scenes
    "cornell": Case(_cfg(scenes.cornell_scene), 32, 32, 16, 6, A, F_FLAT, 0.982, 0.982, wavefront=True),
    "cornell_scan": Case(_cfg(scenes.cornell_scene), 32, 32, 16, 6, A, 0, 0.982, 0.982, env=NO_FLAT),
    "sphere": Case(_cfg(scenes.sphere_scene), 32, 32, 16, 2, A, F_FLAT | F_SMALL, 0.999, 0.999, wavefront=True),
    "sphere_scan": Case(_cfg(scenes.sphere_scene), 32, 32, 16, 2, A, F_SMALL, 0.999, 0.999, env=NO_FLAT),
    "teapot_kd": Case(_cfg(scenes.teapot_scene), 32, 32, 16, 2, K, F_TREE, 0.999, 0.999, wavefront=True),
    "teapot_bvh": Case(_cfg(scenes.teapot_scene), 32, 32, 16, 2, B, F_TREE | F_BVH, 0.999, 0.999, wavefront=True),
    "glass": Case(_cfg(lambda: scenes.glass_scene(64, 32)), 32, 32, 16, 12, A, F_TRANSP | F_HDRI | F_SMALL, 0.974, 0.974, wavefront=True),
    "glass_deep": Case(_glass_lit, 32, 32, 16, 40, A, F_TRANSP | F_HDRI, 0.968, 0.968, env=NO_SMALL, wavefront=True),
    "fractal_spheres": Case(_cfg(lambda: scenes.fractal_spheres_scene(3)), 32, 32, 16, 2, A, F_EVERY, 0.997, 0.997),
    "fractal_teapots_kd": Case(_cfg(lambda: scenes.fractal_teapots_scene(3)), 32, 32, 16, 2, K, F_EVERY, 0.997, 0.997),
    "fractal_teapots_bvh": Case(_cfg(lambda: scenes.fractal_teapots_scene(3)), 32, 32, 16, 2, B, F_EVERY | F_BVH, 0.997, 0.997),
    "monomial_glass": Case(_cfg(lambda: scenes.monomial_glass_scene(64, 32)), 32, 32, 16, 3, A, F_EVERY, 0.990, 0.990),
    # the f32-only rules
    "clamp": Case(_clamp, 32, 32, 16, 6, A, F_FLAT | F_SMALL, 0.998, 0.998, ev=-1.0, wavefront=True),
    "clamp_glass": Case(_clamp_glass, 48, 32, 24, 8, A, F_ALL, 0.9965, 0.9965, wavefront=True),
    "lights_lens": Case(_lights, 37, 23, 20, 3, A, F_FLAT, 0.999, 0.999, wavefront=True),
    "smooth_kd": Case(_smooth(False), 32, 32, 16, 3, K, F_TREE, 0.999, 0.999, wavefront=True),
    "smooth_glass_bvh": Case(_smooth(True), 32, 32, 16, 4, B, F_ALL | F_BVH, 0.995, 0.995, wavefront=True),
}

# ------------------------------------------------------------------------------------------------ list schedule ---
# Adaptive sampling renders through the list-scheduled twins of the variants above (render_list_kernel, F_LIST).  The
# matrix of (case, precision, collect_stats) both tiers run it on (test_hostemu_paths.py checks that it reaches every
# list variant pick_render_list can return, test_gpu_list_matrix.py runs it): every case in f32 without counters, f64
# on one case per f64 variant, and the counting variants on cases with meshes, kd-trees and a BVH.
LIST_MATRIX = ([(name, capi.PRECISION_F32, 0) for name in sorted(CASES)] + [
    ("fractal_teapots_bvh", capi.PRECISION_F32, 1),   # STATS F_EVERY | F_BVH
    ("fractal_teapots_bvh", capi.PRECISION_F32, 2),   # STATS F_EVERY over the reference-shaped kd-trees
    ("teapot_kd", capi.PRECISION_F32, 1),             # STATS F_EVERY
    ("sphere", capi.PRECISION_F64, 0),                # F_ALL / 16
    ("fractal_spheres", capi.PRECISION_F64, 0),       # F_EVERY / 16
    ("glass_deep", capi.PRECISION_F64, 0),            # F_EVERY / 64 (40 bounces)
    ("monomial_glass", capi.PRECISION_F64, 1),        # STATS F_EVERY / 16
    ("glass_deep", capi.PRECISION_F64, 2),            # STATS F_EVERY / 64
])

TILE_W, TILE_H = 16, 8   # a CTA's tile; its four warps each take an 8x4 block (tile.h)


def list_mask(w: int, h: int, seed: int = 0) -> np.ndarray:
    """(h, w) bool: about half the pixels at random, with the ragged last row and column on, tile (0, 0) wholly off and
    a listed tile (the next one) whose first 8x4 warp block is off.  Needs at least two tiles."""
    rng = np.random.default_rng(seed)
    m = rng.random((h, w)) < 0.5
    m[-1, :] = True
    m[:, -1] = True
    m[:TILE_H, :TILE_W] = False
    y0, x0 = (0, TILE_W) if w > TILE_W else (TILE_H, 0)
    assert y0 < h and x0 < w, "list_mask needs two tiles"
    m[y0:y0 + 4, x0:x0 + 8] = False
    m[min(y0 + 4, h - 1), min(x0 + 8, w - 1)] = True
    return m


def edge_masks(w: int, h: int) -> Dict[str, np.ndarray]:
    """The masks where a list schedule goes wrong first, as (h, w) bool: nothing, everything, the last pixel (in the
    last, ragged tile), only the pixels of ragged tiles, a checkerboard of 8x4 warp blocks, every other tile."""
    y, x = np.mgrid[0:h, 0:w]
    tiles_x = -(-w // TILE_W)
    last = np.zeros((h, w), bool)
    last[-1, -1] = True
    return {
        "none": np.zeros((h, w), bool),
        "all": np.ones((h, w), bool),
        "last_pixel": last,
        "ragged": (x >= w // TILE_W * TILE_W) | (y >= h // TILE_H * TILE_H),
        "warp_checker": (x // 8 + y // 4) % 2 == 0,
        "tile_checker": ((y // TILE_H) * tiles_x + x // TILE_W) % 2 == 0,
    }


# ------------------------------------------------------------------------------------------------ placements ------
# The same world geometry placed where the f32 path's magnitude-dependent rules are stretched: meshes whose vertices
# sit far from their own origin and are pulled back by the object's transform (scanned, CAD and georeferenced files
# arrive like this), scenes scaled by 1e-3 and 1e3, a small instance seen from far away, a scene far from the world
# origin.  Each case either has its base's world geometry exactly, or is its base scaled uniformly with the point
# lights' intensities times s^2, so that the oracle's image is the base's.
def moved(make, m: np.ndarray, s: float = 1.0):
    """make() with every shape, point light and the camera mapped by the 4x4 similarity m of uniform scale s."""
    def moved_make():
        scene, cam = make()
        seen = set()
        for o in list(scene.objects) + [l.object for l in scene.lights if l.object is not None]:
            if id(o) not in seen:
                seen.add(id(o))
                o.shape = o.shape.transform(m)
        for l in scene.lights:
            if l.kind == capi.LIGHT_POINT:
                l.vec = (m @ np.append(l.vec, 1.0))[:3]
                l.color = l.color * s * s
        cam.eye = (m @ np.append(cam.eye, 1.0))[:3]
        cam.focal_distance *= s
        cam.aperture *= s
        return scene, cam
    return moved_make


def _translation(v) -> np.ndarray:
    m = np.eye(4)
    m[:3, 3] = v
    return m


def _teapot_at(d: float, group: bool = False):
    """A specular teapot on a diffuse floor under a point light, its vertices shifted by d along x in object space and
    pulled back by translate(-d) (d = 0: the unshifted mesh, no extra transform).  group: the teapot is the one child
    of a kd-tree of shapes."""
    def make():
        tris = scenes.teapot_triangles().copy()
        tris[:, 0:9:3] += d
        mesh = api.Mesh(tris)
        shape = (mesh.translate(api.vec3(-d, 0.0, 0.0)) if d else mesh).scale(api.vec3(0.5, 0.5, 0.5)).translate(api.vec3(0.0, -1.0, 0.0))
        scene = api.Scene()
        scene.add(api.Object(api.KdTree([shape]) if group else shape).material(api.Material.specular(api.hex_color(0xCC4422), 0.3)))
        scene.add(api.Object(api.plane(api.vec3(0, 1, 0), -1.0)).material(api.Material.diffuse(api.hex_color(0xAAAAAA))))
        scene.add(api.Light.Ambient(api.vec3(0.02, 0.02, 0.02)))
        scene.add(api.Light.Point(api.vec3(60.0, 60.0, 60.0), api.vec3(0.0, 5.0, 5.0)))
        return scene, api.Camera.default()
    return make


def _quad_plane_at(d: float):
    """A diffuse floor quad (two triangles, one leaf) whose vertices sit at d along x and z in object space, and a back
    wall plane(n, -2 + d) translated back by -d n; a red ball and a point light: the packed primitive table's mesh and
    plane records with large object-space coordinates."""
    def make():
        v = [api.vec3(-3 + d, -1, -3 + d), api.vec3(-3 + d, -1, 3 + d), api.vec3(3 + d, -1, 3 + d), api.vec3(3 + d, -1, -3 + d)]
        quad = api.polygon(v)
        scene = api.Scene()
        scene.add(api.Object(quad.translate(api.vec3(-d, 0.0, -d)) if d else quad).material(api.Material.diffuse(api.hex_color(0xAAAAAA))))
        wall = api.plane(api.vec3(0, 0, 1), -2.0 + d)
        scene.add(api.Object(wall.translate(api.vec3(0, 0, -d)) if d else wall).material(api.Material.diffuse(api.hex_color(0x88AACC))))
        scene.add(api.Object(api.sphere().scale(api.vec3(0.7, 0.7, 0.7)).translate(api.vec3(0.3, -0.3, 0.0)))
                  .material(api.Material.specular(api.hex_color(0xCC3333), 0.2)))
        scene.add(api.Light.Point(api.vec3(40.0, 40.0, 40.0), api.vec3(-2.0, 4.0, 4.0)))
        return scene, api.Camera.look_at(api.vec3(0, 1.5, 6), api.vec3(0, -0.3, 0), api.vec3(0, 1, 0), 0.8)
    return make


def _far_instance(shape: str, far: float):
    """A teapot or a sphere of size ~1e-2 at the origin on a floor, seen from `far` through a field of view narrowed to
    match: object-space ray origins lie 1e4 - 1e5 extents from the object."""
    def make():
        k = 1e-2
        if shape == "teapot":
            obj = api.Mesh(scenes.teapot_triangles()).scale(api.vec3(0.5 * k, 0.5 * k, 0.5 * k))
        else:
            obj = api.sphere().scale(api.vec3(0.8 * k, 0.8 * k, 0.8 * k))
        scene = api.Scene()
        scene.add(api.Object(obj).material(api.Material.specular(api.hex_color(0x3366CC), 0.2)))
        scene.add(api.Object(api.plane(api.vec3(0, 1, 0), -0.8 * k)).material(api.Material.diffuse(api.hex_color(0xAAAAAA))))
        scene.add(api.Light.Point(api.vec3(40.0, 40.0, 40.0) * k * k, api.vec3(-2.0, 4.0, 4.0) * k))
        return scene, api.Camera.look_at(api.vec3(0, 0.3 * far, far), api.vec3(0, 0, 0), api.vec3(0, 1, 0), 3.0 * k / far)
    return make


def _scaled(make, s):
    return make if s == 1.0 else moved(make, np.diag([s, s, s, 1.0]), s)


_TEAPOT = dict(w=32, h=32, spp=16, max_bounces=3)
_SMALL = dict(w=32, h=32, spp=16)
_D = (("1e2", 1e2), ("1e3", 1e3), ("1e4", 1e4))
# off-center teapot: (floor, slack below the base's floor) per shift; 1e4 is the measured limit (test_hostemu_placement.py)
_OFF = {"1e2": (0.999, 0.0), "1e3": (0.998, 0.0), "1e4": (0.982, 0.014)}


def _teapots(prefix, accel, feat, group, shifts, **kw):
    out = {prefix + "_0": Case(_teapot_at(0.0, group), **_TEAPOT, accel=accel, feat=feat, floor=0.999, gpu_floor=0.998, **kw)}
    for t, d in shifts:
        fl, slack = _OFF[t]
        out["%s_%s" % (prefix, t)] = Case(_teapot_at(d, group), **_TEAPOT, accel=accel, feat=feat, floor=fl, gpu_floor=fl - 0.002,
                                          base=prefix + "_0", base_slack=slack, **kw)
    return out


def _far(shp, t, far, s, floor, bias):
    return Case(_scaled(_far_instance(shp, far), s), **_SMALL, max_bounces=3, accel=(B if shp == "teapot" else A),
                feat=(F_TREE | F_BVH if shp == "teapot" else F_FLAT | F_SMALL), floor=floor, gpu_floor=floor - 0.02, bias=bias,
                base="" if s != 1.0 else "far_%s_%s_x100" % (shp, t), degrades=True)


PLACEMENTS: Dict[str, Case] = {
    # name: Case(scene, width, height, spp, max_bounces, accel, FEAT, floor, gpu_floor, ..., base=)
    # off-center meshes: the world geometry of the *_0 case, vertices at 1e2 .. 1e4 in object space
    **_teapots("teapot_kd", K, F_TREE, False, _D, wavefront=True),
    **_teapots("teapot_bvh", B, F_TREE | F_BVH, False, _D),
    **_teapots("teapot_group", K, F_EVERY, True, _D),
    **_teapots("teapot_group_bvh", B, F_EVERY | F_BVH, True, _D),
    # the packed table's one-leaf mesh and plane, coordinates at 1e4 in object space
    "quad_plane_0": Case(_quad_plane_at(0.0), **_SMALL, max_bounces=3, accel=A, feat=F_FLAT | F_SMALL, floor=0.999, gpu_floor=0.998),
    "quad_plane_1e4": Case(_quad_plane_at(1e4), **_SMALL, max_bounces=3, accel=A, feat=F_FLAT | F_SMALL, floor=0.976, gpu_floor=0.974,
                           bias=4e-5, base="quad_plane_0", base_slack=0.02),
    # uniform scale, camera included (point lights x s^2); at s = 1e3 the oracle's own image moves (F64_FLOOR)
    "cornell_1": Case(_cfg(scenes.cornell_scene), **_SMALL, max_bounces=6, accel=A, feat=F_FLAT, floor=0.982, gpu_floor=0.980),
    "cornell_s1e-3": Case(_scaled(_cfg(scenes.cornell_scene), 1e-3), **_SMALL, max_bounces=6, accel=A, feat=F_FLAT, floor=0.998,
                          gpu_floor=0.996, base="cornell_1"),
    "cornell_s1e3": Case(_scaled(_cfg(scenes.cornell_scene), 1e3), **_SMALL, max_bounces=6, accel=A, feat=F_FLAT, floor=0.775,
                         gpu_floor=0.765, base="cornell_1", degrades=True),
    "glass_1": Case(_cfg(lambda: scenes.glass_scene(64, 32)), **_SMALL, max_bounces=12, accel=A, feat=F_TRANSP | F_HDRI | F_SMALL,
                    floor=0.974, gpu_floor=0.972),
    "glass_s1e-3": Case(_scaled(_cfg(lambda: scenes.glass_scene(64, 32)), 1e-3), **_SMALL, max_bounces=12, accel=A,
                        feat=F_TRANSP | F_HDRI | F_SMALL, floor=0.974, gpu_floor=0.972, base="glass_1"),
    "glass_s1e3": Case(_scaled(_cfg(lambda: scenes.glass_scene(64, 32)), 1e3), **_SMALL, max_bounces=12, accel=A,
                       feat=F_TRANSP | F_HDRI | F_SMALL, floor=0.889, gpu_floor=0.88, base="glass_1", degrades=True),
    # a small instance (1e-2) seen from 1e2 and 1e3 world units; its base is the same view scaled by 1e2 (the instance of
    # size ~1 seen from 1e4 and 1e5), which puts the object-space origins as far out but moves the absolute thresholds
    "far_teapot_1e2": _far("teapot", "1e2", 1e2, 1.0, 0.821, 1e-4),
    "far_teapot_1e2_x100": _far("teapot", "1e2", 1e2, 1e2, 0.785, 1e-4),
    "far_teapot_1e3": _far("teapot", "1e3", 1e3, 1.0, 0.341, 3e-4),
    "far_teapot_1e3_x100": _far("teapot", "1e3", 1e3, 1e2, 0.370, 3e-4),
    "far_sphere_1e2": _far("sphere", "1e2", 1e2, 1.0, 0.822, 1e-4),
    "far_sphere_1e2_x100": _far("sphere", "1e2", 1e2, 1e2, 0.824, 1e-4),
    "far_sphere_1e3": _far("sphere", "1e3", 1e3, 1.0, 0.294, 3e-4),
    "far_sphere_1e3_x100": _far("sphere", "1e3", 1e3, 1e2, 0.341, 3e-4),
    # far from the world origin: the f32 offset is 32 ulp of 1e4 there, 0.03 units, and agreement drops by design
    "cornell_far": Case(moved(_cfg(scenes.cornell_scene), _translation((1e4, 0.0, 0.0))), **_SMALL, max_bounces=6, accel=A,
                        feat=F_FLAT, floor=0.921, gpu_floor=0.91, bias=2e-5, base="cornell_1", degrades=True),
}
