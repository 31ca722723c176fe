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
    wavefront: bool = False        # also rendered through ENGINE_WAVEFRONT on the GPU (kd-tree scenes)


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
    "cornell": Case(_cfg(scenes.cornell_scene), 32, 32, 16, 6, A, F_FLAT, 0.982, 0.982),
    "cornell_scan": Case(_cfg(scenes.cornell_scene), 32, 32, 16, 6, A, 0, 0.982, 0.982, env=NO_FLAT),
    "sphere": Case(_cfg(scenes.sphere_scene), 32, 32, 16, 2, A, F_FLAT | F_SMALL, 0.999, 0.999),
    "sphere_scan": Case(_cfg(scenes.sphere_scene), 32, 32, 16, 2, A, F_SMALL, 0.999, 0.999, env=NO_FLAT),
    "teapot_kd": Case(_cfg(scenes.teapot_scene), 32, 32, 16, 2, K, F_TREE, 0.999, 0.999, wavefront=True),
    "teapot_bvh": Case(_cfg(scenes.teapot_scene), 32, 32, 16, 2, B, F_TREE | F_BVH, 0.999, 0.999),
    "glass": Case(_cfg(lambda: scenes.glass_scene(64, 32)), 32, 32, 16, 12, A, F_TRANSP | F_HDRI | F_SMALL, 0.974, 0.974),
    "glass_deep": Case(_glass_lit, 32, 32, 16, 40, A, F_TRANSP | F_HDRI, 0.968, 0.968, env=NO_SMALL),
    "fractal_spheres": Case(_cfg(lambda: scenes.fractal_spheres_scene(3)), 32, 32, 16, 2, A, F_EVERY, 0.997, 0.997),
    "fractal_teapots_kd": Case(_cfg(lambda: scenes.fractal_teapots_scene(3)), 32, 32, 16, 2, K, F_EVERY, 0.997, 0.997),
    "fractal_teapots_bvh": Case(_cfg(lambda: scenes.fractal_teapots_scene(3)), 32, 32, 16, 2, B, F_EVERY | F_BVH, 0.997, 0.997),
    "monomial_glass": Case(_cfg(lambda: scenes.monomial_glass_scene(64, 32)), 32, 32, 16, 3, A, F_EVERY, 0.990, 0.990),
    # the f32-only rules
    "clamp": Case(_clamp, 32, 32, 16, 6, A, F_FLAT | F_SMALL, 0.998, 0.998, ev=-1.0),
    "clamp_glass": Case(_clamp_glass, 48, 32, 24, 8, A, F_ALL, 0.9965, 0.9965),
    "lights_lens": Case(_lights, 37, 23, 20, 3, A, F_FLAT, 0.999, 0.999),
    "smooth_kd": Case(_smooth(False), 32, 32, 16, 3, K, F_TREE, 0.999, 0.999, wavefront=True),
    "smooth_glass_bvh": Case(_smooth(True), 32, 32, 16, 4, B, F_ALL | F_BVH, 0.995, 0.995),
}
