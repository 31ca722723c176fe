"""GPU parity tests (-m gpu) for SURVEY 8f row N4: kd-trees over whole shapes (two-level instancing) and
MonomialSurface, through the C ABI, against the CPU oracle on the same inputs and random streams.
Tolerances are those stated at the top of tests/test_gpu_parity.py; what differs is noted inline."""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import util
from tests.test_gpu_parity import F32, F64, _gpu_render, _oracle_render
from tests.test_hostemu import scene_rays

pytestmark = pytest.mark.gpu

# name: (w, h, spp, max_bounces).  The fractal examples render with max_bounces 0 (their three lights do the
# work); one bounce is added here so the kd-tree of shapes is also entered by scattered rays.
SMALL = {
    "fractal_spheres": (96, 72, 16, 1),
    "fractal_teapots": (96, 72, 8, 1),
    "monomial_glass": (96, 72, 32, 1),
    "mixed": (80, 60, 16, 2),
}


@pytest.fixture(scope="module")
def cfgs(gpu_ok):
    cache = {}

    def get(name):
        if name not in cache:
            if name == "mixed":
                scene, rays, _ = scene_rays("mixed")
                camera = api.Camera.look_at(api.vec3(3.0, 6.0, 14.0), api.vec3(0.0, 1.0, 0.0), api.vec3(0.0, 1.0, 0.0), 0.9)
                cfg = scenes.Config("mixed", scene, camera, 80, 60, 16, 2)
            else:
                cfg = {"fractal_spheres": lambda: scenes.fractal_spheres_scene(5),
                       "fractal_teapots": lambda: scenes.fractal_teapots_scene(4),
                       "monomial_glass": lambda: scenes.monomial_glass_scene(256, 128)}[name]()
                rays = None
            flat = api.FlatScene(cfg.scene)
            cache[name] = (cfg, flat, api.DeviceScene(flat), rays)
        return cache[name]

    yield get
    for _, _, ds, _ in cache.values():
        ds.close()


@pytest.mark.parametrize("name", sorted(SMALL))
def test_closest_hit_parity(orc, cfgs, name):
    cfg, flat, ds, rays = cfgs(name)
    osc = orc.OracleScene(flat)
    rng = np.random.default_rng(21)
    if rays is None:
        rays = np.concatenate([util.camera_rays(cfg.camera, 60000, rng, spread=0.35),
                               util.interior_rays([-2.5, -2.5, -2.5], [2.5, 2.5, 2.5], 40000, rng)])
    t0, o0, n0, s0 = osc.closest_hit(rays)
    assert (o0 >= 0).mean() > 0.3
    # f64 gate: same trees, same cells, same t_min handed to every child -> the reference's hit, bit for bit
    t1, o1, n1, s1 = ds.closest_hit(rays, precision=F64, want_stats=True)
    assert (o1 == o0).all()
    np.testing.assert_array_equal(t1, t0)
    np.testing.assert_allclose(n1, n0, atol=1e-15)
    assert abs(s1["node_visits"] - s0["node_visits"]) <= 0.01 * max(s0["node_visits"], 1)
    assert abs(s1["tri_tests"] - s0["tri_tests"]) <= 0.01 * max(s0["tri_tests"], 1)
    # f32 product path
    t2, o2, n2, _ = ds.closest_hit(rays, precision=F32, want_stats=True)
    agree = o2 == o0
    with np.errstate(invalid="ignore"):  # inf - inf on rays that miss in both
        tie = (o2 >= 0) & (o0 >= 0) & (np.abs(t2 - t0) <= 1e-5 * np.abs(t0))
    assert (agree | tie).mean() >= 0.999, (agree | tie).mean()
    assert agree.mean() >= 0.995
    hit = agree & (o0 >= 0)
    rel = np.abs(t2[hit] - t0[hit]) / np.abs(t0[hit])
    q = np.quantile(rel, [0.5, 0.99, 0.999])
    # MonomialSurface is found by bisection on a quartic: a grazing ray's root is worse conditioned than a
    # triangle's, hence 1e-3 on the last per mille
    assert q[0] <= 3e-7 and q[1] <= 2e-5 and q[2] <= 1e-3, q
    assert np.quantile(np.abs(n2[hit] - n0[hit]).max(axis=1), 0.99) <= 2e-3


@pytest.mark.parametrize("name", sorted(SMALL))
def test_render_parity_same_stream(orc, cfgs, name):
    cfg, flat, ds, _ = cfgs(name)
    w, h, spp, mb = SMALL[name]
    ref, st0 = _oracle_render(orc, cfg, flat, w, h, spp, mb, 1)
    ref2, _ = _oracle_render(orc, cfg, flat, w, h, spp, mb, 2)
    cl = lambda a: np.clip(a, 0.0, 1.0)
    noise = util.rmse(cl(ref), cl(ref2))
    assert noise > 0 and cl(ref).mean() > 0.02
    g64, st64 = _gpu_render(cfg, ds, w, h, spp, mb, 1, F64, stats=1)
    assert st64["engine"] == capi.ENGINE_MEGAKERNEL
    rel = np.abs(g64 - ref) / np.maximum(np.abs(ref), 1e-6)
    assert (rel.max(axis=1) < 1e-9).mean() >= 0.98
    assert abs(st64["segments"] - st0["segments"]) <= 2e-3 * st0["segments"]
    assert abs(st64["rays"] - st0["rays"]) <= 2e-3 * st0["rays"]
    # (node visits are not compared here: shadow rays are any-hit queries on the device, full closest-hit
    # queries in the reference -- same answer, fewer nodes; test_closest_hit_parity compares the counters)
    assert util.rmse(cl(g64), cl(ref)) <= 0.05 * noise
    g32, st32 = _gpu_render(cfg, ds, w, h, spp, mb, 1, F32)
    assert np.isfinite(g32).all()
    assert util.rmse(cl(g32), cl(ref)) <= 0.25 * noise, (util.rmse(cl(g32), cl(ref)), noise)
    assert abs(cl(g32).mean() - cl(ref).mean()) <= 5e-3 * cl(ref).mean()
    assert 0.85 * st0["segments"] <= st32["segments"] <= 1.001 * st0["segments"]
    g32b, _ = _gpu_render(cfg, ds, w, h, spp, mb, 2, F32)
    assert util.rmse(cl(g32b), cl(ref)) <= 1.25 * noise


def test_stats_kernel_and_plain_kernel_agree(cfgs):
    cfg, flat, ds, _ = cfgs("fractal_teapots")
    w, h, spp, mb = SMALL["fractal_teapots"]
    a, _ = _gpu_render(cfg, ds, w, h, spp, mb, 3, F32, stats=0)
    b, st = _gpu_render(cfg, ds, w, h, spp, mb, 3, F32, stats=1)
    relab = np.abs(b - a) / np.maximum(np.abs(a), 1e-4)   # two instantiations of the same code: FMA contraction may differ
    assert np.quantile(relab.max(axis=1), 0.999) < 1e-5
    # the group's kd-tree over the instances counts as kd nodes; the instances' triangles are reached through the BVH
    assert st["node_visits"] > 0 and st["bvh_tri_tests"] > 0 and st["bvh_node_visits"] > 0 and st["object_tests"] > st["rays"]
    c, st2 = _gpu_render(cfg, ds, w, h, spp, mb, 3, F32, stats=2)   # the reference-shaped trees all the way down
    assert st2["tri_tests"] > st["bvh_tri_tests"] and st2["bvh_node_visits"] == 0
    rel = np.abs(c - a) / np.maximum(np.abs(a), 1e-4)
    assert np.quantile(rel.max(axis=1), 0.99) < 1e-4


@pytest.mark.parametrize("precision", [F32, F64])
def test_shards_sum_to_the_full_image_bit_exact(cfgs, precision):
    cfg, flat, ds, _ = cfgs("mixed")
    w, h, spp, mb = SMALL["mixed"]
    full, _ = _gpu_render(cfg, ds, w, h, spp, mb, 5, precision)
    parts = [_gpu_render(cfg, ds, w, h, spp, mb, 5, precision, shard=(i, 3))[0] for i in range(3)]
    np.testing.assert_array_equal(parts[0] + parts[1] + parts[2], full)


def test_wavefront_request_falls_back_to_the_megakernel(cfgs):
    """The wavefront engine's trace kernel only knows triangle kd-trees; a scene with a kd-tree of shapes or
    a MonomialSurface is always rendered by the megakernel, whatever `engine` asks for."""
    cfg, flat, ds, _ = cfgs("fractal_spheres")
    w, h, spp, mb = SMALL["fractal_spheres"]
    r = api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).seed(1).engine(capi.ENGINE_WAVEFRONT)
    p = r.params(spp, collect_stats=1)
    cam = cfg.camera.to_c()
    out = np.empty((w * h, 3))
    st = capi.Stats()
    capi.check(capi.lib().rptb_render_samples(ds.handle, C.byref(cam), C.byref(p), out.ctypes.data_as(capi.c_double_p),
                                              C.byref(st)), "rptb_render_samples")
    assert st.engine == capi.ENGINE_MEGAKERNEL
    ref, _ = _gpu_render(cfg, ds, w, h, spp, mb, 1, F32, stats=1)
    np.testing.assert_array_equal(out, ref)


def test_full_size_fractal_teapots_example(cfgs):
    """examples/fractal_teapots.rs at its own size (800x600, 1 spp, max_bounces 0) with all five levels:
    781 instances of one 2 256-triangle kd-tree.  Properties only (the oracle needs minutes for this)."""
    cfg = scenes.fractal_teapots_scene(5)
    flat = api.FlatScene(cfg.scene)
    assert [int(flat.groups[i].nchildren) for i in range(5)] == [1, 6, 30, 150, 750] and flat.desc.nmeshes == 1
    with api.DeviceScene(flat) as ds:
        assert ds.device_bytes() < 4 << 20                      # instancing: one teapot on the device, not 937
        img, st = _gpu_render(cfg, ds, cfg.width, cfg.height, 4, 0, 1, F32, stats=1)
        img2, _ = _gpu_render(cfg, ds, cfg.width, cfg.height, 4, 0, 1, F32)
        img3, _ = _gpu_render(cfg, ds, cfg.width, cfg.height, 4, 0, 1, F32)
    np.testing.assert_array_equal(img2, img3)                   # deterministic
    rel = np.abs(img - img2) / np.maximum(np.abs(img2), 1e-4)   # the counting instantiation: same code, FMA contraction may differ
    assert np.quantile(rel.max(axis=1), 0.999) < 1e-4
    assert np.isfinite(img).all() and (img.max(axis=1) > 0).mean() > 0.95
    assert st["segments"] == cfg.width * cfg.height * 4 and st["mesh_hits"] > 0.1 * st["segments"]


def test_cpp_host_mirror_builds_the_same_kd_trees_of_shapes(gpu_ok, tmp_path):
    """examples/fractal_spheres.cpp (include/rpt.hpp: rpt::KdTree over transformed spheres) against the Python
    host on the same scene, size and seed: byte-identical image."""
    import os
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "fractal_spheres_cpp")
    libdir = os.path.join(root, "rpt_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-o", exe, os.path.join(root, "examples", "fractal_spheres.cpp"),
                           "-L" + libdir, "-lrpt_b200", "-Wl,-rpath," + libdir])
    ppm = str(tmp_path / "out.ppm")
    out = subprocess.run([exe, ppm, "small"], capture_output=True, text=True, check=True).stdout
    assert "Level 4: 750 spheres" in out and "rendered 96x72" in out
    data = open(ppm, "rb").read().split(b"\n255\n", 1)[1]
    img_cpp = np.frombuffer(data, np.uint8).reshape(72, 96, 3)
    cfg = scenes.fractal_spheres_scene(5)
    r = api.Renderer(cfg.scene, cfg.camera).width(96).height(72).seed(1)
    img_py = r.render()
    r.close()
    np.testing.assert_array_equal(img_cpp, img_py)


@pytest.mark.parametrize("name", ["fractal_spheres", "fractal_teapots", "monomial_glass"])
def test_gpu_matches_committed_golden(gpu_ok, name):
    """The f64 gate reproduces the committed oracle fixtures of the row-N4 scenes (tests/golden,
    tools/make_golden.py) -- this test needs no oracle on the GPU machine."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", f"{name}_render.npz"))
    cfg = util.golden_config(name)
    with api.DeviceScene(api.FlatScene(cfg.scene)) as ds:
        img, st = _gpu_render(cfg, ds, int(g["width"]), int(g["height"]), int(g["spp"]), int(g["max_bounces"]), int(g["seed"]), F64)
        img32, _ = _gpu_render(cfg, ds, int(g["width"]), int(g["height"]), int(g["spp"]), int(g["max_bounces"]), int(g["seed"]), F32)
    rel = np.abs(img - g["image"]) / np.maximum(np.abs(g["image"]), 1e-6)
    assert (rel.max(axis=1) < 1e-9).mean() >= 0.98
    assert abs(st["segments"] - int(g["segments"])) <= 2e-3 * int(g["segments"])
    cl = lambda a: np.clip(a, 0.0, 1.0)
    assert abs(cl(img32).mean() - cl(g["image"]).mean()) <= 1e-2 * cl(g["image"]).mean()
