"""The fan-out of Renderer::sample (src/renderer.rs:117-129: rayon over rows) behind the C ABI: a handle created with
rptb_scene_create_multi renders through the SAME rptb_render_samples call on every listed GPU, each owning the pixel
tiles t with t % ndevices == i -- bit-identical images for any device count.  Also here: the point-wise
Light::illuminate entry point (src/light.rs:23-47 + Shape::sample) and the ordering of calls that leave work on a
caller's stream."""
import ctypes as C
import math

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from rpt_b200.api import Light, Material, Object, Scene, cube, hex_color, plane, sphere, vec3
from tests import util

pytestmark = pytest.mark.gpu
F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64


def _render(ds, cfg, w, h, spp, mb, seed, precision=F32, shard=(0, 1), first_sample=0, stats=0):
    r = api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).seed(seed).precision(precision)
    p = r.params(spp, first_sample, shard[0], shard[1], collect_stats=stats)
    cam = cfg.camera.to_c()
    out = np.full((w * h, 3), np.nan)
    st = capi.Stats()
    capi.check(capi.lib().rptb_render_samples(ds.handle, C.byref(cam), C.byref(p), out.ctypes.data_as(capi.c_double_p), C.byref(st)),
               "rptb_render_samples")
    return out, st.as_dict()


@pytest.mark.parametrize("name,w,h,spp,mb", [("cornell", 200, 136, 70, 4), ("teapot", 203, 117, 8, 0), ("glass", 160, 90, 130, 12)])
def test_multi_device_handle_is_bit_identical(gpu_ok, monkeypatch, name, w, h, spp, mb):
    """Every list of util.replica_lists (1 to 8 replicas, a repeated device being a replica of its own): same bits
    through the same call; ragged image sizes, more than one sample chunk, both precisions; counters add up."""
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")
    cfg = scenes.glass_scene(256, 128) if name == "glass" else scenes.CONFIGS[name]()
    flat = api.FlatScene(cfg.scene)
    with api.DeviceScene(flat, 0) as one:
        assert one.device_count() == 1
        ref32, st32 = _render(one, cfg, w, h, spp, mb, 7)
        ref64, st64 = _render(one, cfg, w, h, min(spp, 8), mb, 7, F64)
        assert np.isfinite(ref32).all() and ref32.mean() > 0
        # the caller's own sharding still works on top (pixels of the other shards read as zero)
        parts = [_render(one, cfg, w, h, spp, mb, 7, shard=(i, 3))[0] for i in range(3)]
        np.testing.assert_array_equal(parts[0] + parts[1] + parts[2], ref32)
        assert all((p == 0).any() for p in parts)
    tested = []
    for devices in util.replica_lists(gpu_ok):
        n = len(devices)
        with api.DeviceScene(flat, devices) as multi:
            assert multi.device_count() == n
            a, sa = _render(multi, cfg, w, h, spp, mb, 7)
            np.testing.assert_array_equal(a, ref32)
            assert sa["segments"] == st32["segments"] and sa["rays"] == st32["rays"]
            b, sb = _render(multi, cfg, w, h, min(spp, 8), mb, 7, F64)
            np.testing.assert_array_equal(b, ref64)
            assert sb["segments"] == st64["segments"]
            if n > 1:
                # outer shards of a multi-device handle: tiles t % (2 n) == shard * n + device
                q = [_render(multi, cfg, w, h, spp, mb, 7, shard=(i, 2))[0] for i in range(2)]
                np.testing.assert_array_equal(q[0] + q[1], ref32)
                out = np.empty(w * h * 3, np.float32)
                # device-resident output is per device by design
                import torch
                t = torch.empty(w * h * 3, dtype=torch.float32, device="cuda:0")
                r = api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb)
                p = r.params(spp)
                cam = cfg.camera.to_c()
                rc = capi.lib().rptb_render_samples_device(multi.handle, C.byref(cam), C.byref(p), C.c_void_p(t.data_ptr()), None, None)
                assert rc == -5  # RPTB_ERR_UNSUPPORTED
        tested.append(n)
    assert tested[0] == 1 and max(tested) == 8


def test_multi_device_create_rejects_bad_device_lists(gpu_ok):
    cfg = scenes.sphere_scene()
    flat = api.FlatScene(cfg.scene)
    h = C.c_void_p()
    lib = capi.lib()
    for devs in ([0, 0], [gpu_ok], [-1]):
        arr = (C.c_int * len(devs))(*devs)
        assert lib.rptb_scene_create_multi(C.byref(flat.desc), arr, len(devs), C.byref(h)) == -1 and not h
    assert lib.rptb_scene_create_multi(C.byref(flat.desc), None, 0, C.byref(h)) == -1
    assert lib.rptb_scene_create_multi(C.byref(flat.desc), None, 1, C.byref(h)) == 0  # NULL list = devices 0..n-1
    assert lib.rptb_scene_device_count(h) == 1
    lib.rptb_scene_destroy(h)


def _light_scene():
    """Every Light kind and every sampled shape: point, directional, ambient, sphere / cube / mesh object lights,
    bare and transformed."""
    scene = Scene()
    scene.add(Object(plane(vec3(0.0, 1.0, 0.0), -1.0)).material(Material.diffuse(hex_color(0xAAAAAA))))
    scene.add(Light.Point(vec3(10.0, 20.0, 30.0), vec3(1.0, 5.0, -2.0)))
    scene.add(Light.Ambient(vec3(0.1, 0.2, 0.3)))
    scene.add(Light.Directional(vec3(0.5, 0.6, 0.7), vec3(0.3, -1.0, 0.2)))
    scene.add(Light.Object(Object(sphere()).material(Material.light(hex_color(0xFFFFFF), 3.0))))
    scene.add(Light.Object(Object(sphere().scale(vec3(2.0, 0.5, 1.5)).rotate_y(0.7).translate(vec3(0.0, 6.0, 1.0)))
                           .material(Material.light(hex_color(0xFFAA88), 40.0))))
    scene.add(Light.Object(Object(cube().scale(vec3(1.0, 2.0, 0.5)).rotate_y(-0.4).translate(vec3(-3.0, 4.0, 0.0)))
                           .material(Material.light(hex_color(0x88AAFF), 25.0))))
    tris = scenes.teapot_triangles()[::7]
    scene.add(Light.Object(Object(api.Mesh(tris).scale(vec3(0.5, 0.5, 0.5)).translate(vec3(2.0, 3.0, -1.0)))
                           .material(Material.light(hex_color(0xFFFFFF), 10.0))))
    return scene


def test_illuminate_pointwise_against_the_oracle(orc, gpu_ok):
    """rptb_illuminate == oracle_illuminate draw for draw (row a17/a18: Light::illuminate, Sphere / Cube / KdTree /
    Triangle / Transformed::sample): f64 to the last bits, f32 within single precision."""
    scene = _light_scene()
    flat = api.FlatScene(scene)
    osc = orc.OracleScene(flat)
    rng = np.random.default_rng(4)
    pos = rng.uniform([-4, -1, -4], [4, 3, 4], (20000, 3))
    with api.DeviceScene(flat) as ds:
        for li in range(7):
            i0, w0, d0 = osc.illuminate(li, pos, seed=9)
            i1, w1, d1 = ds.illuminate(li, pos, seed=9, precision=F64)
            np.testing.assert_allclose(i1, i0, rtol=1e-12, atol=1e-300)
            np.testing.assert_allclose(w1, w0, rtol=0, atol=1e-14)
            np.testing.assert_allclose(d1, d0, rtol=1e-14)
            i2, w2, d2 = ds.illuminate(li, pos, seed=9, precision=F32)
            assert np.isfinite(i2).all() and np.isfinite(w2).all()
            if li == 2:  # directional: infinite distance
                assert np.isinf(d2).all() and np.isinf(d0).all()
            else:
                rel_d = np.abs(d2 - d0) / np.maximum(np.abs(d0), 1e-30) if li != 1 else np.abs(d2 - d0)
                assert np.quantile(rel_d, 0.999) <= 2e-5   # (a rejection loop may take another turn in f32: a handful of draws)
            good = np.abs(w2 - w0).max(axis=1) <= 1e-4
            assert good.mean() >= 0.999
            rel_i = np.abs(i2 - i0).max(axis=1) / np.maximum(np.abs(i0).max(axis=1), 1e-12)
            assert np.quantile(rel_i[good], 0.99) <= 2e-4
        assert capi.lib().rptb_illuminate(ds.handle, 7, pos.ctypes.data_as(capi.c_double_p), 1, 0, F32,
                                          pos.ctypes.data_as(capi.c_double_p), pos.ctypes.data_as(capi.c_double_p),
                                          pos.ctypes.data_as(capi.c_double_p)) == -1
    # the reference's values for the non-random kinds, stated outright (light.rs:25-31)
    i0, w0, d0 = osc.illuminate(0, pos[:4], seed=0)
    disp = np.array([1.0, 5.0, -2.0]) - pos[:4]
    ln = np.linalg.norm(disp, axis=1)
    np.testing.assert_allclose(i0, np.array([10.0, 20.0, 30.0])[None, :] / (ln * ln)[:, None], rtol=1e-14)
    np.testing.assert_allclose(d0, ln, rtol=1e-15)
    ia, wa, da = osc.illuminate(1, pos[:4], seed=0)
    assert (ia == np.array([0.1, 0.2, 0.3])).all() and (wa == 0).all() and (da == 0).all()
    osc.close()


def test_renders_left_on_caller_streams_do_not_share_scratch(gpu_ok):
    """rptb_render_samples_device on a caller's stream returns while the kernels still run; the next call -- on another
    stream, or a host render through the library's own stream, or one that has to regrow the chunk scratch -- must
    not touch that render's scratch before it has finished (ADVICE r1: per-scene scratch shared by every call)."""
    import torch

    cfg = scenes.cornell_scene()
    w, h, mb = 256, 256, 6
    r = api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).seed(3)
    cam = cfg.camera.to_c()
    dev = torch.device("cuda:0")
    with api.DeviceScene(api.FlatScene(cfg.scene)) as ds:
        def device_call(spp, first, stream, out):
            p = r.params(spp, first)
            capi.check(capi.lib().rptb_render_samples_device(ds.handle, C.byref(cam), C.byref(p), C.c_void_p(out.data_ptr()),
                                                             C.c_void_p(stream.cuda_stream), None), "rptb_render_samples_device")
        # serial references
        refs = {}
        s0 = torch.cuda.Stream(dev)
        for key, (spp, first) in {"a": (200, 0), "b": (330, 1000), "c": (130, 5000)}.items():
            out = torch.zeros(w * h * 3, dtype=torch.float32, device=dev)
            device_call(spp, first, s0, out)
            s0.synchronize()
            refs[key] = out.cpu().numpy().copy()
        # back to back on two streams, growing chunk counts (4 chunks, then 6: the scratch has to be reallocated), then a
        # host render on the library's stream while both may still be running
        s1, s2 = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        for rep in range(3):
            oa = torch.zeros(w * h * 3, dtype=torch.float32, device=dev)
            ob = torch.zeros(w * h * 3, dtype=torch.float32, device=dev)
            device_call(200, 0, s1, oa)
            device_call(330, 1000, s2, ob)
            host, _ = _render(ds, cfg, w, h, 130, mb, 3, first_sample=5000)
            s1.synchronize()
            s2.synchronize()
            np.testing.assert_array_equal(oa.cpu().numpy(), refs["a"])
            np.testing.assert_array_equal(ob.cpu().numpy(), refs["b"])
            np.testing.assert_array_equal(host.astype(np.float32).ravel(), refs["c"])
