"""The device-resident Buffer (rptb_buffer) against the host Buffer on the GPU: the same sums bit for bit, the same
image bytes, the same variance to rounding, for any split of the samples and any device count."""
import ctypes as C
import math

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64


def _renderer(cfg, w, h, mb, prec=F32, radius=1, seed=3, accel=capi.ACCEL_AUTO, engine=capi.ENGINE_AUTO, device=0):
    return (api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).seed(seed).precision(prec)
            .filter(api.Filter.Box(radius)).accel(accel).engine(engine).device(device))


def _both(make, splits):
    """The same renders (same seed, same first_sample sequence) into a host Buffer and a DeviceBuffer."""
    rh, rd = make(), make()
    host = api.Buffer(rh._width, rh._height, rh._filter)
    dev = rd.device_buffer()
    for n in splits:
        rh.sample(n, host)
        rd.sample(n, dev, want_stats=False)
    return rh, rd, host, dev


def _check_same(host, dev):
    assert dev.entries == len(host.batches)
    assert np.array_equal(dev.sums(), np.sum(host.batches, axis=0))
    np.testing.assert_array_equal(dev.image(), host.image())
    np.testing.assert_allclose(dev.variance(), host.variance(), rtol=1e-12)


CASES = {
    # name: (config, w, h, max_bounces, precision, radius, splits, extra renderer settings)
    "sphere_f32": (scenes.sphere_scene, 64, 40, 2, F32, 1, [4, 4, 2], {}),
    "sphere_f64": (scenes.sphere_scene, 48, 32, 2, F64, 0, [1] * 12, {}),
    "cornell_f32": (scenes.cornell_scene, 48, 48, 3, F32, 3, [4, 4, 2], {}),
    "cornell_f64": (scenes.cornell_scene, 32, 32, 3, F64, 1, [4, 4, 2], {}),
    "glass": (lambda: scenes.glass_scene(256, 128), 64, 40, 4, F32, 1, [4, 4, 2], {}),
    "teapot_bvh": (scenes.teapot_scene, 64, 40, 1, F32, 1, [1] * 12, {"accel": capi.ACCEL_BVH}),
    "teapot_kdtree_wavefront": (scenes.teapot_scene, 64, 40, 2, F32, 1, [4, 4, 2],
                                {"accel": capi.ACCEL_KDTREE, "engine": capi.ENGINE_WAVEFRONT}),
    "ragged_203x117": (scenes.sphere_scene, 203, 117, 2, F32, 3, [4, 4, 2], {}),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_buffer_is_the_host_buffer(gpu_ok, name):
    make_cfg, w, h, mb, prec, radius, splits, extra = CASES[name]
    cfg = make_cfg()
    rh, rd, host, dev = _both(lambda: _renderer(cfg, w, h, mb, prec, radius, **extra), splits)
    if "engine" in extra:
        rd.sample(1, dev)  # the schedule asked for is the one that rendered
        rh.sample(1, host)
        assert rd.last_stats["engine"] == capi.ENGINE_WAVEFRONT
    _check_same(host, dev)
    dev.close()
    rh.close()
    rd.close()


def test_one_entry_is_nan_variance_and_none_is_an_error(gpu_ok):
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 32, 16, 1)
    dev = r.device_buffer()
    with pytest.raises(capi.RptbError, match="Pixel found with no samples"):
        dev.image()
    assert not dev.sums().any()
    r.sample(2, dev)
    assert math.isnan(dev.variance())
    host = api.Buffer(32, 16, r._filter)
    r2 = _renderer(cfg, 32, 16, 1)
    r2.sample(2, host)
    np.testing.assert_array_equal(dev.image(), host.image())
    dev.close()
    r.close()
    r2.close()


def test_host_entries_match_the_oracle(orc, gpu_ok):
    """add_samples of host entries: the tolerances of test_film_resolve_matches_oracle_bytes and
    test_film_variance_matches_oracle."""
    rng = np.random.default_rng(31)
    w, h, nb = 70, 41, 5
    batches = rng.uniform(0, 2, (nb, w * h, 3))
    ds = api.DeviceScene(scenes.sphere_scene().scene)
    for radius in (0, 1, 3):
        dev = api.DeviceBuffer(ds, w, h, api.Filter.Box(radius))
        for b in batches:
            dev.add_samples(b)
        assert np.array_equal(dev.sums(), np.sum(batches, axis=0))
        out = dev.image()
        ref = orc.film_resolve(np.sum(batches, axis=0), nb, w, h, radius)
        assert (np.abs(out.astype(int) - ref.astype(int)) <= 1).all()
        assert (out == ref).mean() > 0.999
        np.testing.assert_allclose(dev.variance(), orc.variance(batches), rtol=1e-12)
        dev.close()
    ds.close()


def test_host_and_device_entries_mix(gpu_ok):
    cfg = scenes.sphere_scene()
    rh, rd, host, dev = _both(lambda: _renderer(cfg, 40, 24, 2), [3])
    extra = np.random.default_rng(5).uniform(0, 1, (40 * 24, 3))
    host.add_samples(extra)
    dev.add_samples(extra)
    rh.sample(2, host)
    rd.sample(2, dev, want_stats=False)
    _check_same(host, dev)
    dev.close()
    rh.close()
    rd.close()


def test_iterative_render_with_a_device_buffer(gpu_ok):
    cfg = scenes.sphere_scene()
    make = lambda: _renderer(cfg, 64, 36, 2).num_samples(10)  # noqa: E731
    host_calls, dev_calls = [], []
    make().iterative_render(4, lambda it, buf: host_calls.append((it, buf.image(), buf.variance())))
    r = make()
    dev = r.device_buffer()
    r.iterative_render(4, lambda it, buf: dev_calls.append((it, buf.image(), buf.variance())), buffer=dev)
    assert [c[0] for c in dev_calls] == [4, 8, 10] == [c[0] for c in host_calls]
    for (_, ih, vh), (_, idv, vd) in zip(host_calls, dev_calls):
        np.testing.assert_array_equal(idv, ih)
        if math.isnan(vh):
            assert math.isnan(vd)
        else:
            np.testing.assert_allclose(vd, vh, rtol=1e-12)
    assert dev.entries == 3
    dev.close()
    r.close()


def test_any_device_count_gives_the_same_bits(gpu_ok):
    cfg = scenes.cornell_scene()
    w, h = 203, 117
    ref = None
    for n in range(1, min(gpu_ok, 8) + 1):
        r = _renderer(cfg, w, h, 3, device=list(range(n)))
        dev = r.device_buffer()
        for k in (4, 4, 2):
            r.sample(k, dev, want_stats=False)
        got = (dev.sums(), dev.image(), dev.variance())
        assert dev.variance() == got[2]  # the reduction has a fixed order
        if ref is None:
            ref = got
        else:
            assert np.array_equal(got[0], ref[0])
            np.testing.assert_array_equal(got[1], ref[1])
            assert got[2] == ref[2], n
        dev.close()
        r.close()


def test_buffer_outlives_its_scene(gpu_ok):
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 48, 32, 2)
    dev = r.device_buffer()
    r.sample(4, dev, want_stats=False)  # still running when the scene goes
    r.close()
    img, var = dev.image(), dev.variance()
    r2 = _renderer(cfg, 48, 32, 2)
    host = api.Buffer(48, 32, r2._filter)
    r2.sample(4, host)
    np.testing.assert_array_equal(img, host.image())
    assert math.isnan(var)
    dev.close()
    r2.close()


def test_buffers_give_their_device_memory_back(gpu_ok):
    """50 buffers of 1920x1080 (~150 MB each) keep less than 32 MB of device memory between them.  The free memory
    cudaMemGetInfo reports is the whole device's, which other processes share: one that starts on the GPU while this
    runs takes ~0.5 GB for its CUDA context in a single step.  A buffer that keeps memory does so at every step, so the
    free memory is read after each buffer, and the check is on the 50 smallest of 51 steps."""
    torch = pytest.importorskip("torch")
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 1920, 1080, 0)
    warm = r.device_buffer()
    r.sample(1, warm, want_stats=False)
    warm.image()
    warm.close()  # the scene's own scratch for this size now exists
    torch.cuda.synchronize()
    free = [torch.cuda.mem_get_info(0)[0]]
    for _ in range(51):
        b = r.device_buffer()
        r.sample(1, b, want_stats=False)
        b.image()
        b.close()
        free.append(torch.cuda.mem_get_info(0)[0])
    steps = -np.diff(np.array(free, dtype=np.int64))  # device memory taken over each buffer's life
    kept = int(np.sort(steps)[:-1].sum())
    assert kept <= (32 << 20), (kept / 2**20, (steps / 2**20).tolist())  # one buffer at this size holds ~150 MB
    r.close()


def test_error_statuses(gpu_ok):
    lib = capi.lib()
    cfg = scenes.sphere_scene()
    r = _renderer(cfg, 32, 16, 1)
    ds = r.device_scene()
    dev = r.device_buffer()
    cam = cfg.camera.to_c()
    p = r.params(1)
    wrong = r.params(1)
    wrong.width = 33
    assert lib.rptb_sample_into(ds.handle, C.byref(cam), C.byref(wrong), dev.handle, None) == capi.ERR_BAD_ARG
    sharded = r.params(1, shard_index=0, shard_count=2)
    assert lib.rptb_sample_into(ds.handle, C.byref(cam), C.byref(sharded), dev.handle, None) == capi.ERR_UNSUPPORTED
    assert lib.rptb_sample_into(None, C.byref(cam), C.byref(p), dev.handle, None) == capi.ERR_BAD_ARG
    assert lib.rptb_sample_into(ds.handle, None, C.byref(p), dev.handle, None) == capi.ERR_BAD_ARG
    assert lib.rptb_sample_into(ds.handle, C.byref(cam), None, dev.handle, None) == capi.ERR_BAD_ARG
    assert lib.rptb_sample_into(ds.handle, C.byref(cam), C.byref(p), None, None) == capi.ERR_BAD_ARG
    assert lib.rptb_buffer_image(dev.handle, None) == capi.ERR_BAD_ARG
    assert lib.rptb_buffer_variance(dev.handle, None) == capi.ERR_BAD_ARG
    assert lib.rptb_buffer_sums(dev.handle, None, None) == capi.ERR_BAD_ARG
    assert lib.rptb_buffer_add_samples(dev.handle, None) == capi.ERR_BAD_ARG
    h = C.c_void_p()
    assert lib.rptb_buffer_create(ds.handle, 0, 16, 0, C.byref(h)) == capi.ERR_BAD_ARG and not h
    assert lib.rptb_buffer_create(ds.handle, 32, 16, 0, None) == capi.ERR_BAD_ARG
    assert dev.entries == 0  # nothing was added by the refused calls
    assert lib.rptb_sample_into(ds.handle, C.byref(cam), C.byref(p), dev.handle, None) == capi.OK
    dev.entries += 1
    assert dev.sums().any()
    dev.close()
    r.close()


def test_buffer_refuses_a_scene_on_other_devices(gpu_ok):
    if gpu_ok < 2:
        pytest.skip("needs two GPUs for two different device lists")
    lib = capi.lib()
    cfg = scenes.sphere_scene()
    r0 = _renderer(cfg, 32, 16, 1, device=0)
    r1 = _renderer(cfg, 32, 16, 1, device=1)
    r01 = _renderer(cfg, 32, 16, 1, device=[0, 1])
    dev = r0.device_buffer()
    cam, p = cfg.camera.to_c(), r0.params(1)
    for other in (r1, r01):
        assert lib.rptb_sample_into(other.device_scene().handle, C.byref(cam), C.byref(p), dev.handle, None) == capi.ERR_BAD_ARG
    dev.close()
    for r in (r0, r1, r01):
        r.close()
