"""Reprojection into shard buffers (rptb_buffer_reproject_shard) against rptb_buffer_reproject into one whole buffer:
the shards, gathered, hold the whole buffer's pixel state and features bit for bit, their reused counts add up to the
whole call's, and two adaptive entries later the image, variance and denoised image are still the same bits -- for any
shard count, including shards that own no tile, and for a source of another size or one gathered from shards.  The
gathered buffer is a reprojected one (the exchange header carries the flag), and every refusal is checked.  The
all-gather is stood in for by torch.cat of the shards' exports on one device, as in tests/test_gpu_shard_buffer.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from rpt_b200.distributed import ShardBuffer
from tests.test_reproject import orbit

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
CRIT = api.Adaptive(0.05, 1e-3, 4)
CENTER = (0.0, 0.5, 0.0)  # above the sphere: the upper part of the view sees the environment


def _cameras(angle=0.07):
    cfg = scenes.sphere_scene()
    a = api.Camera.look_at(api.vec3(0.3, 0.6, 4.5), np.asarray(CENTER), api.vec3(0.0, 1.0, 0.0), 0.7)
    return cfg, a, orbit(a, CENTER, angle, lift=0.05)


def _renderer(cfg, cam, w, h, prec):
    return api.Renderer(cfg.scene, cam).width(w).height(h).max_bounces(2).seed(5).precision(prec)


def _gather(shards, dst, with_features=True):
    """torch.cat of every shard's export (what all_gather_into_tensor gives), imported into `dst`."""
    blocks = []
    for s in shards:
        out = torch.empty(s.block_bytes(with_features), dtype=torch.uint8, device="cuda:0")
        s.export(out, with_features)
        blocks.append(out)
    gathered = torch.cat(blocks)
    torch.cuda.synchronize()
    rc = capi.lib().rptb_buffer_import_shards(dst.handle, C.c_void_p(gathered.data_ptr()), len(shards), 1 if with_features else 0)
    assert rc == capi.OK, capi.lib().rptb_last_error()
    return dst


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


def _source(r, cam, w, h, ds):
    """A whole buffer through `cam` at w x h: three plain entries and 16 feature rays."""
    own = (r.camera, r._width, r._height)
    r.camera, r._width, r._height = cam, w, h
    r._next_sample = 0
    src = api.DeviceBuffer(ds, w, h)
    for _ in range(3):
        r.sample(4, src, want_stats=False)
    r.sample_features(16, src)
    r.camera, r._width, r._height = own
    return src


def _reprojected(r, dst, src):
    """dst given 16 feature rays through the renderer's camera, then src's history; returns the reused count."""
    r.sample_features(16, dst)
    return dst.reproject_from(src)


def _two_adaptive(r, buf):
    r._next_sample = 100
    for _ in range(2):
        r.sample(4, buf, want_stats=False, adaptive=CRIT)


def _compare(r, ds, src, n, w, h):
    whole = api.DeviceBuffer(ds, w, h)
    want = _reprojected(r, whole, src)
    shards = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
    got = [_reprojected(r, s, src) for s in shards]
    assert sum(got) == want and 0 < want, (got, want)
    assert all(s.entries == api.Reproject().max_history for s in shards)
    g = _gather(shards, api.DeviceBuffer(ds, w, h))
    for a, b in zip(g.pixel_stats(), whole.pixel_stats()):
        assert _bits(a) == _bits(b)
    for a, b in zip(g.features(), whole.features()):
        assert _bits(a) == _bits(b)
    _two_adaptive(r, whole)
    for s in shards:
        _two_adaptive(r, s)
    g2 = _gather(shards, api.DeviceBuffer(ds, w, h))
    for fn in ("pixel_stats", "image", "variance", "denoise"):
        a, b = getattr(g2, fn)(), getattr(whole, fn)()
        if fn == "pixel_stats":
            assert all(_bits(x) == _bits(y) for x, y in zip(a, b))
        else:
            assert _bits(np.float64(a) if fn == "variance" else a) == _bits(np.float64(b) if fn == "variance" else b), fn
    for b in shards + [whole, g, g2]:
        b.close()
    return want


# dst size, src size: 20x10 is 4 tiles, so shards 4.. of 5 and 8 own none; 97x61 takes a source of another size
SIZES = [((128, 96), (128, 96)), ((97, 61), (80, 70)), ((20, 10), (24, 14))]


@pytest.mark.parametrize("prec", [F32, F64])
@pytest.mark.parametrize("dsize,ssize", SIZES)
def test_shards_reproject_like_the_whole_buffer(gpu_ok, dsize, ssize, prec):
    (w, h), (sw, sh) = dsize, ssize
    cfg, a, b = _cameras()
    r = _renderer(cfg, b, w, h, prec)
    ds = r.device_scene()
    src = _source(r, a, sw, sh, ds)
    for n in (1, 2, 3, 5, 8):
        _compare(r, ds, src, n, w, h)
    src.close()
    r.close()


def test_source_gathered_from_shards(gpu_ok):
    w, h = 97, 61
    cfg, a, b = _cameras()
    r = _renderer(cfg, b, w, h, F32)
    ds = r.device_scene()
    whole_src = _source(r, a, w, h, ds)
    own = r.camera
    r.camera = a
    r._next_sample = 0
    parts = [ShardBuffer(ds, w, h, rank=i, world=3) for i in range(3)]
    for s in parts:  # the calls _source makes
        r._next_sample = 0
        for _ in range(3):
            r.sample(4, s, want_stats=False)
        r.sample_features(16, s)
    r.camera = own
    gathered_src = _gather(parts, api.DeviceBuffer(ds, w, h))
    for x, y in zip(gathered_src.pixel_stats(), whole_src.pixel_stats()):
        assert _bits(x) == _bits(y)
    whole = api.DeviceBuffer(ds, w, h)
    want = _reprojected(r, whole, whole_src)
    for n in (2, 5):
        shards = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
        assert sum(_reprojected(r, s, gathered_src) for s in shards) == want
        g = _gather(shards, api.DeviceBuffer(ds, w, h))
        for x, y in zip(g.pixel_stats(), whole.pixel_stats()):
            assert _bits(x) == _bits(y)
        for s in shards + [g]:
            s.close()
    for x in parts + [whole, whole_src, gathered_src]:
        x.close()
    r.close()


def test_the_reprojected_flag_travels(gpu_ok):
    """Disocclusions keep count 0 after the reprojection, 1 after one plain entry: the gathered buffer's denoise()
    refuses as the whole buffer's does, and a gathered buffer that was not reprojected is not flagged."""
    w, h, n = 64, 48, 3
    cfg, a, b = _cameras(angle=0.3)
    r = _renderer(cfg, b, w, h, F32)
    ds = r.device_scene()
    src = _source(r, a, w, h, ds)
    whole = api.DeviceBuffer(ds, w, h)
    reused = _reprojected(r, whole, src)
    assert 0 < reused < w * h
    shards = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
    assert sum(_reprojected(r, s, src) for s in shards) == reused
    for buf in [whole] + shards:
        r._next_sample = 50
        r.sample(2, buf, want_stats=False)
    g = _gather(shards, api.DeviceBuffer(ds, w, h))
    with pytest.raises(capi.RptbError) as want:
        whole.denoise()
    with pytest.raises(capi.RptbError) as got:
        g.denoise()
    assert str(got.value) == str(want.value)
    assert _bits(g.image()) == _bits(whole.image())
    assert np.isnan(g.variance()) and np.isnan(whole.variance())
    # blocks of a reprojected and an unreprojected shard given the same entry count, rays and cameras do not mix
    mixed = ShardBuffer(ds, w, h, rank=0, world=2)
    _reprojected(r, mixed, src)
    r.sample(2, mixed, want_stats=False)
    plain = ShardBuffer(ds, w, h, rank=1, world=2)
    r.sample_features(16, plain)
    for _ in range(api.Reproject().max_history + 1):
        r.sample(2, plain, want_stats=False)
    blocks = []
    for s in (mixed, plain):
        o = torch.empty(s.block_bytes(True), dtype=torch.uint8, device="cuda:0")
        s.export(o, True)
        blocks.append(o)
    t = torch.cat(blocks)
    torch.cuda.synchronize()
    dst = api.DeviceBuffer(ds, w, h)
    assert capi.lib().rptb_buffer_import_shards(dst.handle, C.c_void_p(t.data_ptr()), 2, 1) == capi.ERR_BAD_ARG
    assert "other calls" in capi.lib().rptb_last_error().decode()
    for x in shards + [whole, g, src, plain, mixed, dst]:
        x.close()


def _rc(dst, src, prm=None):
    c = (prm or api.Reproject()).to_c()
    n = C.c_uint64(123)
    rc = capi.lib().rptb_buffer_reproject_shard(dst.handle, src.handle, C.byref(c), C.byref(n))
    return rc, capi.lib().rptb_last_error().decode(), n.value


def test_errors(gpu_ok):
    w, h = 48, 24
    cfg, a, b = _cameras()
    r = _renderer(cfg, b, w, h, F32)
    ds = r.device_scene()
    good = _source(r, a, w, h, ds)

    def shard(features=True, entries=0, cams=None, rank=0, world=2):
        s = ShardBuffer(ds, w, h, rank=rank, world=world)
        for c in cams or [b]:
            if features:
                r.camera = c
                r.sample_features(1, s)
        r.camera = b
        for _ in range(entries):
            r.sample(1, s, want_stats=False)
        return s

    fresh = shard()
    # a shard src: gather first
    other = shard(entries=2, rank=1)
    rc = _rc(fresh, other)
    assert rc[0] == capi.ERR_UNSUPPORTED and "gather the shards" in rc[1], rc
    with pytest.raises(TypeError, match="gather"):
        fresh.reproject_from(other)
    # a whole dst
    whole = api.DeviceBuffer(ds, w, h)
    r.sample_features(1, whole)
    rc = _rc(whole, good)
    assert rc[0] == capi.ERR_BAD_ARG and "not a shard buffer" in rc[1], rc
    # dst with entries, dst without features
    rc = _rc(shard(entries=1), good)
    assert rc[0] == capi.ERR_BAD_ARG and "already holds entries" in rc[1], rc
    assert _rc(shard(features=False), good)[:2] == (capi.ERR_BAD_ARG, "dst holds no features (rptb_buffer_add_features)")
    # src without entries, src without features
    noent = api.DeviceBuffer(ds, w, h)
    r.camera = a
    r.sample_features(1, noent)
    nofeat = api.DeviceBuffer(ds, w, h)
    r.sample(1, nofeat, want_stats=False)
    r.camera = b
    assert _rc(fresh, noent)[:2] == (capi.ERR_BAD_ARG, "src holds no entries")
    assert _rc(fresh, nofeat)[:2] == (capi.ERR_BAD_ARG, "src holds no features (rptb_buffer_add_features)")
    # mixed cameras: src's entries, dst's features
    mixed_src = api.DeviceBuffer(ds, w, h)
    for c in (a, b):
        r.camera = c
        r.sample(1, mixed_src, want_stats=False)
    r.camera = a
    r.sample_features(1, mixed_src)
    r.camera = b
    rc = _rc(fresh, mixed_src)
    assert rc[0] == capi.ERR_BAD_ARG and "entries have no single camera: mixed" in rc[1], rc
    rc = _rc(shard(cams=[a, b]), good)
    assert rc[0] == capi.ERR_BAD_ARG and "dst's features have no single camera: mixed" in rc[1], rc
    # an open aperture
    focused = api.Camera(b.eye, b.direction, b.up, b.fov).focus(np.asarray(CENTER), 0.05)
    rc = _rc(shard(cams=[focused]), good)
    assert rc[0] == capi.ERR_UNSUPPORTED and "aperture" in rc[1], rc
    # the whole call still refuses shards
    c = api.Reproject().to_c()
    assert capi.lib().rptb_buffer_reproject(fresh.handle, good.handle, C.byref(c), None) == capi.ERR_UNSUPPORTED
    # nothing refused touched the shard
    assert fresh.entries == 0 and _rc(fresh, good)[0] == capi.OK
    for x in (fresh, other, whole, noent, nofeat, mixed_src, good):
        x.close()
    r.close()


def test_src_on_another_device(gpu_ok):
    if gpu_ok < 2:
        pytest.skip("needs two GPUs")
    w, h = 32, 16
    cfg, a, b = _cameras()
    r1 = _renderer(cfg, a, w, h, F32).device(1)
    src = _source(r1, a, w, h, r1.device_scene())
    r0 = _renderer(cfg, b, w, h, F32).device(0)
    dst = ShardBuffer(r0.device_scene(), w, h, rank=0, world=2)
    r0.sample_features(1, dst)
    rc = _rc(dst, src)
    assert rc[0] == capi.ERR_BAD_ARG and "device" in rc[1], rc
    for x in (src, dst, r0, r1):
        x.close()


def test_a_shard_with_no_tile(gpu_ok):
    """20x10 is 4 tiles: shard 7 of 8 owns none.  It reprojects with 0 reused, takes the reprojected state, and its
    block imports with the others'."""
    w, h, n = 20, 10, 8
    cfg, a, b = _cameras()
    r = _renderer(cfg, b, w, h, F32)
    ds = r.device_scene()
    src = _source(r, a, w, h, ds)
    whole = api.DeviceBuffer(ds, w, h)
    want = _reprojected(r, whole, src)
    shards = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
    got = [_reprojected(r, s, src) for s in shards]
    assert got[4:] == [0, 0, 0, 0] and sum(got) == want
    rc = _rc(ShardBuffer(ds, w, h, rank=7, world=n), src)
    assert rc[0] == capi.ERR_BAD_ARG and "no features" in rc[1]  # the checks run all the same
    g = _gather(shards, api.DeviceBuffer(ds, w, h))
    for x, y in zip(g.pixel_stats(), whole.pixel_stats()):
        assert _bits(x) == _bits(y)
    for x in shards + [g, whole, src]:
        x.close()
    r.close()


# ---- render_frames_distributed on two ranks (gloo, both on cuda:0; NCCL cannot put two ranks on one GPU) ------------
FW, FH, FSPP = 72, 44, 8  # ragged against the 16x8 tiles
MODES = {"plain": dict(entries=4), "adaptive_denoised": dict(entries=4, adaptive=(0.05, 1e-3, 2), denoise=True)}


def _frames_setup():
    cfg = scenes.sphere_scene()
    cam = api.Camera.look_at(api.vec3(0.3, 0.6, 4.5), np.asarray(CENTER), api.vec3(0.0, 1.0, 0.0), 0.7)
    cams = [orbit(cam, CENTER, 0.05 * i, lift=0.02 * i) for i in range(4)]
    r = api.Renderer(cfg.scene, cam).width(FW).height(FH).max_bounces(2).seed(7).num_samples(FSPP).filter(api.Filter.Box(1)).device(0)
    return r, cams


def _mode_kwargs(mode):
    kw = dict(MODES[mode])
    if "adaptive" in kw:
        kw["adaptive"] = api.Adaptive(*kw["adaptive"])
    if kw.pop("denoise", False):
        kw["denoise"] = api.Denoise()
    return dict(kw, feature_samples=4)


def _frames_worker(rank, world, port, q):
    import os

    import torch.distributed as dist

    from rpt_b200.distributed import render_frames_distributed

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        out = {}
        for mode in MODES:
            r, cams = _frames_setup()
            own = r.camera
            out[mode] = [f.tobytes() for f in render_frames_distributed(r, cams, **_mode_kwargs(mode))]
            assert r.camera is own
            r.close()
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


def test_two_ranks_render_the_frames_of_one_buffer(gpu_ok):
    import socket

    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_frames_worker, args=(rk, world, port, q)) for rk in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=300) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    assert [p.exitcode for p in procs] == [0] * world
    for mode in MODES:
        r, cams = _frames_setup()
        want = [f.tobytes() for f in r.render_frames(cams, **_mode_kwargs(mode))]
        r.close()
        assert len(want) == len(cams)
        assert len(set(want)) == len(want)  # the frames differ: the camera moves
        for rank in range(world):
            assert got[rank][mode] == want, (mode, rank)
