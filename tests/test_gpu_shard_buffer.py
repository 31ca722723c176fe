"""Shard buffers (rptb_buffer_create_shard) gathered into a whole buffer (rptb_buffer_export_shard /
rptb_buffer_import_shards) against one whole buffer given the same calls: the same pixel state, features, image bytes,
variance and denoised image bit for bit, for any shard count -- including shards that own no tile.  The all-gather is
stood in for by torch.cat of the shards' exports on one device."""
import ctypes as C

import numpy as np
import pytest
import torch

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from rpt_b200.distributed import ShardBuffer, shard_block_layout, shard_tiles
from tests import util

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
CRIT = api.Adaptive(0.05, 1e-3, 4)


def _renderer(w, h, prec, seed=5):
    cfg = scenes.sphere_scene()
    return api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(2).seed(seed).precision(prec)


def _calls(r, buf, plain=2, adaptive=3):
    """The sequence every buffer of a case gets, from sample 0: plain entries, a 16-ray feature pass, adaptive entries.
    Returns the active count of each adaptive call."""
    r._next_sample = 0
    for _ in range(plain):
        r.sample(4, buf, want_stats=False)
    r.sample_features(16, buf)
    return [r.sample(4, buf, want_stats=False, adaptive=CRIT) for _ in range(adaptive)]


def _gather(shards, dst, with_features=True):
    """torch.cat of every shard's export (what all_gather_into_tensor gives), imported into `dst`."""
    blocks = []
    for s in shards:
        out = torch.empty(s.block_bytes(with_features), dtype=torch.uint8, device="cuda:0")
        s.export(out, with_features)
        blocks.append(out)
    gathered = torch.cat(blocks)
    torch.cuda.synchronize()
    return capi.lib().rptb_buffer_import_shards(dst.handle, C.c_void_p(gathered.data_ptr()), len(shards),
                                               1 if with_features else 0)


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


_REF = {}


def _reference(w, h, prec):
    """Whole buffers at box radius 0 and 1 given the case's calls, and their adaptive active counts (cached per case)."""
    key = (w, h, prec)
    if key not in _REF:
        r = _renderer(w, h, prec)
        ds = r.device_scene()
        whole = [api.DeviceBuffer(ds, w, h, api.Filter.Box(rad)) for rad in (0, 1)]
        active = [_calls(r, b) for b in whole]
        assert active[0] == active[1]
        _REF[key] = (r, whole, active[0])
    return _REF[key]


CASES = [(w, h, prec, n) for (w, h) in ((128, 96), (97, 61)) for prec in (F32, F64) for n in (1, 2, 3, 5, 8)]
CASES += [(20, 10, F32, n) for n in (3, 5, 8)]  # 4 tiles: shards 4.. of 5 and 8 own none


@pytest.mark.parametrize("w,h,prec,n", CASES)
def test_gathered_shards_are_the_whole_buffer(gpu_ok, w, h, prec, n):
    r, whole, ref_active = _reference(w, h, prec)
    ds = r.device_scene()
    shards = [ShardBuffer(ds, w, h, api.Filter.Box(0), rank=i, world=n) for i in range(n)]
    actives = [_calls(r, s) for s in shards]
    for k, want in enumerate(ref_active):  # the shards' active pixels add up to the whole buffer's, call by call
        assert sum(a[k] for a in actives) == want
    for i, s in enumerate(shards):
        lay = shard_block_layout(w, h, n, True)
        assert s.block_bytes(True) == lay["bytes"] == 256 + 100 * shard_tiles(w, h, 0, n) * 128
        assert s.block_bytes(False) == shard_block_layout(w, h, n, False)["bytes"]
    got = [api.DeviceBuffer(ds, w, h, api.Filter.Box(rad)) for rad in (0, 1)]
    for g in got:
        assert _gather(shards, g) == capi.OK, capi.lib().rptb_last_error()
    for g, ref in zip(got, whole):
        for a, b in zip(g.pixel_stats(), ref.pixel_stats()):
            assert _bits(a) == _bits(b)
        for a, b in zip(g.features(), ref.features()):
            assert _bits(a) == _bits(b)
        assert _bits(g.image()) == _bits(ref.image())
        assert _bits(np.float64(g.variance())) == _bits(np.float64(ref.variance()))
        assert _bits(g.denoise()) == _bits(ref.denoise())
    # the gathered buffer keeps its entries' and features' camera: it reprojects like the whole one
    if n == 3 and prec == F32:
        outs = []
        for src in (got[0], whole[0]):
            dst = r.device_buffer()
            r.sample_features(16, dst)
            dst.reproject_from(src)
            outs.append(dst.pixel_stats())
        for a, b in zip(*outs):
            assert _bits(a) == _bits(b)
    for b in shards + got:
        b.close()


def test_gather_without_features(gpu_ok):
    w, h, n = 97, 61, 3
    r, whole, _ = _reference(w, h, F32)
    ds = r.device_scene()
    shards = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
    for s in shards:
        _calls(r, s)
    dst = api.DeviceBuffer(ds, w, h, api.Filter.Box(1))
    assert _gather(shards, dst, with_features=False) == capi.OK
    for a, b in zip(dst.pixel_stats(), whole[1].pixel_stats()):
        assert _bits(a) == _bits(b)
    assert _bits(dst.image()) == _bits(whole[1].image())
    with pytest.raises(capi.RptbError, match="no features"):
        dst.features()
    # a later feature pass starts from nothing, as on a buffer that never had one
    r.sample_features(16, dst)
    for a, b in zip(dst.features(), whole[1].features()):
        assert _bits(a) == _bits(b)


def test_gather_into_a_buffer_with_state_replaces_it(gpu_ok):
    w, h, n = 64, 40, 2
    r = _renderer(w, h, F64)
    ds = r.device_scene()
    ref = api.DeviceBuffer(ds, w, h)
    _calls(r, ref)
    shards = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
    for s in shards:
        _calls(r, s)
    dst = api.DeviceBuffer(ds, w, h)
    r._next_sample = 100
    for _ in range(3):
        r.sample(2, dst, want_stats=False)  # overwritten by the import
    assert _gather(shards, dst) == capi.OK
    for a, b in zip(dst.pixel_stats(), ref.pixel_stats()):
        assert _bits(a) == _bits(b)
    assert _bits(dst.denoise()) == _bits(ref.denoise())


def _status(fn, *args):
    rc = fn(*args)
    return rc, capi.lib().rptb_last_error().decode()


def test_errors(gpu_ok):
    lib = capi.lib()
    w, h = 48, 24
    r = _renderer(w, h, F32)
    ds = r.device_scene()
    cam = r.camera.to_c()
    hd = C.c_void_p()
    assert lib.rptb_buffer_create_shard(ds.handle, w, h, 0, 2, 2, C.byref(hd)) == capi.ERR_BAD_ARG and not hd
    assert lib.rptb_buffer_create_shard(ds.handle, w, h, 0, 0, 0, C.byref(hd)) == capi.ERR_BAD_ARG and not hd
    assert lib.rptb_buffer_create_shard(ds.handle, 0, h, 0, 0, 1, C.byref(hd)) == capi.ERR_BAD_ARG and not hd
    assert lib.rptb_buffer_create_shard(None, w, h, 0, 0, 1, C.byref(hd)) == capi.ERR_BAD_ARG
    assert lib.rptb_buffer_create_shard(ds.handle, w, h, 0, 0, 1, None) == capi.ERR_BAD_ARG
    s = ShardBuffer(ds, w, h, rank=1, world=2)
    # a render into the shard must name its shard
    crit = CRIT.to_c()
    for idx, cnt in ((0, 2), (1, 3), (0, 1), (0, 0)):
        p = r.params(1, 0, idx, cnt)
        assert lib.rptb_sample_into(ds.handle, C.byref(cam), C.byref(p), s.handle, None) == capi.ERR_BAD_ARG
        assert lib.rptb_sample_into_adaptive(ds.handle, C.byref(cam), C.byref(p), C.byref(crit), s.handle, None,
                                             None) == capi.ERR_BAD_ARG
        assert lib.rptb_buffer_add_features(ds.handle, C.byref(cam), C.byref(p), s.handle, None) == capi.ERR_BAD_ARG
    assert "the buffer holds shard 1 of 2" in lib.rptb_last_error().decode()
    whole = r.device_buffer()
    p = r.params(1, 0, 1, 2)
    assert lib.rptb_sample_into(ds.handle, C.byref(cam), C.byref(p), whole.handle, None) == capi.ERR_UNSUPPORTED
    _calls(r, s)
    assert s.entries == 5 and s.feature_rays == 16
    # whole-image reads of a shard are refused, and say to gather first
    d = api.Denoise().to_c()
    rp = api.Reproject().to_c()
    npix = w * h
    sums, m2, cnt = np.empty(npix * 3), np.empty(npix), np.empty(npix, np.uint32)
    rgb8 = np.empty(npix * 3, np.uint8)
    dbl = C.c_double()
    refused = [
        _status(lib.rptb_buffer_image, s.handle, rgb8.ctypes.data_as(capi.c_u8_p)),
        _status(lib.rptb_buffer_variance, s.handle, C.byref(dbl)),
        _status(lib.rptb_buffer_sums, s.handle, sums.ctypes.data_as(capi.c_double_p), None),
        _status(lib.rptb_buffer_pixel_stats, s.handle, None, None, cnt.ctypes.data_as(capi.c_u32_p)),
        _status(lib.rptb_buffer_features, s.handle, None, m2.ctypes.data_as(capi.c_double_p), None, None),
        _status(lib.rptb_buffer_denoise, s.handle, C.byref(d), sums.ctypes.data_as(capi.c_double_p), None),
        _status(lib.rptb_buffer_reproject, whole.handle, s.handle, C.byref(rp), None),
        _status(lib.rptb_buffer_reproject, s.handle, whole.handle, C.byref(rp), None),
        _status(lib.rptb_buffer_add_samples, s.handle, sums.ctypes.data_as(capi.c_double_p)),
    ]
    for rc, msg in refused:
        assert rc == capi.ERR_UNSUPPORTED and "gather the shards" in msg, msg
    with pytest.raises(capi.RptbError, match="gather the shards"):
        s.image()
    # export: shard buffers only, features only when held
    out = torch.empty(s.block_bytes(True), dtype=torch.uint8, device="cuda:0")
    assert lib.rptb_buffer_shard_bytes(whole.handle, 0) == 0 and lib.rptb_buffer_shard_bytes(None, 0) == 0
    assert lib.rptb_buffer_export_shard(whole.handle, C.c_void_p(out.data_ptr()), 0, None) == capi.ERR_BAD_ARG
    assert lib.rptb_buffer_export_shard(s.handle, None, 0, None) == capi.ERR_BAD_ARG
    bare = ShardBuffer(ds, w, h, rank=0, world=2)
    assert lib.rptb_buffer_export_shard(bare.handle, C.c_void_p(out.data_ptr()), 1, None) == capi.ERR_BAD_ARG
    assert "no features" in lib.rptb_last_error().decode()

    # import: the blocks of shards 0 and 1 of a case both got, then one case at a time broken
    s0 = ShardBuffer(ds, w, h, rank=0, world=2)
    _calls(r, s0)

    def blocks(bufs, wf=1):
        outs = []
        for b in bufs:
            o = torch.empty(b.block_bytes(bool(wf)), dtype=torch.uint8, device="cuda:0")
            b.export(o, bool(wf))
            outs.append(o)
        t = torch.cat(outs)
        torch.cuda.synchronize()
        return t

    def imp(dst, t, n=2, wf=1):
        return _status(lib.rptb_buffer_import_shards, dst.handle, C.c_void_p(t.data_ptr()), n, wf)

    good = blocks([s0, s])
    assert imp(r.device_buffer(), good)[0] == capi.OK
    rc, msg = imp(r.device_buffer(), blocks([s, s0]))
    assert rc == capi.ERR_BAD_ARG and "in order" in msg, msg
    rc, msg = imp(ShardBuffer(ds, w, h, rank=0, world=1), good)
    assert rc == capi.ERR_BAD_ARG and "dst is a shard buffer" in msg, msg
    rc, msg = imp(api.DeviceBuffer(ds, w - 1, h), good)
    assert rc == capi.ERR_BAD_ARG and "dst is" in msg, msg
    rc, msg = imp(r.device_buffer(), good, n=3)
    assert rc == capi.ERR_BAD_ARG, msg
    rc, msg = imp(r.device_buffer(), good, wf=0)
    assert rc == capi.ERR_BAD_ARG and "exported with features" in msg, msg
    assert imp(r.device_buffer(), good, n=0)[0] == capi.ERR_BAD_ARG
    assert _status(lib.rptb_buffer_import_shards, None, C.c_void_p(good.data_ptr()), 2, 1)[0] == capi.ERR_BAD_ARG
    assert _status(lib.rptb_buffer_import_shards, whole.handle, None, 2, 1)[0] == capi.ERR_BAD_ARG
    rc, msg = imp(r.device_buffer(), torch.zeros_like(good))
    assert rc == capi.ERR_BAD_ARG and "not a shard block" in msg, msg
    # shards given different calls: one more entry, more feature rays, another camera
    extra = ShardBuffer(ds, w, h, rank=0, world=2)
    _calls(r, extra, adaptive=4)
    more_rays = ShardBuffer(ds, w, h, rank=0, world=2)
    _calls(r, more_rays)
    r.sample_features(4, more_rays)
    moved = ShardBuffer(ds, w, h, rank=0, world=2)
    r2 = _renderer(w, h, F32)
    r2.camera = api.Camera.look_at(api.vec3(0.1, 0.2, 5.0), api.vec3(0, 0, 0), api.vec3(0, 1, 0), 0.5)
    r2._dev_scene = ds
    _calls(r2, moved)
    r2._dev_scene = None
    for odd in (extra, more_rays, moved):
        rc, msg = imp(r.device_buffer(), blocks([odd, s]))
        assert rc == capi.ERR_BAD_ARG and "other calls" in msg, msg
    for b in (s, s0, bare, extra, more_rays, moved, whole):
        b.close()


def test_multi_replica_scene_is_unsupported(gpu_ok, monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")
    r = _renderer(32, 16, F32).device([0, 0])
    hd = C.c_void_p()
    rc = capi.lib().rptb_buffer_create_shard(r.device_scene().handle, 32, 16, 0, 0, 2, C.byref(hd))
    assert rc == capi.ERR_UNSUPPORTED and not hd
