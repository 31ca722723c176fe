"""Guided adaptive sampling on the error estimate from two half buffers on shard buffers with halves
(rptb_buffer_create_shard_halves, rptb_sample_into_guided_error_shard), the gathered whole buffer with halves kept current
by halves delta blocks, against rptb_sample_into_guided_error on one whole buffer with halves given the same calls.  Bit
for bit: per call the shards' active counts add up to the whole call's; after every delta import the synced whole buffer
equals a fresh full import of the same shards (pixel_stats, half_sums, features, denoise, denoised_variance and
denoised_error); and at the end the gathered shards equal the whole buffer.  v'-guided calls on halves shards give a
plain shard's sums, M2 and counts.  Every refusal, by code and text.  The all-gather is stood in for by torch.cat of the
shards' blocks on one device, as in tests/test_gpu_guided_shard.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from rpt_b200.distributed import ShardBuffer, delta_block_layout, shard_block_layout

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
GUIDE = api.Denoise()
CRIT_E = api.Adaptive(0.05, 1e-3, 3, guide=GUIDE, estimate="halves")
CRIT_V = api.Adaptive(0.05, 1e-3, 3, guide=GUIDE)
CENTER = (0.0, 0.5, 0.0)


def _renderer(w, h, prec):
    cfg = scenes.sphere_scene()
    cam = api.Camera.look_at(api.vec3(0.3, 0.6, 4.5), np.asarray(CENTER), api.vec3(0.0, 1.0, 0.0), 0.7)
    return api.Renderer(cfg.scene, cam).width(w).height(h).max_bounces(2).seed(5).precision(prec)


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


def _blocks(shards, export, nbytes):
    """torch.cat of every shard's block (what all_gather_into_tensor gives), and what each export returned."""
    blocks, rets = [], []
    for s in shards:
        out = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
        rets.append(export(s, out))
        blocks.append(out)
    gathered = torch.cat(blocks)
    torch.cuda.synchronize()
    return gathered, rets


def _full(shards, ds, w, h, halves=True):
    """A new whole buffer (with halves when the shards have them) holding every shard's block with features."""
    gathered, _ = _blocks(shards, lambda s, out: s.export(out, True), shards[0].block_bytes(True))
    dst = api.DeviceBuffer(ds, w, h, halves=halves)
    rc = capi.lib().rptb_buffer_import_shards(dst.handle, C.c_void_p(gathered.data_ptr()), len(shards), 1)
    assert rc == capi.OK, capi.lib().rptb_last_error()
    return dst


def _deltas(shards, capacity):
    return _blocks(shards, lambda s, out: s.export_delta(out, capacity), delta_block_layout(capacity, shards[0].halves)["bytes"])


def _import(whole, gathered, n, capacity):
    return capi.lib().rptb_buffer_import_deltas(whole.handle, C.c_void_p(gathered.data_ptr()), n, capacity)


def _outcome(fn):
    """fn()'s bytes, or its refusal's text."""
    try:
        return _bits(fn())
    except capi.RptbError as e:
        return str(e)


def _same_state(a, b, halves=True):
    for x, y in zip(a.pixel_stats(), b.pixel_stats()):
        assert _bits(x) == _bits(y)
    for x, y in zip(a.features(), b.features()):
        assert _bits(x) == _bits(y)
    reads = [lambda d: d.denoise(GUIDE), lambda d: d.denoised_variance(GUIDE)]
    if halves:
        reads += [lambda d: d.half_sums(), lambda d: d.denoised_error(GUIDE)]
    for read in reads:
        assert _outcome(lambda: read(a)) == _outcome(lambda: read(b))


def _guided_calls(r, ref, shards, ds, w, h, calls, crit, check_every=True):
    """`calls` guided calls of 2 samples on the whole buffer `ref` and on every shard, the shards' filter running over a
    whole buffer kept current by deltas (a full import before the first call that runs the filter).  Returns it and the
    per-call active counts of the shards."""
    n, synced, log = len(shards), None, []
    halves = shards[0].halves
    for c in range(calls):
        r._next_sample = 2 * c
        want = r.sample(2, ref, want_stats=False, adaptive=crit)
        if synced is None and shards[0].entries >= crit.min_entries:
            synced = _full(shards, ds, w, h, halves)
        actives = []
        for s in shards:
            r._next_sample = 2 * c
            actives.append(r.sample(2, s, want_stats=False, adaptive=crit, guide_buffer=synced))
        assert sum(actives) == want, (c, actives, want)
        log.append(actives)
        if synced is None:
            continue
        cap = max(actives)
        gathered, pixels = _deltas(shards, cap)
        assert pixels == actives
        assert _import(synced, gathered, n, cap) == capi.OK, capi.lib().rptb_last_error()
        if check_every or c == calls - 1:
            fresh = _full(shards, ds, w, h, halves)
            _same_state(synced, fresh, halves)
            fresh.close()
    return synced, log


CASES = [(w, h, prec, n) for (w, h) in ((128, 96), (97, 61), (20, 10)) for prec in (F32, F64) for n in (1, 2, 3, 5, 8)]


@pytest.mark.parametrize("w,h,prec,n", CASES)
def test_halves_shards_are_the_whole_error_guided_buffer(gpu_ok, w, h, prec, n):
    r = _renderer(w, h, prec)
    ds = r.device_scene()
    ref = api.DeviceBuffer(ds, w, h, halves=True)
    shards = [ShardBuffer(ds, w, h, rank=i, world=n, halves=True) for i in range(n)]
    assert shards[0].block_bytes(True) == shard_block_layout(w, h, n, True, halves=True)["bytes"]
    for b in [ref] + shards:
        r.sample_features(16, b)
    synced, log = _guided_calls(r, ref, shards, ds, w, h, calls=6, crit=CRIT_E)
    assert any(sum(a) < w * h for a in log)  # E stopped some pixels: the mark ran
    _same_state(synced, ref)
    got = _full(shards, ds, w, h)
    _same_state(got, ref)
    for b in [ref, synced, got] + shards:
        b.close()
    r.close()


def test_halves_shards_at_1080p(gpu_ok):
    w, h, n = 1920, 1080, 3
    r = _renderer(w, h, F32)
    ds = r.device_scene()
    ref = api.DeviceBuffer(ds, w, h, halves=True)
    shards = [ShardBuffer(ds, w, h, rank=i, world=n, halves=True) for i in range(n)]
    for b in [ref] + shards:
        r.sample_features(4, b)
    synced, _ = _guided_calls(r, ref, shards, ds, w, h, calls=5, crit=CRIT_E, check_every=False)
    _same_state(synced, ref)
    for b in [ref, synced] + shards:
        b.close()
    r.close()


@pytest.mark.parametrize("n", [2, 5])
def test_v_guided_halves_shards_only_carry_half(gpu_ok, n):
    """v'-guided calls: halves shards make the plain shards' decisions, and their HALF is a whole halves buffer's."""
    w, h = 97, 61
    r = _renderer(w, h, F32)
    ds = r.device_scene()
    got = {}
    for halves in (False, True):
        ref = api.DeviceBuffer(ds, w, h, halves=halves)
        shards = [ShardBuffer(ds, w, h, rank=i, world=n, halves=halves) for i in range(n)]
        for b in [ref] + shards:
            r.sample_features(16, b)
        synced, log = _guided_calls(r, ref, shards, ds, w, h, calls=5, crit=CRIT_V, check_every=halves)
        whole = _full(shards, ds, w, h, halves)
        got[halves] = (log, whole.pixel_stats(), whole.half_sums() if halves else None, ref.half_sums() if halves else None)
        for b in [ref, synced, whole] + shards:
            b.close()
    assert got[True][0] == got[False][0]
    for x, y in zip(got[True][1], got[False][1]):
        assert _bits(x) == _bits(y)
    assert _bits(got[True][2]) == _bits(got[True][3])
    r.close()


def _refused(fn, code, text):
    with pytest.raises(capi.RptbError) as e:
        fn()
    assert f"status {code}:" in str(e.value) and text in str(e.value), str(e.value)


def _code(rc, code, text):
    assert rc == code, (rc, capi.lib().rptb_last_error())
    assert text in capi.lib().rptb_last_error().decode(), capi.lib().rptb_last_error()


def test_refusals(gpu_ok):
    w, h, n = 40, 24, 2
    r = _renderer(w, h, F32)
    ds = r.device_scene()
    L = capi.lib()
    BAD, UNSUP = capi.ERR_BAD_ARG, capi.ERR_UNSUPPORTED
    crit2 = api.Adaptive(0.05, 1e-3, 2, guide=GUIDE, estimate="halves")

    def new_shards(halves):
        shards = [ShardBuffer(ds, w, h, rank=i, world=n, halves=halves) for i in range(n)]
        for s in shards:
            r.sample_features(4, s)
        return shards

    def entry(shard, whole, crit=crit2, d=GUIDE, engine=None):
        cam, p, c, g = r.camera.to_c(), r.params(2, 0, *shard.shard), crit.to_c(), d.to_c()
        if engine is not None:
            p.engine = engine
        return L.rptb_sample_into_guided_error_shard(ds.handle, C.byref(cam), C.byref(p), C.byref(c), C.byref(g), shard.handle,
                                                     whole.handle if whole is not None else None, None, None)

    hs, ps = new_shards(True), new_shards(False)
    for s in hs + ps:
        r._next_sample = 0
        r.sample(2, s, want_stats=False)
    # whole-image reads of a halves shard
    _refused(lambda: hs[0].half_sums(), UNSUP, "half_sums of a shard buffer")
    _refused(lambda: hs[0].denoised_error(GUIDE), UNSUP, "denoise_error of a shard buffer")
    # the whole-buffer entry keeps refusing a shard
    cam, p, c, g = r.camera.to_c(), r.params(2, 0, 0, n), crit2.to_c(), GUIDE.to_c()
    _code(L.rptb_sample_into_guided_error(ds.handle, C.byref(cam), C.byref(p), C.byref(c), C.byref(g), hs[0].handle, None, None),
          UNSUP, "shard buffer")
    # the shard entry: a plain shard, iterations 0, the wavefront engine, a whole buffer as the shard
    _code(entry(ps[0], None), BAD, "no halves")
    _code(entry(hs[0], None, crit=api.Adaptive(0.05, 1e-3, 2, guide=api.Denoise(iterations=0), estimate="halves"),
                d=api.Denoise(iterations=0)), BAD, "iterations 0")
    _code(entry(hs[0], None, engine=capi.ENGINE_WAVEFRONT), UNSUP, "wavefront")
    plain_whole, halves_whole = _full(ps, ds, w, h, False), _full(hs, ds, w, h)
    cam, p = r.camera.to_c(), r.params(2, 0)
    _code(L.rptb_sample_into_guided_error_shard(ds.handle, C.byref(cam), C.byref(p), C.byref(c), C.byref(g), halves_whole.handle,
                                                halves_whole.handle, None, None), BAD, "not a shard buffer")
    # once the filter runs (min_entries 2: the shards hold 1 entry call, so this one decides with the plain mark) ...
    for s in hs:
        r._next_sample = 2
        r.sample(2, s, want_stats=False, adaptive=crit2, guide_buffer=None)
    _code(entry(hs[0], None), BAD, "null whole buffer")
    _code(entry(hs[0], halves_whole), BAD, "changed since its last export")
    synced = _full(hs, ds, w, h)
    _code(entry(hs[0], hs[1]), BAD, "whole is a shard buffer")
    _code(entry(hs[0], halves_whole), BAD, "does not hold the shard's current state")
    _code(entry(hs[0], plain_whole), BAD, "whole has no halves")
    for whole in (plain_whole, halves_whole):
        whole.close()
    # imports: plain blocks into a halves dst, halves blocks into a plain dst, full and delta
    plain_blocks, _ = _blocks(ps, lambda s, out: s.export(out, True), ps[0].block_bytes(True))
    halves_blocks, _ = _blocks(hs, lambda s, out: s.export(out, True), hs[0].block_bytes(True))
    hdst, pdst = api.DeviceBuffer(ds, w, h, halves=True), api.DeviceBuffer(ds, w, h)
    _code(L.rptb_buffer_import_shards(hdst.handle, C.c_void_p(plain_blocks.data_ptr()), n, 1), UNSUP, "halves")
    _code(L.rptb_buffer_import_shards(pdst.handle, C.c_void_p(halves_blocks.data_ptr()), n, 1), BAD, "halves")
    psynced = _full(ps, ds, w, h, False)
    pacts, hacts = [], []
    for s in ps:
        r._next_sample = 4
        pacts.append(r.sample(2, s, want_stats=False, adaptive=CRIT_V, guide_buffer=psynced))
    for s in hs:
        r._next_sample = 4
        hacts.append(r.sample(2, s, want_stats=False, adaptive=crit2, guide_buffer=synced))
    pd, _ = _deltas(ps, max(pacts))
    hd, _ = _deltas(hs, max(hacts))
    _code(_import(synced, pd, n, max(pacts)), UNSUP, "halves")
    _code(_import(psynced, hd, n, max(hacts)), BAD, "halves")
    assert _import(synced, hd, n, max(hacts)) == capi.OK, L.rptb_last_error()
    # reprojection and merge into a halves shard: history has no halves
    src = _full(ps, ds, w, h, False)
    fresh = ShardBuffer(ds, w, h, rank=0, world=n, halves=True)
    r.sample_features(4, fresh)
    _refused(lambda: fresh.reproject_from(src), UNSUP, "halves")
    for _ in range(2):
        r.sample(2, fresh, want_stats=False)
    _refused(lambda: fresh.merge_history_from(src), UNSUP, "halves")
    # a halves src is fine
    pfresh = ShardBuffer(ds, w, h, rank=0, world=n)
    r.sample_features(4, pfresh)
    assert pfresh.reproject_from(synced) >= 0
    for b in [synced, psynced, hdst, pdst, src, fresh, pfresh] + hs + ps:
        b.close()
    r.close()
