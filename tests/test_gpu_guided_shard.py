"""Guided adaptive sampling on shard buffers (rptb_sample_into_guided_shard), with the gathered whole buffer kept current
by delta blocks (rptb_buffer_export_delta / rptb_buffer_import_deltas), against rptb_sample_into_guided on one whole
buffer given the same calls.  Bit for bit: per call the shards' active counts add up to the whole call's; after every
call the delta-synced whole buffer equals a fresh full import of the same shards (sums, M2, counts, features, image,
denoised image and variance); and at the end the gathered shards equal the whole buffer.  The same after a reprojection
and after a history merge (counts 0 and 1, the reprojected flag), at 1920x1080, and every refusal.  The all-gather is
stood in for by torch.cat of the shards' blocks on one device, as in tests/test_gpu_shard_buffer.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from rpt_b200.distributed import ShardBuffer, delta_block_layout
from tests.test_reproject import orbit

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
GUIDE = api.Denoise()
CRIT = api.Adaptive(0.05, 1e-3, 3, guide=GUIDE)
CENTER = (0.0, 0.5, 0.0)


def _cameras():
    cfg = scenes.sphere_scene()
    a = api.Camera.look_at(api.vec3(0.3, 0.6, 4.5), np.asarray(CENTER), api.vec3(0.0, 1.0, 0.0), 0.7)
    return cfg, a, orbit(a, CENTER, 0.07, lift=0.05)


def _renderer(cfg, cam, w, h, prec):
    return api.Renderer(cfg.scene, cam).width(w).height(h).max_bounces(2).seed(5).precision(prec)


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


def _full(shards, ds, w, h):
    """A new whole buffer holding torch.cat of every shard's export with features (what all_gather_into_tensor gives)."""
    blocks = []
    for s in shards:
        out = torch.empty(s.block_bytes(True), dtype=torch.uint8, device="cuda:0")
        s.export(out, True)
        blocks.append(out)
    gathered = torch.cat(blocks)
    torch.cuda.synchronize()
    dst = api.DeviceBuffer(ds, w, h)
    rc = capi.lib().rptb_buffer_import_shards(dst.handle, C.c_void_p(gathered.data_ptr()), len(shards), 1)
    assert rc == capi.OK, capi.lib().rptb_last_error()
    return dst


def _deltas(shards, capacity):
    """torch.cat of every shard's delta block of `capacity`, and the pixel counts the exports report."""
    blocks, pixels = [], []
    for s in shards:
        out = torch.empty(delta_block_layout(capacity)["bytes"], dtype=torch.uint8, device="cuda:0")
        pixels.append(s.export_delta(out, capacity))
        blocks.append(out)
    gathered = torch.cat(blocks)
    torch.cuda.synchronize()
    return gathered, pixels


def _import(whole, gathered, n, capacity):
    return capi.lib().rptb_buffer_import_deltas(whole.handle, C.c_void_p(gathered.data_ptr()), n, capacity)


def _outcome(fn):
    """fn()'s bytes, or its refusal's text: a buffer with a pixel of 0 or 1 entries refuses image and denoise."""
    try:
        return _bits(fn())
    except capi.RptbError as e:
        return str(e)


def _same_state(a, b):
    for x, y in zip(a.pixel_stats(), b.pixel_stats()):
        assert _bits(x) == _bits(y)
    for x, y in zip(a.features(), b.features()):
        assert _bits(x) == _bits(y)
    for read in (lambda d: d.image(), lambda d: d.denoise(GUIDE), lambda d: d.denoised_variance(GUIDE)):
        assert _outcome(lambda: read(a)) == _outcome(lambda: read(b))


def _guided_calls(r, ref, shards, ds, w, h, calls, first_sample, check_every=True):
    """`calls` guided calls of 2 samples on the whole buffer `ref` and on every shard, the shards' filter running over a
    whole buffer kept current by deltas (a full import before the first call that runs the filter).  Returns it."""
    n, synced = len(shards), None
    for c in range(calls):
        r._next_sample = first_sample + 2 * c
        want = r.sample(2, ref, want_stats=False, adaptive=CRIT)
        if synced is None and shards[0].entries >= CRIT.min_entries:
            synced = _full(shards, ds, w, h)
        actives = []
        for s in shards:
            r._next_sample = first_sample + 2 * c
            actives.append(r.sample(2, s, want_stats=False, adaptive=CRIT, guide_buffer=synced))
        assert sum(actives) == want
        if synced is None:
            continue
        cap = max(actives)
        gathered, pixels = _deltas(shards, cap)
        assert pixels == actives
        assert _import(synced, gathered, n, cap) == capi.OK, capi.lib().rptb_last_error()
        if check_every or c == calls - 1:
            fresh = _full(shards, ds, w, h)
            _same_state(synced, fresh)
            fresh.close()
    return synced


CASES = [(w, h, prec, n) for (w, h) in ((128, 96), (97, 61)) for prec in (F32, F64) for n in (1, 2, 3, 5, 8)]
CASES += [(20, 10, prec, n) for prec in (F32, F64) for n in (1, 2, 3, 5, 8)]  # 4 tiles: shards 4.. of 5 and 8 own none


@pytest.mark.parametrize("w,h,prec,n", CASES)
def test_delta_synced_shards_are_the_whole_guided_buffer(gpu_ok, w, h, prec, n):
    cfg, cam, _ = _cameras()
    r = _renderer(cfg, cam, w, h, prec)
    ds = r.device_scene()
    ref = api.DeviceBuffer(ds, w, h)
    shards = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
    for b in [ref] + shards:
        r.sample_features(16, b)
    synced = _guided_calls(r, ref, shards, ds, w, h, calls=6, first_sample=0)
    _same_state(synced, ref)
    got = _full(shards, ds, w, h)
    _same_state(got, ref)
    for b in [ref, synced, got] + shards:
        b.close()
    r.close()


@pytest.mark.parametrize("merge", [False, True])
@pytest.mark.parametrize("n", [1, 3, 8])
def test_after_reprojection_and_merge(gpu_ok, merge, n):
    """Frame 2 takes frame 1's history (reproject_from, whose pixels hold counts 0 and 1, or two fresh entries and
    merge_history_from): the reprojected flag travels in both blocks, and the guided calls still match the whole
    buffer's."""
    w, h = 97, 61
    cfg, a, b = _cameras()
    r = _renderer(cfg, a, w, h, F32)
    ds = r.device_scene()
    ref1 = api.DeviceBuffer(ds, w, h)
    shards1 = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
    for buf in [ref1] + shards1:
        r.sample_features(16, buf)
    _guided_calls(r, ref1, shards1, ds, w, h, calls=4, first_sample=0, check_every=False).close()
    prev = _full(shards1, ds, w, h)
    r.camera = b
    ref2 = api.DeviceBuffer(ds, w, h)
    shards2 = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
    for buf in [ref2] + shards2:
        r.sample_features(16, buf)
        if merge:
            r._next_sample = 100
            for _ in range(2):
                r.sample(2, buf, want_stats=False)
            buf.merge_history_from(ref1 if buf is ref2 else prev)
        else:
            buf.reproject_from(ref1 if buf is ref2 else prev)
    if not merge:
        assert int(ref2.counts().min()) < 2  # there are pixels with 0 or 1 entries
    synced = _guided_calls(r, ref2, shards2, ds, w, h, calls=4, first_sample=200)
    _same_state(synced, ref2)
    for buf in [ref1, ref2, prev, synced] + shards1 + shards2:
        buf.close()
    r.close()


def test_guided_shards_at_1080p(gpu_ok):
    w, h, n = 1920, 1080, 3
    cfg, cam, _ = _cameras()
    r = _renderer(cfg, cam, w, h, F32)
    ds = r.device_scene()
    ref = api.DeviceBuffer(ds, w, h)
    shards = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
    for b in [ref] + shards:
        r.sample_features(4, b)
    synced = _guided_calls(r, ref, shards, ds, w, h, calls=5, first_sample=0, check_every=False)
    _same_state(synced, ref)
    for b in [ref, synced] + shards:
        b.close()
    r.close()


def _refused(fn, code, text):
    with pytest.raises(capi.RptbError) as e:
        fn()
    assert f"status {code}:" in str(e.value) and text in str(e.value), str(e.value)


def test_refusals(gpu_ok, monkeypatch):
    w, h, n = 40, 24, 2
    cfg, cam, other = _cameras()
    r = _renderer(cfg, cam, w, h, F32)
    ds = r.device_scene()
    L = capi.lib()
    BAD, UNSUP = capi.ERR_BAD_ARG, capi.ERR_UNSUPPORTED
    out = torch.empty(delta_block_layout(w * h)["bytes"], dtype=torch.uint8, device="cuda:0")

    def new_shards():
        shards = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
        for s in shards:
            r.sample_features(4, s)
        return shards

    def err():
        return L.rptb_last_error().decode()

    # no delta: nothing since the last export, a plain entry, a feature pass, two calls since the export
    shards = new_shards()
    _refused(lambda: shards[0].export_delta(out, w * h), BAD, "no delta to export")
    for s in shards:
        r._next_sample = 0
        r.sample(2, s, want_stats=False)
    _refused(lambda: shards[0].export_delta(out, w * h), BAD, "no delta to export")
    _full(shards, ds, w, h).close()
    r.sample_features(4, shards[0])
    _refused(lambda: shards[0].export_delta(out, w * h), BAD, "no delta to export")
    r._next_sample = 2
    r.sample(2, shards[0], want_stats=False, adaptive=CRIT, guide_buffer=None)
    _refused(lambda: shards[0].export_delta(out, w * h), BAD, "no delta to export")
    for s in shards:
        s.close()

    # export: a whole buffer, a null block, a capacity below the pixel count
    shards = new_shards()
    whole = _full(shards, ds, w, h)
    acts = []
    for s in shards:
        r._next_sample = 0
        acts.append(r.sample(2, s, want_stats=False, adaptive=CRIT, guide_buffer=None))
    assert L.rptb_buffer_export_delta(whole.handle, C.c_void_p(out.data_ptr()), 8, None, None) == BAD
    assert L.rptb_buffer_export_delta(shards[0].handle, None, 8, None, None) == BAD
    _refused(lambda: shards[0].export_delta(out, acts[0] - 1), BAD, "capacity")
    cap = max(acts)
    gathered, _ = _deltas(shards, cap)
    blk = delta_block_layout(cap)["bytes"]

    # import: not a delta block, another capacity or shard count, shards out of order, another image size, a null
    # block, a shard dst, n > capacity, blocks of different calls
    zeros = torch.zeros(blk * n, dtype=torch.uint8, device="cuda:0")
    assert _import(whole, zeros, n, cap) == BAD and "not a delta block" in err()
    assert _import(whole, gathered, n, cap + 1) == BAD and "capacity" in err()
    assert _import(whole, gathered, 1, cap) == BAD and "shards but shard_count" in err()
    assert _import(whole, gathered, 0, cap) == BAD
    assert _import(whole, torch.cat([gathered[blk:], gathered[:blk]]), n, cap) == BAD and "order" in err()
    other_size = api.DeviceBuffer(ds, w + 1, h)
    assert _import(other_size, gathered, n, cap) == BAD and "dst is" in err()
    assert L.rptb_buffer_import_deltas(whole.handle, None, n, cap) == BAD
    assert L.rptb_buffer_import_deltas(shards[0].handle, C.c_void_p(gathered.data_ptr()), n, cap) == BAD
    bad = gathered.clone()
    bad[248:252] = torch.tensor([cap + 1], dtype=torch.int32).view(torch.uint8).to(bad.device)  # block 0's pixel count
    assert _import(whole, bad, n, cap) == BAD and "more than its capacity" in err()
    bad = gathered.clone()
    bad[blk + 20:blk + 24] = torch.tensor([99], dtype=torch.int32).view(torch.uint8).to(bad.device)  # shard 1's entries before
    assert _import(whole, bad, n, cap) == BAD and "other calls" in err()
    bad = gathered.clone()
    bad[blk + 28] ^= 1  # shard 1's reprojected flag
    assert _import(whole, bad, n, cap) == BAD and "other calls" in err()
    # a dst not at the blocks' state before the call: never imported, or changed since its import; a dst of two parts
    fresh = api.DeviceBuffer(ds, w, h)
    assert _import(fresh, gathered, n, cap) == BAD and "not last written by an import" in err()
    touched = _full(shards, ds, w, h)  # (the shards' current state, not the "before" one)
    assert _import(touched, gathered, n, cap) == BAD and "not at the shards' state before" in err()
    r.sample_features(1, touched)
    assert _import(touched, gathered, n, cap) == BAD and "not last written by an import" in err()
    monkeypatch.setenv("RPTB_ALLOW_REPEATED_DEVICES", "1")
    ds2 = api.DeviceScene(cfg.scene, [0, 0])
    two = api.DeviceBuffer(ds2, w, h)
    assert _import(two, gathered, n, cap) == UNSUP
    two.close()
    ds2.close()
    # the good import, once: whole is then at the "after" state
    assert _import(whole, gathered, n, cap) == capi.OK, err()
    assert _import(whole, gathered, n, cap) == BAD and "not at the shards' state before" in err()

    # the guided shard entry
    crit2 = api.Adaptive(0.05, 1e-3, 2, guide=GUIDE)  # the shards hold 1 entry call: one more reaches min_entries 2
    for s in shards:
        r._next_sample = 2
        r.sample(2, s, want_stats=False, adaptive=crit2, guide_buffer=None)  # the plain mark decides: no whole needed
    _refused(lambda: r.sample(2, whole, adaptive=crit2, guide_buffer=whole), BAD, "not a shard buffer")
    _refused(lambda: r.sample(2, shards[0], adaptive=crit2, guide_buffer=None), BAD, "null whole buffer")
    _refused(lambda: r.sample(2, shards[0], adaptive=crit2, guide_buffer=whole), BAD, "changed since its last export")
    synced = _full(shards, ds, w, h)
    _refused(lambda: r.sample(2, shards[0], adaptive=crit2, guide_buffer=shards[1]), BAD, "whole is a shard buffer")
    _refused(lambda: r.sample(2, shards[0], adaptive=crit2, guide_buffer=other_size), BAD, "whole is 41x24")
    _refused(lambda: r.sample(2, shards[0], adaptive=crit2, guide_buffer=whole), BAD, "does not hold the shard's current state")
    _refused(lambda: r.sample(2, shards[0], adaptive=crit2, guide_buffer=fresh), BAD, "not last written by an import")
    r.camera = other
    _refused(lambda: r.sample(2, shards[0], adaptive=crit2, guide_buffer=synced), BAD, "another camera")
    r.camera = cam
    # without guide_buffer a shard stays refused, as rptb_sample_into_guided refuses it
    _refused(lambda: r.sample(2, shards[0], adaptive=crit2), UNSUP, "shard buffer")
    assert r.sample(2, shards[0], want_stats=False, adaptive=crit2, guide_buffer=synced) >= 0
    for b in [whole, fresh, touched, other_size, synced] + shards:
        b.close()
    r.close()
