"""Guided adaptive sampling on two ranks (gloo, both on cuda:0) against the whole-buffer loops: render_iterative_distributed
with Adaptive(guide=Denoise()) gathers to iterative_render's bits at every callback and at the end, and stops after the
same batch; render_frames_distributed with a guided criterion gives render_frames' bytes on every frame, with and without
history_test, and makes exactly one full gather per frame -- the deltas keep the rest current.  (NCCL cannot put two
ranks on one GPU.)"""
import os
import socket

import pytest
import torch.multiprocessing as mp

from rpt_b200 import api, scenes
from tests.test_reproject import orbit

pytestmark = pytest.mark.gpu

W, H, SPP, INTERVAL, FEAT = 72, 44, 400, 4, 16  # ragged against the 16x8 tiles
GUIDED = dict(rel_tol=0.2, abs_tol=0.01, min_entries=3)  # loose enough that every pixel converges well before SPP
FRAMES = dict(entries=4, feature_samples=8)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _renderer():
    cfg = scenes.sphere_scene()
    return (api.Renderer(cfg.scene, cfg.camera).width(W).height(H).max_bounces(2).seed(11).num_samples(SPP)
            .filter(api.Filter.Box(1)).device(0))


def _crit():
    return api.Adaptive(guide=api.Denoise(), **GUIDED)


def _path(cam):
    return [cam, orbit(cam, (0.0, 0.0, 0.0), 0.05), orbit(cam, (0.0, 0.0, 0.0), 0.1)]


def _worker(rank, world, port, q):
    import torch.distributed as dist

    from rpt_b200 import distributed
    from rpt_b200.distributed import ShardBuffer, render_frames_distributed, render_iterative_distributed

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        r = _renderer()
        images = []

        def callback(iteration, shard):
            whole = shard.gather()  # a full gather inside the loop does not break the delta chain
            images.append((iteration, whole.image()))
            whole.close()

        buf = render_iterative_distributed(r, INTERVAL, callback, adaptive=_crit(), feature_samples=FEAT)
        whole = buf.gather(with_features=True)
        it = (images, whole.pixel_stats(), whole.image(), whole.denoise())
        whole.close()
        buf.close()
        # frames: count the full gathers
        full = [0]
        gather = ShardBuffer.gather

        def counted(self, *a, **k):
            full[0] += 1
            return gather(self, *a, **k)

        ShardBuffer.gather = counted
        frames = {}
        try:
            for ht in (None, api.HistoryTest()):
                r2 = _renderer().num_samples(8)
                full[0] = 0
                frames[ht is not None] = ([f.tobytes() for f in render_frames_distributed(
                    r2, _path(r2.camera), adaptive=_crit(), denoise=api.Denoise(), history_test=ht, **FRAMES)], full[0])
                r2.close()
        finally:
            ShardBuffer.gather = gather
        assert distributed.ShardBuffer.gather is gather
        q.put((rank, it, frames))
        r.close()
    finally:
        dist.destroy_process_group()


def test_two_ranks_guided(gpu_ok):
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(rk, world, port, q)) for rk in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict((res[0], res[1:]) for res in (q.get(timeout=600) for _ in range(world)))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    assert [p.exitcode for p in procs] == [0] * world

    r = _renderer()
    buf = r.device_buffer()
    images = []
    r.iterative_render(INTERVAL, lambda it, b: images.append((it, b.image())), buffer=buf, adaptive=_crit(), feature_samples=FEAT)
    assert 0 < len(images) < SPP // INTERVAL  # the guided loop stopped early, so the early exit is compared too
    ref_frames = {}
    for ht in (None, api.HistoryTest()):
        r2 = _renderer().num_samples(8)
        ref_frames[ht is not None] = [f.tobytes() for f in r2.render_frames(_path(r2.camera), adaptive=_crit(), denoise=api.Denoise(),
                                                                            history_test=ht, **FRAMES)]
        r2.close()
    for rank in range(world):
        (imgs, stats, img, den), frames = got[rank]
        assert [it for it, _ in imgs] == [it for it, _ in images]
        for (_, a), (_, b) in zip(imgs, images):
            assert a.tobytes() == b.tobytes()
        for a, b in zip(stats, buf.pixel_stats()):
            assert a.tobytes() == b.tobytes()
        assert img.tobytes() == buf.image().tobytes()
        assert den.tobytes() == buf.denoise().tobytes()
        for ht in (False, True):
            got_frames, gathers = frames[ht]
            assert got_frames == ref_frames[ht]
            assert gathers == len(ref_frames[ht])  # one full gather per frame
    buf.close()
    r.close()
