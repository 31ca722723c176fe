"""render_iterative_distributed on two ranks (gloo, both on cuda:0) against Renderer.iterative_render on one whole
buffer: with adaptive sampling, every rank's gathered image at every callback, and its final denoised image, are the
whole buffer's bit for bit, and the loop stops after the same batch.  (NCCL cannot put two ranks on one GPU; the NCCL
path is exercised by tools/shard_buffer_measure.py on a multi-GPU machine.)"""
import os
import socket

import pytest
import torch.multiprocessing as mp

from rpt_b200 import api, scenes

pytestmark = pytest.mark.gpu

W, H, SPP, INTERVAL, FEAT = 72, 44, 400, 4, 16  # ragged against the 16x8 tiles
CRIT = (0.5, 0.05, 3)  # loose enough that every pixel converges well before SPP


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


def _worker(rank, world, port, q):
    import torch.distributed as dist

    from rpt_b200.distributed import ShardBuffer, render_iterative_distributed

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        r = _renderer()
        buf = ShardBuffer(r.device_scene(), W, H, r._filter)
        assert buf.shard == (rank, world)
        r.sample_features(FEAT, buf)
        images = []

        def callback(iteration, shard):
            whole = shard.gather()
            images.append((iteration, whole.image()))
            whole.close()

        render_iterative_distributed(r, INTERVAL, callback, adaptive=api.Adaptive(*CRIT), buffer=buf)
        whole = buf.gather(with_features=True)
        q.put((rank, images, whole.image(), whole.denoise(), whole.entries))
        whole.close()
        buf.close()
        r.close()
    finally:
        dist.destroy_process_group()


def test_two_ranks_gather_the_whole_buffer(gpu_ok):
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(rk, world, port, q)) for rk in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict((res[0], res[1:]) for res in (q.get(timeout=300) for _ in range(world)))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    assert [p.exitcode for p in procs] == [0] * world

    r = _renderer()
    buf = r.device_buffer()
    r.sample_features(FEAT, buf)
    images = []
    r.iterative_render(INTERVAL, lambda it, b: images.append((it, b.image())), buffer=buf, adaptive=api.Adaptive(*CRIT))
    assert 0 < len(images) < SPP // INTERVAL  # the adaptive loop stopped early, so the early exit is compared too
    for rank in range(world):
        imgs, img, den, entries = got[rank]
        assert [it for it, _ in imgs] == [it for it, _ in images]
        for (_, a), (_, b) in zip(imgs, images):
            assert a.tobytes() == b.tobytes()
        assert img.tobytes() == buf.image().tobytes()
        assert den.tobytes() == buf.denoise().tobytes()
        assert entries == int(buf.counts().max())
    r.close()
