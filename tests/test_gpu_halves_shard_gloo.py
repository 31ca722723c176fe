"""Guided adaptive sampling on the error estimate from two half buffers on two and three ranks (gloo, all on cuda:0)
against the whole-buffer loop: render_iterative_distributed with Adaptive(guide=Denoise(), estimate="halves") gives
iterative_render's callback iterations and image bytes on one whole buffer with halves, stops after the same batch, and
ends with the same pixel_stats, half_sums and denoised_error bytes.  (NCCL cannot put two ranks on one GPU.)"""
import os
import socket

import pytest
import torch.multiprocessing as mp

from rpt_b200 import api, scenes

pytestmark = pytest.mark.gpu

W, H, SPP, INTERVAL, FEAT = 72, 44, 400, 4, 16  # ragged against the 16x8 tiles
GUIDED = dict(rel_tol=0.5, abs_tol=0.05, min_entries=3)  # loose enough that every pixel converges on E well before SPP


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
    return api.Adaptive(guide=api.Denoise(), estimate="halves", **GUIDED)


def _worker(rank, world, port, q):
    import torch.distributed as dist

    from rpt_b200.distributed import render_iterative_distributed

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
        assert buf.halves
        whole = buf.gather(with_features=True)
        assert whole.halves
        q.put((rank, images, whole.pixel_stats(), whole.half_sums(), whole.denoised_error(api.Denoise())))
        whole.close()
        buf.close()
        r.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_ranks_guided_on_the_error_estimate(gpu_ok, world):
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
    buf = r.device_buffer(halves=True)
    images = []
    r.iterative_render(INTERVAL, lambda it, b: images.append((it, b.image())), buffer=buf, adaptive=_crit(), feature_samples=FEAT)
    assert 0 < len(images) < SPP // INTERVAL  # the loop stopped early, so the early exit is compared too
    for rank in range(world):
        imgs, stats, half, err = got[rank]
        assert [it for it, _ in imgs] == [it for it, _ in images]
        for (_, a), (_, b) in zip(imgs, images):
            assert a.tobytes() == b.tobytes()
        for a, b in zip(stats, buf.pixel_stats()):
            assert a.tobytes() == b.tobytes()
        assert half.tobytes() == buf.half_sums().tobytes()
        assert err.tobytes() == buf.denoised_error(api.Denoise()).tobytes()
    buf.close()
    r.close()
