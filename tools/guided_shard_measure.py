"""Guided adaptive sampling on shards, kept current by delta blocks (ShardBuffer.gather_delta), measured on the GPU: one
JSON line per measurement, each with the card's name and power limit read in the same run.  BASELINE.md section 3.0g
holds the results.

  kernels  Cornell at 800x600 and 1920x1080 on a world-1 shard with 16 feature rays: runs of 24 adaptive calls of 2
           spp (plain at rel_tol 0.02, 0.1, 0.2 and 0.4, and guided at 0.02; abs_tol 1e-3, min_entries 4), each call
           followed by gather_delta into the whole buffer gathered before the first.  Per call, torch.profiler's CUDA
           kernel records of the export (CUB's select kernels and delta_export_kernel) and of the import
           (delta_import_kernel), beside the call's active fraction; the rows nearest 100 %, 10 % and 1 % active are
           printed.
  bytes    sphere, Cornell, the BVH teapot and glass at 800x600: a guided run (Adaptive(0.02, 1e-3, 4, guide=Denoise()),
           16 feature rays, up to 64 calls of 2 spp) on one whole buffer.  Per call, the active count and the bytes one
           world-1 delta block takes (256 + 40 per active pixel, delta_block_layout) beside the full block a re-gather
           would move (256 + 36 per pixel, without features).  Computed from the layout, not timed.
  ranks    run under `torchrun --nproc_per_node=2` (gloo; both ranks on one GPU, exchanging through host memory -- not
           NCCL scaling): Cornell at 800x600, the same guided run sharded.  Per call after the first full gather, the
           host clock of gather_delta against a full gather(with_features=True) (each ending in a synchronise), and the
           filter's device time on rank 0 from torch.profiler; then the whole guided loop sharded
           (render_iterative_distributed) against iterative_render on one whole buffer, rank 0 alone on the GPU.

python tools/guided_shard_measure.py [--quick] [--only kernels,bytes]
torchrun --standalone --nproc_per_node=2 tools/guided_shard_measure.py --only ranks [--quick]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from rpt_b200 import _capi as capi  # noqa: E402
from rpt_b200 import api, distributed, scenes  # noqa: E402

SPP = 2
GUIDE = api.Denoise()


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def configs(quick):
    out = [("sphere", scenes.sphere_scene, None, {}), ("cornell", scenes.cornell_scene, None, {}),
           ("teapot", scenes.teapot_scene, 4, {"accel": capi.ACCEL_BVH}), ("glass", lambda: scenes.glass_scene(512, 256), None, {})]
    return out[:2] if quick else out


def renderer(cfg, w, h, mb=None, extra=None):
    r = api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(cfg.max_bounces if mb is None else mb).seed(1)
    if extra and "accel" in extra:
        r.accel(extra["accel"])
    return r


def kernel_ms(prof, names):
    total = 0.0
    for e in prof.key_averages():
        if any(k in e.key for k in names):
            total += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
    return total / 1e3


def kernels(gpu, quick):
    # runs that reach every active fraction: plain criteria of several tolerances (a plain run stays above 90 % active at
    # 0.02), and the guided one, which falls to a few per cent after min_entries calls
    crits = [api.Adaptive(rel, 1e-3, 4) for rel in (0.02, 0.1, 0.2, 0.4)] + [api.Adaptive(0.02, 1e-3, 4, guide=GUIDE)]
    for w, h in [(64, 48)] if quick else [(800, 600), (1920, 1080)]:
        r = renderer(scenes.cornell_scene(), w, h)
        rows = []
        for crit in crits:
            r._next_sample = 0
            shard = distributed.ShardBuffer(r.device_scene(), w, h, rank=0, world=1)
            r.sample_features(16, shard)
            whole = shard.gather(with_features=True)
            for call in range(8 if quick else 24):
                kw = {"guide_buffer": whole} if crit.guide is not None else {}
                active = r.sample(SPP, shard, want_stats=False, adaptive=crit, **kw)
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    shard.gather_delta(whole, active)
                    torch.cuda.synchronize()
                rows.append({"criterion": "guided" if crit.guide is not None else "plain", "rel_tol": crit.rel_tol, "call": call,
                             "active": active, "fraction": active / (w * h),
                             "export_ms": round(kernel_ms(prof, ("delta_export_kernel", "DeviceSelect", "DeviceCompact")), 4),
                             "import_ms": round(kernel_ms(prof, ("delta_import_kernel",)), 4)})
            whole.close()
            shard.close()
        for target in (1.0, 0.1, 0.01):
            best = min(rows, key=lambda x: abs(x["fraction"] - target))
            print(json.dumps({"what": "kernels", "size": [w, h], "target_fraction": target, **best, "gpu": gpu}), flush=True)
        r.close()


def bytes_per_call(gpu, quick):
    w, h = (64, 48) if quick else (800, 600)
    crit = api.Adaptive(0.02, 1e-3, 4, guide=GUIDE)
    full = distributed.shard_block_layout(w, h, 1)["bytes"]
    for name, make, mb, extra in configs(quick):
        r = renderer(make(), w, h, mb, extra)
        buf = r.device_buffer()
        r.sample_features(16, buf)
        actives = []
        for _ in range(64):
            actives.append(r.sample(SPP, buf, want_stats=False, adaptive=crit))
            if actives[-1] == 0:
                break
        delta = [distributed.delta_block_layout(a)["bytes"] for a in actives]
        print(json.dumps({"what": "bytes", "scene": name, "size": [w, h], "calls": len(actives), "active": actives,
                          "delta_bytes": delta, "full_block_bytes": full, "delta_bytes_total": sum(delta),
                          "full_bytes_total": full * len(actives), "median_delta_over_full": statistics.median(delta) / full,
                          "gpu": gpu}), flush=True)
        buf.close()
        r.close()


def ranks(gpu, quick):
    import torch.distributed as dist

    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    w, h = (64, 48) if quick else (800, 600)
    crit = api.Adaptive(0.02, 1e-3, 4, guide=GUIDE)
    r = renderer(scenes.cornell_scene(), w, h).num_samples(128)
    shard = distributed.ShardBuffer(r.device_scene(), w, h, group=None)
    r.sample_features(16, shard)
    # _GuidedShard.sample's steps, one by one, to time each
    guided = distributed._GuidedShard(r, shard, crit)
    t_delta, t_full, filt, actives = [], [], [], []
    for _ in range(64):
        s = shard
        if guided.whole is None and s.entries >= crit.min_entries:
            guided.whole = s.gather(with_features=True)
        torch.cuda.synchronize()
        if guided.whole is not None and rank == 0:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                active = r.sample(SPP, s, want_stats=False, adaptive=crit, guide_buffer=guided.whole)
                torch.cuda.synchronize()
            filt.append(kernel_ms(prof, ("buffer_scatter", "buffer_move", "features_resolve", "denoise_demodulate", "denoise_pass",
                                         "guided_mark")))
        else:
            active = r.sample(SPP, s, want_stats=False, adaptive=crit, guide_buffer=guided.whole)
        out = torch.empty(world, dtype=torch.int64)
        dist.all_gather_into_tensor(out, torch.tensor([active], dtype=torch.int64))
        counts = out.tolist()
        actives.append(sum(counts))
        if guided.whole is not None:
            dist.barrier()
            t = time.perf_counter()
            s.gather_delta(guided.whole, max(counts))
            torch.cuda.synchronize()
            t_delta.append((time.perf_counter() - t) * 1e3)
            dist.barrier()
            t = time.perf_counter()
            g = s.gather(with_features=True)
            torch.cuda.synchronize()
            t_full.append((time.perf_counter() - t) * 1e3)
            g.close()
        if sum(counts) == 0:
            break
    guided.close()
    shard.close()
    if rank == 0:
        print(json.dumps({"what": "sync", "size": [w, h], "world": world, "backend": "gloo, both ranks on one GPU through host memory",
                          "calls": len(actives), "active": actives, "delta_ms_median": round(statistics.median(t_delta), 3),
                          "full_gather_with_features_ms_median": round(statistics.median(t_full), 3),
                          "delta_ms": [round(x, 3) for x in t_delta], "full_ms": [round(x, 3) for x in t_full],
                          "filter_device_ms_median_rank0": round(statistics.median(filt), 3) if filt else None,
                          "nccl_across_gpus": "not measured", "gpu": gpu}), flush=True)
    # the whole loop: sharded, then on one whole buffer with rank 0 alone on the GPU
    dist.barrier()
    torch.cuda.synchronize()
    t = time.perf_counter()
    r._next_sample = 0
    buf = distributed.render_iterative_distributed(r, SPP, lambda i, b: None, adaptive=crit)
    torch.cuda.synchronize()
    dist.barrier()
    sharded_s = time.perf_counter() - t
    buf.close()
    if rank == 0:
        r1 = renderer(scenes.cornell_scene(), w, h).num_samples(r._num_samples)
        b = r1.device_buffer()
        torch.cuda.synchronize()
        t = time.perf_counter()
        r1.iterative_render(SPP, lambda i, bb: None, buffer=b, adaptive=crit)
        torch.cuda.synchronize()
        whole_s = time.perf_counter() - t
        b.close()
        r1.close()
        print(json.dumps({"what": "loop", "size": [w, h], "world": world, "backend": "gloo, both ranks on one GPU through host memory",
                          "spp_cap": r._num_samples, "sharded_s": round(sharded_s, 3), "whole_s": round(whole_s, 3), "gpu": gpu}),
              flush=True)
    dist.barrier()
    r.close()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes: a rehearsal, not a measurement")
    ap.add_argument("--only", default="kernels,bytes")
    a = ap.parse_args()
    gpu = card()
    only = a.only.split(",")
    if "kernels" in only:
        kernels(gpu, a.quick)
    if "bytes" in only:
        bytes_per_call(gpu, a.quick)
    if "ranks" in only:
        ranks(gpu, a.quick)


if __name__ == "__main__":
    main()
