"""Guided adaptive sampling on the error estimate E over shards with halves (ShardBuffer(halves=True),
rptb_sample_into_guided_error_shard), measured on the GPU: one JSON line per measurement, each with the card's name and
power limit read in the same run.  BASELINE.md section 3.0i holds the results.

  bytes    sphere, Cornell, the BVH teapot and glass at 800x600: a guided run on E (Adaptive(0.05, 1e-3, 4,
           guide=Denoise(), estimate="halves"), 16 feature rays, up to 64 calls of 2 spp) on one whole buffer with
           halves.  Per call, the active count and the bytes one world-1 halves delta block takes (256 + 64 per active
           pixel, delta_block_layout(m, halves=True)) beside the plain layout's (256 + 40) and the full halves block a
           re-gather would move (256 + 124 per pixel with features, 256 + 60 without).  Computed from the layout, not
           timed.
  kernels  Cornell at 800x600 and 1920x1080 on world-1 shards, one plain and one with halves, given the same plain
           adaptive calls (Adaptive(0.1, 1e-3, 4): the same pixels change in both), each call followed by gather_delta
           into the whole buffer gathered before the first.  Per call, torch.profiler's CUDA kernel records of the
           export's copy kernel (delta_export_kernel / delta_export_halves_kernel) and of the import
           (delta_import_kernel / delta_import_halves_kernel), beside the call's active count.
  ranks    run under `torchrun --nproc_per_node=2` (gloo; both ranks on one GPU, exchanging through host memory -- not
           NCCL scaling): Cornell at 800x600, the guided run on E sharded.  Per call after the first full gather, the
           host clock of gather_delta (ending in a synchronise); then the whole loop sharded (render_iterative_distributed)
           against iterative_render on one whole buffer with halves, rank 0 alone on the GPU.

python tools/halves_shard_measure.py [--quick] [--only bytes,kernels]
torchrun --standalone --nproc_per_node=2 tools/halves_shard_measure.py --only ranks [--quick]"""
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
CRIT_E = api.Adaptive(0.05, 1e-3, 4, guide=GUIDE, estimate="halves")


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


def bytes_per_call(gpu, quick):
    w, h = (64, 48) if quick else (800, 600)
    full = distributed.shard_block_layout(w, h, 1, True, halves=True)["bytes"]
    full_nf = distributed.shard_block_layout(w, h, 1, halves=True)["bytes"]
    for name, make, mb, extra in configs(quick):
        r = renderer(make(), w, h, mb, extra)
        buf = r.device_buffer(halves=True)
        r.sample_features(16, buf)
        actives = []
        for _ in range(64):
            actives.append(r.sample(SPP, buf, want_stats=False, adaptive=CRIT_E))
            if actives[-1] == 0:
                break
        delta = [distributed.delta_block_layout(a, halves=True)["bytes"] for a in actives]
        plain = [distributed.delta_block_layout(a)["bytes"] for a in actives]
        print(json.dumps({"what": "bytes", "scene": name, "size": [w, h], "criterion": "E, rel_tol 0.05", "calls": len(actives),
                          "active": actives, "delta_bytes": delta, "delta_bytes_total": sum(delta),
                          "plain_layout_bytes_total": sum(plain), "full_block_bytes_with_features": full,
                          "full_block_bytes_without_features": full_nf, "full_bytes_total": full * len(actives),
                          "median_delta_over_full": statistics.median(delta) / full, "gpu": gpu}), flush=True)
        buf.close()
        r.close()


def kernels(gpu, quick):
    crit = api.Adaptive(0.1, 1e-3, 4)
    names = {False: ("delta_export_kernel", "delta_import_kernel"), True: ("delta_export_halves_kernel", "delta_import_halves_kernel")}
    for w, h in [(64, 48)] if quick else [(800, 600), (1920, 1080)]:
        r = renderer(scenes.cornell_scene(), w, h)
        rows = {}
        for halves in (False, True):
            r._next_sample = 0
            shard = distributed.ShardBuffer(r.device_scene(), w, h, rank=0, world=1, halves=halves)
            r.sample_features(16, shard)
            whole = shard.gather(with_features=True)
            rows[halves] = []
            for _ in range(8 if quick else 24):
                active = r.sample(SPP, shard, want_stats=False, adaptive=crit)
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    shard.gather_delta(whole, max(active, 1))
                    torch.cuda.synchronize()
                rows[halves].append((active, kernel_ms(prof, names[halves][:1]), kernel_ms(prof, names[halves][1:])))
            whole.close()
            shard.close()
        assert [a for a, _, _ in rows[False]] == [a for a, _, _ in rows[True]]  # the same pixels changed
        full = [i for i, (a, _, _) in enumerate(rows[False]) if a == w * h]
        part = [i for i, (a, _, _) in enumerate(rows[False]) if 0 < a < w * h]
        for label, idx in (("every pixel", full), ("part of the image", part)):
            if not idx:
                continue
            out = {"what": "kernels", "size": [w, h], "calls": label, "n_calls": len(idx),
                   "active_median": statistics.median(rows[False][i][0] for i in idx)}
            for halves in (False, True):
                key = "halves" if halves else "plain"
                out[key + "_export_ms_median"] = round(statistics.median(rows[halves][i][1] for i in idx), 4)
                out[key + "_import_ms_median"] = round(statistics.median(rows[halves][i][2] for i in idx), 4)
            print(json.dumps({**out, "gpu": gpu}), flush=True)
        r.close()


def ranks(gpu, quick):
    import torch.distributed as dist

    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    w, h = (64, 48) if quick else (800, 600)
    r = renderer(scenes.cornell_scene(), w, h).num_samples(128)
    shard = distributed.ShardBuffer(r.device_scene(), w, h, group=None, halves=True)
    r.sample_features(16, shard)
    # _GuidedShard.sample's steps, one by one, to time the delta exchange
    guided = distributed._GuidedShard(r, shard, CRIT_E)
    t_delta, actives, caps = [], [], []
    for _ in range(64):
        if guided.whole is None and shard.entries >= CRIT_E.min_entries:
            guided.whole = shard.gather(with_features=True)
        active = r.sample(SPP, shard, want_stats=False, adaptive=CRIT_E, guide_buffer=guided.whole)
        out = torch.empty(world, dtype=torch.int64)
        dist.all_gather_into_tensor(out, torch.tensor([active], dtype=torch.int64))
        counts = out.tolist()
        actives.append(sum(counts))
        if guided.whole is not None:
            dist.barrier()
            torch.cuda.synchronize()
            t = time.perf_counter()
            shard.gather_delta(guided.whole, max(counts))
            torch.cuda.synchronize()
            t_delta.append((time.perf_counter() - t) * 1e3)
            caps.append(max(counts))
        if sum(counts) == 0:
            break
    guided.close()
    shard.close()
    if rank == 0:
        print(json.dumps({"what": "sync", "size": [w, h], "world": world, "backend": "gloo, both ranks on one GPU through host memory",
                          "calls": len(actives), "active": actives, "capacity": caps,
                          "delta_block_bytes": [distributed.delta_block_layout(c, halves=True)["bytes"] for c in caps],
                          "gather_delta_ms_median": round(statistics.median(t_delta), 3) if t_delta else None,
                          "gather_delta_ms": [round(x, 3) for x in t_delta], "nccl_across_gpus": "not measured", "gpu": gpu}),
              flush=True)
    dist.barrier()
    torch.cuda.synchronize()
    t = time.perf_counter()
    r._next_sample = 0
    buf = distributed.render_iterative_distributed(r, SPP, lambda i, b: None, adaptive=CRIT_E)
    torch.cuda.synchronize()
    dist.barrier()
    sharded_s = time.perf_counter() - t
    buf.close()
    if rank == 0:
        r1 = renderer(scenes.cornell_scene(), w, h).num_samples(r._num_samples)
        b = r1.device_buffer(halves=True)
        torch.cuda.synchronize()
        t = time.perf_counter()
        r1.iterative_render(SPP, lambda i, bb: None, buffer=b, adaptive=CRIT_E)
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
    ap.add_argument("--only", default="bytes,kernels")
    a = ap.parse_args()
    gpu = card()
    only = a.only.split(",")
    if "bytes" in only:
        bytes_per_call(gpu, a.quick)
    if "kernels" in only:
        kernels(gpu, a.quick)
    if "ranks" in only:
        ranks(gpu, a.quick)


if __name__ == "__main__":
    main()
