"""Reprojection into shard buffers and the sharded frame loop, measured on the GPU (one JSON line per measurement, each
with the card's name and power limit read in the same run).

  kernels  single process: reproject_part_kernel summed over the n = 1, 2, 4, 8 shards of one destination (all
           simulated in this process), against the same kernel on the whole destination, at 800x600 and 1920x1080
           (Cornell, a 0.02 rad orbit step), per call from torch.profiler's CUDA kernel records over --reps calls after
           warm-up.  Also the source's gather and feature-resolve kernels, which every shard's call runs once (one per
           rank in a real run; n times here).
  frames   under torchrun, --backend gloo (every rank on cuda:0) or nccl (rank i on cuda:i): per frame of a 16-frame
           orbit (tools/reproject_measure.py's orbit_cameras) at 800x600, the host-clock wall time of
           render_frames_distributed and of Renderer.render_frames on one whole buffer (rank 0 alone, the other ranks
           waiting), and the loop's phases -- feature pass, reprojection, entries, gather (export + all-gather +
           import), image -- each ended by a device synchronise, from a copy of the loop.  The frames of both are
           compared byte for byte.

  python tools/shard_frames_measure.py --what kernels
  torchrun --nproc_per_node=2 tools/shard_frames_measure.py --what frames --backend gloo
  torchrun --nproc_per_node=N tools/shard_frames_measure.py --what frames --backend nccl     (N GPUs)"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from reproject_measure import MAX_BOUNCES, orbit_cameras  # noqa: E402
from rpt_b200 import _capi as capi  # noqa: E402
from rpt_b200 import api  # noqa: E402
from rpt_b200.distributed import ShardBuffer, render_frames_distributed  # noqa: E402


def card(dev):
    try:
        line = subprocess.check_output(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
        return [s.strip() for s in line.split(",")]
    except Exception as e:  # noqa: BLE001
        return [torch.cuda.get_device_name(dev), "unknown (%s)" % e]


def _kernel_ms(prof, reps):
    part = src = 0.0
    for e in prof.key_averages():
        us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if "reproject_part_kernel" in e.key:
            part += us
        elif "buffer_scatter" in e.key or "features_resolve" in e.key:
            src += us
    return part / 1e3 / reps, src / 1e3 / reps


def kernels(args, gpu):
    sizes = [(64, 48)] if args.quick else [(800, 600), (1920, 1080)]
    cfg, cams = orbit_cameras("cornell", 2, 0.02)
    prm = api.Reproject().to_c()
    n_out = C.c_uint64(0)
    for w, h in sizes:
        r = api.Renderer(cfg.scene, cams[0]).width(w).height(h).max_bounces(2).seed(1)
        ds = r.device_scene()
        src = r.device_buffer()
        for _ in range(4):
            r.sample(1, src, want_stats=False)
        r.sample_features(4, src)
        r.camera = cams[1]

        def dst(shard=None):
            b = r.device_buffer() if shard is None else ShardBuffer(ds, w, h, rank=shard[0], world=shard[1])
            r.sample_features(4, b)
            return b

        wholes = [dst() for _ in range(args.reps + 3)]
        for b in wholes[:3]:
            capi.check(capi.lib().rptb_buffer_reproject(b.handle, src.handle, C.byref(prm), C.byref(n_out)), "rptb_buffer_reproject")
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for b in wholes[3:]:
                capi.check(capi.lib().rptb_buffer_reproject(b.handle, src.handle, C.byref(prm), C.byref(n_out)), "rptb_buffer_reproject")
        torch.cuda.synchronize()
        whole_ms, whole_src_ms = _kernel_ms(prof, args.reps)
        reused_whole = int(n_out.value)
        for b in wholes:
            b.close()
        for n in (1, 2, 4, 8):
            sets = [[dst((i, n)) for i in range(n)] for _ in range(args.reps + 3)]
            for s in sets[0]:
                s.reproject_from(src)
            reused = []
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for shards in sets[3:]:
                    reused.append(sum(s.reproject_from(src) for s in shards))
            torch.cuda.synchronize()
            part_ms, src_ms = _kernel_ms(prof, args.reps)
            print(json.dumps({"what": "kernels", "size": [w, h], "shards": n, "reproject_part_kernel_ms_summed": round(part_ms, 4),
                              "reproject_part_kernel_ms_whole": round(whole_ms, 4),
                              "source_gather_resolve_ms_per_shard_call": round(src_ms / n, 4),
                              "source_gather_resolve_ms_whole_call": round(whole_src_ms, 4),
                              "reused_sum_equals_whole": all(x == reused_whole for x in reused), "gpu": gpu}), flush=True)
            for shards in sets:
                for s in shards:
                    s.close()
        src.close()
        r.close()


def _sync(dev, t):
    torch.cuda.synchronize(dev)
    return time.perf_counter() - t


def frames(args, gpu, rank, world, dev):
    w, h = (64, 48) if args.quick else (800, 600)
    entries, fspp, spp = 4, 8, args.spp
    for name in ("sphere", "cornell"):
        cfg, cams = orbit_cameras(name, args.frames, 0.02)

        def renderer():
            return api.Renderer(cfg.scene, cams[0]).width(w).height(h).max_bounces(MAX_BOUNCES[name]).seed(1).num_samples(spp).device(dev)

        # one whole buffer, rank 0 alone (a warm-up orbit first: module loads, first allocations)
        single_ms, want = [], []
        if rank == 0:
            for keep in (False, True):
                r = renderer()
                t = time.perf_counter()
                for img in r.render_frames(cams, entries=entries, feature_samples=fspp):
                    if keep:
                        single_ms.append(_sync(dev, t) * 1e3)
                        want.append(img.tobytes())
                    t = time.perf_counter()
                r.close()
        if world > 1:
            dist.barrier()
        # render_frames_distributed as it stands, after a warm-up orbit
        dist_ms, same = [], True
        for keep in (False, True):
            r = renderer()
            t = time.perf_counter()
            for i, img in enumerate(render_frames_distributed(r, cams, entries=entries, feature_samples=fspp)):
                if keep:
                    dist_ms.append(_sync(dev, t) * 1e3)
                    same = same and (rank != 0 or img.tobytes() == want[i])
                t = time.perf_counter()
            r.close()
        # its phases, from a copy of its loop with a synchronise after each
        r = renderer()
        phases = {k: [] for k in ("features", "reproject", "entries", "gather", "image")}
        prev = None
        for cam in cams:
            r.camera = cam
            buf = ShardBuffer(r.device_scene(), w, h, r._filter)
            t = time.perf_counter()
            r.sample_features(fspp, buf)
            phases["features"].append(_sync(dev, t))
            t = time.perf_counter()
            if prev is not None:
                buf.reproject_from(prev)
            phases["reproject"].append(_sync(dev, t))
            t = time.perf_counter()
            for _ in range(entries):
                r.sample(spp // entries, buf, want_stats=False)
            phases["entries"].append(_sync(dev, t))
            t = time.perf_counter()
            whole = buf.gather(with_features=True)
            phases["gather"].append(_sync(dev, t))
            buf.close()
            t = time.perf_counter()
            whole.image()
            phases["image"].append(_sync(dev, t))
            if prev is not None:
                prev.close()
            prev = whole
        prev.close()
        r.close()
        if rank == 0:
            med = {k + "_ms": round(statistics.median(v[1:]) * 1e3, 3) for k, v in phases.items()}
            print(json.dumps({"what": "frames", "scene": name, "size": [w, h], "world": world, "backend": args.backend,
                              "frames": args.frames, "spp_per_frame": spp, "feature_samples": fspp,
                              "render_frames_ms_median_1on": round(statistics.median(single_ms[1:]), 3),
                              "render_frames_distributed_ms_median_1on": round(statistics.median(dist_ms[1:]), 3),
                              "phases_median_1on": med, "same_bytes": same, "gpu": gpu}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes, for a rehearsal")
    ap.add_argument("--what", default="kernels", choices=["kernels", "frames"])
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl"])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--spp", type=int, default=16)
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = int(os.environ.get("LOCAL_RANK", "0")) if args.backend == "nccl" else 0
    torch.cuda.set_device(dev)
    gpu = card(dev)
    if args.what == "kernels":
        kernels(args, gpu)
        return
    if world > 1:
        if args.backend == "nccl":
            dist.init_process_group("nccl", device_id=torch.device("cuda", dev))
        else:
            dist.init_process_group("gloo")
    try:
        frames(args, gpu, rank, world, dev)
        if rank == 0 and args.backend == "gloo":
            visible = torch.cuda.device_count()
            print(json.dumps({"what": "frames", "backend": "nccl", "result": "not measured" if visible < 2 else
                              "run with --backend nccl (%d GPUs visible)" % visible}), flush=True)
    finally:
        if world > 1:
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
