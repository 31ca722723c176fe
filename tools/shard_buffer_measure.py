"""The exchange of a sharded device Buffer, measured on the GPU: ShardBuffer export + all_gather_into_tensor + import
into a whole buffer (what ShardBuffer.gather does), at 800x600 and 1920x1080, with and without the feature sums.  One
JSON line per size and feature choice, each with the card's name and power limit read in the same run.

Per call, after --warmup calls, the median over --reps of:
  export_ms   CUDA events around rptb_buffer_export_shard on the current stream (device-to-device copies)
  gather_ms   CUDA events around all_gather_into_tensor (NCCL; none at world 1, reported as 0)
  import_ms   host clock of rptb_buffer_import_shards: it reads the headers, runs the scatter / compact kernels and
              returns when it has read the gathered bytes
and the block size per rank and in total.

  python tools/shard_buffer_measure.py                                   world 1
  torchrun --nproc_per_node=N tools/shard_buffer_measure.py              world N, one GPU per rank, NCCL

World sizes the run did not have GPUs for are reported as not measured."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from rpt_b200 import _capi as capi  # noqa: E402
from rpt_b200 import api, scenes  # noqa: E402
from rpt_b200.distributed import ShardBuffer  # noqa: E402

SIZES = [(800, 600), (1920, 1080)]


def card(dev):
    try:
        line = subprocess.check_output(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
        name, limit = (s.strip() for s in line.split(","))
        return name, limit
    except Exception as e:  # noqa: BLE001
        return torch.cuda.get_device_name(dev), "unknown (%s)" % e


def measure(rank, world, dev, w, h, with_features, warmup, reps):
    cfg = scenes.sphere_scene()
    r = api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(2).seed(1).device(dev)
    buf = ShardBuffer(r.device_scene(), w, h, rank=rank, world=world)
    for _ in range(2):
        r.sample(1, buf, want_stats=False)
    r.sample_features(1, buf)
    nbytes = buf.block_bytes(with_features)
    mine = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    gathered = torch.empty(nbytes * world, dtype=torch.uint8, device=dev) if world > 1 else mine
    whole = api.DeviceBuffer(r.device_scene(), w, h)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    wf = 1 if with_features else 0
    rows = []
    for i in range(warmup + reps):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)
        ev[0].record()
        buf.export(mine, with_features)
        ev[1].record()
        if world > 1:
            dist.all_gather_into_tensor(gathered, mine)
        ev[2].record()
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        capi.check(capi.lib().rptb_buffer_import_shards(whole.handle, C.c_void_p(gathered.data_ptr()), world, wf),
                   "rptb_buffer_import_shards")
        t1 = time.perf_counter()
        if i >= warmup:
            rows.append((ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), (t1 - t0) * 1e3))
    whole.close()
    buf.close()
    r.close()
    med = [statistics.median(c) for c in zip(*rows)]
    return {"export_ms": round(med[0], 4), "gather_ms": round(med[1], 4) if world > 1 else 0.0,
            "import_ms": round(med[2], 4), "block_bytes": nbytes, "gathered_bytes": nbytes * world,
            "bytes_per_pixel": round(nbytes / (w * h), 3)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", dev))
    name, limit = card(dev)
    for (w, h) in SIZES:
        for wf in (False, True):
            res = measure(rank, world, dev, w, h, wf, a.warmup, a.reps)
            if rank == 0:
                print(json.dumps({"what": "shard_buffer_gather", "card": name, "power_limit": limit, "world": world,
                                  "width": w, "height": h, "with_features": wf, **res}), flush=True)
    if rank == 0:
        visible = torch.cuda.device_count()
        for n in (2, 4, 8):
            if n != world:
                why = "not measured" + ("" if n <= visible else " (%d GPU%s visible)" % (visible, "" if visible == 1 else "s"))
                print(json.dumps({"what": "shard_buffer_gather", "world": n, "result": why}), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
