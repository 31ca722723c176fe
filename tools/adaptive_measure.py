"""Adaptive sampling on the device Buffer, measured on the GPU (prints one JSON line per measurement; --out FILE
also writes every figure, the per-call rows included, to FILE).

  overhead   an always-active adaptive call (select + list-scheduled render + masked accumulate) against
             rptb_sample_into (render + accumulate) at the bench sizes of sphere and Cornell: host clock around each
             call, which ends in a device synchronise (both calls are given a stats struct), median of --reps
  scaling    per adaptive call while the active fraction falls: device time, segments, active pixels, listed warp
             blocks and active lanes per listed warp (active pixels / (32 x listed blocks), from the counts)
  tolerance  device time until every pixel meets the criterion, against uniform sampling at the spp the slowest pixel
             needed (that many plain calls, timed the same way), capped at 64 calls; plus a call with no pixel
             active (the select, a grid of CTAs that all leave at once, and the accumulate)

python tools/adaptive_measure.py [--quick] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C  # noqa: E402

from rpt_b200 import _capi as capi  # noqa: E402
from rpt_b200 import api, scenes  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def renderer(cfg, w, h):
    return api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(cfg.max_bounces).seed(1)


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t) * 1e3, out


def adaptive_call(r, n, buf, crit):
    ds, p, cam, c = r.device_scene(), r.params(n, r._next_sample), r.camera.to_c(), crit.to_c()
    active, st = C.c_uint64(0), capi.Stats()
    capi.check(capi.lib().rptb_sample_into_adaptive(ds.handle, C.byref(cam), C.byref(p), C.byref(c), buf.handle, C.byref(active),
                                                    C.byref(st)), "rptb_sample_into_adaptive")
    r._next_sample += n
    return int(active.value), st.as_dict()


def listed_blocks(taken, w, h):
    """8x4 warp blocks with at least one pixel that took the entry."""
    hp, wp = (h + 7) // 8 * 8, (w + 15) // 16 * 16
    m = np.zeros((hp, wp), bool)
    m[:h, :w] = taken.reshape(h, w)
    return int(m.reshape(hp // 4, 4, wp // 8, 8).any(axis=(1, 3)).sum())


def overhead(name, reps):
    cfg = scenes.CONFIGS[name]()
    r = renderer(cfg, cfg.width, cfg.height)
    always = api.Adaptive(0.0, 0.0, 1 << 30)
    plain_buf, ad_buf = r.device_buffer(), r.device_buffer()
    r.sample(cfg.spp, plain_buf)  # warm-up of both paths
    adaptive_call(r, cfg.spp, ad_buf, always)
    tp, ta, gp, ga = [], [], [], []
    for _ in range(reps):
        ms, _ = timed(lambda: r.sample(cfg.spp, plain_buf))
        tp.append(ms)
        gp.append(r.last_stats["gpu_ms"])
        ms, (_, st) = timed(lambda: adaptive_call(r, cfg.spp, ad_buf, always))
        ta.append(ms)
        ga.append(st["gpu_ms"])
    mp, ma = statistics.median(tp), statistics.median(ta)
    out = {"config": "%s %dx%d, %d spp per call, max_bounces %d" % (name, cfg.width, cfg.height, cfg.spp, cfg.max_bounces),
           "plain_call_ms": mp, "adaptive_call_ms": ma, "overhead_pct": 100.0 * (ma - mp) / mp,
           "plain_render_gpu_ms": statistics.median(gp), "adaptive_select_render_accumulate_gpu_ms": statistics.median(ga),
           "plain_ms_all": tp, "adaptive_ms_all": ta}
    plain_buf.close(), ad_buf.close(), r.close()
    return out


def tolerance(name, w, h, spp, crit, max_calls):
    cfg = scenes.glass_scene() if name == "glass" else scenes.CONFIGS[name]()
    r = renderer(cfg, w, h)
    buf = r.device_buffer()
    calls, total_ms = [], 0.0
    prev = np.zeros(w * h, np.uint32)
    for _ in range(max_calls):
        ms, (active, st) = timed(lambda: adaptive_call(r, spp, buf, crit))
        counts = buf.counts().reshape(-1)
        taken = counts > prev
        prev = counts
        blocks = listed_blocks(taken, w, h)
        calls.append({"active_fraction": active / (w * h), "call_ms": ms, "gpu_ms": st["gpu_ms"], "segments": st["segments"],
                      "listed_blocks": blocks, "active_lanes_per_listed_warp": 32.0 * active / (32 * blocks) if blocks else 0.0})
        total_ms += ms
        if active == 0:
            break
    converged = calls[-1]["active_fraction"] == 0.0
    # a call with no pixel active: the select, the grid of CTAs that leave at once, and the accumulate
    ms, (active, st) = timed(lambda: adaptive_call(r, spp, buf, api.Adaptive(0.0, 1e30, 2)))
    empty = {"active": active, "call_ms": ms, "gpu_ms": st["gpu_ms"], "segments": st["segments"]}
    slowest = int(prev.max())
    uni = r.device_buffer()
    ru = renderer(cfg, w, h)
    uni_ms = 0.0
    for _ in range(slowest):
        ms, _ = timed(lambda: ru.sample(spp, uni))
        uni_ms += ms
    seg_adaptive = sum(c["segments"] for c in calls)
    out = {"config": "%s %dx%d, %d spp per call, max_bounces %d" % (name, w, h, spp, cfg.max_bounces),
           "criterion": vars(crit), "converged": converged, "calls": len(calls), "slowest_pixel_entries": slowest,
           "mean_entries": float(prev.mean()), "adaptive_total_ms": total_ms, "uniform_ms_at_slowest_spp": uni_ms,
           "adaptive_segments": seg_adaptive, "empty_call": empty, "per_call": calls}
    buf.close(), uni.close(), r.close(), ru.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes: a rehearsal, not a measurement")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write all results, per-call rows included, as JSON to this file")
    a = ap.parse_args()
    res = {"card": card(), "overhead": [], "tolerance": []}
    if not a.quick:
        for name in ("cornell", "sphere"):
            res["overhead"].append(overhead(name, a.reps))
            print(json.dumps({k: v for k, v in res["overhead"][-1].items() if not k.endswith("_all")}), flush=True)
    crit = api.Adaptive(0.05, 2e-3, 4)
    sizes = {"sphere": (480, 270, 16), "cornell": (400, 400, 32), "glass": (480, 270, 32)}
    for name, (w, h, spp) in sizes.items():
        if a.quick:
            w, h, spp = w // 8, h // 8, 4
        t = tolerance(name, w, h, spp, crit, 12 if a.quick else 64)
        res["tolerance"].append(t)
        print(json.dumps({k: v for k, v in t.items() if k != "per_call"}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print("card:", res["card"])


if __name__ == "__main__":
    main()
