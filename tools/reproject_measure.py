"""Reprojection of the device Buffer across camera moves, measured on the GPU (one JSON line per measurement, each with the
card's name and power limit read in the same run).

  quality  a --frames orbit (--step radians per frame about the vertical axis through the scene's centre) of sphere,
           Cornell, the BVH teapot and glass at 800x600, at 4 and 16 fresh spp per frame (4 entries of spp / 4, 8 feature
           samples per frame).  Modes: fresh (a new buffer per frame), reprojected (the previous frame's buffer
           reprojected into the new one first), reprojected + adaptive (the entries are adaptive ones, Adaptive(0.05,
           1e-3, 4), so they go to the disocclusions and the noisy pixels first), tested and tested + adaptive (the default
           HistoryTest(): its fresh_entries plain entries first, the history merged where it agrees with them
           (rptb_buffer_reproject_merge), then the other entries, plain or adaptive); each also denoised (Denoise()).  Per
           frame: MSE of the clamped mean image against a --ref-spp render of that frame with another seed, the fraction
           of pixels reused, and the fresh samples actually rendered per pixel.
  sweep    the reprojected mode, raw and denoised, at 4 and 16 spp on the same orbits for a grid of rptb_reproject
           parameter sets (the defaults' evidence)
  tsweep   the tested mode, raw and denoised, at 4 and 16 spp on the same orbits for HistoryTest gamma in {2, 3, 4, 6}
           x fresh_entries in {2, 4} (the default gamma's evidence), with the fresh spp rendered and the rejected fraction
  timing   rptb_buffer_reproject after warm-up, --reps calls, at 800x600 and 1920x1080 (Cornell): the device time of the
           reprojection kernel (reproject_part_kernel), of the source's gather / feature-resolve kernels before it and of
           the call's kernels together, per call, from torch.profiler's CUDA kernel records; and the host clock of the whole
           call with out_reused (median).  The same for rptb_buffer_reproject_merge into buffers holding two fresh entries
           (its kernel reproject_merge_part_kernel).

python tools/reproject_measure.py [--quick] [--ref-spp N] [--frames N] [--step RAD] [--reps N]
                                  [--what timing,quality,sweep,tsweep]"""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402  (torch.profiler: the library's kernels show up among the CUDA activity records)

from rpt_b200 import _capi as capi  # noqa: E402
from rpt_b200 import api, scenes  # noqa: E402

CENTER = {"sphere": (0.0, -0.25, 0.0), "cornell": (278.0, 273.0, 280.0), "teapot": (0.0, 0.0, 0.0), "glass": (0.0, 0.0, 0.0)}
MAKE = {"sphere": scenes.sphere_scene, "cornell": scenes.cornell_scene, "teapot": scenes.teapot_scene,
        "glass": lambda: scenes.glass_scene(512, 256)}
MAX_BOUNCES = {"sphere": 4, "cornell": 6, "teapot": 4, "glass": 12}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def orbit_cameras(name, frames, step):
    cfg = MAKE[name]()
    c = np.asarray(CENTER[name])
    d = cfg.camera.eye - c
    out = []
    for i in range(frames):
        a = step * i
        eye = c + np.array([math.cos(a) * d[0] + math.sin(a) * d[2], d[1], -math.sin(a) * d[0] + math.cos(a) * d[2]])
        out.append(api.Camera.look_at(eye, c, api.vec3(0.0, 1.0, 0.0), cfg.camera.fov))
    return cfg, out


def frames_run(r, cams, spp, reproject, adaptive, d, truth, test=None):
    """One orbit: per frame (mse raw, mse denoised, reused fraction, fresh samples per pixel, rejected fraction).  With
    `test` (an api.HistoryTest) the frame is render_frames(history_test=test)'s: fresh plain entries, the merge, the rest."""
    prev, rows = None, []
    entries = 4
    for cam, t in zip(cams, truth):
        r.camera = cam
        buf = r.device_buffer()
        r.sample_features(8, buf)
        h, w = t.shape[:2]
        reused = rejected = rendered = 0
        first = 0
        if test is not None:
            first = test.fresh_entries
            for _ in range(first):
                r.sample(spp // entries, buf, want_stats=False)
            rendered = first * w * h
            if prev is not None:
                reused, rejected = buf.merge_history_from(prev, reproject, test)
        elif prev is not None and reproject is not None:
            reused = buf.reproject_from(prev, reproject)
        before = int(buf.counts().sum())
        for _ in range(entries - first):
            r.sample(spp // entries, buf, want_stats=False, adaptive=adaptive)
        sums, _, counts = buf.pixel_stats()
        fresh = float((rendered + int(counts.sum()) - before) * (spp // entries)) / (w * h)
        raw = np.clip(sums.reshape(h, w, 3) / counts.reshape(h, w, 1), 0, 1)
        den = np.clip(buf.denoise(d), 0, 1)
        rows.append((float(np.mean((raw - t) ** 2)), float(np.mean((den - t) ** 2)), reused / (w * h), fresh, rejected / (w * h)))
        if prev is not None:
            prev.close()
        prev = buf
    prev.close()
    return rows


def quality(args, gpu):
    w, h = (64, 48) if args.quick else (800, 600)
    names = ["sphere", "cornell"] if args.quick else ["sphere", "cornell", "teapot", "glass"]
    d = api.Denoise()
    for name in names:
        cfg, cams = orbit_cameras(name, args.frames, args.step)
        mb = MAX_BOUNCES[name]
        rr = api.Renderer(cfg.scene, cams[0]).width(w).height(h).max_bounces(mb).seed(777)
        per = max(1, args.ref_spp // 16)
        truth = []
        for cam in cams:
            rr.camera = cam
            b = rr.device_buffer()
            for _ in range(16):
                rr.sample(per, b, want_stats=False)
            truth.append(np.clip(b.sums().reshape(h, w, 3) / 16.0, 0, 1))
            b.close()
        rr.close()
        crit, test = api.Adaptive(0.05, 1e-3, 4), api.HistoryTest()
        modes = {"fresh": (None, None, None), "reprojected": (api.Reproject(), None, None),
                 "reprojected_adaptive": (api.Reproject(), crit, None), "tested": (api.Reproject(), None, test),
                 "tested_adaptive": (api.Reproject(), crit, test)}
        for spp in (4, 16) if "quality" in args.what else ():
            for mode, (rep, ad, ht) in modes.items():
                r = api.Renderer(cfg.scene, cams[0]).width(w).height(h).max_bounces(mb).seed(1)
                rows = frames_run(r, cams, spp, rep, ad, d, truth, ht)
                r.close()
                raw, den, reused, fresh, rejected = (list(x) for x in zip(*rows))
                out = {"what": "quality", "scene": name, "size": [w, h], "spp_per_frame": spp, "mode": mode, "frames": args.frames,
                       "step_rad": args.step, "ref_spp": per * 16, "mse_raw": raw, "mse_denoised": den, "reused": reused,
                       "rejected": rejected, "fresh_spp": fresh, "mse_raw_mean_1on": float(np.mean(raw[1:])),
                       "mse_denoised_mean_1on": float(np.mean(den[1:])), "fresh_spp_mean_1on": float(np.mean(fresh[1:])),
                       "reprojection": vars(rep) if rep else None, "history_test": vars(ht) if ht else None, "gpu": gpu}
                print(json.dumps(out), flush=True)
        grid = [(dt, 0.9, mh) for dt in (0.01, 0.02, 0.05) for mh in (8, 16, 32)] + [(0.02, 0.5, 16), (0.02, 0.97, 16), (0.2, 0.9, 16)]
        for spp in (4, 16) if "sweep" in args.what else ():
            for prm in (api.Reproject(*g) for g in grid):
                r = api.Renderer(cfg.scene, cams[0]).width(w).height(h).max_bounces(mb).seed(1)
                rows = frames_run(r, cams, spp, prm, None, d, truth)
                r.close()
                raw, den, reused = (list(x) for x in list(zip(*rows))[:3])
                print(json.dumps({"what": "sweep", "scene": name, "size": [w, h], "spp_per_frame": spp, "reprojection": vars(prm),
                                  "mse_raw_mean_1on": float(np.mean(raw[1:])), "mse_denoised_mean_1on": float(np.mean(den[1:])),
                                  "reused_mean_1on": float(np.mean(reused[1:])), "gpu": gpu}), flush=True)
        for spp in (4, 16) if "tsweep" in args.what else ():
            for gamma in (2.0, 3.0, 4.0, 6.0):
                for fe in (2, 4):
                    ht = api.HistoryTest(gamma, fe)
                    r = api.Renderer(cfg.scene, cams[0]).width(w).height(h).max_bounces(mb).seed(1)
                    rows = frames_run(r, cams, spp, api.Reproject(), None, d, truth, ht)
                    r.close()
                    raw, den, reused, fresh, rejected = (list(x) for x in zip(*rows))
                    print(json.dumps({"what": "tsweep", "scene": name, "size": [w, h], "spp_per_frame": spp, "history_test": vars(ht),
                                      "mse_raw_mean_1on": float(np.mean(raw[1:])), "mse_denoised_mean_1on": float(np.mean(den[1:])),
                                      "reused_mean_1on": float(np.mean(reused[1:])), "rejected_mean_1on": float(np.mean(rejected[1:])),
                                      "fresh_spp_mean_1on": float(np.mean(fresh[1:])), "gpu": gpu}), flush=True)


def timing(args, gpu):
    sizes = [(64, 48)] if args.quick else [(800, 600), (1920, 1080)]
    cfg, cams = orbit_cameras("cornell", 2, 0.02)
    for w, h in sizes:
        r = api.Renderer(cfg.scene, cams[0]).width(w).height(h).max_bounces(2).seed(1)
        src = r.device_buffer()
        for _ in range(4):
            r.sample(1, src, want_stats=False)
        r.sample_features(4, src)
        r.camera = cams[1]
        dsts = []
        for _ in range(args.reps + 3):
            b = r.device_buffer()
            r.sample_features(4, b)
            dsts.append(b)
        prm = api.Reproject().to_c()
        n = C.c_uint64(0)
        for b in dsts[:3]:  # warm-up: first allocations of both buffers' planes
            capi.check(capi.lib().rptb_buffer_reproject(b.handle, src.handle, C.byref(prm), C.byref(n)), "rptb_buffer_reproject")
        times = []
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for b in dsts[3:]:
                t = time.perf_counter()
                capi.check(capi.lib().rptb_buffer_reproject(b.handle, src.handle, C.byref(prm), C.byref(n)), "rptb_buffer_reproject")
                times.append((time.perf_counter() - t) * 1e3)
        kern = gather = 0.0
        for e in prof.key_averages():
            us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if "reproject_part_kernel" in e.key:
                kern += us
            elif "buffer_scatter" in e.key or "features_resolve" in e.key:
                gather += us
        print(json.dumps({"what": "timing", "size": [w, h], "reproject_part_kernel_ms": round(kern / 1e3 / args.reps, 4),
                          "gather_resolve_kernels_ms": round(gather / 1e3 / args.reps, 4), "call_kernels_ms": round((kern + gather) / 1e3 / args.reps, 4),
                          "call_ms_host_clock": round(statistics.median(times), 3), "reused": int(n.value), "gpu": gpu}), flush=True)
        for b in dsts:
            b.close()
        # the merge: into buffers holding their features and two fresh entries
        dsts = []
        for _ in range(args.reps + 3):
            b = r.device_buffer()
            r.sample_features(4, b)
            for _ in range(2):
                r.sample(1, b, want_stats=False)
            dsts.append(b)
        gamma, j = api.HistoryTest().gamma, C.c_uint64(0)
        for b in dsts[:3]:
            capi.check(capi.lib().rptb_buffer_reproject_merge(b.handle, src.handle, C.byref(prm), gamma, C.byref(n), C.byref(j)),
                       "rptb_buffer_reproject_merge")
        times = []
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for b in dsts[3:]:
                t = time.perf_counter()
                capi.check(capi.lib().rptb_buffer_reproject_merge(b.handle, src.handle, C.byref(prm), gamma, C.byref(n), C.byref(j)),
                           "rptb_buffer_reproject_merge")
                times.append((time.perf_counter() - t) * 1e3)
        kern = gather = 0.0
        for e in prof.key_averages():
            us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if "reproject_merge_part_kernel" in e.key:
                kern += us
            elif "buffer_scatter" in e.key or "features_resolve" in e.key:
                gather += us
        print(json.dumps({"what": "timing_merge", "size": [w, h], "reproject_merge_part_kernel_ms": round(kern / 1e3 / args.reps, 4),
                          "gather_resolve_kernels_ms": round(gather / 1e3 / args.reps, 4), "call_kernels_ms": round((kern + gather) / 1e3 / args.reps, 4),
                          "call_ms_host_clock": round(statistics.median(times), 3), "reused": int(n.value), "rejected": int(j.value),
                          "gamma": gamma, "gpu": gpu}), flush=True)
        for b in dsts:
            b.close()
        src.close()
        r.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes, for a rehearsal")
    ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--step", type=float, default=0.02)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--what", default="timing,quality,sweep", help="comma-separated: timing, quality, sweep, tsweep")
    args = ap.parse_args()
    args.what = set(args.what.split(","))
    gpu = card()
    if "timing" in args.what:
        timing(args, gpu)
    if args.what & {"quality", "sweep", "tsweep"}:
        quality(args, gpu)


if __name__ == "__main__":
    main()
