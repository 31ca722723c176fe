"""Reprojected history with halves, measured on the GPU (one JSON line per measurement, each with the card's name and power
limit read in the same run).

  timing   the halves reprojection and merge kernels (reproject_halves_part_kernel, reproject_merge_halves_part_kernel)
           against the plain ones (reproject_part_kernel, reproject_merge_part_kernel) at 800x600 and 1920x1080
           (Cornell), --reps calls each after warm-up: device time per call from torch.profiler's CUDA kernel records.
  quality  the section 3.0c orbits (--frames frames, --step radians per frame) of sphere, Cornell, the BVH teapot and
           glass at 800x600 with 16 fresh spp per frame (4 entries of 4 spp, 8 feature samples per frame), each frame's
           history merged where the HistoryTest() agrees with its 2 plain fresh entries, then 2 more entries:
             error_guided   buffers with halves, the 2 entries guided on E (Adaptive(0.05, 1e-3, 4, Denoise(), "halves"))
             filter_guided  plain buffers, the same criterion on v' (estimate="filter")
             uniform        plain buffers, 2 plain entries
           Per mode: the denoised (Denoise()) MSE against a --ref-spp render of each frame with another seed, and the
           fresh samples rendered per pixel, both averaged over frames 1 on.
  calib    on reprojected frames: per --seeds seed, frame 0 (4 entries of 4 spp) reprojected into frame 1, then 2 entries
           of 2 spp; the median over pixels of (mean of E over the seeds) / (variance of c' over the seeds), and the same
           for v' (sphere, Cornell; 128x128).

python tools/reproject_halves_measure.py [--quick] [--ref-spp N] [--frames N] [--step RAD] [--reps N] [--seeds N]
                                         [--what timing,quality,calib]"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402  (torch.profiler: the library's kernels show up among the CUDA activity records)

from rpt_b200 import _capi as capi  # noqa: E402
from rpt_b200 import api  # noqa: E402
from reproject_measure import MAX_BOUNCES, card, orbit_cameras  # noqa: E402

GUIDE = api.Denoise()


def _kernel_ms(prof, names, reps):
    us = 0.0
    for e in prof.key_averages():
        if any(n in e.key for n in names):
            us += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
    return round(us / 1e3 / reps, 4)


def timing(args, gpu):
    sizes = [(64, 48)] if args.quick else [(800, 600), (1920, 1080)]
    cfg, cams = orbit_cameras("cornell", 2, 0.02)
    prm, gamma = api.Reproject().to_c(), api.HistoryTest().gamma
    n, j = C.c_uint64(0), C.c_uint64(0)
    L = capi.lib()
    for w, h in sizes:
        r = api.Renderer(cfg.scene, cams[0]).width(w).height(h).max_bounces(2).seed(1)
        out = {"what": "timing", "size": [w, h], "reps": args.reps, "gpu": gpu}
        for halves in (False, True):
            r.camera = cams[0]
            src = r.device_buffer(halves=halves)
            for _ in range(4):
                r.sample(1, src, want_stats=False)
            r.sample_features(4, src)
            r.camera = cams[1]
            for merge in (False, True):
                dsts = []
                for _ in range(args.reps + 3):
                    b = r.device_buffer(halves=halves)
                    r.sample_features(4, b)
                    for _ in range(2 if merge else 0):
                        r.sample(1, b, want_stats=False)
                    dsts.append(b)

                def call(b):
                    if merge:
                        capi.check(L.rptb_buffer_reproject_merge(b.handle, src.handle, C.byref(prm), gamma, C.byref(n), C.byref(j)), "merge")
                    else:
                        capi.check(L.rptb_buffer_reproject(b.handle, src.handle, C.byref(prm), C.byref(n)), "reproject")

                for b in dsts[:3]:  # warm-up: first allocations of both buffers' planes
                    call(b)
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for b in dsts[3:]:
                        call(b)
                    torch.cuda.synchronize()
                kern = ("reproject_merge_halves_part_kernel" if merge else "reproject_halves_part_kernel") if halves else \
                    ("reproject_merge_part_kernel" if merge else "reproject_part_kernel")
                key = ("merge" if merge else "reproject") + ("_halves" if halves else "_plain")
                out[key + "_kernel_ms"] = _kernel_ms(prof, [kern + "("], args.reps)
                out[key + "_call_kernels_ms"] = _kernel_ms(prof, ["rptb::"], args.reps)
                for b in dsts:
                    b.close()
            src.close()
        r.close()
        print(json.dumps(out), flush=True)


def _frames(r, cams, truth, mode, spp=16):
    """One orbit in `mode`: per frame (denoised MSE, fresh spp per pixel)."""
    halves = mode == "error_guided"
    crit = {"error_guided": api.Adaptive(0.05, 1e-3, 4, guide=GUIDE, estimate="halves"),
            "filter_guided": api.Adaptive(0.05, 1e-3, 4, guide=GUIDE), "uniform": None}[mode]
    test, prm = api.HistoryTest(), api.Reproject()
    prev, rows = None, []
    per = spp // 4
    for cam, t in zip(cams, truth):
        r.camera = cam
        buf = r.device_buffer(halves=halves)
        r.sample_features(8, buf)
        h, w = t.shape[:2]
        for _ in range(test.fresh_entries):
            r.sample(per, buf, want_stats=False)
        rendered = test.fresh_entries * per * w * h
        if prev is not None:
            buf.merge_history_from(prev, prm, test)
        for _ in range(4 - test.fresh_entries):
            before = int(buf.counts().sum())
            r.sample(per, buf, want_stats=False, adaptive=crit)
            rendered += (int(buf.counts().sum()) - before) * per
        den = np.clip(buf.denoise(GUIDE), 0, 1)
        rows.append((float(np.mean((den - t) ** 2)), rendered / (w * h)))
        if prev is not None:
            prev.close()
        prev = buf
    prev.close()
    return rows


def quality(args, gpu):
    w, h = (64, 48) if args.quick else (800, 600)
    for name in (["sphere", "cornell"] if args.quick else ["sphere", "cornell", "teapot", "glass"]):
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
        out = {"what": "quality", "scene": name, "size": [w, h], "spp_per_frame": 16, "frames": args.frames, "step_rad": args.step,
               "ref_spp": per * 16, "gpu": gpu}
        for mode in ("error_guided", "filter_guided", "uniform"):
            r = api.Renderer(cfg.scene, cams[0]).width(w).height(h).max_bounces(mb).seed(1)
            mse, fresh = zip(*_frames(r, cams, truth, mode))
            r.close()
            out[mode] = {"mse_denoised_mean_1on": float(np.mean(mse[1:])), "fresh_spp_mean_1on": float(np.mean(fresh[1:]))}
        print(json.dumps(out), flush=True)


def calib(args, gpu):
    w = h = 64 if args.quick else 128
    for name in ("sphere", "cornell"):
        cfg, cams = orbit_cameras(name, 2, args.step)
        cs, Es, vs = [], [], []
        for k in range(args.seeds):
            r = api.Renderer(cfg.scene, cams[0]).width(w).height(h).max_bounces(MAX_BOUNCES[name]).seed(1000 + k)
            src = r.device_buffer(halves=True)
            for _ in range(4):
                r.sample(4, src, want_stats=False)
            r.sample_features(16, src)
            r.camera = cams[1]
            b = r.device_buffer(halves=True)
            r.sample_features(16, b)
            b.reproject_from(src)
            for _ in range(2):
                r.sample(2, b, want_stats=False)  # every pixel: 2 entries or more
            cs.append(b.denoise(GUIDE))
            Es.append(b.denoised_error(GUIDE))
            vs.append(b.denoised_variance(GUIDE))
            for x in (src, b):
                x.close()
            r.close()
        emp = np.var(np.stack(cs), axis=0, ddof=1).mean(-1)
        Ebar, vbar = np.mean(Es, 0), np.mean(vs, 0)
        ok = np.isfinite(emp) & (emp > 0) & np.isfinite(Ebar) & np.isfinite(vbar)
        print(json.dumps({"what": "calib", "scene": name, "size": [w, h], "seeds": args.seeds, "step_rad": args.step,
                          "median_E_over_var_c": float(np.median(Ebar[ok] / emp[ok])),
                          "median_vprime_over_var_c": float(np.median(vbar[ok] / emp[ok])), "gpu": gpu}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes, for a rehearsal")
    ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--step", type=float, default=0.02)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--seeds", type=int, default=16)
    ap.add_argument("--what", default="timing,quality,calib", help="comma-separated: timing, quality, calib")
    args = ap.parse_args()
    args.what = set(args.what.split(","))
    gpu = card()
    if "timing" in args.what:
        timing(args, gpu)
    if "quality" in args.what:
        quality(args, gpu)
    if "calib" in args.what:
        calib(args, gpu)


if __name__ == "__main__":
    main()
