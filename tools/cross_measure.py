"""The cross-filtered denoiser with a smoothed selection map (rptb_buffer_denoise_cross), measured on the GPU: one JSON
line per measurement, each with the card's name and power limit read in the same run.  BASELINE.md section 3.0l holds
the results.

  cost         Cornell at 800x600 and 1920x1080, 8 entries of 2 spp and 16 feature rays in a buffer with halves, Denoise()
               (5 passes): the device time per call of every kernel of denoise_cross() against denoised_error() and
               denoise_select(), from torch.profiler's CUDA kernel records (copies excluded), after warm-up; --runs
               profiles of --reps calls each, alternating the three calls, for the spread
  quality      section 3.0k's protocol: sphere, Cornell, the BVH teapot and glass at 800x600 with their own max_bounces,
               16 / 64 / 256 spp as 8 equal entries with 16 feature rays; MSE (clamped to [0, 1]) against a --ref-spp
               render with another seed, of the raw mean, denoise(Denoise()), denoise_select(Denoise()) and
               denoise_cross(Denoise()); and the histogram of k*
  calibration  --seeds seeds at 128x128 (8 entries of 2 spp, 16 feature rays) per scene: per pixel, the mean over the
               seeds of M^ against the empirical MSE of the cross output (unclamped) around a --ref-spp render with
               another seed; the median ratio and the ratio of the image means
  levels       the quality protocol at 16 spp: the MSE of every candidate level O_k of the cross filter (tests/cross_ref.py
               on the buffer's read-backs) beside that of denoise(iterations = k), to tell the candidates' own error
               from the choice among them

python tools/cross_measure.py [--quick] [--ref-spp N] [--reps N] [--runs N] [--seeds N] [--only cost,quality,calibration,levels]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402  (torch.profiler: the library's kernels show up among the CUDA activity records)

from rpt_b200 import api, scenes  # noqa: E402

D = api.Denoise()
CONFIGS = [("sphere", scenes.sphere_scene), ("cornell", scenes.cornell_scene), ("teapot", scenes.teapot_scene),
           ("glass", lambda: scenes.glass_scene(512, 256))]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def renderer(cfg, w, h, seed):
    return api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(cfg.max_bounces).seed(seed)


def filled(r, spp, entries=8, features=16):
    b = r.device_buffer(halves=True)
    for _ in range(entries):
        r.sample(spp // entries, b, want_stats=False)
    r.sample_features(features, b)
    return b


def reference(cfg, w, h, ref_spp):
    rr = renderer(cfg, w, h, 777)
    per = max(1, ref_spp // 16)
    with rr.device_buffer() as b:
        for _ in range(16):
            rr.sample(per, b, want_stats=False)
        truth = b.sums().reshape(h, w, 3) / 16.0
    rr.close()
    return truth, per * 16


def kernels_ms(fn, reps):
    """Device time per call of every kernel fn() launches (copies and sets excluded), in total and by name."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    by = {}
    for e in prof.key_averages():
        if e.key.startswith("Memcpy") or e.key.startswith("Memset"):
            continue
        us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        name = e.key.split("(")[0].replace("void ", "").replace("rptb::", "")
        by[name] = by.get(name, 0.0) + us / 1e3 / reps
    return round(sum(by.values()), 4), {k: round(v, 4) for k, v in sorted(by.items()) if v > 0}


def cost(gpu, quick, reps, runs):
    cfg = scenes.cornell_scene()
    for w, h in [(64, 48)] if quick else [(800, 600), (1920, 1080)]:
        r = renderer(cfg, w, h, 1)
        b = filled(r, 16)
        calls = {"denoised_error": lambda: b.denoised_error(D), "denoise_select": lambda: b.denoise_select(D),
                 "denoise_cross": lambda: b.denoise_cross(D)}
        for _ in range(3):  # warm-up, and the planes' first allocation
            for fn in calls.values():
                fn()
        totals, by = {k: [] for k in calls}, {}
        for _ in range(runs):
            for name, fn in calls.items():
                t, per = kernels_ms(fn, reps)
                totals[name].append(t)
                by[name] = per
        row = {"what": "cost", "size": [w, h], "iterations": D.iterations, "reps": reps, "runs": runs, "gpu": gpu}
        for name, ts in totals.items():
            row[name + "_kernels_ms"] = round(float(np.median(ts)), 4)
            row[name + "_kernels_ms_runs"] = ts
        row["denoise_cross_by_kernel"] = by["denoise_cross"]
        print(json.dumps(row), flush=True)
        b.close()
        r.close()


def quality(gpu, quick, ref_spp):
    for name, mk in CONFIGS[:2] if quick else CONFIGS:
        cfg = mk()
        w, h = (64, 48) if quick else (800, 600)
        truth, used = reference(cfg, w, h, ref_spp)
        truth = np.clip(truth, 0, 1)

        def mse(x):
            return float(np.mean((np.clip(x, 0, 1) - truth) ** 2))

        for spp in (16, 64, 256):
            r = renderer(cfg, w, h, 1)
            b = filled(r, spp)
            sums, _, counts = b.pixel_stats()
            raw = sums.reshape(h, w, 3) / counts.reshape(h, w, 1)
            sel, _, _ = b.denoise_select(D)
            rgb, level, _ = b.denoise_cross(D)
            row = {"what": "quality", "scene": name, "size": [w, h], "spp": spp, "ref_spp": used, "mse_raw": mse(raw),
                   "mse_denoised": mse(b.denoise(D)), "mse_selected": mse(sel), "mse_cross": mse(rgb),
                   "levels": np.bincount(level.reshape(-1), minlength=D.iterations + 1).tolist(), "gpu": gpu}
            row["raw_over_denoised"] = round(row["mse_raw"] / row["mse_denoised"], 3)
            row["raw_over_cross"] = round(row["mse_raw"] / row["mse_cross"], 3)
            row["denoised_over_cross"] = round(row["mse_denoised"] / row["mse_cross"], 3)
            row["denoised_over_selected"] = round(row["mse_denoised"] / row["mse_selected"], 3)
            print(json.dumps(row), flush=True)
            b.close()
            r.close()


def calibration(gpu, quick, seeds, ref_spp):
    w = h = 32 if quick else 128
    for name, mk in CONFIGS[:3]:
        cfg = mk()
        truth, used = reference(cfg, w, h, ref_spp)
        errs, Ms, levels = [], [], []
        for k in range(seeds):
            r = renderer(cfg, w, h, 1000 + k)
            b = filled(r, 16)
            rgb, level, M = b.denoise_cross(D)
            errs.append(((rgb - truth) ** 2).mean(-1))
            Ms.append(M)
            levels.append(level)
            b.close()
            r.close()
        emp, Mbar = np.mean(errs, 0), np.mean(Ms, 0)
        ok = np.isfinite(emp) & np.isfinite(Mbar) & (Mbar > 0)
        print(json.dumps({"what": "calibration", "scene": name, "size": [w, h], "seeds": seeds, "ref_spp": used,
                          "median_emp_over_M": round(float(np.median(emp[ok] / Mbar[ok])), 3),
                          "mean_emp_over_mean_M": round(float(emp[ok].mean() / Mbar[ok].mean()), 3),
                          "levels": np.bincount(np.stack(levels).reshape(-1), minlength=D.iterations + 1).tolist(), "gpu": gpu}),
              flush=True)


def levels(gpu, quick, ref_spp):
    from tests import cross_ref as xref

    for name, mk in CONFIGS[:2] if quick else CONFIGS:
        cfg = mk()
        w, h = (64, 48) if quick else (800, 600)
        truth, used = reference(cfg, w, h, ref_spp)
        truth = np.clip(truth, 0, 1)

        def mse(x):
            return float(np.mean((np.clip(x, 0, 1) - truth) ** 2))

        r = renderer(cfg, w, h, 1)
        b = filled(r, 16)
        sums, m2, counts = b.pixel_stats()
        nrm, z, albedo, _ = b.features()
        state = (sums.reshape(h, w, 3), m2.reshape(h, w), b.half_sums().reshape(h, w, 3), counts.reshape(h, w), nrm, z, albedo)
        lv = xref.levels(*state, D)
        plain = [mse(b.denoise(api.Denoise(iterations=k))) for k in range(D.iterations + 1)]
        print(json.dumps({"what": "levels", "scene": name, "size": [w, h], "spp": 16, "ref_spp": used,
                          "mse_cross_level": [mse(o) for o, _, _ in lv], "mse_plain_level": plain, "gpu": gpu}), flush=True)
        b.close()
        r.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes, for a rehearsal")
    ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--seeds", type=int, default=16)
    ap.add_argument("--only", default="cost,quality,calibration,levels")
    args = ap.parse_args()
    gpu = card()
    only = args.only.split(",")
    if "cost" in only:
        cost(gpu, args.quick, args.reps, args.runs)
    if "quality" in only:
        quality(gpu, args.quick, args.ref_spp)
    if "calibration" in only:
        calibration(gpu, args.quick, args.seeds, args.ref_spp)
    if "levels" in only:
        levels(gpu, args.quick, args.ref_spp)


if __name__ == "__main__":
    main()
