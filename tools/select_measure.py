"""The choice of each pixel's number of filter passes (rptb_buffer_denoise_select), measured on the GPU: one JSON line per
measurement, each with the card's name and power limit read in the same run.  BASELINE.md section 3.0k holds the results.

  cost         Cornell at 800x600 and 1920x1080, 8 entries of 2 spp and 16 feature rays in a buffer with halves, Denoise()
               (5 passes): the device time per call of every kernel of denoise_select() against denoised_error(), from
               torch.profiler's CUDA kernel records (copies excluded), after warm-up
  quality      section 3.0b's protocol: sphere, Cornell, the BVH teapot and glass at 800x600 with their own max_bounces,
               16 / 64 / 256 spp as 8 equal entries with 16 feature rays; MSE (clamped to [0, 1]) against a --ref-spp
               render with another seed, of the raw mean, denoise(Denoise()) and denoise_select(Denoise()); and the
               histogram of the chosen levels
  calibration  --seeds seeds at 128x128 (8 entries of 2 spp, 16 feature rays) per scene: per pixel, the mean over the
               seeds of M at the chosen level against the empirical MSE of the selected output (unclamped) around a
               --ref-spp render with another seed; the median ratio and the ratio of the image means

python tools/select_measure.py [--quick] [--ref-spp N] [--reps N] [--seeds N] [--only cost,quality,calibration]"""
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


def cost(gpu, quick, reps):
    cfg = scenes.cornell_scene()
    for w, h in [(64, 48)] if quick else [(800, 600), (1920, 1080)]:
        r = renderer(cfg, w, h, 1)
        b = filled(r, 16)
        for _ in range(3):  # warm-up, and the planes' first allocation
            b.denoise_select(D)
            b.denoised_error(D)
        err_total, err_by = kernels_ms(lambda: b.denoised_error(D), reps)
        sel_total, sel_by = kernels_ms(lambda: b.denoise_select(D), reps)
        print(json.dumps({"what": "cost", "size": [w, h], "iterations": D.iterations, "denoised_error_kernels_ms": err_total,
                          "denoise_select_kernels_ms": sel_total, "denoised_error_by_kernel": err_by,
                          "denoise_select_by_kernel": sel_by, "reps": reps, "gpu": gpu}), flush=True)
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
            rgb, level, _ = b.denoise_select(D)
            row = {"what": "quality", "scene": name, "size": [w, h], "spp": spp, "ref_spp": used, "mse_raw": mse(raw),
                   "mse_denoised": mse(b.denoise(D)), "mse_selected": mse(rgb),
                   "levels": np.bincount(level.reshape(-1), minlength=D.iterations + 1).tolist(), "gpu": gpu}
            row["raw_over_denoised"] = round(row["mse_raw"] / row["mse_denoised"], 3)
            row["raw_over_selected"] = round(row["mse_raw"] / row["mse_selected"], 3)
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
            rgb, level, M = b.denoise_select(D)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes, for a rehearsal")
    ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--seeds", type=int, default=16)
    ap.add_argument("--only", default="cost,quality,calibration")
    args = ap.parse_args()
    gpu = card()
    only = args.only.split(",")
    if "cost" in only:
        cost(gpu, args.quick, args.reps)
    if "quality" in only:
        quality(gpu, args.quick, args.ref_spp)
    if "calibration" in only:
        calibration(gpu, args.quick, args.seeds, args.ref_spp)


if __name__ == "__main__":
    main()
