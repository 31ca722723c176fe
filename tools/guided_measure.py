"""Adaptive sampling guided by the denoiser (rptb_sample_into_guided), measured on the GPU: one JSON line per measurement,
each with the card's name and power limit read in the same run.  BASELINE.md section 3.0f holds the results.

  cost         Cornell at 800x600 and 1920x1080, 8 entries and 16 feature rays, guide Denoise() (5 passes): the device
               time per call of the guide's kernels (gather, resolve, demodulate, passes, mark) from torch.profiler's
               CUDA kernel records, and the host clock (median of --reps, each ending in a device synchronise) of a whole
               guided call against a plain adaptive call, both with rel_tol = abs_tol = 0 so that (nearly) every pixel is
               active in both -- the active counts are printed beside the times.
  calibration  32 seeds of the same buffer state (8 entries of 2 spp, 16 feature rays) per scene: the per-pixel variance
               over the seeds of the denoised colour c' (the channel mean of the per-channel variances, the units of v')
               against the mean over the seeds of v' (DeviceBuffer.denoised_variance).  The median ratio over all pixels
               with v' > 0 and over the edge band (pixels whose 4-neighbourhood has a normal turn of more than 25 degrees,
               a 5 % depth step, or a partial hit fraction).  The same ratio for the raw mean and its variance of the mean
               is printed as a control (it should be close to 1).
  quality      the section 3.0b protocol: the denoised image clamped to [0, 1] against a --ref-spp render with another seed.
               Uniform runs of 2, 4, 8, 16, 32 and 64 calls of 2 spp; plain adaptive and guided runs (min_entries 4, abs_tol
               1e-3, up to 64 calls of 2 spp) over a rel_tol sweep.  Each adaptive run is compared with the uniform runs
               at the call counts on either side of its mean spp, interpolated in log-log (MSE and wall time).

Scenes: sphere, Cornell, the BVH teapot (max_bounces 4) and glass at 800x600.

python tools/guided_measure.py [--quick] [--ref-spp N] [--reps N] [--seeds N] [--only cost,calibration,quality]"""
import argparse
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

GUIDE = api.Denoise()
SPP = 2  # samples per call in every run


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


def renderer(cfg, w, h, mb, seed, extra):
    r = api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(cfg.max_bounces if mb is None else mb).seed(seed)
    if "accel" in extra:
        r.accel(extra["accel"])
    return r


def sync():
    torch.cuda.synchronize()


def cost(gpu, quick, reps):
    sizes = [(64, 48)] if quick else [(800, 600), (1920, 1080)]
    for w, h in sizes:
        cfg = scenes.cornell_scene()
        r = renderer(cfg, w, h, None, 1, {})
        bufs = []
        for _ in range(2):
            b = r.device_buffer()
            r.sample_features(16, b)
            for _ in range(8):
                r.sample(SPP, b, want_stats=False)
            bufs.append(b)
        guided, plain = api.Adaptive(0.0, 0.0, 4, guide=GUIDE), api.Adaptive(0.0, 0.0, 4)
        for _ in range(2):  # warm-up
            r.sample(SPP, bufs[0], want_stats=False, adaptive=guided)
            r.sample(SPP, bufs[1], want_stats=False, adaptive=plain)
        tg, tp, ag, ap_ = [], [], [], []
        for _ in range(reps):  # alternated, each call ends in a synchronise (the active count is read back)
            t = time.perf_counter()
            ag.append(r.sample(SPP, bufs[0], want_stats=False, adaptive=guided))
            tg.append((time.perf_counter() - t) * 1e3)
            t = time.perf_counter()
            ap_.append(r.sample(SPP, bufs[1], want_stats=False, adaptive=plain))
            tp.append((time.perf_counter() - t) * 1e3)
        kinds = {"buffer_scatter": 0.0, "features_resolve": 0.0, "denoise_demodulate": 0.0, "denoise_pass": 0.0, "guided_mark": 0.0}
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                r.sample(SPP, bufs[0], want_stats=False, adaptive=guided)
            sync()
        for e in prof.key_averages():
            us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            for k in kinds:
                if k in e.key:
                    kinds[k] += us
        row = {"what": "cost", "size": [w, h], "iterations": GUIDE.iterations,
               "guide_kernels_ms": {k: round(v / 1e3 / reps, 4) for k, v in kinds.items()},
               "guide_kernels_total_ms": round(sum(kinds.values()) / 1e3 / reps, 3),
               "guided_call_ms_host_clock": round(statistics.median(tg), 3), "plain_call_ms_host_clock": round(statistics.median(tp), 3),
               "guided_active_median": int(statistics.median(ag)), "plain_active_median": int(statistics.median(ap_)),
               "pixels": w * h, "gpu": gpu}
        print(json.dumps(row), flush=True)
        for b in bufs:
            b.close()
        r.close()


def edge_band(N, z, f):
    """Pixels whose 4-neighbourhood turns the normal by more than 25 degrees, steps the depth by 5 %, or that a
    silhouette crosses (a hit fraction strictly between 0 and 1)."""
    H, W = z.shape
    band = (f > 0.0) & (f < 1.0)
    for dy, dx in ((0, 1), (1, 0)):
        a, b = (slice(0, H - dy), slice(0, W - dx)), (slice(dy, H), slice(dx, W))
        with np.errstate(invalid="ignore"):
            turn = (N[a] * N[b]).sum(-1) < math.cos(math.radians(25.0))
            step = np.abs(z[a] - z[b]) > 0.05 * np.minimum(z[a], z[b])
        e = turn | (step & np.isfinite(z[a]) & np.isfinite(z[b])) | (np.isfinite(z[a]) != np.isfinite(z[b]))
        band[a] |= e
        band[b] |= e
    return band


def calibration(gpu, quick, seeds):
    w, h = (64, 48) if quick else (800, 600)
    for name, mk, mb, extra in configs(quick):
        cfg = mk()
        r = None
        mean_c = m2_c = mean_raw = m2_raw = None
        vsum, rawv_sum = np.zeros((h, w)), np.zeros((h, w))
        band = None
        for k in range(seeds):
            r = renderer(cfg, w, h, mb, 1000 + k, extra)
            b = r.device_buffer()
            for _ in range(8):
                r.sample(SPP, b, want_stats=False)
            r.sample_features(16, b)
            c = b.denoise(GUIDE)
            v = b.denoised_variance(GUIDE)
            sums, m2, counts = b.pixel_stats()
            raw = sums.reshape(h, w, 3) / counts.reshape(h, w, 1)
            rawv = b.denoised_variance(api.Denoise(iterations=0))
            if band is None:
                N, z, _, f = b.features()
                band = edge_band(N, z, f)
                mean_c, m2_c, mean_raw, m2_raw = np.zeros_like(c), np.zeros_like(c), np.zeros_like(c), np.zeros_like(c)
            # Welford over the seeds, per pixel and channel
            d = c - mean_c
            mean_c += d / (k + 1)
            m2_c += d * (c - mean_c)
            d = raw - mean_raw
            mean_raw += d / (k + 1)
            m2_raw += d * (raw - mean_raw)
            vsum += v
            rawv_sum += rawv
            b.close()
            r.close()
        emp = (m2_c / (seeds - 1)).mean(-1)
        emp_raw = (m2_raw / (seeds - 1)).mean(-1)
        vbar, rawbar = vsum / seeds, rawv_sum / seeds
        ok = np.isfinite(vbar) & (vbar > 0) & np.isfinite(emp)
        ok_raw = np.isfinite(rawbar) & (rawbar > 0) & np.isfinite(emp_raw)
        ratio, ratio_raw = emp / np.where(ok, vbar, 1.0), emp_raw / np.where(ok_raw, rawbar, 1.0)
        row = {"what": "calibration", "scene": name, "size": [w, h], "seeds": seeds, "iterations": GUIDE.iterations,
               "median_empirical_over_v": round(float(np.median(ratio[ok])), 3),
               "median_empirical_over_v_edge_band": round(float(np.median(ratio[ok & band])), 3),
               "edge_band_fraction": round(float(band.mean()), 4),
               "raw_control_median_ratio": round(float(np.median(ratio_raw[ok_raw])), 3), "gpu": gpu}
        print(json.dumps(row), flush=True)


def run(cfg, w, h, mb, extra, calls, crit=None):
    """One run from an empty buffer: features, then up to `calls` calls of SPP samples (adaptive ones stop once a call
    renders nothing).  -> (mean spp per pixel, denoised image, wall ms, calls made)."""
    r = renderer(cfg, w, h, mb, 1, extra)
    b = r.device_buffer()
    sync()
    t = time.perf_counter()
    r.sample_features(16, b)
    made = 0
    for _ in range(calls):
        made += 1
        if crit is None:
            r.sample(SPP, b, want_stats=False)
        elif r.sample(SPP, b, want_stats=False, adaptive=crit) == 0:
            break
    img = b.denoise(GUIDE)  # ends in a synchronise
    ms = (time.perf_counter() - t) * 1e3
    spp = float(b.counts().mean()) * SPP
    b.close()
    r.close()
    return spp, img, ms, made


def loglog(x, xs, ys):
    """ys at x, interpolated in log-log between the neighbouring xs (None outside their range)."""
    for (x0, y0), (x1, y1) in zip(zip(xs, ys), zip(xs[1:], ys[1:])):
        if x0 <= x <= x1:
            u = (math.log(x) - math.log(x0)) / (math.log(x1) - math.log(x0))
            return math.exp(math.log(y0) + u * (math.log(y1) - math.log(y0)))
    return None


def quality(gpu, quick, ref_spp):
    w, h = (64, 48) if quick else (800, 600)
    uniform_calls = [2, 4, 8, 16, 32, 64]
    sweep_plain, sweep_guided = [0.02, 0.05, 0.1], [0.0025, 0.005, 0.01, 0.02, 0.05, 0.1]
    max_calls = 64
    for name, mk, mb, extra in configs(quick):
        cfg = mk()
        rr = renderer(cfg, w, h, mb, 777, extra)
        ref_buf = rr.device_buffer()
        per = max(1, ref_spp // 16)
        for _ in range(16):
            rr.sample(per, ref_buf, want_stats=False)
        truth = np.clip(ref_buf.sums().reshape(h, w, 3) / 16.0, 0, 1)
        ref_buf.close()
        rr.close()

        def mse(x):
            return float(np.mean((np.clip(x, 0, 1) - truth) ** 2))

        run(cfg, w, h, mb, extra, 2)  # warm-up
        us, um, ut = [], [], []
        for calls in uniform_calls:
            spp, img, ms, _ = run(cfg, w, h, mb, extra, calls)
            us.append(spp)
            um.append(mse(img))
            ut.append(ms)
            print(json.dumps({"what": "quality", "scene": name, "size": [w, h], "run": "uniform", "calls": calls, "mean_spp": spp,
                              "mse_denoised": um[-1], "wall_ms": round(ms, 1), "ref_spp": per * 16, "gpu": gpu}), flush=True)
        for kind, sweep in (("adaptive", sweep_plain), ("guided", sweep_guided)):
            for rel in sweep:
                crit = api.Adaptive(rel, 1e-3, 4, guide=GUIDE if kind == "guided" else None)
                spp, img, ms, made = run(cfg, w, h, mb, extra, max_calls, crit)
                m = mse(img)
                mu, tu = loglog(spp, us, um), loglog(spp, us, ut)
                print(json.dumps({"what": "quality", "scene": name, "size": [w, h], "run": kind, "rel_tol": rel, "mean_spp": round(spp, 3),
                                  "mse_denoised": m, "wall_ms": round(ms, 1), "calls": made,
                                  "uniform_mse_at_equal_spp": mu, "uniform_wall_ms_at_equal_spp": None if tu is None else round(tu, 1),
                                  "gain_over_uniform": None if mu is None else round(mu / m, 3), "ref_spp": per * 16, "gpu": gpu}),
                      flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes: a rehearsal, not a measurement")
    ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--seeds", type=int, default=32)
    ap.add_argument("--only", default="cost,calibration,quality")
    args = ap.parse_args()
    gpu = card()
    parts = args.only.split(",")
    if "cost" in parts:
        cost(gpu, args.quick, args.reps)
    if "calibration" in parts:
        calibration(gpu, args.quick, args.seeds)
    if "quality" in parts:
        quality(gpu, args.quick, args.ref_spp)


if __name__ == "__main__":
    main()
