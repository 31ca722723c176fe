"""The device Buffer's feature pass and denoiser, measured on the GPU (one JSON line per measurement, each with the card's
name and power limit read in the same run).

  features   device time of rptb_buffer_add_features (events around the launch) per camera ray sample, 16 samples
  denoise    rptb_buffer_denoise at 5 iterations after warm-up, --reps calls: the device time of the filter's kernels
             (demodulate, the five passes, remodulate) and of the gather / feature-resolve kernels before them, per call,
             from torch.profiler's CUDA kernel records; and the host clock around the whole call, which ends in a device
             synchronise (median)
  quality    MSE against a --ref-spp render with another seed, of the raw mean, Box(1) and the denoised image (clamped
             to [0, 1]), at 16, 64 and 256 spp as 8 equal entries with 16 feature samples

Scenes: sphere, Cornell, the BVH teapot and glass at 800x600, Cornell at 1920x1080, each with its own max_bounces.

python tools/denoise_measure.py [--quick] [--ref-spp N] [--reps N]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402  (torch.profiler: the library's kernels show up among the CUDA activity records)

from rpt_b200 import api, scenes  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def box(mean, radius):
    H, W, _ = mean.shape
    pad = np.pad(mean, ((radius, radius), (radius, radius), (0, 0)))
    ones = np.pad(np.ones((H, W, 1)), ((radius, radius), (radius, radius), (0, 0)))
    s, c = np.zeros_like(mean), np.zeros((H, W, 1))
    for dy in range(2 * radius + 1):
        for dx in range(2 * radius + 1):
            s += pad[dy:dy + H, dx:dx + W]
            c += ones[dy:dy + H, dx:dx + W]
    return s / c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes, for a rehearsal")
    ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    gpu = card()
    configs = [("sphere", scenes.sphere_scene, 800, 600), ("cornell", scenes.cornell_scene, 800, 600),
               ("teapot", scenes.teapot_scene, 800, 600), ("glass", lambda: scenes.glass_scene(512, 256), 800, 600),
               ("cornell", scenes.cornell_scene, 1920, 1080)]
    if args.quick:
        configs = [(n, mk, 64, 48) for n, mk, _, _ in configs[:2]]
    for name, mk, w, h in configs:
        cfg = mk()

        def renderer(seed):
            return api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(cfg.max_bounces).seed(seed)

        r = renderer(1)
        buf = r.device_buffer()
        r.sample(2, buf, want_stats=False)
        r.sample(2, buf, want_stats=False)
        r.sample_features(1, buf)  # warm-up
        r.sample_features(16, buf, want_stats=True)
        feat_ms = r.last_stats["gpu_ms"] / 16
        d = api.Denoise()
        for _ in range(3):
            buf.denoise(d)
        times = []
        dc = d.to_c()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                t = time.perf_counter()
                api.capi.check(api.capi.lib().rptb_buffer_denoise(buf.handle, api.C.byref(dc), None, None), "rptb_buffer_denoise")
                times.append((time.perf_counter() - t) * 1e3)
        filt = other = 0.0
        for e in prof.key_averages():
            us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if "denoise_" in e.key:
                filt += us
            elif "buffer_scatter" in e.key or "features_resolve" in e.key:
                other += us
        print(json.dumps({"what": "timing", "scene": name, "size": [w, h], "feature_ms_per_sample": round(feat_ms, 4),
                          "filter_kernels_ms_5it": round(filt / 1e3 / args.reps, 3), "gather_resolve_kernels_ms": round(other / 1e3 / args.reps, 3),
                          "call_ms_host_clock": round(statistics.median(times), 3), "gpu": gpu}), flush=True)
        buf.close()
        rr = renderer(777)
        ref_buf = rr.device_buffer()
        per = max(1, args.ref_spp // 16)
        for _ in range(16):
            rr.sample(per, ref_buf, want_stats=False)
        truth = np.clip(ref_buf.sums().reshape(h, w, 3) / 16.0, 0, 1)
        ref_buf.close()
        for spp in (16, 64, 256):
            r = renderer(1)
            b = r.device_buffer()
            for _ in range(8):
                r.sample(spp // 8, b, want_stats=False)
            r.sample_features(16, b)
            sums, _, counts = b.pixel_stats()
            raw = sums.reshape(h, w, 3) / counts.reshape(h, w, 1)

            def mse(x):
                return float(np.mean((np.clip(x, 0, 1) - truth) ** 2))

            row = {"what": "quality", "scene": name, "size": [w, h], "spp": spp, "ref_spp": per * 16, "mse_raw": mse(raw),
                   "mse_box1": mse(box(raw, 1)), "mse_denoised": mse(b.denoise(d)), "gpu": gpu}
            row["raw_over_denoised"] = round(row["mse_raw"] / row["mse_denoised"], 3)
            row["box1_over_denoised"] = round(row["mse_box1"] / row["mse_denoised"], 3)
            print(json.dumps(row), flush=True)
            b.close()
        r.close()


if __name__ == "__main__":
    main()
