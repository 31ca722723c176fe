"""The denoised image's error from two half buffers (rptb_buffer_denoise_error, rptb_sample_into_guided_error), measured on
the GPU: one JSON line per measurement, each with the card's name and power limit read in the same run.  BASELINE.md
section 3.0h holds the results.  The protocols are tools/guided_measure.py's (section 3.0f), whose helpers this reuses.

  cost         Cornell at 800x600 and 1920x1080, 8 entries and 16 feature rays, guide Denoise() (5 passes): per call, the
               device time of the accumulate kernels of a plain entry into a buffer with and without halves, and of the
               guide's kernels of a guided call on E against one on v' (torch.profiler's CUDA kernel records), with
               rel_tol = abs_tol = 0 so that every pixel is active; and the bytes per pixel of each buffer's planes.
  calibration  --seeds seeds of the same buffer state (8 entries of 2 spp, 16 feature rays) per scene, in a buffer with
               halves: the per-pixel variance over the seeds of c' against the mean of E and, as in section 3.0f, of v';
               the median ratio over all pixels and over the edge band.
  quality      section 3.0f's protocol for Adaptive(guide=Denoise(), estimate="filter") and estimate="halves" over a
               rel_tol sweep, against uniform runs at equal spp; each run reports its mean spp and calls (cap 64).

python tools/halves_measure.py [--quick] [--ref-spp N] [--reps N] [--seeds N] [--only cost,calibration,quality]"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import guided_measure as gm  # noqa: E402
import torch  # noqa: E402

from rpt_b200 import api  # noqa: E402

GUIDE = gm.GUIDE
SPP = gm.SPP


def _kernel_ms(fn, reps, names):
    """Device time per call of the kernels whose names contain each of `names`, over `reps` calls of fn()."""
    out = {k: 0.0 for k in names}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        gm.sync()
    for e in prof.key_averages():
        us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        for k in names:
            if k in e.key:
                out[k] += us
    return {k: round(v / 1e3 / reps, 4) for k, v in out.items()}


def cost(gpu, quick, reps):
    sizes = [(64, 48)] if quick else [(800, 600), (1920, 1080)]
    cfg = gm.scenes.cornell_scene()
    for w, h in sizes:
        r = gm.renderer(cfg, w, h, None, 1, {})
        bufs = {}
        for halves in (False, True):
            b = r.device_buffer(halves=halves)
            r.sample_features(16, b)
            for _ in range(8):
                r.sample(SPP, b, want_stats=False)
            bufs[halves] = b
        filt = api.Adaptive(0.0, 0.0, 4, guide=GUIDE)
        err = api.Adaptive(0.0, 0.0, 4, guide=GUIDE, estimate="halves")
        for _ in range(2):  # warm-up
            r.sample(SPP, bufs[True], want_stats=False, adaptive=err)
            r.sample(SPP, bufs[True], want_stats=False, adaptive=filt)
            r.sample(SPP, bufs[False], want_stats=False)
        acc = ["buffer_accumulate_kernel"]  # plain or halves: the buffer decides the instantiation
        plain = _kernel_ms(lambda: r.sample(SPP, bufs[False], want_stats=False), reps, acc)
        halves = _kernel_ms(lambda: r.sample(SPP, bufs[True], want_stats=False), reps, acc)
        guide = ["buffer_scatter", "features_resolve", "denoise_demodulate", "denoise_pass", "halves_demodulate",
                 "halves_pass", "halves_error", "guided_mark"]
        on_v = _kernel_ms(lambda: r.sample(SPP, bufs[True], want_stats=False, adaptive=filt), reps, guide)
        on_e = _kernel_ms(lambda: r.sample(SPP, bufs[True], want_stats=False, adaptive=err), reps, guide)
        row = {"what": "cost", "size": [w, h], "iterations": GUIDE.iterations,
               "accumulate_ms_plain_buffer": plain["buffer_accumulate_kernel"],
               "accumulate_ms_halves_buffer": halves["buffer_accumulate_kernel"],
               "guide_kernels_ms_filter": on_v, "guide_total_ms_filter": round(sum(on_v.values()), 3),
               "guide_kernels_ms_halves": on_e, "guide_total_ms_halves": round(sum(on_e.values()), 3),
               "buffer_bytes_per_pixel": {"plain": 3 * 8 + 8 + 4, "halves": 3 * 8 + 8 + 4 + 24}, "gpu": gpu}
        print(json.dumps(row), flush=True)
        for b in bufs.values():
            b.close()
        r.close()


def calibration(gpu, quick, seeds):
    w, h = (64, 48) if quick else (800, 600)
    for name, mk, mb, extra in gm.configs(quick):
        cfg = mk()
        n = 0
        mean_c = m2_c = None
        Esum, vsum = np.zeros((h, w)), np.zeros((h, w))
        band = None
        for k in range(seeds):
            r = gm.renderer(cfg, w, h, mb, 1000 + k, extra)
            b = r.device_buffer(halves=True)
            for _ in range(8):
                r.sample(SPP, b, want_stats=False)
            r.sample_features(16, b)
            c = b.denoise(GUIDE)
            Esum += b.denoised_error(GUIDE)
            vsum += b.denoised_variance(GUIDE)
            if band is None:
                N, z, _, f = b.features()
                band = gm.edge_band(N, z, f)
                mean_c, m2_c = np.zeros_like(c), np.zeros_like(c)
            n += 1
            d = c - mean_c
            mean_c += d / n
            m2_c += d * (c - mean_c)
            b.close()
            r.close()
        emp = (m2_c / (seeds - 1)).mean(-1)
        Ebar, vbar = Esum / seeds, vsum / seeds
        ok = np.isfinite(emp) & np.isfinite(Ebar) & (Ebar > 0) & np.isfinite(vbar) & (vbar > 0)
        rE, rv = emp / np.where(ok, Ebar, 1.0), emp / np.where(ok, vbar, 1.0)
        row = {"what": "calibration", "scene": name, "size": [w, h], "seeds": seeds, "iterations": GUIDE.iterations,
               "median_empirical_over_E": round(float(np.median(rE[ok])), 3),
               "median_empirical_over_E_edge_band": round(float(np.median(rE[ok & band])), 3),
               "median_empirical_over_v": round(float(np.median(rv[ok])), 3),
               "median_empirical_over_v_edge_band": round(float(np.median(rv[ok & band])), 3),
               "edge_band_fraction": round(float(band.mean()), 4), "gpu": gpu}
        print(json.dumps(row), flush=True)


def run(cfg, w, h, mb, extra, calls, crit=None):
    """gm.run in a buffer with halves (the uniform runs too, so that every run does the same accumulate work)."""
    r = gm.renderer(cfg, w, h, mb, 1, extra)
    b = r.device_buffer(halves=True)
    gm.sync()
    t = time.perf_counter()
    r.sample_features(16, b)
    made = 0
    for _ in range(calls):
        made += 1
        if crit is None:
            r.sample(SPP, b, want_stats=False)
        elif r.sample(SPP, b, want_stats=False, adaptive=crit) == 0:
            break
    img = b.denoise(GUIDE)
    ms = (time.perf_counter() - t) * 1e3
    spp = float(b.counts().mean()) * SPP
    b.close()
    r.close()
    return spp, img, ms, made


def quality(gpu, quick, ref_spp, sweep):
    w, h = (64, 48) if quick else (800, 600)
    uniform_calls = [2, 4, 8, 16, 32, 64]
    max_calls = 64
    for name, mk, mb, extra in gm.configs(quick):
        cfg = mk()
        rr = gm.renderer(cfg, w, h, mb, 777, extra)
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
        us, um = [], []
        for calls in uniform_calls:
            spp, img, ms, _ = run(cfg, w, h, mb, extra, calls)
            us.append(spp)
            um.append(mse(img))
        for estimate in ("filter", "halves"):
            for rel in sweep:
                crit = api.Adaptive(rel, 1e-3, 4, guide=GUIDE, estimate=estimate)
                spp, img, ms, made = run(cfg, w, h, mb, extra, max_calls, crit)
                m = mse(img)
                mu = gm.loglog(spp, us, um)
                print(json.dumps({"what": "quality", "scene": name, "size": [w, h], "estimate": estimate, "rel_tol": rel,
                                  "mean_spp": round(spp, 3), "mse_denoised": m, "wall_ms": round(ms, 1), "calls": made,
                                  "ended_before_cap": made < max_calls,
                                  "uniform_mse_at_equal_spp": mu, "gain_over_uniform": None if mu is None else round(mu / m, 3),
                                  "ref_spp": per * 16, "gpu": gpu}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes: a rehearsal, not a measurement")
    ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--seeds", type=int, default=32)
    ap.add_argument("--sweep", default="0.005,0.01,0.02,0.05,0.1")
    ap.add_argument("--only", default="cost,calibration,quality")
    args = ap.parse_args()
    gpu = gm.card()
    parts = args.only.split(",")
    if "cost" in parts:
        cost(gpu, args.quick, args.reps)
    if "calibration" in parts:
        calibration(gpu, args.quick, args.seeds)
    if "quality" in parts:
        quality(gpu, args.quick, args.ref_spp, [float(x) for x in args.sweep.split(",")])


if __name__ == "__main__":
    main()
