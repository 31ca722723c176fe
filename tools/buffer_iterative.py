"""Renderer.iterative_render with a callback that calls image() and variance(), through the host Buffer and
through the DeviceBuffer, on three configs:

    python tools/buffer_iterative.py [cornell sphere dragon]

Each (config, buffer) pair runs in its own process so that the peak host RSS is its own.  Printed per pair:
wall time per callback (mean and last) and in total, and the peak RSS.  Then, per config, the device time of
buffer_accumulate_kernel (kernel durations as CUPTI records them, through torch.profiler) and its achieved
bandwidth at 84 B per pixel: 12 B of f32 entry read, 36 B of sums + M2 + entry count read and 36 B written.  The card's name
and power limit are printed in the same run."""
import json
import os
import resource
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# name: (scene, width, height, max_bounces, spp, callback interval, box radius)
CONFIGS = {
    "cornell": ("cornell_scene", 1024, 1024, 2, 100, 10, 1),
    "sphere": ("sphere_scene", 800, 600, 6, 1000, 10, 0),
    "dragon": ("dragon_scene", 1200, 1200, 8, 10, 1, 0),
}
HBM_TBS = 3.35  # H100 SXM5 HBM3 peak


def renderer(name):
    from rpt_b200 import api, scenes
    scene, w, h, mb, spp, k, radius = CONFIGS[name]
    cfg = getattr(scenes, scene)()
    r = (api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).num_samples(spp).seed(1)
         .filter(api.Filter.Box(radius)))
    r.device_scene()  # scene upload (and the dragon's BVH build) outside the timed region
    return r, k


def rss_mb():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) / 1024.0
    return float("nan")


def run_one(name, mode):
    r, k = renderer(name)
    rss0 = rss_mb()
    times = []

    def cb(it, buf):
        t0 = time.perf_counter()
        buf.image()
        buf.variance()
        times.append(time.perf_counter() - t0)

    t0 = time.perf_counter()
    r.iterative_render(k, cb, buffer=r.device_buffer() if mode == "device" else None)
    total = time.perf_counter() - t0
    print(json.dumps({"config": name, "buffer": mode, "callbacks": len(times), "callback_ms_mean": 1e3 * sum(times) / len(times),
                      "callback_ms_last": 1e3 * times[-1], "total_s": total, "rss_before_render_mb": rss0,
                      "peak_rss_mb": resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0}), flush=True)


def run_kernel(name):
    import torch
    from torch.profiler import ProfilerActivity, profile
    r, _ = renderer(name)
    buf = r.device_buffer()
    r.sample(1, buf, want_stats=False)
    buf.image()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(10):
            r.sample(1, buf, want_stats=False)
        buf.image()
        torch.cuda.synchronize()
    us = [e.time_range.elapsed_us() for e in prof.events()
          if "buffer_accumulate_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
    w, h = CONFIGS[name][1], CONFIGS[name][2]
    mean_us = sum(us) / len(us) if us else float("nan")
    gbs = w * h * 84 / (mean_us * 1e-6) / 1e9 if us else float("nan")
    print(json.dumps({"config": name, "accumulate_launches": len(us), "accumulate_us_mean": mean_us,
                      "accumulate_us_min": min(us) if us else None, "accumulate_GBps": gbs,
                      "of_peak": gbs / (HBM_TBS * 1e3)}), flush=True)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--one":
        return run_one(sys.argv[2], sys.argv[3])
    if len(sys.argv) > 2 and sys.argv[1] == "--kernel":
        return run_kernel(sys.argv[2])
    if len(sys.argv) > 1 and sys.argv[1] == "--card":
        name, q = card()
        return print(f"card: {name}; power limit, max SM clock: {q}", flush=True)
    names = sys.argv[1:] or list(CONFIGS)
    me = os.path.abspath(__file__)
    # ru_maxrss survives fork and exec: this process stays small (no CUDA, no torch) so that each child's peak
    # RSS is its own
    subprocess.check_call([sys.executable, me, "--card"])
    for n in names:
        for mode in ("host", "device"):
            subprocess.check_call([sys.executable, me, "--one", n, mode])
        subprocess.check_call([sys.executable, me, "--kernel", n])


if __name__ == "__main__":
    main()
