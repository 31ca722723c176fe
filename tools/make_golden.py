"""Generate tests/golden/*_render.npz and *_hits.npz from the CPU oracle (no GPU needed).

The reference holds no golden vectors for this path (SURVEY 8c) and is not built by this
project (it is Rust), so these fixtures pin the ORACLE against regressions; they are not outputs
of rpt itself.  Regenerate only when the oracle is deliberately changed:

    python tools/make_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle_py as orc  # noqa: E402
from rpt_b200 import api, scenes  # noqa: E402
from tests import util  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

RENDERS = {  # name: (width, height, spp, max_bounces)
    "sphere": (48, 27, 8, 2),
    "cornell": (32, 32, 8, 6),
    "teapot": (48, 27, 4, 0),
    "glass": (48, 27, 8, 12),
    # SURVEY 8f row N4 (kd-trees over whole shapes, MonomialSurface)
    "fractal_spheres": (48, 36, 4, 1),
    "fractal_teapots": (48, 36, 4, 1),
    "monomial_glass": (48, 36, 8, 1),
}


def main():
    only = set(sys.argv[1:])  # e.g. `python tools/make_golden.py fractal_spheres` adds one fixture, leaves the rest
    os.makedirs(OUT, exist_ok=True)
    for name, (w, h, spp, mb) in RENDERS.items():
        if only and name not in only:
            continue
        cfg = util.golden_config(name)
        osc = orc.OracleScene(api.FlatScene(cfg.scene))
        r = api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(mb).seed(1)
        img, st = osc.render(cfg.camera, r.params(spp))
        np.savez_compressed(os.path.join(OUT, f"{name}_render.npz"), image=img, width=w, height=h, spp=spp,
                            max_bounces=mb, seed=1, segments=st["segments"], rays=st["rays"])
        print(name, img.mean(0), st["segments"], st["rays"])
    rng = np.random.default_rng(42)
    for name in ("cornell", "teapot"):
        if only:  # regenerating single render fixtures: leave the hit fixtures (and their ray stream) alone
            continue
        cfg = scenes.CONFIGS[name]()
        osc = orc.OracleScene(api.FlatScene(cfg.scene))
        if name == "cornell":
            rays = np.concatenate([util.camera_rays(cfg.camera, 1500, rng), util.interior_rays([1, 1, 1], [555, 548, 559], 1500, rng)])
        else:
            rays = np.concatenate([util.camera_rays(cfg.camera, 2000, rng, spread=0.4), util.interior_rays([-2, -1, -2], [2, 1.5, 2], 1000, rng)])
        t, o, n, _ = osc.closest_hit(rays)
        np.savez_compressed(os.path.join(OUT, f"{name}_hits.npz"), rays=rays, t=t, obj=o, normal=n)
        print(name, "hits", (o >= 0).mean())


if __name__ == "__main__":
    main()
