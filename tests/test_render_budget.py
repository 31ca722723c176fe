"""The packed-table render kernels' register budget, and the renders without counters.

The Cornell and sphere configs run render_kernel<float, 16, false, F_FLAT[| F_SMALL]>, a loop bound by instruction
issue.  A render given no counters (RenderArgs::counters null: bench.py's timed steps, rptb_sample_into without stats)
runs the F_NOCOUNT twin, which has the counting compiled out and is built for RPTB_MIN_BLOCKS_FLAT resident CTAs per SM;
a render given counters runs the counting variant, at RPTB_MIN_BLOCKS_LITE.

CPU: ptxas's report of what the build made (build/obj/kernels_f32.ptxas.log) holds each of these kernels to its
register cap and to the spill stores it has today, so that state added to the loop fails here rather than at benchmark
time (that every pick, with counters or without, is a compiled variant is a static_assert in launch.h).  GPU: the two
variants give the same bits, in the tile schedule and in the list schedule."""
import os
import re

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "build", "obj", "kernels_f32.ptxas.log")
INTEGRATOR = os.path.join(ROOT, "rpt_b200", "csrc", "integrator.cuh")
F_SMALL, F_FLAT, F_LIST, F_NOCOUNT = 8, 128, 256, 512

# spill stores (bytes) ptxas reports for each packed-table render kernel (sm_90a, CUDA 12.9): (FEAT, list schedule) -> bytes.
# Not yet 0: 64 registers without spills needs less loop-carried state (integrator.cuh, RPTB_MIN_BLOCKS_FLAT).
SPILL_STORES = {
    (F_FLAT | F_NOCOUNT, False): 384, (F_FLAT | F_SMALL | F_NOCOUNT, False): 360,
    (F_FLAT | F_NOCOUNT, True): 396, (F_FLAT | F_SMALL | F_NOCOUNT, True): 372,
    (F_FLAT, False): 320, (F_FLAT | F_SMALL, False): 292,
    (F_FLAT, True): 332, (F_FLAT | F_SMALL, True): 304,
}


def min_blocks(name):
    m = re.search(r"#define %s (\d+)" % name, open(INTEGRATOR).read())
    assert m, name
    return int(m.group(1))


def ptxas_report():
    """{(FEAT, list schedule): (registers, spill store bytes, spill load bytes)} of the f32 render kernels"""
    if not os.path.exists(LOG):
        pytest.fail("%s is missing: build() writes it" % LOG)
    out = {}
    for block in re.split(r"Compiling entry function '", open(LOG).read())[1:]:
        name = block.split("'")[0]
        m = re.match(r"_ZN4rptb(13render_kernel|18render_list_kernel)IfLi16ELb0ELi(\d+)E", name)
        if not m:
            continue
        regs = re.search(r"Used (\d+) registers", block)
        sp = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
        feat = int(m.group(2))
        out[(feat & ~F_LIST, (feat & F_LIST) != 0)] = (int(regs.group(1)), int(sp.group(1)), int(sp.group(2)))
    return out


@pytest.mark.parametrize("key", sorted(SPILL_STORES))
def test_packed_table_kernels_keep_their_budget(key):
    rep = ptxas_report()
    assert key in rep, sorted(rep)
    regs, stores, _ = rep[key]
    blocks = min_blocks("RPTB_MIN_BLOCKS_FLAT" if key[0] & F_NOCOUNT else "RPTB_MIN_BLOCKS_LITE")
    assert regs <= 65536 // (128 * blocks), (key, regs, blocks)
    assert stores <= SPILL_STORES[key], (key, stores)


def small(cfg, w, h):
    return api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(cfg.max_bounces).seed(1)


CASES = [("cornell", 72, 40, 40), ("cornell", 72, 40, 130), ("sphere", 96, 56, 70)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,w,h,spp", CASES)
def test_counting_and_silent_renders_are_the_same_bits(gpu_ok, name, w, h, spp):
    """rptb_sample_into without stats runs the F_NOCOUNT variant, with stats the counting one (one chunk at 40 spp, chunk
    sums at 70 and 130): the same sums, bit for bit, entry after entry; and the counting one still counts."""
    cfg = scenes.CONFIGS[name]()
    runs = []
    for want_stats in (False, True):
        r = small(cfg, w, h).engine(capi.ENGINE_MEGAKERNEL)
        trace = []
        with r.device_buffer() as db:
            for _ in range(2):
                r.sample(spp, db, want_stats=want_stats)
                trace.append(db.sums().copy())
                if want_stats:
                    assert r.last_stats["segments"] >= w * h * spp and r.last_stats["rays"] >= r.last_stats["segments"]
        r.close()
        runs.append(trace)
    for s0, s1 in zip(*runs):
        assert np.isfinite(s0).all()
        assert np.array_equal(s0, s1), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cornell", "sphere"])
def test_counting_and_silent_list_renders_are_the_same_bits(gpu_ok, name):
    """adaptive entries (the list schedule) with and without stats: the same sums and counts after every entry"""
    cfg = scenes.CONFIGS[name]()
    w, h = 80, 48
    crit = api.Adaptive(rel_tol=0.2, abs_tol=1e-3, min_entries=2)
    runs = []
    for want_stats in (False, True):
        r = small(cfg, w, h).engine(capi.ENGINE_MEGAKERNEL)
        trace = []
        with r.device_buffer() as db:
            for _ in range(4):
                r.sample(16, db, want_stats=want_stats, adaptive=crit)
                trace.append((db.sums().copy(), db.counts().copy()))
        r.close()
        runs.append(trace)
    for (s0, c0), (s1, c1) in zip(*runs):
        assert np.array_equal(c0, c1)
        assert np.array_equal(s0, s1)
