"""The f32 megakernel body against the oracle path by path, without a GPU.

tests/pathwise.py renders every scene of its matrix one sample at a time (iterations = 1, first_sample = s) through the
emulated megakernel in f32 and through the oracle, on the same Philox streams, and compares the S * W * H paths one by
one.  Per scene:
  (a) the fraction of paths within 1e-3 (relative, see pathwise.compare) is at least a measured floor;
  (b) the signed bias sum(f32 - f64) / sum|f64| of those paths is within 1e-5;
  (c) the f32 path never traces more segments than the oracle (it skips zero-weight subtrees and dead vertices).

Measured on the host emulation (16 384 paths per scene; 17 020 for lights_lens, 36 864 for clamp_glass).  Each floor is
the measurement less three to five binomial standard deviations:

    scene                FEAT  agree    floor   >1e-1    bias
    cornell              128   0.98724  0.982   0.0056   +1.4e-6
    cornell_scan           0   0.98724  0.982   0.0056   +1.4e-6
    sphere               136   0.99988  0.999   0.00006  +1.3e-7
    sphere_scan            8   0.99988  0.999   0.00006  +1.3e-7
    teapot_kd              1   0.99988  0.999   0        +8.7e-7
    teapot_bvh            65   0.99988  0.999   0        +8.7e-7
    glass                 14   0.97943  0.974   0.00012  +1.9e-6
    glass_deep             6   0.97443  0.968   0.00043  -5.5e-6
    fractal_spheres       55   0.99902  0.997   0.00031  +3.1e-7
    fractal_teapots_kd    55   0.99896  0.997   0        +7.5e-7
    fractal_teapots_bvh  119   0.99896  0.997   0        +7.5e-7
    monomial_glass        55   0.99371  0.990   0.00006  +3.4e-6
    clamp                136   0.99927  0.998   0        -6.7e-7
    clamp_glass            7   0.99778  0.9965  0.00003  +3.0e-6
    lights_lens          128   0.99988  0.999   0        -2.9e-7
    smooth_kd              1   0.99976  0.999   0        +2.1e-7
    smooth_glass_bvh      71   0.99744  0.995   0.00012  +1.6e-6

What each f32-only rule looks like when it is wrong, and which scene sees it (each change applied alone to the source):
  * clamp composite `min(100 W, C) - W a` instead of `min(100 W, C - W a)`: clamp drops to ~0.62, clamp_glass to 0.991;
  * fwdC computed from fwdT after fwdT is multiplied by w: clamp ~0.93, clamp_glass 0.987;
  * `dead` decided by the face normal ng instead of the shading normal n: smooth_kd and smooth_glass_bvh lose 15 % of
    their paths (their meshes are wound both ways; a mesh wound consistently with its normals cannot show it);
  * the shadow `skip` taken for transparent materials too: clamp_glass 0.9936 (its back-lit frosted pane);
  * offset_origin's delta at 4096 ulp instead of 32, or a factor 1 + 1e-3 on the f32 sample_f pdf: every scene fails,
    through its agreement fraction or its bias.
Of the other host-emulation tests only the vertex-at-once bit-equality test sees the `dead` change, and only the
image-statistics tests see the offset change; none sees the other four.

The divergent tail, traced event by event (hit object, light sample, shadow verdict, sample_f lobe and direction) in
both precisions through a printf build of the host emulation, where Real = double is the oracle bit for bit:
  * Cornell (0.56 % of paths off by more than 10 %): 7 of 8 traced paths part where the oracle's shadow or
    continuation ray hits the very face it starts on, at t = 1.1e-12 .. 1.9e-11.  The reference restarts rays exactly
    at the hit point with EPSILON = 1e-12 (renderer.rs:14), and at Cornell's coordinates (~500) the rounding of the hit
    point is of that order: shadow acne of the reference, which the f32 path avoids by design (offset_origin).  The
    eighth path reached the edge of the small box on a ray that had drifted by 2e-4 over three diffuse bounces.
  * glass (2 % off by more than 1e-3): the first difference is always the direction sampled from the roughness-1e-4
    Beckmann lobe.  Its microfacet angle is ~1e-4 rad, which f32 resolves to ~1e-3 of itself; the reflected direction
    then moves by ~3e-5 rad and the synthetic HDRI's narrow lamps turn that into 0.1 - 1 % of the path's radiance.
    The pdf differs by up to 100x there, but the weight f |cos| / pdf does not.
Both are rounding at a threshold or ill-conditioned geometry, not a rule of the f32 path.
"""
import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api
from tests import pathwise as pw
from tests.hostemu import emu

F_LIST = 256
_CACHE = {}


def emulated(orc, name):
    """(PathStats, FEAT of the variant that rendered) of CASES[name] through the emulated megakernel."""
    if name not in _CACHE:
        c = pw.CASES[name]
        scene, cam = c.make()
        with pw.scene_env(c.env):
            e = emu.EmuScene(api.FlatScene(scene, accel=c.accel))
        # the library sends every feature bit to the launchers (api.cu): a kd-tree of shapes over BVH meshes runs
        # F_EVERY | F_BVH
        ext_bvh = (e.features & pw.F_BVH) != 0
        r = pw.renderer(c, scene, cam, 1, capi.PRECISION_F32)
        feats = set()

        def render(s):
            img, st, feat = e.render(cam, r.params(1, s), ext_bvh=ext_bvh)
            feats.add(feat)
            return img, st

        f32, seg32 = pw.stack_paths(render, c.spp)
        f64, seg64 = pw.oracle_paths(orc, c, scene, cam)
        e.close()
        assert len(feats) == 1
        _CACHE[name] = (pw.compare(f32, f64, seg32, seg64), feats.pop())
    return _CACHE[name]


@pytest.mark.parametrize("name", sorted(pw.CASES))
def test_f32_paths_are_the_oracles(orc, name):
    c = pw.CASES[name]
    st, feat = emulated(orc, name)
    print(st.line(name, feat))
    assert feat == c.feat
    assert st.rel.size >= pw.MIN_PATHS
    assert np.isfinite(st.rel).all(), "non-finite f32 path"
    assert st.agree >= c.floor, st.line(name, feat)
    assert abs(st.bias) <= c.bias, st.line(name, feat)
    assert st.seg32 <= st.seg64, st.line(name, feat)


def test_the_matrix_reaches_every_f32_variant():
    """Every variant pick_render returns for an f32 render without counters, over every feature set, is served by a
    scene of the matrix -- and the list in pathwise is exactly that set."""
    reachable = set()
    for features in range(256):
        (stats, feat, _), compiled = emu.pick_variant(emu.ENGINE_RENDER, features, 0, capi.PRECISION_F32, 6)
        assert compiled and not stats
        reachable.add(feat)
    assert reachable == pw.F32_RENDER_VARIANTS
    served = {}
    for name, c in pw.CASES.items():
        scene, _ = c.make()
        with pw.scene_env(c.env):
            e = emu.EmuScene(api.FlatScene(scene, accel=c.accel))
        (_, feat, _), _ = emu.pick_variant(emu.ENGINE_RENDER, e.features, 0, capi.PRECISION_F32, c.max_bounces)
        e.close()
        assert feat == c.feat, name
        served.setdefault(feat, []).append(name)
    assert set(served) == pw.F32_RENDER_VARIANTS, sorted(pw.F32_RENDER_VARIANTS - set(served))


def test_the_list_matrix_reaches_every_list_variant():
    """Adaptive sampling's list-scheduled variants (pick_render_list): every one returned for any feature set, counting
    pass, precision and depth is compiled, and pathwise.LIST_MATRIX, the matrix test_gpu_list_matrix.py runs, reaches
    exactly that set."""
    reachable = set()
    for features in range(256):
        for stats in (0, 1, 2):
            for precision in (capi.PRECISION_F32, capi.PRECISION_F64):
                for max_bounces in (6, 40):
                    v, compiled = emu.pick_render_list(features, stats, precision, max_bounces)
                    assert compiled, (features, stats, precision, max_bounces, v)
                    assert v[1] & F_LIST and v[0] == (stats != 0)
                    reachable.add((precision,) + v)
    served = {}
    for name, precision, stats in pw.LIST_MATRIX:
        c = pw.CASES[name]
        scene, _ = c.make()
        with pw.scene_env(c.env):
            e = emu.EmuScene(api.FlatScene(scene, accel=c.accel))
        v, _ = emu.pick_render_list(e.features, stats, precision, c.max_bounces)
        e.close()
        served.setdefault((precision,) + v, []).append((name, stats))
    for k in sorted(reachable):
        print("%s STATS %d FEAT %3d MAXD %2d  %s" % ("f64" if k[0] == capi.PRECISION_F64 else "f32", k[1], k[2], k[3], served.get(k)))
    assert set(served) == reachable, sorted(reachable ^ set(served))
    # the f32 ones are the twins of every compiled f32 render variant; f64 never picks F_BVH
    assert len([k for k in reachable if k[0] == capi.PRECISION_F32]) == 14
    assert len([k for k in reachable if k[0] == capi.PRECISION_F64]) == 5
