"""The f32 render kernels on the GPU against the oracle away from the unit box (-m gpu).

The placement matrix of tests/pathwise.py (PLACEMENTS), rendered one sample at a time through rptb_render_samples:
the megakernel for every case, and the wavefront engine as well for the cases traced through kd-trees of meshes.
The criteria are test_hostemu_placement.py's (a) -- agreement >= Case.gpu_floor, |signed bias| <= Case.bias, no more
segments than the oracle -- and its (b): the f32 agreement of an off-center case meets its base case's on the same
engine within binomial error.  The floors are the host emulation's less 0.002 (0.01 - 0.02 where the oracle's own image
moves or the instance is far away).  Measured on one H100 80GB HBM3 at a 700 W power limit, megakernel (mk) and
wavefront (wf), 16 384 paths per case:

    case                      agree    bias        case                      agree    bias
    teapot_kd_0 (mk, wf)      0.99994  +4.8e-7     teapot_bvh_0              0.99994  +4.8e-7
    teapot_kd_1e2 (mk, wf)    0.99994  +5.3e-7     teapot_bvh_1e2            0.99994  +5.3e-7
    teapot_kd_1e3 (mk, wf)    0.99890  +1.3e-6     teapot_bvh_1e3            0.99890  +1.3e-6
    teapot_kd_1e4 (mk, wf)    0.98572  +2.5e-6     teapot_bvh_1e4            0.98572  +2.5e-6
    teapot_group(_bvh)_0      0.99994  +4.8e-7     teapot_group(_bvh)_1e4    0.98572  +2.5e-6
    quad_plane_0              0.99976  +2.7e-7     quad_plane_1e4            0.97943  +3.1e-5
    cornell_1                 0.98730  +1.5e-6     cornell_s1e-3             0.99933  +1.0e-6
    cornell_s1e3              0.78485  +4.1e-6     cornell_far               0.92712  +1.5e-5
    glass_1                   0.97949  +1.4e-6     glass_s1e-3               0.97961  +3.7e-7
    glass_s1e3                0.89612  +1.6e-6
    far_teapot_1e2            0.83405  +1.2e-5     far_teapot_1e2_x100       0.79785  -5.3e-5
    far_teapot_1e3            0.35834  +1.2e-4     far_teapot_1e3_x100       0.39850  +3.3e-5
    far_sphere_1e2            0.83228  +7.2e-6     far_sphere_1e2_x100       0.83160  -5.1e-5
    far_sphere_1e3            0.31073  +1.6e-4     far_sphere_1e3_x100       0.37598  +5.2e-5
"""
import numpy as np
import pytest

from rpt_b200 import _capi as capi
from tests import pathwise as pw
from tests.test_gpu_paths import _device_paths

pytestmark = pytest.mark.gpu

ENGINES = [(name, capi.ENGINE_MEGAKERNEL) for name in sorted(pw.PLACEMENTS)] + \
          [(name, capi.ENGINE_WAVEFRONT) for name in sorted(pw.PLACEMENTS) if pw.PLACEMENTS[name].wavefront]
_CACHE = {}


def _stats(orc, name, engine):
    if (name, engine) not in _CACHE:
        c = pw.PLACEMENTS[name]
        scene, cam = c.make()
        f32, seg32, feat, compiled = _device_paths(c, scene, cam, engine)
        f64, seg64 = pw.oracle_paths(orc, c, scene, cam)
        _CACHE[(name, engine)] = (pw.compare(f32, f64, seg32, seg64), feat, compiled, f32)
    return _CACHE[(name, engine)]


def _id(n, e):
    return "%s-%s" % (n, "wf" if e == capi.ENGINE_WAVEFRONT else "mk")


@pytest.mark.parametrize("name,engine", ENGINES, ids=[_id(n, e) for n, e in ENGINES])
def test_f32_paths_on_the_gpu_away_from_the_unit_box(orc, gpu_ok, name, engine):
    c = pw.PLACEMENTS[name]
    st, feat, compiled, f32 = _stats(orc, name, engine)
    print(st.line(_id(name, engine), feat))
    assert compiled and feat == c.feat
    assert np.isfinite(f32).all(), "non-finite f32 path"
    assert st.agree >= c.gpu_floor, st.line(name, feat)
    assert abs(st.bias) <= c.bias, st.line(name, feat)
    assert st.seg32 <= st.seg64, st.line(name, feat)


BASED = [(n, e) for n, e in ENGINES if pw.PLACEMENTS[n].base and not pw.PLACEMENTS[n].degrades]


@pytest.mark.parametrize("name,engine", BASED, ids=[_id(n, e) for n, e in BASED])
def test_placement_on_the_gpu_keeps_the_base_scenes_agreement(orc, gpu_ok, name, engine):
    c = pw.PLACEMENTS[name]
    st = _stats(orc, name, engine)[0]
    bst = _stats(orc, c.base, engine)[0]
    sigma = np.sqrt(st.agree * (1.0 - st.agree) / st.rel.size)
    print("%-24s agree %.5f  base %.5f" % (_id(name, engine), st.agree, bst.agree))
    base_floor = pw.PLACEMENTS[c.base].gpu_floor
    assert st.agree >= base_floor - c.base_slack - 3.0 * max(sigma, 1.0 / st.rel.size), (st.line(name, 0), bst.line(c.base, 0))
