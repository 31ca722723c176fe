"""The f32 render kernels on the GPU against the oracle, path by path (-m gpu).

The scene matrix of tests/pathwise.py, rendered one sample at a time through rptb_render_samples: the megakernel for
every scene, and the wavefront engine as well for every scene it serves (all but the kd-trees of shapes and the
MonomialSurface, which it hands to the megakernel).  The criteria are those
of test_hostemu_paths.py -- (a) agreement fraction >= a measured floor, (b) |signed bias| of the agreeing paths
<= 1e-5, (c) no more segments than the oracle -- with floors (Case.gpu_floor) checked against the H100's own
measurement, since the compiled kernels use the SFU approximations of --use_fast_math and contract multiply-adds,
which the host emulation does not.  The variant that
serves each scene is the one pick_render chooses for the scene's features (the library and the emulation share that
dispatch; test_hostemu_paths.py checks the matrix reaches every variant).

Measured on one H100 80GB HBM3, megakernel (mk) at a 400 W power limit and wavefront (wf) at 700 W (agreement does not
depend on the clock); the floors are those of the host emulation, which the H100 meets within one binomial standard
deviation everywhere.  Both engines give the same agreement and bias on every scene, to the digits shown:

    scene                        agree    floor   bias
    cornell (mk, wf) / _scan     0.98730  0.982   +1.5e-6
    sphere (mk, wf) / _scan      0.99988  0.999   +2.0e-7
    teapot_kd (mk, wf)           0.99988  0.999   +8.9e-7
    teapot_bvh (mk, wf)          0.99988  0.999   +8.9e-7
    glass (mk, wf)               0.97949  0.974   +1.4e-6
    glass_deep (mk, wf)          0.97443  0.968   -5.3e-6
    fractal_spheres              0.99896  0.997   +2.3e-7
    fractal_teapots_kd/bvh       0.99896  0.997   +5.2e-7
    monomial_glass               0.99365  0.990   +3.5e-6
    clamp (mk, wf)               0.99927  0.998   +3.0e-7
    clamp_glass (mk, wf)         0.99778  0.9965  +3.3e-6
    lights_lens (mk, wf)         0.99988  0.999   -2.3e-7
    smooth_kd (mk, wf)           0.99976  0.999   +2.1e-7
    smooth_glass_bvh (mk, wf)    0.99750  0.995   +1.7e-6
"""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api
from tests import pathwise as pw
from tests.hostemu import emu

pytestmark = pytest.mark.gpu

ENGINES = [(name, capi.ENGINE_MEGAKERNEL) for name in sorted(pw.CASES)] + \
          [(name, capi.ENGINE_WAVEFRONT) for name in sorted(pw.CASES) if pw.CASES[name].wavefront]
_ORACLE = {}


def _oracle(orc, name, scene, cam):
    if name not in _ORACLE:
        _ORACLE[name] = pw.oracle_paths(orc, pw.CASES[name], scene, cam)
    return _ORACLE[name]


def _device_paths(case, scene, cam, engine):
    with pw.scene_env(case.env):
        flat = api.FlatScene(scene, accel=case.accel)
        ds = api.DeviceScene(flat, accel=case.accel)
        features = emu.EmuScene(flat).features
    (_, feat, _), compiled = emu.pick_variant(emu.ENGINE_RENDER, features, 0, capi.PRECISION_F32, case.max_bounces)
    r = pw.renderer(case, scene, cam, 1, capi.PRECISION_F32, engine)
    c_cam = cam.to_c()
    out = np.empty((case.w * case.h, 3))

    def render(s):
        st = capi.Stats()
        capi.check(capi.lib().rptb_render_samples(ds.handle, C.byref(c_cam), C.byref(r.params(1, s)),
                                                  out.ctypes.data_as(capi.c_double_p), C.byref(st)), "rptb_render_samples")
        d = st.as_dict()
        assert d["engine"] == engine
        return out.copy(), d

    try:
        f32, seg = pw.stack_paths(render, case.spp)
    finally:
        ds.close()
    return f32, seg, feat, compiled


@pytest.mark.parametrize("name,engine", ENGINES, ids=["%s-%s" % (n, "wf" if e == capi.ENGINE_WAVEFRONT else "mk") for n, e in ENGINES])
def test_f32_paths_on_the_gpu_are_the_oracles(orc, gpu_ok, name, engine):
    c = pw.CASES[name]
    scene, cam = c.make()
    f32, seg32, feat, compiled = _device_paths(c, scene, cam, engine)
    f64, seg64 = _oracle(orc, name, scene, cam)
    st = pw.compare(f32, f64, seg32, seg64)
    print(st.line(name + ("-wf" if engine == capi.ENGINE_WAVEFRONT else ""), feat))
    assert compiled and feat == c.feat
    assert st.rel.size >= pw.MIN_PATHS
    assert np.isfinite(f32).all(), "non-finite f32 path"
    assert st.agree >= c.gpu_floor, st.line(name, feat)
    assert abs(st.bias) <= c.bias, st.line(name, feat)
    assert st.seg32 <= st.seg64, st.line(name, feat)
