"""The device-resident Buffer (rptb_buffer) without a GPU: its C ABI, the streaming variance it computes
restated in numpy against the oracle's two-pass Buffer::variance, and the C++ mirror compiling."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from rpt_b200 import _capi as capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUFFER_SYMBOLS = {"rptb_buffer_create", "rptb_buffer_destroy", "rptb_sample_into", "rptb_buffer_add_samples",
                  "rptb_buffer_image", "rptb_buffer_variance", "rptb_buffer_sums"}


def test_buffer_symbols_are_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "rpt_b200.h")).read()
    declared = set(re.findall(r"\b(rptb_[a-z0-9_]+)\s*\(", header))
    bound = {name for name, _, _ in capi.SYMBOLS}
    assert BUFFER_SYMBOLS <= declared and BUFFER_SYMBOLS <= bound
    lib = capi.lib()
    for name in BUFFER_SYMBOLS:
        assert hasattr(lib, name)


def test_buffer_entry_points_return_a_status_instead_of_aborting():
    lib = capi.lib()
    h = C.c_void_p()
    assert lib.rptb_buffer_create(None, 8, 8, 1, C.byref(h)) == capi.ERR_BAD_ARG
    assert not h
    assert "null" in lib.rptb_last_error().decode()
    rgb = np.zeros((64, 3))
    out8 = np.zeros(64 * 3, np.uint8)
    v = C.c_double(0.0)
    n = C.c_uint32(0)
    cam, p = capi.Camera(), capi.RenderParams()
    p.width = p.height = 8
    p.iterations = 1
    assert lib.rptb_sample_into(None, C.byref(cam), C.byref(p), None, None) == capi.ERR_BAD_ARG
    assert lib.rptb_buffer_add_samples(None, rgb.ctypes.data_as(capi.c_double_p)) == capi.ERR_BAD_ARG
    assert lib.rptb_buffer_image(None, out8.ctypes.data_as(capi.c_u8_p)) == capi.ERR_BAD_ARG
    assert lib.rptb_buffer_variance(None, C.byref(v)) == capi.ERR_BAD_ARG
    assert lib.rptb_buffer_sums(None, rgb.ctypes.data_as(capi.c_double_p), C.byref(n)) == capi.ERR_BAD_ARG
    lib.rptb_buffer_destroy(None)
    if lib.rptb_device_count() <= 0:
        # no scene can exist without a device, so no buffer either
        from rpt_b200 import api, scenes
        cfg = scenes.sphere_scene()
        with pytest.raises(capi.RptbError, match="status -3"):
            api.DeviceScene(cfg.scene)


def welford(batches):
    """What buffer_accumulate_kernel computes per entry, and rptb_buffer_variance from it (film.cu)."""
    nb, npix, _ = batches.shape
    s = np.zeros((npix, 3))
    m2 = np.zeros(npix)
    for n, x in enumerate(batches, 1):
        if n == 1:
            s = x.copy()
            continue
        new = s + x
        d = (x - s / (n - 1)) * (x - new / n)
        m2 += d[:, 0] + d[:, 1] + d[:, 2]
        s = new
    return s, (np.mean(m2 / (nb - 1)) if nb > 1 else float("nan"))


def fireflies(rng, nb, npix):
    b = rng.uniform(0, 1, (nb, npix, 3))
    hot = rng.random((nb, npix)) < 0.002  # rare paths that hit the light: a few entries far above the rest
    b[hot] *= rng.uniform(1e2, 1e5, (int(hot.sum()), 1))
    return b


@pytest.mark.parametrize("nb", [2, 3, 17, 300])
def test_streaming_variance_matches_two_pass_oracle(orc, nb):
    rng = np.random.default_rng(nb)
    batches = fireflies(rng, nb, 20000 if nb < 100 else 4000)
    sums, var = welford(batches)
    np.testing.assert_allclose(var, orc.variance(batches), rtol=1e-12)
    # the running sum is the sequential one np.sum takes along axis 0
    assert np.array_equal(sums, np.sum(list(batches), axis=0))


def test_streaming_variance_is_nan_below_two_entries():
    assert np.isnan(welford(np.ones((1, 4, 3)))[1])


CPP = r"""
#include "rpt.hpp"
int main(int argc, char**) {
    rpt::Scene scene;
    scene.add(rpt::Object(rpt::sphere()));
    rpt::Renderer r(scene, rpt::Camera{});
    r.width(32).height(16).num_samples(10).filter(rpt::Filter::Box(1));
    if (argc > 1) {
        rpt::DeviceBuffer buffer = r.device_buffer();
        double v = 0;
        r.iterative_render(4, buffer, [&](uint32_t, const rpt::DeviceBuffer& b) {
            std::vector<uint8_t> img = b.image();
            v = b.variance();
            (void)img;
        });
        std::vector<double> sums = buffer.sums();
        return sums.size() == 32u * 16u * 3u && v >= 0 ? 0 : 1;
    }
    return 0;
}
"""


def test_cpp_device_buffer_compiles(tmp_path):
    src = tmp_path / "device_buffer.cpp"
    src.write_text(CPP)
    libdir = os.path.join(ROOT, "rpt_b200", "lib")
    exe = str(tmp_path / "device_buffer")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                           "-o", exe, "-L" + libdir, "-lrpt_b200", "-Wl,-rpath," + libdir])
    assert subprocess.run([exe]).returncode == 0  # without an argument it touches no device
