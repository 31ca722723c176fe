"""The wavefront engine's step loop and sample chunks on the GPU (-m gpu).

The wavefront engine (wavefront.cuh, run_wavefront_f32) advances every path by one vertex per step inside a CUDA graph
WHILE loop, and a path sums the sample chunks g, g + G, g + 2G, ... of its pixel.  These tests pin what that schedule
must get exactly right, whatever the image and the sample count:

  * exact answers: scenes whose every sample ends at a vertex with nothing left to trace (an ambient-lit plane, a
    closed emissive sphere seen from inside, a plane whose only sampled light is behind it, a closed room of planes at
    max depth) or at a miss, so that every pixel has a closed form.  A lost sample or a stale chunk sum moves a pixel
    by a whole sample's share;
  * the three regimes of paths per pixel slot against sample chunks (G == nchunks, 1 < G < nchunks, G == 1 < nchunks);
  * recomposition, bit for bit: with exposure 0 an N-spp render is the chunk-ordered float64 sum of the 1-spp renders
    with first_sample = 0 .. N-1, divided by N.  That holds whatever FMA contraction does, so it pins the scheduling
    (chunks, groups, shards, the Buffer's entry) exactly, and it holds for the megakernel too;
  * scratch reuse: a render on a handle gives the same bits as on a fresh handle after megakernel renders, after
    renders of other sizes and while renders on other streams are in flight;
  * sampled-light slots: 0, 1 and 8 sampled lights against the oracle; a ninth is refused.
"""
import ctypes as C

import numpy as np
import pytest

from rpt_b200 import _capi as capi
from rpt_b200 import api, scenes
from tests import pathwise as pw

pytestmark = pytest.mark.gpu
F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
MK, WF, AUTO = capi.ENGINE_MEGAKERNEL, capi.ENGINE_WAVEFRONT, capi.ENGINE_AUTO
TILE_W, TILE_H = 16, 8

AMB = np.array([0.25, 0.5, 0.75])     # the ambient light
ALB = np.array([0.8, 0.6, 0.4])       # the diffuse plane's colour
ENV = np.array([0.3, 0.2, 0.1])       # the environment of the half-and-half scene
LE = 0.2 * np.array([0.5, 0.6, 0.7])  # the emissive sphere's emittance * colour

SIZES = [(1, 1), (7, 3), (203, 117)]
SPPS = [1, 16, 130]


# ------------------------------------------------------------------------------------ the schedule, restated ------
def sample_chunks(n):
    """scene_dev.cuh sample_chunks: chunk = max(64, ceil(n / 32)) -> (nchunks, chunk)."""
    chunk = max(64, -(-n // 32))
    return -(-n // chunk), chunk


def wavefront_groups(npix, nchunks):
    """kernels_f32.cu wavefront_groups: paths per owned pixel slot, ~2M paths in flight, at most nchunks."""
    if npix == 0:
        return 1
    return max(1, min(-(-2000000 // npix), nchunks))


def pixel_slots(w, h):
    """Pixel slots a one-shard render owns: 128 per 16x8 tile."""
    return -(-w // TILE_W) * -(-h // TILE_H) * 128


def recompose(singles, n, f32):
    """The N-spp image from its 1-spp images: each chunk's samples summed in sample order from 0.0, the chunk sums in
    chunk order from 0.0, divided by N, cast to the output type.  An explicit loop: np.sum is pairwise."""
    nch, chunk = sample_chunks(n)
    total = np.zeros_like(singles[0])
    for c in range(nch):
        cs = np.zeros_like(singles[0])
        for i in range(c * chunk, min((c + 1) * chunk, n)):
            cs = cs + singles[i]
        total = total + cs
    out = total / n
    return out.astype(np.float32).astype(np.float64) if f32 else out


# ------------------------------------------------------------------------------------------------ calls ------------
def params(scene, cam, w, h, spp, mb, engine, precision=F32, first=0, shard=(0, 1), seed=1):
    r = api.Renderer(scene, cam).width(w).height(h).max_bounces(mb).seed(seed).precision(precision).engine(engine)
    return r.params(spp, first, shard[0], shard[1])


def render(ds, scene, cam, w, h, spp, mb, engine=WF, precision=F32, first=0, shard=(0, 1), seed=1):
    """rptb_render_samples -> ((w*h, 3) float64, stats dict); checks that `engine` (if not AUTO) rendered it."""
    p = params(scene, cam, w, h, spp, mb, engine, precision, first, shard, seed)
    c_cam = cam.to_c()
    out = np.full((w * h, 3), np.nan)
    st = capi.Stats()
    capi.check(capi.lib().rptb_render_samples(ds.handle, C.byref(c_cam), C.byref(p), out.ctypes.data_as(capi.c_double_p),
                                              C.byref(st)), "rptb_render_samples")
    d = st.as_dict()
    if engine != AUTO:
        assert d["engine"] == engine
    return out, d


def singles(ds, scene, cam, w, h, n, mb, engine=WF, precision=F32):
    return [render(ds, scene, cam, w, h, 1, mb, engine, precision, first=i)[0] for i in range(n)]


def device_scene(scene, accel=capi.ACCEL_AUTO):
    return api.DeviceScene(api.FlatScene(scene, accel=accel), accel=accel)


def rel_err(got, want):
    return np.abs(got - want) / np.abs(want)


# ------------------------------------------------------------------------------------------------ scenes -----------
def ambient_plane(point_lights=()):
    """A diffuse plane z = 0 filling the view of the default camera, lit by one ambient light (and `point_lights`)."""
    scene = api.Scene()
    scene.add(api.Object(api.plane(api.vec3(0, 0, 1), 0.0)).material(api.Material.diffuse(ALB)))
    scene.add(api.Light.Ambient(AMB))
    for c, pos in point_lights:
        scene.add(api.Light.Point(c, pos))
    return scene, api.Camera.default()


def backlit_plane():
    """The ambient plane with a point light behind it: the light is sampled and never sends a shadow ray."""
    return ambient_plane([(api.vec3(50, 50, 50), api.vec3(0.5, 0.3, -4.0))])


def half_plane():
    """The floor y = -1 seen level from y = 0: rows above the horizon miss (environment), rows below hit the floor,
    lit by the ambient light only; the middle row of an odd height mixes both."""
    scene = api.Scene()
    scene.add(api.Object(api.plane(api.vec3(0, 1, 0), -1.0)).material(api.Material.diffuse(ALB)))
    scene.add(api.Light.Ambient(AMB))
    scene.environment = api.Environment.Color(ENV)
    return scene, api.Camera(eye=api.vec3(0, 0, 0), direction=api.vec3(0, 0, -1), up=api.vec3(0, 1, 0))


def emissive_interior():
    """test_gpu_edge_cases' closed emissive sphere, seen from inside: every vertex is dead (an opaque surface from
    behind), so the f32 path ends there with Le."""
    scene = api.Scene()
    scene.add(api.Object(api.sphere().scale(api.vec3(5.0, 5.0, 5.0))).material(api.Material.light(api.vec3(0.5, 0.6, 0.7), 0.2)))
    return scene, api.Camera(eye=api.vec3(0, 0, 0), direction=api.vec3(0, 0, -1), up=api.vec3(0, 1, 0), fov=1.0)


def room():
    """A closed box of six inward-facing diffuse planes lit by an ambient light only: every bounce hits a wall and no
    vertex sends a shadow ray, so every sample ends at a vertex at max depth with nothing to trace."""
    scene = api.Scene()
    for n, col in (((0, 1, 0), 0xAAAAAA), ((0, -1, 0), 0x8899AA), ((1, 0, 0), 0xBC4444), ((-1, 0, 0), 0x44BC44),
                   ((0, 0, 1), 0x9999CC), ((0, 0, -1), 0xCCCC99)):
        scene.add(api.Object(api.plane(api.vec3(*n), -2.0)).material(api.Material.diffuse(api.hex_color(col))))
    scene.add(api.Light.Ambient(AMB))
    return scene, api.Camera.look_at(api.vec3(0.3, -0.2, 1.0), api.vec3(-0.4, -0.5, -2.0), api.vec3(0, 1, 0), 1.0)


@pytest.fixture(scope="module")
def handles(gpu_ok):
    cache = {}

    def get(name, make, accel=capi.ACCEL_AUTO):
        if name not in cache:
            scene, cam = make()
            cache[name] = (scene, cam, device_scene(scene, accel))
        return cache[name]

    yield get
    for _, _, ds in cache.values():
        ds.close()


def _check_counts(st_wf, st_mk, w, h, spp, exact_segments):
    assert st_wf["segments"] == st_mk["segments"], (st_wf["segments"], st_mk["segments"])
    assert st_wf["rays"] == st_mk["rays"], (st_wf["rays"], st_mk["rays"])
    if exact_segments:
        assert st_wf["segments"] == w * h * spp


# -------------------------------------------------------------------------------------------- exact answers -------
ONE_VERTEX = {
    # name: (scene, max_bounces, closed form per pixel)
    "ambient_plane": (ambient_plane, 0, AMB * ALB),
    "backlit_plane_ks1": (backlit_plane, 0, AMB * ALB),
    "emissive_interior_mb0": (emissive_interior, 0, LE),
    "emissive_interior_mb1": (emissive_interior, 1, LE),
    "emissive_interior_mb40": (emissive_interior, 40, LE),
}


@pytest.mark.parametrize("spp", SPPS)
@pytest.mark.parametrize("w,h", SIZES, ids=["%dx%d" % s for s in SIZES])
@pytest.mark.parametrize("name", sorted(ONE_VERTEX))
def test_one_vertex_scene_is_its_closed_form(orc, handles, name, w, h, spp):
    """Every sample is one camera ray to a vertex that traces nothing more: the pixel is the closed form, and there is
    exactly one segment and one ray per sample."""
    make, mb, want = ONE_VERTEX[name]
    scene, cam, ds = handles(name.rsplit("_mb", 1)[0], make)
    got, st = render(ds, scene, cam, w, h, spp, mb)
    _, st_mk = render(ds, scene, cam, w, h, spp, mb, MK)
    assert rel_err(got, want[None, :]).max() <= 1e-6, (got.min(axis=0), got.max(axis=0), want)
    _check_counts(st, st_mk, w, h, spp, exact_segments=True)
    assert st["rays"] == w * h * spp
    if mb == 0:  # the f64 oracle bounces on from a dead vertex (test_one_pixel_image_and_many_bounces)
        _, st0 = orc.OracleScene(api.FlatScene(scene)).render(cam, params(scene, cam, w, h, spp, mb, WF, F64))
        assert st0["segments"] == w * h * spp


@pytest.mark.parametrize("spp", SPPS)
@pytest.mark.parametrize("w,h", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_half_environment_half_plane(orc, handles, w, h, spp):
    """Misses finish in one step, hits in two.  Rows wholly above or below the horizon are the closed form; in the
    horizon row every pixel is k samples of the plane and spp - k of the environment for a whole k, and equals the
    oracle on the same Philox streams unless some sample's hit decision differs between f32 and f64."""
    scene, cam, ds = handles("half_plane", half_plane)
    got, st = render(ds, scene, cam, w, h, spp, 0)
    _, st_mk = render(ds, scene, cam, w, h, spp, 0, MK)
    ref, st0 = orc.OracleScene(api.FlatScene(scene)).render(cam, params(scene, cam, w, h, spp, 0, WF, F64))
    _check_counts(st, st_mk, w, h, spp, exact_segments=True)
    assert st["rays"] == w * h * spp and st0["segments"] == w * h * spp
    # row y's camera rays have dir.y = yn + jitter, yn = (h - 2y - 1) / max(w, h), jitter in [-1, 1) / max(w, h)
    a = (h - 2 * np.arange(h) - 1)[:, None] * np.ones((1, w), int)
    a = a.reshape(-1)
    P, E = AMB * ALB, ENV
    assert rel_err(got[a >= 2], E).max(initial=0) <= 1e-6
    assert rel_err(got[a <= -2], P).max(initial=0) <= 1e-6
    mixed = np.abs(a) <= 1

    def hits(img):  # whole number of plane samples behind each mixed pixel, checked on every channel
        k = np.rint(spp * (img[:, 0] - E[0]) / (P[0] - E[0]))
        assert ((k >= 0) & (k <= spp)).all()
        recon = (k[:, None] * P + (spp - k)[:, None] * E) / spp
        assert rel_err(img, recon).max(initial=0) <= 1e-6
        return k

    k32, k64 = hits(got[mixed]), hits(ref[mixed])
    agree = rel_err(got[mixed], ref[mixed]).max(axis=1) <= 1e-6
    flips = k32 != k64
    assert (agree | flips).all()
    print("%dx%d %d spp: %d horizon pixels, %d with a flipped hit decision" % (w, h, spp, mixed.sum(), flips.sum()))
    # dir.y is the jitter itself in the horizon row: f32 and f64 disagree on a hit only where it is within rounding of 0
    assert flips.sum() <= 2


@pytest.mark.parametrize("spp", SPPS)
@pytest.mark.parametrize("w,h", SIZES, ids=["%dx%d" % s for s in SIZES])
@pytest.mark.parametrize("mb", [0, 3, 64])
def test_room_at_max_depth(handles, mb, w, h, spp):
    """Every vertex below max depth sends only its bounce ray, the last one nothing: the sample needs its whole step
    budget but one.  No closed form: the image is its own 1-spp renders recomposed, bit for bit, and has the
    megakernel's mean (the two engines differ by FMA contraction, which moves single paths, not the mean)."""
    scene, cam, ds = handles("room", room)
    got, st = render(ds, scene, cam, w, h, spp, mb)
    mk, st_mk = render(ds, scene, cam, w, h, spp, mb, MK)
    assert np.isfinite(got).all() and (got > 0).all()
    np.testing.assert_array_equal(got, recompose(singles(ds, scene, cam, w, h, spp, mb), spp, True))
    n = w * h * spp
    assert st["rays"] == st["segments"]
    assert abs(st["segments"] - st_mk["segments"]) <= 1e-4 * st_mk["segments"]
    if mb == 0:
        assert st["segments"] == st_mk["segments"] == n
        np.testing.assert_allclose(got, mk, rtol=1e-6)
    else:
        assert st["segments"] <= n * (mb + 1)
        assert abs(got.mean() - mk.mean()) <= (1e-3 if n >= 1000 else 3e-2) * mk.mean()


# -------------------------------------------------------------------------------------------- path groups ---------
REGIMES = [
    ("G_eq_nchunks", 7, 3, 130, 3, 3),
    ("G_eq_nchunks", 203, 117, 130, 3, 3),
    ("G_between", 257, 255, 2100, 29, 32),
    ("G_one", 1920, 1080, 130, 1, 3),
]


@pytest.mark.parametrize("regime,w,h,spp,G,nchunks", REGIMES, ids=["%s-%dx%d-%dspp" % r[:4] for r in REGIMES])
def test_path_group_regimes(handles, regime, w, h, spp, G, nchunks):
    """The ambient plane (exact) in each regime of paths per pixel slot: G == nchunks (each path one chunk),
    1 < G < nchunks (paths 0 .. nchunks - G - 1 sum two chunks), G == 1 < nchunks (one path sums every chunk)."""
    nch, chunk = sample_chunks(spp)
    assert (nch, wavefront_groups(pixel_slots(w, h), nch)) == (nchunks, G)
    if regime == "G_between":
        assert chunk == 66 and 1 < G < nchunks
    scene, cam, ds = handles("ambient_plane", ambient_plane)
    got, st = render(ds, scene, cam, w, h, spp, 0)
    assert rel_err(got, (AMB * ALB)[None, :]).max() <= 1e-6
    assert st["segments"] == st["rays"] == w * h * spp


# -------------------------------------------------------------------------------------------- recomposition -------
def _teapot_kd():
    cfg = scenes.teapot_scene()
    return cfg.scene, cfg.camera


def _dragon0():
    cfg = scenes.dragon_scene(level=0)
    return cfg.scene, cfg.camera


def _cfg(name):
    def make():
        cfg = scenes.glass_scene(256, 128) if name == "glass" else scenes.CONFIGS[name]()
        return cfg.scene, cfg.camera
    return make


PRODUCT = {
    # name: (scene, accel, max_bounces)
    "teapot_kd": (_teapot_kd, capi.ACCEL_KDTREE, 2),
    "dragon0_kd": (_dragon0, capi.ACCEL_KDTREE, 2),
    "cornell": (_cfg("cornell"), capi.ACCEL_AUTO, 6),
    "glass": (_cfg("glass"), capi.ACCEL_AUTO, 12),
    "lights": (pw._lights, capi.ACCEL_AUTO, 3),
}
RW, RH = 37, 19  # 3 x 3 tiles, ragged in both directions


@pytest.mark.parametrize("n", [16, 130])
@pytest.mark.parametrize("name", sorted(PRODUCT))
def test_wavefront_recomposes_bit_for_bit(handles, name, n):
    """N spp == the chunk-ordered sum of the N 1-spp renders, bit for bit; so are 3 and 7 shards added up and a
    DeviceBuffer's entry."""
    make, accel, mb = PRODUCT[name]
    scene, cam, ds = handles(name, make, accel)
    full, st = render(ds, scene, cam, RW, RH, n, mb)
    assert np.isfinite(full).all() and full.mean() > 0
    np.testing.assert_array_equal(full, recompose(singles(ds, scene, cam, RW, RH, n, mb), n, True))
    for shards in (3, 7):
        parts = [render(ds, scene, cam, RW, RH, n, mb, shard=(i, shards)) for i in range(shards)]
        np.testing.assert_array_equal(sum(p for p, _ in parts), full)
        assert sum(s["segments"] for _, s in parts) == st["segments"]
    buf = api.DeviceBuffer(ds, RW, RH)
    try:
        p, c_cam = params(scene, cam, RW, RH, n, mb, WF), cam.to_c()
        capi.check(capi.lib().rptb_sample_into(ds.handle, C.byref(c_cam), C.byref(p), buf.handle, None), "rptb_sample_into")
        np.testing.assert_array_equal(buf.sums(), full)
    finally:
        buf.close()


@pytest.mark.parametrize("precision", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", sorted(PRODUCT))
def test_megakernel_recomposes_bit_for_bit(handles, name, precision):
    make, accel, mb = PRODUCT[name]
    scene, cam, ds = handles(name, make, accel)
    for n in (16, 130):
        full, _ = render(ds, scene, cam, RW, RH, n, mb, MK, precision)
        np.testing.assert_array_equal(full, recompose(singles(ds, scene, cam, RW, RH, n, mb, MK, precision), n, precision == F32))


@pytest.mark.parametrize("engine,precision", [(WF, F32), (MK, F32), (MK, F64)], ids=["wf", "mk-f32", "mk-f64"])
def test_recomposes_at_2100_spp(handles, engine, precision):
    """32 chunks of 66 samples, the last of 54, on one 16x8 tile (the wavefront then has G = nchunks)."""
    scene, cam, ds = handles("cornell", _cfg("cornell"))
    w, h, n, mb = 16, 8, 2100, 6
    assert sample_chunks(n) == (32, 66)
    full, _ = render(ds, scene, cam, w, h, n, mb, engine, precision)
    np.testing.assert_array_equal(full, recompose(singles(ds, scene, cam, w, h, n, mb, engine, precision), n, precision == F32))


# -------------------------------------------------------------------------------------------- scratch reuse -------
def test_scratch_reuse_matches_a_fresh_handle(gpu_ok):
    """On one handle, chunk sums left by a 32-chunk megakernel render and path scratch grown for a bigger image change
    nothing: every wavefront render equals the same render on a fresh handle."""
    make, accel, mb = PRODUCT["teapot_kd"]
    scene, cam = make()
    big, small = (640, 360, 130), (24, 16, 70)  # 3 x 230 400 and 2 x 768 paths

    def fresh(w, h, n):
        with device_scene(scene, accel) as d:
            return render(d, scene, cam, w, h, n, mb)[0]

    ref_big, ref_small = fresh(*big), fresh(*small)
    with device_scene(scene, accel) as ds:
        render(ds, scene, cam, 64, 40, 2100, mb, MK)
        np.testing.assert_array_equal(render(ds, scene, cam, *small, mb)[0], ref_small)
        np.testing.assert_array_equal(render(ds, scene, cam, *big, mb)[0], ref_big)  # regrows the path scratch
        np.testing.assert_array_equal(render(ds, scene, cam, *small, mb)[0], ref_small)
        np.testing.assert_array_equal(render(ds, scene, cam, *big, mb)[0], ref_big)


def test_wavefront_renders_left_on_caller_streams_do_not_share_scratch(gpu_ok):
    """test_gpu_multi's stream test through the wavefront engine on the kd-tree teapot: renders left running on two
    caller streams and a host render on the library's stream, with growing chunk counts (4, 6, 3)."""
    import torch

    scene, cam = _teapot_kd()
    w, h, mb = 256, 256, 2
    c_cam = cam.to_c()
    dev = torch.device("cuda:0")
    with device_scene(scene, capi.ACCEL_KDTREE) as ds:
        def device_call(spp, first, stream, out):
            p = params(scene, cam, w, h, spp, mb, WF, first=first, seed=3)
            capi.check(capi.lib().rptb_render_samples_device(ds.handle, C.byref(c_cam), C.byref(p), C.c_void_p(out.data_ptr()),
                                                             C.c_void_p(stream.cuda_stream), None), "rptb_render_samples_device")
        refs = {}
        s0 = torch.cuda.Stream(dev)
        for key, (spp, first) in {"a": (200, 0), "b": (330, 1000), "c": (130, 5000)}.items():
            out = torch.zeros(w * h * 3, dtype=torch.float32, device=dev)
            device_call(spp, first, s0, out)
            s0.synchronize()
            refs[key] = out.cpu().numpy().copy()
        s1, s2 = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        for rep in range(3):
            oa = torch.zeros(w * h * 3, dtype=torch.float32, device=dev)
            ob = torch.zeros(w * h * 3, dtype=torch.float32, device=dev)
            device_call(200, 0, s1, oa)
            device_call(330, 1000, s2, ob)
            host, _ = render(ds, scene, cam, w, h, 130, mb, first=5000, seed=3)
            s1.synchronize()
            s2.synchronize()
            np.testing.assert_array_equal(oa.cpu().numpy(), refs["a"])
            np.testing.assert_array_equal(ob.cpu().numpy(), refs["b"])
            np.testing.assert_array_equal(host.astype(np.float32).ravel(), refs["c"])


# -------------------------------------------------------------------------------------------- light slots ---------
def lit_plane(ks):
    """The diffuse plane at max_bounces 0 under `ks` point lights in front of it, no occluders; ambient lights first,
    between the sampled lights and last."""
    scene = api.Scene()
    scene.add(api.Object(api.plane(api.vec3(0, 0, 1), 0.0)).material(api.Material.diffuse(ALB)))
    rng = np.random.default_rng(ks)
    pts = [api.Light.Point(rng.uniform(2.0, 8.0, 3), np.array([rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(1, 4)]))
           for _ in range(ks)]
    lights = [api.Light.Ambient(0.2 * AMB)] + pts[:ks // 2] + [api.Light.Ambient(0.1 * AMB)] + pts[ks // 2:] + \
        [api.Light.Ambient(api.vec3(0.0, 0.02, 0.0))]
    for l in lights:
        scene.add(l)
    return scene, api.Camera.default()


@pytest.mark.parametrize("ks", [0, 1, 8])
def test_sampled_light_slots(orc, ks):
    scene, cam = lit_plane(ks)
    w, h, spp = 48, 32, 16
    with device_scene(scene) as ds:
        got, st = render(ds, scene, cam, w, h, spp, 0)
        _, st_mk = render(ds, scene, cam, w, h, spp, 0, MK)
    ref, _ = orc.OracleScene(api.FlatScene(scene)).render(cam, params(scene, cam, w, h, spp, 0, WF, F64))
    np.testing.assert_allclose(got, ref, rtol=1e-5)
    assert st["rays"] == st_mk["rays"] == w * h * spp * (1 + ks)
    assert st["segments"] == w * h * spp


def test_ninth_sampled_light_is_refused_and_auto_takes_the_megakernel(gpu_ok):
    """Eight sampled lights are the wavefront's limit (9 ray slots per path).  A kd-tree scene that ENGINE_AUTO sends to
    the wavefront with 8 lights goes to the megakernel with 9, and ENGINE_WAVEFRONT refuses it."""
    mesh = scenes.dragon_mesh(0)
    w, h = 32, 16
    for ks, engine in ((8, WF), (9, MK)):
        scene = api.Scene()
        scene.add(api.Object(mesh.scale(api.vec3(3.4, 3.4, 3.4))).material(api.Material.specular(api.hex_color(0xB7CA79), 0.1)))
        scene.add(api.Object(api.plane(api.vec3(0, 1, 0), -1.0)).material(api.Material.diffuse(ALB)))
        for i in range(ks):
            scene.add(api.Light.Point(api.vec3(5, 5, 5), api.vec3(i - 4.0, 5.0, 4.0)))
        cam = api.Camera.look_at(api.vec3(-2.5, 4.0, 6.5), api.vec3(0, 0, 0), api.vec3(0, 1, 0), 0.5)
        with device_scene(scene, capi.ACCEL_KDTREE) as ds:
            auto, st = render(ds, scene, cam, w, h, 2, 1, AUTO)
            assert st["engine"] == engine
            np.testing.assert_array_equal(auto, render(ds, scene, cam, w, h, 2, 1, engine)[0])
            if ks == 9:
                p, c_cam, out = params(scene, cam, w, h, 2, 1, WF), cam.to_c(), np.empty((w * h, 3))
                assert capi.lib().rptb_render_samples(ds.handle, C.byref(c_cam), C.byref(p), out.ctypes.data_as(capi.c_double_p),
                                                      None) == capi.ERR_UNSUPPORTED
