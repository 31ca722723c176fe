"""ctypes binding of tests/hostemu/_build/libhostemu.so -- TEST INFRASTRUCTURE, NOT PRODUCT.

The device geometry functions (rpt_b200/csrc/geometry.cuh, shading.cuh) compiled for the host; see
hostemu.cu.  Nothing under rpt_b200/ imports this."""
import ctypes as C
import os
import subprocess

import numpy as np

from rpt_b200 import _capi as capi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_build", "libhostemu.so")
_lib = None
dp = capi.c_double_p


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "hostemu"], cwd=os.path.dirname(os.path.dirname(_HERE)))
        L = C.CDLL(LIB_PATH)
        L.hostemu_scene_create.restype = C.c_void_p
        L.hostemu_scene_create.argtypes = [C.POINTER(capi.SceneDesc), C.c_char_p, C.c_size_t]
        L.hostemu_scene_destroy.argtypes = [C.c_void_p]
        L.hostemu_scene_features.argtypes = [C.c_void_p]
        L.hostemu_closest_hit.argtypes = [C.c_void_p, dp, C.c_uint64, C.c_double, C.c_uint32, dp, capi.c_i32_p, dp,
                                          capi.c_u32_p, dp, C.POINTER(capi.Stats)]
        L.hostemu_flat_table.restype = None
        L.hostemu_flat_table.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), capi.c_u32_p, C.POINTER(C.c_float), C.POINTER(C.c_float)]
        L.hostemu_pick_variant.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_uint32, capi.c_i32_p]
        L.hostemu_render.argtypes = [C.c_void_p, C.POINTER(capi.Camera), C.POINTER(capi.RenderParams), C.c_int, dp, C.POINTER(capi.Stats)]
        L.hostemu_occluded.argtypes = [C.c_void_p, dp, dp, C.c_uint64, C.c_double, C.c_uint32, C.c_int, capi.c_i32_p]
        L.hostemu_bvh_check.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64)]
        L.hostemu_bvh8_probe.argtypes = [C.c_void_p, C.c_uint32, dp, C.c_uint64, C.c_int, dp, C.POINTER(C.c_int64), C.POINTER(C.c_uint64)]
        L.hostemu_bvh4_probe.argtypes = L.hostemu_bvh8_probe.argtypes
        L.hostemu_draws.restype = None
        L.hostemu_draws.argtypes = [C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
        L.hostemu_illuminate.argtypes = [C.c_void_p, C.c_uint32, dp, C.c_uint64, C.c_uint64, C.c_uint32, dp, dp, dp]
        _lib = L
    return _lib


LIST_LIB_PATH = os.path.join(_HERE, "_build", "libhostemu_list.so")
_list_lib = None


def list_lib():
    """tests/hostemu/_build/libhostemu_list.so: this emulation plus adaptive sampling's list schedule and criterion
    (hostemu_list.cu)."""
    global _list_lib
    if _list_lib is None:
        lib()  # `make hostemu` builds both emulation libraries
        L = C.CDLL(LIST_LIB_PATH)
        L.hostemu_scene_create.restype = C.c_void_p
        L.hostemu_scene_create.argtypes = [C.POINTER(capi.SceneDesc), C.c_char_p, C.c_size_t]
        L.hostemu_scene_destroy.argtypes = [C.c_void_p]
        L.hostemu_scene_features.argtypes = [C.c_void_p]
        L.hostemu_render.argtypes = [C.c_void_p, C.POINTER(capi.Camera), C.POINTER(capi.RenderParams), C.c_int, dp, C.POINTER(capi.Stats)]
        L.hostemu_render_list.argtypes = [C.c_void_p, C.POINTER(capi.Camera), C.POINTER(capi.RenderParams), C.c_int,
                                          C.POINTER(C.c_uint8), dp, C.POINTER(capi.Stats)]
        L.hostemu_adaptive_active.restype = None
        L.hostemu_adaptive_active.argtypes = [capi.c_u32_p, dp, dp, C.c_uint64, C.POINTER(capi.Adaptive), C.POINTER(C.c_uint8)]
        L.hostemu_pick_render_list.argtypes = [C.c_int, C.c_int, C.c_uint32, C.c_uint32, capi.c_i32_p]
        _list_lib = L
    return _list_lib


def pick_render_list(features, stats, precision, max_bounces):
    """The list-scheduled variant launch_render_list_impl picks (pick_render_list, launch.h): ((STATS, FEAT, MAXD), whether
    it is in RenderListVariantsF32 / F64)."""
    out = (C.c_int32 * 3)()
    compiled = list_lib().hostemu_pick_render_list(features, stats, precision, max_bounces, out)
    return (bool(out[0]), int(out[1]), int(out[2])), bool(compiled)


ENGINE_RENDER, ENGINE_VX, ENGINE_CLOSEST_HIT = 0, 1, 2


def pick_variant(engine, features, stats, precision, max_bounces):
    """The kernel variant the launchers pick (launch.h): ((STATS, FEAT, MAXD), whether it is compiled)."""
    out = (C.c_int32 * 3)()
    compiled = lib().hostemu_pick_variant(engine, features, stats, precision, max_bounces, out)
    return (bool(out[0]), int(out[1]), int(out[2])), bool(compiled)


def draws(seed, pixel, sample, n, ensure_every=0):
    """(u64[n], u32[4, n]): the stream as the f64 generator and as the four f32 buffers of rng.cuh hand it out."""
    o64 = np.empty(n, np.uint64)
    o32 = np.empty((4, n), np.uint32)
    lib().hostemu_draws(seed, pixel, sample, n, ensure_every, o64.ctypes.data_as(C.POINTER(C.c_uint64)), o32.ctypes.data_as(C.POINTER(C.c_uint32)))
    return o64, o32


class EmuScene:
    def __init__(self, flat):
        self.flat = flat
        err = C.create_string_buffer(512)
        self.handle = C.c_void_p(lib().hostemu_scene_create(C.byref(flat.desc), err, 512))
        if not self.handle:
            raise ValueError(err.value.decode())

    def close(self):
        if self.handle:
            lib().hostemu_scene_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def features(self) -> int:
        return int(lib().hostemu_scene_features(self.handle))

    def render(self, camera, params, ext_bvh: bool = False):
        """Renderer::sample through the emulated megakernel -> ((w*h, 3) float64, stats dict, FEAT bits of the variant)."""
        out = np.empty((params.width * params.height, 3))
        st = capi.Stats()
        cam = camera.to_c() if hasattr(camera, "to_c") else camera
        feat = lib().hostemu_render(self.handle, C.byref(cam), C.byref(params), 1 if ext_bvh else 0, out.ctypes.data_as(dp), C.byref(st))
        if feat < -0:
            raise ValueError("bad render parameters")
        return out, st.as_dict(), int(feat)

    def occluded(self, rays, tmax, t_min=1e-12, precision=capi.PRECISION_F32, use_bvh=True):
        """Any-hit shadow queries: 1 where something lies in [t_min, tmax) on the ray."""
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        tmax = np.ascontiguousarray(np.broadcast_to(np.asarray(tmax, dtype=np.float64), (rays.shape[0],)))
        out = np.empty(rays.shape[0], np.int32)
        if lib().hostemu_occluded(self.handle, rays.ctypes.data_as(dp), tmax.ctypes.data_as(dp), rays.shape[0], t_min, precision,
                                  1 if use_bvh else 0, out.ctypes.data_as(capi.c_i32_p)) < 0:
            raise RuntimeError("occluded: the variant the launchers pick is not compiled")
        return out

    def bvh_check(self, mesh: int = 0):
        """{nodes, leaves, max_leaf, depth, distinct, violations} of the BVH of mesh `mesh`, or None if it has none."""
        out = (C.c_uint64 * 6)()
        if lib().hostemu_bvh_check(self.handle, mesh, out) != 0:
            return None
        return dict(zip(("nodes", "leaves", "max_leaf", "depth", "distinct", "violations"), [int(v) for v in out]))

    def bvh8_probe(self, mesh, rays, any_hit=False):
        """Mesh-local rays through the binary BVH and through its eight-wide collapse: (t[n, 2], tri[n, 2], info) or None."""
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        n = rays.shape[0]
        t = np.empty((n, 2))
        tri = np.empty((n, 2), np.int64)
        info = (C.c_uint64 * 5)()
        if lib().hostemu_bvh8_probe(self.handle, mesh, rays.ctypes.data_as(dp), n, 1 if any_hit else 0, t.ctypes.data_as(dp),
                                    tri.ctypes.data_as(C.POINTER(C.c_int64)), info) != 0:
            return None
        return t, tri, dict(zip(("nodes8", "max_children", "empty_slots", "visits2", "visits8"), [int(v) for v in info]))

    def bvh4_probe(self, mesh, rays, any_hit=False):
        """Mesh-local rays through the binary BVH and through its four-wide collapse: (t[n, 2], tri[n, 2], info) or None."""
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        n = rays.shape[0]
        t = np.empty((n, 2))
        tri = np.empty((n, 2), np.int64)
        info = (C.c_uint64 * 6)()
        if lib().hostemu_bvh4_probe(self.handle, mesh, rays.ctypes.data_as(dp), n, 1 if any_hit else 0, t.ctypes.data_as(dp),
                                    tri.ctypes.data_as(C.POINTER(C.c_int64)), info) != 0:
            return None
        return t, tri, dict(zip(("nodes4", "empty_slots", "visits2", "visits4", "tris2", "tris4"), [int(v) for v in info]))

    def closest_hit(self, rays, t_min=1e-12, precision=capi.PRECISION_F64):
        t, obj, nrm, _, _, st = self.closest_hit_detail(rays, t_min, precision)
        return t, obj, nrm, st

    def closest_hit_detail(self, rays, t_min=1e-12, precision=capi.PRECISION_F64):
        """closest_hit plus Hit::aux (the triangle or cube face hit) and the barycentrics (v, w) as (n, 2)."""
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        n = rays.shape[0]
        t = np.empty(n)
        obj = np.empty(n, np.int32)
        nrm = np.empty((n, 3))
        aux = np.empty(n, np.uint32)
        bvw = np.empty((n, 2))
        st = capi.Stats()
        if lib().hostemu_closest_hit(self.handle, rays.ctypes.data_as(dp), n, t_min, precision, t.ctypes.data_as(dp),
                                     obj.ctypes.data_as(capi.c_i32_p), nrm.ctypes.data_as(dp), aux.ctypes.data_as(capi.c_u32_p),
                                     bvw.ctypes.data_as(dp), C.byref(st)) < 0:
            raise RuntimeError("closest_hit: the variant the launchers pick is not compiled")
        return t, obj, nrm, aux, bvw, st.as_dict()

    def flat_table(self):
        """The packed primitive table as built (scene_dev.cuh): (words as uint32 (nwords, 4), flat_ok, inverse-transform
        rows of every f32 object record as float32 (nobjects, 3, 4), tri48 of every mesh's triangles as float32
        (ntris over all meshes, 3, 4), meshes in order)."""
        info = (C.c_uint64 * 4)()
        lib().hostemu_flat_table(self.handle, info, None, None, None)
        nwords, ok, nobj, ntris = (int(v) for v in info)
        words = np.zeros((nwords, 4), np.uint32)
        inv = np.zeros((nobj, 3, 4), np.float32)
        tri48 = np.zeros((ntris, 3, 4), np.float32)
        fp = C.POINTER(C.c_float)
        lib().hostemu_flat_table(self.handle, info, words.ctypes.data_as(capi.c_u32_p), inv.ctypes.data_as(fp), tri48.ctypes.data_as(fp))
        return words, bool(ok), inv, tri48

    def illuminate(self, light, pos, seed=0, precision=capi.PRECISION_F64):
        pos = np.ascontiguousarray(pos, dtype=np.float64).reshape(-1, 3)
        n = pos.shape[0]
        inten, wi, dist = np.empty((n, 3)), np.empty((n, 3)), np.empty(n)
        lib().hostemu_illuminate(self.handle, light, pos.ctypes.data_as(dp), n, seed, precision, inten.ctypes.data_as(dp),
                                 wi.ctypes.data_as(dp), dist.ctypes.data_as(dp))
        return inten, wi, dist
