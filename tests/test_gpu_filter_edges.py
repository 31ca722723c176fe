"""The device Buffer's five filter entry points on programmed edge-case states: rptb_buffer_denoise (and its bytes),
rptb_buffer_denoise_variance, rptb_buffer_denoise_error, rptb_buffer_denoise_select, rptb_buffer_denoise_cross and the
guided marks (rptb_sample_into_guided / _guided_error).  Rendered buffers are finite, have continuous features and hold
counts >= 2; these states are not: NaN and +-inf sums, inf M2, NaN HALF, clusters of them on corners and borders, a pixel
whose every neighbour is non-finite, zero variance, all-miss regions (z = inf, N = 0, albedo 1), black albedo, negative
means, depth steps and constant-depth planes -- at 1x1, 1x7, 7x1, 2x2 and 3x5 (every tap, the 3x3 prefilter, the
gradients and the 5x5 smoothing off the image), around the 32x8 block (31x9, 32x8, 33x7) and at 97x61.

Each state is programmed without rendering it: one plain entry and the features are rendered into a world-1 shard with
halves (so its header records the entry and feature cameras, which the guided calls check), its exchange block is
exported, its planes (sums, M2, counts, HALF and the four feature sums) are overwritten on the host through
distributed.shard_block_layout(..., halves=True), and it is imported into a whole buffer with halves.

Checks: every output against the numpy restatements (tests/denoise_ref.py, halves_ref.py, select_ref.py, cross_ref.py,
guided_ref.py) on the buffer's own read-backs, within 1e-12 of the largest finite value, with NaN at the same places and
infinities equal; and properties no restatement shares -- scale covariance, the locality of a non-finite pixel, scratch
reuse across the entry points, replicas, and finite colours for every albedo_eps the parameters accept.  Breaking any one
of the filter's rules for non-finite values -- the keep rule, the non-finite tap skip, the 3x3 prefilter's finiteness
test, select_smooth's finiteness test or the cross blend's `first` flag -- fails the "nonfinite" cases of
test_entry_points_match_numpy.  On one H100 80GB HBM3 at 700 W the whole file ran in 59 s."""
import ctypes as C

import numpy as np
import pytest
import torch

from rpt_b200 import _capi as capi
from rpt_b200 import api, distributed, scenes
from rpt_b200.distributed import ShardBuffer
from tests import cross_ref as xref
from tests import denoise_ref as dr
from tests import guided_ref as gref
from tests import halves_ref as href
from tests import select_ref as sref
from tests import util

pytestmark = pytest.mark.gpu

HEADER_ENTRIES = 24  # byte offset of ShardHeader::entries (rpt_b200/csrc/api.cu)
RAYS = 4  # feature rays of every programmed state


@pytest.fixture(autouse=True)
def _repeated_devices(monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")


def _renderer(w, h, devices=(0,)):
    cfg = scenes.sphere_scene()
    return (api.Renderer(cfg.scene, cfg.camera).width(w).height(h).max_bounces(1).seed(7).precision(capi.PRECISION_F32)
            .device(list(devices)))


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


class HalvesBlock:
    """A genuine world-1 shard block with halves and features, editable per pixel on the host: the renderer (of size
    w x h) first adds one plain entry and RAYS feature rays, so the header records both cameras."""

    def __init__(self, r, w, h):
        self.w, self.h = w, h
        self.lay = distributed.shard_block_layout(w, h, 1, True, halves=True)
        self.slot = distributed.gather_permutation(w, h, 1)  # pixel p (row-major) -> its slot in the block
        s = ShardBuffer(r.device_scene(), w, h, rank=0, world=1, halves=True)
        r.sample(1, s, want_stats=False)
        r.sample_features(RAYS, s)
        dev = torch.empty(s.block_bytes(True), dtype=torch.uint8, device="cuda:0")
        assert dev.numel() == self.lay["bytes"]
        s.export(dev, True)
        torch.cuda.synchronize()
        self.feature_rays = s.feature_rays
        s.close()
        self.host = dev.cpu().numpy().copy()
        self.dev = dev

    def _plane(self, name, dtype, values):
        n = self.lay["slots"]
        a = self.host[self.lay[name]:self.lay[name] + n * values * np.dtype(dtype).itemsize].view(dtype)
        return a.reshape(n, values) if values > 1 else a

    def program(self, st):
        """The state's per-pixel planes into the block's slots, its largest count into the header's entry count."""
        npix = self.w * self.h
        self._plane("sums", np.float64, 3)[self.slot] = st["sums"].reshape(npix, 3)
        self._plane("m2", np.float64, 1)[self.slot] = st["m2"].reshape(npix)
        self._plane("counts", np.uint32, 1)[self.slot] = st["counts"].reshape(npix)
        self._plane("half", np.float64, 3)[self.slot] = st["half"].reshape(npix, 3)
        n = self.lay["slots"]
        f = self.host[self.lay["features"]:self.lay["counts"]].view(np.float64)
        f[:3 * n].reshape(n, 3)[self.slot] = st["sn"].reshape(npix, 3)
        f[3 * n:6 * n].reshape(n, 3)[self.slot] = st["sa"].reshape(npix, 3)
        f[6 * n:7 * n][self.slot] = st["hits"].reshape(npix)
        f[7 * n:8 * n][self.slot] = st["sz"].reshape(npix)
        self.host[HEADER_ENTRIES:HEADER_ENTRIES + 4].view(np.uint32)[0] = int(st["counts"].max())
        self.dev.copy_(torch.from_numpy(self.host))
        torch.cuda.synchronize()
        return self

    def import_into(self, buf):
        capi.check(capi.lib().rptb_buffer_import_shards(buf.handle, C.c_void_p(self.dev.data_ptr()), 1, 1), "rptb_buffer_import_shards")
        buf.feature_rays = self.feature_rays
        buf.entries = int(self.host[HEADER_ENTRIES:HEADER_ENTRIES + 4].view(np.uint32)[0])
        return buf


# ---- the states ----------------------------------------------------------------------------------------------------
def _base(w, h, rng, lo=0.0, hi=2.0):
    """Finite random values: counts 2-9 (odd ones and n = 2, n_B = 1, among them), sums n * mean, HALF about n_B / n of
    them, M2 >= 0; every ray a hit, unit normals near +z, depths 1-9, albedo 0-1."""
    counts = rng.integers(2, 10, (h, w)).astype(np.uint32)
    counts.reshape(-1)[::3] = 2
    n = counts.astype(np.float64)[..., None]
    nb = (counts >> 1).astype(np.float64)[..., None]
    mean = rng.uniform(lo, hi, (h, w, 3))
    sums = mean * n
    half = mean * nb + rng.normal(0.0, 0.3, (h, w, 3)) * np.sqrt(nb)
    m2 = rng.uniform(0.0, 3.0, (h, w)) * counts
    hits = np.full((h, w), float(RAYS))
    nrm = np.stack([rng.normal(0, 0.2, (h, w)), rng.normal(0, 0.2, (h, w)), np.ones((h, w))], -1)
    nrm /= np.linalg.norm(nrm, axis=-1, keepdims=True)
    return {"sums": sums, "half": half, "m2": m2, "counts": counts, "hits": hits, "sn": nrm * RAYS,
            "sz": rng.uniform(1.0, 9.0, (h, w)) * RAYS, "sa": rng.uniform(0.0, 1.0, (h, w, 3)) * RAYS}


def _cells(w, h, rng, k):
    """k random pixels (row, column), at most every pixel."""
    p = rng.choice(w * h, size=min(k, w * h), replace=False)
    return p // w, p % w


def state_baseline(w, h, rng):
    return _base(w, h, rng)


def state_nonfinite(w, h, rng):
    """NaN and +-inf sums (all channels or one), inf M2 and NaN HALF: isolated, in a 2x2 cluster, on the four corners
    and a border; one pixel whose 8 neighbours are all non-finite (its one finite tap is itself at step 1); and sums inf
    with M2 finite, whose v still enters its neighbours' prefiltered variance g."""
    st = _base(w, h, rng)
    S, M2, HF = st["sums"], st["m2"], st["half"]
    bad = [np.nan, np.inf, -np.inf]
    for k, (y, x) in enumerate(zip(*_cells(w, h, rng, max(1, w * h // 12)))):
        kind = k % 5
        if kind == 0:
            S[y, x] = bad[k % 3]
        elif kind == 1:
            S[y, x, k % 3] = bad[(k + 1) % 3]
        elif kind == 2:
            M2[y, x] = np.inf
        elif kind == 3:
            HF[y, x, k % 3] = np.nan
        else:
            S[y, x, 1] = np.inf  # M2 stays finite: v finite, i not
    for y, x in ((0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1)):
        S[y, x, 0] = bad[(x + y) % 3]
    S[h // 2, 0] = np.nan  # the left border
    if w >= 2 and h >= 2:
        y0, x0 = (h - 2) // 3, (w - 2) // 2
        S[y0:y0 + 2, x0:x0 + 2] = np.inf
        M2[y0 + 1, x0] = np.inf
    if w >= 3 and h >= 3:
        cy, cx = h - 2, w - 2
        ring = [(cy + dy, cx + dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if dy or dx]
        for k, (y, x) in enumerate(ring):
            if k % 2:
                S[y, x] = bad[k % 3]
            else:
                M2[y, x] = np.inf
        S[cy, cx], M2[cy, cx], HF[cy, cx] = st["counts"][cy, cx] * 0.5, 1.0, 0.25 * (st["counts"][cy, cx] >> 1)
    return st


def state_flat(w, h, rng):
    """M2 = 0 on the left part, over equal colours in its top rows and unequal ones below."""
    st = _base(w, h, rng)
    xs = slice(0, max(1, w // 2))
    st["m2"][:, xs] = 0.0
    top = slice(0, max(1, h // 2))
    c = np.array([0.3, 0.6, 0.9])
    st["sums"][top, xs] = c * st["counts"][top, xs, None]
    st["half"][top, xs] = c * (st["counts"][top, xs, None] >> 1)
    st["sa"][top, xs] = 0.5 * RAYS
    return st


def state_flat_all(w, h, rng):
    """M2 = 0 everywhere: every lden is eps_l alone."""
    st = _base(w, h, rng)
    st["m2"][:] = 0.0
    st["sums"][::2] = 0.7 * st["counts"][::2, :, None]
    return st


def state_misses(w, h, rng):
    """hits = 0 (z = inf, N = 0, albedo 1) on a block of columns and a random tenth of pixels, next to hits, some of them
    partial (0 < hits < rays)."""
    st = _base(w, h, rng)
    miss = np.zeros((h, w), bool)
    miss[:, w // 3:max(w // 3 + 1, (2 * w) // 3)] = True
    miss |= rng.random((h, w)) < 0.1
    part = ~miss & (rng.random((h, w)) < 0.3)
    st["hits"][part] = rng.integers(1, RAYS, int(part.sum()))
    for k in ("sn", "sa"):
        st[k][part] *= (st["hits"][part] / RAYS)[:, None]
    st["sz"][part] *= st["hits"][part] / RAYS
    st["hits"][miss], st["sn"][miss], st["sz"][miss], st["sa"][miss] = 0.0, 0.0, 0.0, 0.0
    return st


def state_all_miss(w, h, rng):
    st = _base(w, h, rng)
    st["hits"][:], st["sn"][:], st["sz"][:], st["sa"][:] = 0.0, 0.0, 0.0, 0.0
    return st


def state_black(w, h, rng):
    """A zero albedo channel (Sa = 0 with hits = rays) on half the pixels, with sums 0 on some of them and > 0 on the
    rest; and a fully black albedo on a quarter."""
    st = _base(w, h, rng)
    black = rng.random((h, w)) < 0.5
    ch = rng.integers(0, 3, (h, w))
    for c in range(3):
        st["sa"][black & (ch == c), c] = 0.0
    full = rng.random((h, w)) < 0.25
    st["sa"][full] = 0.0
    zero = (black | full) & (rng.random((h, w)) < 0.5)
    st["sums"][zero], st["half"][zero] = 0.0, 0.0
    return st


def state_negative(w, h, rng):
    """Negative means (a signed cosine's glass quirk), a third of them within 1e-6 of 0, so the guided tolerance
    t = rel_tol m' + abs_tol goes negative."""
    st = _base(w, h, rng, -2.0, 0.5)
    near = rng.random((h, w)) < 0.33
    n = st["counts"].astype(np.float64)
    st["sums"][near] = rng.uniform(-1e-6, 1e-6, (int(near.sum()), 3)) * n[near, None]
    st["half"][near] = 0.5 * st["sums"][near]
    return st


def state_depth(w, h, rng):
    """Constant-depth planes (zero gradients, ties between the forward and backward differences) with a step between
    them, one column and one row at a third depth, and normals all +z."""
    st = _base(w, h, rng)
    z = np.where(np.arange(w)[None, :] < w // 2, 2.0, 6.0) * np.ones((h, 1))
    z[h // 2, :] = 4.0
    z[:, (3 * w) // 4] = 3.0
    st["sz"] = z * RAYS
    st["sn"][:] = 0.0
    st["sn"][..., 2] = RAYS
    return st


STATES = {f.__name__[6:]: f for f in (state_baseline, state_nonfinite, state_flat, state_flat_all, state_misses, state_all_miss,
                                      state_black, state_negative, state_depth)}
SHAPES = [(1, 1), (1, 7), (7, 1), (2, 2), (3, 5), (31, 9), (32, 8), (33, 7), (97, 61)]
PARAMS = [api.Denoise(iterations=1), api.Denoise(iterations=5), api.Denoise(iterations=12), api.Denoise(iterations=5, sigma_luminance=0.0),
          api.Denoise(iterations=5, sigma_depth=0.0), api.Denoise(iterations=5, sigma_normal=0), api.Denoise(iterations=5, sigma_normal=1),
          api.Denoise(iterations=5, albedo_eps=1e-12), api.Denoise(iterations=1, albedo_eps=1.0),
          api.Denoise(iterations=12, sigma_luminance=0.0, albedo_eps=1e-12)]


def _state(name, w, h, seed=0):
    return STATES[name](w, h, np.random.default_rng([seed, w, h, len(name)]))


def _with(d, **kw):
    p = dict(iterations=d.iterations, sigma_normal=d.sigma_normal, sigma_depth=d.sigma_depth, sigma_luminance=d.sigma_luminance,
             albedo_eps=d.albedo_eps)
    p.update(kw)
    return api.Denoise(**p)


def _setup(st, w, h, devices=(0,)):
    """The state's block (made on one part: a shard is refused on a scene with replicas) and a buffer with halves on
    `devices` holding it, with that buffer's renderer."""
    r1 = _renderer(w, h)
    b = HalvesBlock(r1, w, h).program(st)
    if list(devices) == [0]:
        r = r1
    else:
        r1.close()
        r = _renderer(w, h, devices)
    return r, b, b.import_into(r.device_buffer(halves=True))


def _readback(buf):
    """(sums, m2, half, counts, nrm, z, albedo) as the restatements take them, from the buffer's own read-backs."""
    h, w = buf.height, buf.width
    sums, m2, counts = buf.pixel_stats()
    nrm, z, albedo, _ = buf.features()
    return (sums.reshape(h, w, 3), m2.reshape(h, w), buf.half_sums().reshape(h, w, 3), counts.reshape(h, w), nrm, z, albedo)


def _close(got, want, rel=1e-12):
    """NaN at the same places, infinities equal, the finite values within rel of the largest finite value."""
    assert np.array_equal(np.isnan(got), np.isnan(want)), np.argwhere(np.isnan(got) != np.isnan(want))[:8]
    inf = np.isinf(want)
    assert np.array_equal(np.isinf(got), inf) and np.array_equal(got[inf], want[inf]), np.argwhere(np.isinf(got) != inf)[:8]
    fin = np.isfinite(want)
    scale = np.max(np.abs(want[fin]), initial=0.0)
    assert np.max(np.abs(got[fin] - want[fin]), initial=0.0) <= rel * scale, (np.max(np.abs(got[fin] - want[fin])), scale)


def _bytes(c):
    """The film resolve of one entry at radius 0 (film.cu): fmin(fmax(c, 0), 1), so NaN gives 0, +inf 255, -inf 0; then
    gamma 1/2.2 and the truncating cast."""
    v = np.fmin(np.fmax(c, 0.0), 1.0)
    return (v ** (1.0 / 2.2) * 255.0).astype(np.uint8)


# ---- the route itself ----------------------------------------------------------------------------------------------
def test_programmed_halves_state_is_what_the_buffer_reads(gpu_ok):
    """Random colour, HALF and feature planes (non-finite ones included), programmed into a 97x61 block with halves, read
    back through pixel_stats() and half_sums() bit for bit and through features() as tests/denoise_ref.py resolves them,
    on one part and on three."""
    w, h = 97, 61
    st = _state("nonfinite", w, h)
    st["hits"] = np.random.default_rng(3).integers(0, RAYS + 1, (h, w)).astype(np.float64)
    st["sn"] *= (st["hits"] / RAYS)[..., None]
    st["sa"] *= (st["hits"] / RAYS)[..., None]
    st["sz"] *= st["hits"] / RAYS
    npix = w * h
    wn, wz, wa, wf = dr.features_resolve(st["hits"], st["sn"], st["sz"], st["sa"], float(RAYS))
    for devices in ([0], [0, 0, 0]):
        r, b, buf = _setup(st, w, h, devices)
        assert b.feature_rays == RAYS
        gs, gm, gc = buf.pixel_stats()
        assert _bits(gs) == _bits(st["sums"].reshape(npix, 3)) and _bits(gm) == _bits(st["m2"].reshape(npix))
        assert _bits(gc) == _bits(st["counts"].reshape(npix))
        assert _bits(buf.half_sums()) == _bits(st["half"].reshape(npix, 3))
        for g, want in zip(buf.features(), (wn, wz, wa, wf)):
            assert _bits(g) == _bits(np.asarray(want)), devices
        buf.close()
        r.close()


# ---- every entry point against numpy -------------------------------------------------------------------------------
def _check_denoise(buf, st, d):
    c, v = dr.denoise(st[0], st[1], st[3], st[4], st[5], st[6], d, return_variance=True)
    got = buf.denoise(d)
    _close(got, c)
    _close(buf.denoised_variance(d), v)
    img = buf.denoised_image(d)
    want = _bytes(got)
    assert (np.abs(img.astype(int) - want.astype(int)) <= 1).all()
    assert np.array_equal(img[~np.isfinite(got)], want[~np.isfinite(got)])  # NaN 0, +inf 255, -inf 0, exactly
    return got


def _check_error(buf, st, d):
    _, _, E = href.error(*st, d)
    _close(buf.denoised_error(d), E)


def _check_select(buf, st, d):
    rgb, level, mse = buf.denoise_select(d)
    assert level.max() <= d.iterations
    wrgb, wlevel, wM = sref.select(*st, d)
    near = sref.ties(*st, d)
    assert np.array_equal(level[~near], wlevel[~near]), np.argwhere((level != wlevel) & ~near)[:8]
    same = level == wlevel
    _close(np.where(same, mse, 0.0), np.where(same, wM, 0.0))
    _close(np.where(same[..., None], rgb, 0.0), np.where(same[..., None], wrgb, 0.0))
    img = buf.selected_image(d)
    for k in range(d.iterations + 1):  # every pixel is its level's denoise output, bit for bit
        at = level == k
        if at.any():
            assert _bits(rgb[at]) == _bits(buf.denoise(_with(d, iterations=k))[at]), k
            assert np.array_equal(img[at], buf.denoised_image(_with(d, iterations=k))[at]), k


def _check_cross(buf, st, d):
    """tests/test_gpu_denoise_cross.py's _check on states with non-finite values: the blend over the device's k* and,
    where no neighbour's k* differs from numpy's, over numpy's; level 0 bit for bit where the whole 5x5 neighbourhood
    chose it, and each level k where both this call and one with k passes chose k there; and the convex bound where the
    colour and every blended level are finite."""
    rgb, level, mse = buf.denoise_cross(d)
    assert level.max() <= d.iterations
    lv = xref.levels(*st, d)
    wlevel = xref.argmin([M for _, _, M in lv])
    near = xref.ties(lv)
    assert np.array_equal(level[~near], wlevel[~near]), np.argwhere((level != wlevel) & ~near)[:8]
    wrgb, wM = xref.blend(lv, level)
    _close(rgb, wrgb)
    _close(mse, wM)
    same = ~xref.dilate(level != wlevel)
    wrgb2, wM2 = xref.blend(lv, wlevel)
    _close(np.where(same[..., None], rgb, 0.0), np.where(same[..., None], wrgb2, 0.0))
    _close(np.where(same, mse, 0.0), np.where(same, wM2, 0.0))
    sums, counts = st[0], st[3]
    at = ~xref.dilate(level != 0)
    with np.errstate(invalid="ignore"):
        assert _bits(rgb[at]) == _bits((sums / counts.astype(np.float64)[..., None])[at])
    for k in range(1, d.iterations):
        rgb_k, level_k, _ = buf.denoise_cross(_with(d, iterations=k))
        at = ~xref.dilate(level != k) & ~xref.dilate(level_k != k)
        assert _bits(rgb[at]) == _bits(rgb_k[at]), k
    used = np.stack([xref.beta(level, k)[0] > 0.0 for k in range(d.iterations + 1)])
    O = np.stack([o for o, _, _ in lv])
    ok = np.isfinite(rgb) & np.where(used[..., None], np.isfinite(O), True).all(0)
    lo = np.where(used[..., None], O, np.inf).min(0)
    hi = np.where(used[..., None], O, -np.inf).max(0)
    tol = 1e-11 * np.max(np.abs(O[np.isfinite(O)]), initial=0.0)
    assert (rgb[ok] >= lo[ok] - tol).all() and (rgb[ok] <= hi[ok] + tol).all()


def _params(i):
    return [PARAMS[i % len(PARAMS)], PARAMS[(i + 4) % len(PARAMS)]]


CASES = [pytest.param(name, w, h, id=f"{name}-{w}x{h}") for name in STATES for w, h in SHAPES]


@pytest.mark.parametrize("name,w,h", CASES)
def test_entry_points_match_numpy(gpu_ok, name, w, h):
    """denoise, denoised_variance and denoised_image; denoised_error; denoise_select; denoise_cross -- on one state and
    shape, with two of PARAMS (every parameter set is met on every state across the shapes)."""
    st = _state(name, w, h)
    r, _, buf = _setup(st, w, h)
    rb = _readback(buf)
    i = list(STATES).index(name) * len(SHAPES) + SHAPES.index((w, h))
    for d in _params(i):
        _check_denoise(buf, rb, d)
        _check_error(buf, rb, d)
        _check_select(buf, rb, d)
        _check_cross(buf, rb, d)
    buf.close()
    r.close()


def _guided(r, buf, crit):
    """One guided call; the pixels that took an entry."""
    before = buf.counts().reshape(-1)
    r._next_sample = 50
    active = r.sample(1, buf, want_stats=False, adaptive=crit)
    took = buf.counts().reshape(-1) != before
    assert active == int(took.sum())
    return took


@pytest.mark.parametrize("name", list(STATES))
@pytest.mark.parametrize("w,h", [(1, 7), (3, 5), (33, 7), (97, 61)], ids=["1x7", "3x5", "33x7", "97x61"])
def test_guided_decisions_match_numpy(gpu_ok, name, w, h):
    """One guided call on v' and one on E add an entry exactly where guided_ref.active / halves_ref.active say, outside
    borderline -- each on a fresh import of the state."""
    st = _state(name, w, h)
    r, b, buf = _setup(st, w, h)
    rb = _readback(buf)
    sums, m2, half, counts, nrm, z, albedo = rb
    for k, d in enumerate((api.Denoise(iterations=3), api.Denoise(iterations=5, albedo_eps=1e-12, sigma_normal=1))):
        crit = api.Adaptive(0.05, 1e-3, 3, guide=d)
        c, v = gref.filtered(sums, m2, counts, nrm, z, albedo, d)
        want, near = gref.active(counts, c, v, crit).reshape(-1), gref.borderline(counts, c, v, crit).reshape(-1)
        took = _guided(r, b.import_into(buf), crit)
        assert not np.any((took != want) & ~near), np.flatnonzero((took != want) & ~near)[:8]
        crit = api.Adaptive(0.05, 1e-3, 3, guide=d, estimate="halves")
        c, _, E = href.error(*rb, d)
        want, near = href.active(counts, c, E, crit).reshape(-1), href.borderline(counts, c, E, crit).reshape(-1)
        took = _guided(r, b.import_into(buf), crit)
        assert not np.any((took != want) & ~near), np.flatnonzero((took != want) & ~near)[:8]
    buf.close()
    r.close()


# ---- properties that need no restatement ---------------------------------------------------------------------------
def _outputs(buf, d):
    """Every filter output of one parameter set: colour, v', bytes, E, select's (rgb, level, mse), cross's."""
    out = {"denoise": buf.denoise(d), "variance": buf.denoised_variance(d), "image": buf.denoised_image(d), "error": buf.denoised_error(d)}
    out.update(zip(("select rgb", "select level", "select mse"), buf.denoise_select(d)))
    out.update(zip(("cross rgb", "cross level", "cross mse"), buf.denoise_cross(d)))
    return out


SCALE_STATES = ["baseline", "nonfinite", "misses", "black", "negative", "depth"]


@pytest.mark.parametrize("name", SCALE_STATES)
@pytest.mark.parametrize("s", [20, -20])
def test_scale_covariance(gpu_ok, name, s):
    """S and HALF times 2^s, M2 times 4^s (exact in binary): colours scale by 2^s, v', E, select's M and cross's M^ by
    4^s, and k* stays outside numpy's ties.  eps_l (1e-10) is the one term that does not scale, so the state is first
    lifted to 2^40 (its prefiltered sqrt(g) is then ~2^20 even at s = -20), and numpy's own covariance on it -- where only
    eps_l breaks it -- is asserted within the tolerance before the kernels are.  The zero-variance states are left out:
    there lden is eps_l alone and no scale covariance holds."""
    w, h = 33, 7
    base = _state(name, w, h)
    for k in ("sums", "half"):
        base[k] = base[k] * 2.0 ** 40
    base["m2"] = base["m2"] * 4.0 ** 40
    scaled = dict(base, sums=base["sums"] * 2.0 ** s, half=base["half"] * 2.0 ** s, m2=base["m2"] * 4.0 ** s)
    d = api.Denoise(iterations=5)
    got = []
    for st in (base, scaled):
        r, _, buf = _setup(st, w, h)
        got.append((_outputs(buf, d), _readback(buf)))
        buf.close()
        r.close()
    (o0, rb0), (o1, rb1) = got
    c0, v0 = dr.denoise(*(rb0[i] for i in (0, 1, 3, 4, 5, 6)), d, return_variance=True)
    c1, v1 = dr.denoise(*(rb1[i] for i in (0, 1, 3, 4, 5, 6)), d, return_variance=True)
    _close(c1, c0 * 2.0 ** s)  # eps_l's effect on these states stays below the tolerance
    _close(v1, v0 * 4.0 ** s)
    _close(href.error(*rb1, d)[2], href.error(*rb0, d)[2] * 4.0 ** s)
    for k in ("denoise", "select rgb", "cross rgb"):
        _close(o1[k], o0[k] * 2.0 ** s)
    for k in ("variance", "error"):
        _close(o1[k], o0[k] * 4.0 ** s)
    near = sref.ties(*rb0, d)
    assert np.array_equal(o1["select level"][~near], o0["select level"][~near])
    same = o1["select level"] == o0["select level"]
    _close(np.where(same, o1["select mse"], 0.0), np.where(same, o0["select mse"] * 4.0 ** s, 0.0))
    near = xref.ties(xref.levels(*rb0, d))
    assert np.array_equal(o1["cross level"][~near], o0["cross level"][~near])
    same = ~xref.dilate(o1["cross level"] != o0["cross level"])
    _close(np.where(same, o1["cross mse"], 0.0), np.where(same, o0["cross mse"] * 4.0 ** s, 0.0))


@pytest.mark.parametrize("w,h,y,x", [(7, 1, 0, 3), (3, 5, 0, 0), (33, 7, 3, 16), (97, 61, 60, 96)],
                         ids=["7x1", "3x5-corner", "33x7", "97x61-corner"])
def test_a_non_finite_pixel_is_local(gpu_ok, w, h, y, x):
    """Pixel p's sums switched among NaN, +inf and -inf, its M2 and HALF held finite: every other pixel's outputs from
    all five entry points keep their bits.  From the rules: p's v (from M2 and n) is the same finite value, so every
    prefiltered g is; p's i, u and i_A are non-finite in all three cases, so as a neighbour's tap p has w = 0 (its i) in
    the filter, the estimate and chain A, and p keeps its own; i_B (from HALF) is finite, so chain B weighs p as before,
    and p's payload X_A, non-finite, is skipped from every payload sum; p's m_k (select and cross) is NaN or inf in all
    three cases and select_smooth skips it, so every M_k is unchanged -- p's own k* included, which is why the cross
    blend of p's neighbours keeps its bits.  The guided decisions follow from c', v' and E.  p's own colour differs
    (it keeps its non-finite i), and so may its bytes."""
    st = _state("baseline", w, h)
    p = y * w + x
    d_all = [api.Denoise(iterations=3), api.Denoise(iterations=12, albedo_eps=1e-12)]
    others = np.arange(w * h) != p
    ref = None
    r, b, buf = _setup(st, w, h)
    for bad in (np.nan, np.inf, -np.inf):
        st["sums"][y, x] = bad
        b.program(st).import_into(buf)
        outs = [_outputs(buf, d) for d in d_all]
        marks = []
        for d in d_all:
            for est in ("filter", "halves"):
                marks.append(_guided(r, b.import_into(buf), api.Adaptive(0.05, 1e-3, 3, guide=d, estimate=est)))
        got = ([{k: v.reshape(w * h, -1)[others] for k, v in o.items()} for o in outs], [m[others] for m in marks])
        if ref is None:
            ref = got
            continue
        for o, o_ref in zip(got[0], ref[0]):
            for k in o:
                assert _bits(o[k]) == _bits(o_ref[k]), (bad, k)
        for m, m_ref in zip(got[1], ref[1]):
            assert np.array_equal(m, m_ref), bad
    buf.close()
    r.close()


@pytest.mark.parametrize("name,w,h", [("nonfinite", 33, 7), ("black", 97, 61), ("misses", 31, 9)])
def test_scratch_reuse(gpu_ok, name, w, h):
    """On one buffer: cross(5), select(2), error(12), a host entry, denoise(3), cross(1), denoised_variance(5) -- every
    result the same bits as the same call on a freshly imported buffer of the same state (and the same host entry), so
    no entry point reads what another left in the shared scratch planes."""
    st = _state(name, w, h)
    entry = np.random.default_rng(5).uniform(-0.5, 2.0, (w * h, 3))
    D = api.Denoise
    calls = [("cross", D(iterations=5), False), ("select", D(iterations=2), False), ("error", D(iterations=12), False),
             ("denoise", D(iterations=3), True), ("cross", D(iterations=1), True), ("variance", D(iterations=5), True)]

    def run(buf, what, d):
        f = {"cross": buf.denoise_cross, "select": buf.denoise_select, "error": buf.denoised_error, "denoise": buf.denoise,
             "variance": buf.denoised_variance}[what]
        out = f(d)
        return [_bits(a) for a in (out if isinstance(out, tuple) else (out,))]

    r, b, buf = _setup(st, w, h)
    added = False
    for what, d, after in calls:
        if after and not added:
            buf.add_samples(entry)
            added = True
        got = run(buf, what, d)
        fresh = b.import_into(r.device_buffer(halves=True))
        if after:
            fresh.add_samples(entry)
        assert got == run(fresh, what, d), (what, d.iterations)
        fresh.close()
    buf.close()
    r.close()


@pytest.mark.parametrize("name,w,h", [("nonfinite", 97, 61), ("misses", 33, 7)])
def test_replicas_give_the_same_bits(gpu_ok, name, w, h):
    """One state imported into [0] and into [0, 0, 0]: the same bits from all five entry points, guided marks included."""
    st = _state(name, w, h)
    got = []
    for devices in ([0], [0, 0, 0]):
        r, b, buf = _setup(st, w, h, devices)
        outs = [_outputs(buf, d) for d in (api.Denoise(iterations=4), api.Denoise(iterations=12, sigma_luminance=0.0))]
        for est in ("filter", "halves"):
            _guided(r, b.import_into(buf), api.Adaptive(0.05, 1e-3, 3, guide=api.Denoise(iterations=4), estimate=est))
            outs.append(buf.pixel_stats() + (buf.half_sums(),))
        got.append(outs)
        buf.close()
        r.close()
    for x, y in zip(*got):
        if isinstance(x, dict):
            assert all(_bits(x[k]) == _bits(y[k]) for k in x)
        else:
            assert all(_bits(a) == _bits(c) for a, c in zip(x, y))


@pytest.mark.parametrize("eps", [1e-12, 1e-3, 1.0])
def test_black_albedo_gives_finite_colours(gpu_ok, eps):
    """albedo_eps >= 1e-12, entries within +-1e6 and every S, M2 and HALF finite: every entry point's colour (and v', E,
    M) is finite everywhere, the black-albedo pixels with a raw mean of 0 and of 1e6 included; albedo_eps 0, which
    divided such a pixel by 0 and made it NaN, is refused before any device work."""
    w, h = 33, 7
    st = state_black(w, h, np.random.default_rng(11))
    n = st["counts"].astype(np.float64)[..., None]
    big = np.random.default_rng(12).random((h, w)) < 0.3
    st["sums"][big] = 1e6 * n[big]
    st["sums"][~big] = np.clip(st["sums"][~big], -1e6, 1e6)
    st["half"] = np.clip(st["half"], -1e6 * n, 1e6 * n)
    st["sums"][0, 0], st["half"][0, 0], st["sa"][0, 0] = 0.0, 0.0, 0.0  # raw mean 0 on a black albedo
    st["sums"][h - 1, w - 1], st["sa"][h - 1, w - 1] = -1e6 * n[h - 1, w - 1], 0.0
    r, _, buf = _setup(st, w, h)
    assert (buf.features()[2] == 0.0).any()
    for it in (1, 5, 12):
        d = api.Denoise(iterations=it, albedo_eps=eps)
        o = _outputs(buf, d)
        for k in ("denoise", "variance", "error", "select rgb", "select mse", "cross rgb", "cross mse"):
            assert np.isfinite(o[k]).all(), (k, it)
    for bad in (0.0, -0.0):
        with pytest.raises(capi.RptbError, match="albedo_eps"):
            buf.denoise(api.Denoise(albedo_eps=bad))
        with pytest.raises(capi.RptbError, match="albedo_eps"):
            r.sample(1, buf, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 3, guide=api.Denoise(albedo_eps=bad)))
    buf.close()
    r.close()
