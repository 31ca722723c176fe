"""The device Buffer's kernels at the image sizes it is used at (800x600, 1920x1080, 3840x2160) and at the sizes where a
kernel's code changes path: the variance reduction's chunk boundary (4096 px) and its second pass over the block
partials (more than 256 partials, 1,048,576 px); the least count's grid-stride loop (more than 1024 x 256 threads,
262,144 px); the adaptive select over tens of thousands of warp-block flags; the denoiser's wide passes (step 2^k up
to 2^11); and the multi-thousand-block grids of the resolve, the reprojection, the merge and the part copies.

Every check is against a reference that does not share the kernel's code:
  1. variance: bit for bit against a numpy restatement of the documented fixed order, against math.fsum within a
     bound derived from that order's depth, NaN from one single-entry pixel anywhere, the same bits on every read;
  2. the least count of a reprojected buffer (image "no samples", variance NaN, denoise refusing) against numpy min;
  3. adaptive selection at 1080p and 2160p against the numpy criterion, pixel for pixel, on one and three parts;
  4. image bytes at 1080p with mixed counts against test_gpu_adaptive.py's reference Buffer, edge rows included;
  5. denoise against tests/denoise_ref.py at 1080p (rendered state) and on a 4200x9 strip with 12 passes;
  6. reprojection and history merge at 1080p against tests/reproject_ref.py / reproject_merge_ref.py, whole and as
     gathered shards;
  7. parts [0], [0, 0, 0] and [0] * 8 at 1080p giving the same bits, and a host round trip of a 1080p block.

A per-pixel state at any size is programmed without rendering it: a world-1 shard block is exported
(rptb_buffer_export_shard), its planes are edited on the host through distributed.shard_block_layout, and it is imported
into a whole buffer (rptb_buffer_import_shards).  The header keeps what the import checks (magic, size, shard count,
feature choice); only its entry-call count and its "reprojected" flag are set.  test_programmed_state_is_what_the_buffer_reads
checks this route against pixel_stats() and features().  Each test prints how long its checks took; on one H100 80GB
HBM3 the whole file ran in about 190 s, 82 s of it the numpy denoiser at 1080p."""
import contextlib
import ctypes as C
import math
import time

import numpy as np
import pytest
import torch

from rpt_b200 import _capi as capi
from rpt_b200 import api, distributed, scenes
from rpt_b200.distributed import ShardBuffer
from tests import denoise_ref
from tests import reproject_merge_ref as mref
from tests import reproject_ref
from tests import util
from tests.test_gpu_adaptive import _reference_buffer
from tests.test_reproject import orbit

pytestmark = pytest.mark.gpu

F32, F64 = capi.PRECISION_F32, capi.PRECISION_F64
EPS = float(np.finfo(np.float64).eps)
HEADER_ENTRIES, HEADER_FLAGS = 24, 28  # byte offsets of ShardHeader::entries / ::flags (rpt_b200/csrc/api.cu)
REPROJECTED = 1


@pytest.fixture(autouse=True)
def _repeated_devices(monkeypatch):
    monkeypatch.setenv(util.REPEATED_DEVICES, "1")


@contextlib.contextmanager
def _timed(what):
    t0 = time.perf_counter()
    yield
    print(f"{what}: {time.perf_counter() - t0:.2f} s")


def _renderer(w, h, prec=F32, devices=(0,), mb=1, seed=3, cam=None):
    cfg = scenes.sphere_scene()
    return (api.Renderer(cfg.scene, cam or cfg.camera).width(w).height(h).max_bounces(mb).seed(seed).precision(prec)
            .device(list(devices)))


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


class Block:
    """A genuine world-1 shard block of w x h, editable per pixel on the host and imported into whole buffers.  With
    features, the shard first takes `feature_rays` rays from the renderer (whose size must be w x h)."""

    def __init__(self, r, w, h, with_features=False, feature_rays=1):
        self.w, self.h, self.with_features = w, h, with_features
        self.lay = distributed.shard_block_layout(w, h, 1, with_features)
        self.slot = distributed.gather_permutation(w, h, 1)  # pixel p (row-major) -> its slot in the block
        s = ShardBuffer(r.device_scene(), w, h, rank=0, world=1)
        if with_features:
            r.sample_features(feature_rays, s)
        self.feature_rays = s.feature_rays
        dev = torch.empty(s.block_bytes(with_features), dtype=torch.uint8, device="cuda:0")
        assert dev.numel() == self.lay["bytes"]
        s.export(dev, with_features)
        torch.cuda.synchronize()
        s.close()
        self.host = dev.cpu().numpy().copy()
        self.dev = dev

    def plane(self, name, dtype, values=1):
        lay, slots = self.lay, self.lay["slots"]
        a = self.host[lay[name]:lay[name] + slots * values * np.dtype(dtype).itemsize].view(dtype)
        return a.reshape(slots, values) if values > 1 else a

    def features(self):
        """The feature sums' planes (normal (slots, 3), albedo (slots, 3), hits, depth), as views."""
        f = self.host[self.lay["features"]:self.lay["counts"]].view(np.float64)
        n = self.lay["slots"]
        return f[:3 * n].reshape(n, 3), f[3 * n:6 * n].reshape(n, 3), f[6 * n:7 * n], f[7 * n:8 * n]

    def program(self, sums=None, m2=None, counts=None, entries=None, flags=None):
        """Row-major per-pixel state into the block's slots; entries / flags into the header."""
        if sums is not None:
            self.plane("sums", np.float64, 3)[self.slot] = sums
        if m2 is not None:
            self.plane("m2", np.float64)[self.slot] = m2
        if counts is not None:
            self.plane("counts", np.uint32)[self.slot] = counts
        if entries is not None:
            self.host[HEADER_ENTRIES:HEADER_ENTRIES + 4].view(np.uint32)[0] = entries
        if flags is not None:
            self.host[HEADER_FLAGS:HEADER_FLAGS + 4].view(np.uint32)[0] = flags
        return self

    def upload(self):
        self.dev.copy_(torch.from_numpy(self.host))
        torch.cuda.synchronize()
        return self

    def poke(self, p, sums, m2, count):
        """One pixel's state, on the host and the device copy (a few bytes each)."""
        e = int(self.slot[p])
        for name, dtype, values, v in (("sums", np.float64, 3, sums), ("m2", np.float64, 1, m2), ("counts", np.uint32, 1, count)):
            off = self.lay[name] + e * values * np.dtype(dtype).itemsize
            raw = np.asarray(v, dtype).reshape(values).view(np.uint8)
            self.host[off:off + raw.size] = raw
            self.dev[off:off + raw.size].copy_(torch.from_numpy(raw.copy()))
        torch.cuda.synchronize()

    def import_into(self, buf):
        capi.check(capi.lib().rptb_buffer_import_shards(buf.handle, C.c_void_p(self.dev.data_ptr()), 1, 1 if self.with_features else 0),
                   "rptb_buffer_import_shards")
        buf.feature_rays = self.feature_rays if self.with_features else 0
        buf.entries = int(self.host[HEADER_ENTRIES:HEADER_ENTRIES + 4].view(np.uint32)[0])
        return buf


def _sizes(ids):
    return [pytest.param(w, h, id=f"{w}x{h}") for w, h in ids]


# ---- the route itself ----------------------------------------------------------------------------------------------
def test_programmed_state_is_what_the_buffer_reads(gpu_ok):
    """Random colour and feature planes, programmed into a 513x512 block, read back through pixel_stats() bit for bit
    and through features() as tests/denoise_ref.py resolves them, on one part and on three."""
    w, h = 513, 512
    npix = w * h
    rng = np.random.default_rng(1)
    with _timed("programmed route 513x512"):
        r = _renderer(w, h)
        b = Block(r, w, h, with_features=True, feature_rays=4)
        sums, m2, counts = rng.uniform(0, 4, (npix, 3)), rng.uniform(0, 2, npix), rng.integers(2, 9, npix).astype(np.uint32)
        b.program(sums, m2, counts, entries=8)
        rays = float(b.feature_rays)
        hits = rng.integers(0, b.feature_rays + 1, npix).astype(np.float64)
        sn, sa, sz = rng.normal(size=(npix, 3)) * hits[:, None], rng.uniform(0, 1, (npix, 3)) * hits[:, None], rng.uniform(1, 9, npix) * hits
        fn, fa, fh, fz = b.features()
        fn[b.slot], fa[b.slot], fh[b.slot], fz[b.slot] = sn, sa, hits, sz
        b.upload()
        wn, wz, wa, wf = denoise_ref.features_resolve(hits, sn, sz, sa, rays)
        for devices in ([0], [0, 0, 0]):
            rd = _renderer(w, h, devices=devices)
            buf = b.import_into(api.DeviceBuffer(rd.device_scene(), w, h))
            gs, gm, gc = buf.pixel_stats()
            assert _bits(gs) == _bits(sums) and _bits(gm) == _bits(m2) and _bits(gc) == _bits(counts), devices
            gn, gz, ga, gf = buf.features()
            for g, want in ((gn, wn), (gz, wz), (ga, wa), (gf, wf)):
                assert _bits(g.reshape(-1)) == _bits(np.asarray(want).reshape(-1)), devices
            buf.close()
            rd.close()
        r.close()


# ---- 1. variance ---------------------------------------------------------------------------------------------------
CHUNK, THREADS = 4096, 256  # buffer_variance_partial_kernel: pixels per block partial, threads per block


def _tree(a):
    """block_sum_fixed over the last axis (256): sh[t] += sh[t + s] for s = 128, 64, ..., 1."""
    s = a.shape[-1] // 2
    while s:
        a = a[..., :s] + a[..., s:2 * s]
        s //= 2
    return a[..., 0]


def _variance_fixed_order(m2, counts):
    """The documented order: block b sums pixels [4096 b, 4096 (b + 1)), thread t its pixels t, t + 256, ... in order,
    then the fixed tree; one block then sums the partials the same way; the total is divided by the pixel count."""
    npix = m2.size
    with np.errstate(divide="ignore", invalid="ignore"):
        t = m2 / (counts.astype(np.float64) - 1.0)
    nb = -(-npix // CHUNK)
    x = np.zeros(nb * CHUNK)
    x[:npix] = t  # past the end nothing is added; adding +0.0 to a sum of non-negative terms changes no bit
    x = x.reshape(nb, CHUNK // THREADS, THREADS)
    v = np.zeros((nb, THREADS))
    for k in range(CHUNK // THREADS):
        v = v + x[:, k, :]
    partial = _tree(v)
    nf = -(-nb // THREADS)
    y = np.zeros(nf * THREADS)
    y[:nb] = partial
    u = np.zeros(THREADS)
    for k in range(nf):
        u = u + y[k * THREADS:(k + 1) * THREADS]
    return _tree(u) / float(npix), t, nb


VARIANCE_SIZES = [(64, 64), (4095, 1), (4096, 1), (4097, 1), (512, 512), (513, 512), (1024, 1024), (1024, 1025), (800, 600),
                  (1920, 1080), (3840, 2160)]


@pytest.mark.parametrize("w,h", _sizes(VARIANCE_SIZES))
def test_variance_at_size(gpu_ok, w, h):
    """(a) bit for bit against the fixed order restated in numpy.  (b) Against math.fsum of the same terms
    m2 / (n - 1): every term is >= 0, and along the fixed order each term meets at most 16 (thread) + 8 (tree) +
    ceil(partials / 256) (final thread) + 8 (tree) additions and one division, d roundings in all; so the relative
    error is at most gamma_d = d u / (1 - d u) <= d eps (u = eps / 2).  The test allows d eps.  (c) One pixel with one
    entry (M2 0: the term is 0/0) at 0, 4095, 4096, 1,048,575, 1,048,576 or the last pixel makes the result NaN, and
    removing it restores the bits.  (d) Every read gives the same bits."""
    npix = w * h
    rng = np.random.default_rng(npix)
    m2, counts = rng.uniform(0.0, 3.0, npix), rng.integers(2, 10, npix).astype(np.uint32)
    sums = rng.uniform(0.0, 1.0, (npix, 3))
    r = _renderer(w, h)
    with _timed(f"variance {w}x{h} program"):
        b = Block(r, w, h).program(sums, m2, counts, entries=9).upload()
        buf = b.import_into(r.device_buffer())
    with _timed(f"variance {w}x{h} checks"):
        want, terms, nb = _variance_fixed_order(m2, counts)
        got = buf.variance()
        assert _bits(np.float64(got)) == _bits(np.float64(want)), (got, want, nb)
        exact = math.fsum(terms.tolist()) / npix
        depth = 16 + 8 + -(-nb // THREADS) + 8 + 1
        assert abs(got - exact) <= depth * EPS * exact, (got, exact, depth)
        print(f"variance {w}x{h}: {nb} partials, |error| / fsum {abs(got - exact) / exact:.3g}, bound {depth * EPS:.3g}")
        for _ in range(3):
            assert _bits(np.float64(buf.variance())) == _bits(np.float64(got))
        for p in sorted({q for q in (0, 4095, 4096, 1048575, 1048576, npix - 1) if q < npix}):
            b.poke(p, sums[p], 0.0, 1)
            b.import_into(buf)
            assert math.isnan(buf.variance()), p
            b.poke(p, sums[p], m2[p], counts[p])
            b.import_into(buf)
            assert _bits(np.float64(buf.variance())) == _bits(np.float64(got)), p
    buf.close()
    r.close()


@pytest.mark.parametrize("prec", [F32, F64], ids=["f32", "f64"])
def test_variance_of_rendered_entries_at_1080p(gpu_ok, prec):
    """The same restatement on entries the renderer added (the f32 and f64 accumulate kernels), with one adaptive call
    so the counts differ."""
    w, h = 1920, 1080
    r = _renderer(w, h, prec, mb=1)
    buf = r.device_buffer()
    with _timed(f"rendered variance 1080p {'f32' if prec == F32 else 'f64'}"):
        for _ in range(2):
            r.sample(1, buf, want_stats=False)
        r.sample(1, buf, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 2))
        _, m2, counts = buf.pixel_stats()
        assert counts.min() == 2 and counts.max() == 3
        want, _, _ = _variance_fixed_order(m2, counts)
        assert _bits(np.float64(buf.variance())) == _bits(np.float64(want))
    buf.close()
    r.close()


# ---- 2. the least count of a reprojected buffer --------------------------------------------------------------------
LEAST_SIZES = [(512, 512), (513, 512), (1024, 1024), (1920, 1080), (3840, 2160)]


@pytest.mark.parametrize("w,h", _sizes(LEAST_SIZES))
def test_least_count_of_a_reprojected_buffer(gpu_ok, w, h):
    """A reprojected block (the header's flag) with every count >= 2 reads; one pixel with count 0 at 0, 255, 262,143,
    262,144, 524,288 or the last pixel makes image() and denoise() raise "no samples" and variance() NaN; with count 1
    variance() is NaN, denoise() refuses and image() still reads.  numpy min of the programmed counts is the
    reference for which of these happens."""
    npix = w * h
    rng = np.random.default_rng(npix + 7)
    sums, m2 = rng.uniform(0.0, 4.0, (npix, 3)), rng.uniform(0.0, 2.0, npix)
    counts = rng.integers(2, 9, npix).astype(np.uint32)
    r = _renderer(w, h, mb=0)
    one = api.Denoise(iterations=1)
    with _timed(f"least count {w}x{h} program"):
        b = Block(r, w, h, with_features=True).program(sums, m2, counts, entries=8, flags=REPROJECTED).upload()
        buf = b.import_into(r.device_buffer())
    with _timed(f"least count {w}x{h} checks"):
        assert counts.min() >= 2
        base = buf.image()
        assert np.isfinite(buf.variance()) and np.isfinite(buf.denoise(one)).all()
        for p in sorted({q for q in (0, 255, 262143, 262144, 524288, npix - 1) if q < npix}):
            for n in (0, 1):
                b.poke(p, sums[p] if n else np.zeros(3), 0.0, n)
                b.import_into(buf)
                least = int(np.min(b.plane("counts", np.uint32)[b.slot]))
                assert least == n
                if least == 0:
                    with pytest.raises(capi.RptbError, match="no samples"):
                        buf.image()
                    with pytest.raises(capi.RptbError, match="no samples"):
                        buf.denoise(one)
                else:
                    assert buf.image().shape == (h, w, 3)
                    with pytest.raises(capi.RptbError, match="fewer than 2 entries"):
                        buf.denoise(one)
                assert math.isnan(buf.variance()), (p, n)
            b.poke(p, sums[p], m2[p], counts[p])
            b.import_into(buf)
            assert np.isfinite(buf.variance()) and _bits(buf.image()) == _bits(base), p
    buf.close()
    r.close()


# ---- 3. adaptive selection -----------------------------------------------------------------------------------------
CRIT = api.Adaptive(0.05, 1e-3, 4)


def _adaptive_states(w, h, rng):
    """name -> the active mask (row-major) each programmed state should give."""
    npix = w * h
    slot = distributed.gather_permutation(w, h, 1)
    slots = distributed.shard_block_layout(w, h, 1)["slots"]

    def from_slots(on):
        m = np.zeros(slots, bool)
        m[on] = True
        return m[slot]

    blocks = slots // 32  # 8x4 warp blocks, slot 32 b + lane
    every7 = np.arange(0, blocks, 7)
    return {
        "all": np.ones(npix, bool),
        "none": np.zeros(npix, bool),
        "first tile": from_slots([77]),
        "last tile": from_slots([slots - 128 + 50]),
        "every 7th warp block": from_slots(32 * every7 + every7 % 32),
        "random half": rng.random(npix) < 0.5,
    }


def _adaptive_program(mask, rng):
    """A state the criterion splits by `mask`: inactive pixels hold 5 entries that agree (M2 0); active ones 5 entries
    that do not (M2 100) or, for one in four, fewer than min_entries."""
    npix = mask.size
    sums = rng.uniform(0.2, 1.0, (npix, 3)) * 5.0
    counts = np.full(npix, 5, np.uint32)
    m2 = np.where(mask, 100.0, 0.0)
    few = mask & (rng.random(npix) < 0.25)
    counts[few] = rng.integers(2, 4, int(few.sum()))
    return sums, m2, counts


@pytest.mark.parametrize("prec", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("w,h", _sizes([(1920, 1080), (3840, 2160)]))
def test_adaptive_selection_at_size(gpu_ok, w, h, prec):
    """One adaptive call (Renderer.sample(1, buf, adaptive=...), rptb_sample_into_adaptive) on each programmed state:
    out_active is the numpy criterion's count, the counts grow by the numpy mask pixel for pixel, the inactive pixels'
    sums and M2 keep their bits -- on one part and on three, which give the same bits."""
    rng = np.random.default_rng(w + h + prec)
    mb = 0 if prec == F32 else 1
    r1 = _renderer(w, h, prec, mb=mb)
    b = Block(r1, w, h)
    r3 = _renderer(w, h, prec, devices=[0, 0, 0], mb=mb)
    for name, mask in _adaptive_states(w, h, rng).items():
        sums, m2, counts = _adaptive_program(mask, rng)
        b.program(sums, m2, counts, entries=5).upload()
        want = CRIT.active(counts, sums, m2)
        assert np.array_equal(want, mask), name
        with _timed(f"adaptive {w}x{h} {name}"):
            outs = []
            for r in (r1, r3):
                buf = b.import_into(r.device_buffer())
                r._next_sample = 10
                active = r.sample(1, buf, want_stats=False, adaptive=CRIT)
                s1, m1, c1 = buf.pixel_stats()
                assert active == int(want.sum()), (name, r._device, active)
                assert np.array_equal(c1.astype(np.int64) - counts, want.astype(np.int64)), (name, r._device)
                assert _bits(s1[~want]) == _bits(sums[~want]) and _bits(m1[~want]) == _bits(m2[~want]), (name, r._device)
                outs.append((s1, m1, c1))
                buf.close()
            assert all(_bits(x) == _bits(y) for x, y in zip(*outs)), name
    r1.close()
    r3.close()


# ---- 4. image bytes with mixed counts ------------------------------------------------------------------------------
@pytest.mark.parametrize("radius", [0, 1, 3])
def test_image_bytes_with_mixed_counts_at_1080p(gpu_ok, radius):
    """Per-pixel counts 1..6 and the sums of that many random entries, against test_gpu_adaptive.py's reference Buffer
    (per-pixel entry lists, get_filtered_color's order): every byte within 1 (the device's pow against numpy's), and
    the bottom row, the top row and the left and right columns each exact in more than 99 % of their bytes."""
    w, h, k = 1920, 1080, 6
    npix = w * h
    rng = np.random.default_rng(40 + radius)
    entries = rng.uniform(0.0, 1.2, (k, npix, 3))
    counts = rng.integers(1, k + 1, npix).astype(np.uint32)
    takes = np.arange(k)[:, None] < counts[None, :]
    sums = np.zeros((npix, 3))
    for e, t in zip(entries, takes):  # the reference's own order of addition
        sums[t] = sums[t] + e[t]
    r = _renderer(w, h)
    b = Block(r, w, h).program(sums, np.zeros(npix), counts, entries=k).upload()
    buf = b.import_into(api.DeviceBuffer(r.device_scene(), w, h, api.Filter.Box(radius)))
    with _timed(f"image 1080p radius {radius}"):
        with np.errstate(all="ignore"):
            want, _ = _reference_buffer(entries, takes, w, h, radius)
        got = buf.image()
        assert (np.abs(got.astype(int) - want.astype(int)) <= 1).all()
        for edge in (got[-1] == want[-1], got[0] == want[0], got[:, 0] == want[:, 0], got[:, -1] == want[:, -1]):
            assert edge.mean() > 0.99
        assert (got == want).mean() > 0.999
    buf.close()
    r.close()


# ---- 5. denoise ----------------------------------------------------------------------------------------------------
def _check_denoise(buf, d, w, h):
    sums, m2, counts = buf.pixel_stats()
    N, z, a, _ = buf.features()
    want = denoise_ref.denoise(sums.reshape(h, w, 3), m2.reshape(h, w), counts.reshape(h, w), N, z, a, d)
    got = buf.denoise(d)
    assert np.isfinite(got).all()
    assert np.max(np.abs(got - want)) <= 1e-12 * np.abs(want).max()
    return want, (sums, m2, counts, N, z, a)


def test_denoise_at_1080p(gpu_ok):
    """A rendered state (three entries, features from sample_features) through 5 passes, against the numpy restatement
    at the tolerance of test_gpu_denoise.py (1e-12 of the largest value)."""
    w, h = 1920, 1080
    r = _renderer(w, h, F64, mb=1)
    buf = r.device_buffer()
    for _ in range(3):
        r.sample(1, buf, want_stats=False)
    r.sample_features(2, buf)
    with _timed("denoise 1080p 5 passes"):
        _check_denoise(buf, api.Denoise(iterations=5), w, h)
    buf.close()
    r.close()


def test_denoise_wide_strip_with_12_passes(gpu_ok):
    """4200x9 (a ragged right tile) with 12 passes, so the steps 1024 and 2048 land taps inside the image.  Every
    pixel sees the same flat surface (normal weight 1, depth weight 1) and noisy colour with a large variance, so the
    wide taps carry weight: the numpy result after 12 passes is far from the one after 10, whose last two passes would
    be all a filter that dropped the taps at |offset| >= 1024 computes."""
    w, h = 4200, 9
    npix = w * h
    rng = np.random.default_rng(9)
    r = _renderer(w, h, mb=0)
    b = Block(r, w, h, with_features=True, feature_rays=4)
    rays = float(b.feature_rays)
    fn, fa, fh, fz = b.features()
    fn[:] = 0.0
    fn[:, 2] = rays
    fa[:] = 0.5 * rays
    fh[:] = rays
    fz[:] = 5.0 * rays
    b.program(rng.uniform(0.0, 4.0, (npix, 3)), np.full(npix, 3.0), np.full(npix, 4, np.uint32), entries=4).upload()
    buf = b.import_into(r.device_buffer())
    d = api.Denoise(iterations=12)
    with _timed("denoise 4200x9 12 passes"):
        want, st = _check_denoise(buf, d, w, h)
        sums, m2, counts, N, z, a = st
        ten = denoise_ref.denoise(sums.reshape(h, w, 3), m2.reshape(h, w), counts.reshape(h, w), N, z, a, api.Denoise(iterations=10))
        assert np.max(np.abs(want - ten)) > 1e-6 * np.abs(want).max()
    buf.close()
    r.close()


# ---- 6. reprojection and history merge -----------------------------------------------------------------------------
CENTER = (0.0, -0.25, 0.0)


def _gather_into(shards, dst, with_features=True):
    blocks = []
    for s in shards:
        out = torch.empty(s.block_bytes(with_features), dtype=torch.uint8, device="cuda:0")
        s.export(out, with_features)
        blocks.append(out)
    g = torch.cat(blocks)
    torch.cuda.synchronize()
    capi.check(capi.lib().rptb_buffer_import_shards(dst.handle, C.c_void_p(g.data_ptr()), len(shards), 1 if with_features else 0),
               "rptb_buffer_import_shards")
    return dst


def test_reprojection_and_merge_at_1080p(gpu_ok):
    """A 1080p source through camera A (3 entries, 4 feature rays) reprojected onto an orbited camera B, plainly and
    merged into 2 fresh entries, against the numpy restatements bit for bit; then as 1, 3 and 8 shards, whose gather
    gives the whole buffer's bits and whose reused / rejected counts add up to the whole call's."""
    w, h = 1920, 1080
    cfg = scenes.sphere_scene()
    scam = api.Camera.look_at(cfg.camera.eye, np.asarray(CENTER), api.vec3(0.0, 1.0, 0.0), cfg.camera.fov)
    dcam = orbit(scam, CENTER, -0.05, lift=0.03)
    r = _renderer(w, h, F32, mb=1, cam=scam)
    ds = r.device_scene()
    src = r.device_buffer()
    for _ in range(3):
        r.sample(1, src, want_stats=False)
    r.sample_features(4, src)
    r.camera = dcam
    prm = api.Reproject()
    gamma = api.HistoryTest().gamma
    ssum, sm2, scnt = src.pixel_stats()
    sN, sz, _, sf = src.features()

    def fresh(buf, entries):
        r.sample_features(4, buf)
        r._next_sample = 100
        for _ in range(entries):
            r.sample(1, buf, want_stats=False)
        return buf

    with _timed("reproject 1080p whole"):
        plain = fresh(api.DeviceBuffer(ds, w, h), 0)
        dN, dz, _, df = plain.features()
        want = reproject_ref.reproject(dcam, dN, dz, df, scam, ssum.reshape(h, w, 3), sm2.reshape(h, w), scnt.reshape(h, w), sN, sz, sf, prm)
        reused = plain.reproject_from(src, prm)
        got = plain.pixel_stats()
        assert _bits(got[2].reshape(h, w)) == _bits(want[2])
        assert _bits(got[0].reshape(h, w, 3)) == _bits(want[0]) and _bits(got[1].reshape(h, w)) == _bits(want[1])
        assert reused == int((want[2] > 0).sum()) and 0 < reused < w * h
    with _timed("merge 1080p whole"):
        merged = fresh(api.DeviceBuffer(ds, w, h), 2)
        fs, fm, fc = merged.pixel_stats()
        mN, mz, _, mf = merged.features()
        wm = mref.reproject_merge(dcam, mN, mz, mf, scam, ssum.reshape(h, w, 3), sm2.reshape(h, w), scnt.reshape(h, w), sN, sz, sf, prm,
                                  gamma, fs.reshape(h, w, 3), fm.reshape(h, w), fc.reshape(h, w))
        tally = merged.merge_history_from(src, prm, api.HistoryTest(gamma))
        got_m = merged.pixel_stats()
        assert _bits(got_m[2].reshape(h, w)) == _bits(wm[2])
        assert _bits(got_m[0].reshape(h, w, 3)) == _bits(wm[0]) and _bits(got_m[1].reshape(h, w)) == _bits(wm[1])
        assert tally == (int((wm[3] == mref.REUSED).sum()), int((wm[3] == mref.REJECTED).sum()))
        assert tally[0] > 0 and sum(tally) == reused
    for n in (1, 3, 8):
        with _timed(f"reproject and merge 1080p as {n} shards"):
            for merge in (False, True):
                shards = [ShardBuffer(ds, w, h, rank=i, world=n) for i in range(n)]
                counts = []
                for s in shards:
                    fresh(s, 2 if merge else 0)
                    counts.append(s.merge_history_from(src, prm, api.HistoryTest(gamma)) if merge else s.reproject_from(src, prm))
                whole = _gather_into(shards, api.DeviceBuffer(ds, w, h))
                g = whole.pixel_stats()
                assert all(_bits(x) == _bits(y) for x, y in zip(g, got_m if merge else got)), (n, merge)
                if merge:
                    assert tuple(map(sum, zip(*counts))) == tally, n
                else:
                    assert sum(counts) == reused, n
                for s in shards:
                    s.close()
                whole.close()
    for x in (src, plain, merged):
        x.close()
    r.close()


# ---- 7. parts ------------------------------------------------------------------------------------------------------
def _calls(r, buf):
    r._next_sample = 0
    for _ in range(2):
        r.sample(1, buf, want_stats=False)
    r.sample_features(2, buf)
    for _ in range(2):
        r.sample(1, buf, want_stats=False, adaptive=api.Adaptive(0.05, 1e-3, 2))


def _reads(buf):
    out = dict(zip(("sums", "m2", "counts"), buf.pixel_stats()))
    out.update(zip(("normal", "depth", "albedo", "hit fraction"), buf.features()))
    out["image"] = buf.image()
    out["variance"] = np.float64(buf.variance())
    out["denoise"] = buf.denoise(api.Denoise())
    return out


def _same(got, want, where):
    for k in want:
        assert _bits(got[k]) == _bits(want[k]), (where, k)


def test_parts_at_1080p(gpu_ok):
    """Two plain entries, features and two adaptive entries on [0], [0, 0, 0] and [0] * 8: the same sums, M2, counts,
    features, image, variance and denoising, bit for bit.  Then the same calls on a world-1 shard, whose 207 MB block
    with features goes to the host and back and is imported: the buffer again, bit for bit."""
    w, h = 1920, 1080
    want = None
    for devices in ([0], [0, 0, 0], [0] * 8):
        with _timed(f"parts 1080p {devices}"):
            r = _renderer(w, h, devices=devices)
            buf = r.device_buffer()
            _calls(r, buf)
            got = _reads(buf)
            if want is None:
                want = got
                assert 0 < got["counts"].min() < got["counts"].max()
            else:
                _same(got, want, devices)
            buf.close()
            r.close()
    with _timed("host round trip of the 1080p block"):
        r = _renderer(w, h)
        s = ShardBuffer(r.device_scene(), w, h, rank=0, world=1)
        _calls(r, s)
        dev = torch.empty(s.block_bytes(True), dtype=torch.uint8, device="cuda:0")
        s.export(dev, True)
        torch.cuda.synchronize()
        assert dev.numel() == distributed.shard_block_layout(w, h, 1, True)["bytes"] > 200e6
        back = torch.from_numpy(dev.cpu().numpy().copy()).to("cuda:0")
        torch.cuda.synchronize()
        buf = r.device_buffer()
        capi.check(capi.lib().rptb_buffer_import_shards(buf.handle, C.c_void_p(back.data_ptr()), 1, 1), "rptb_buffer_import_shards")
        buf.feature_rays = s.feature_rays
        _same(_reads(buf), want, "round trip")
        buf.close()
        s.close()
        r.close()
