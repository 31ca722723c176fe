"""numpy restatement of the guided adaptive criterion (guided_active / guided_slot in rpt_b200/csrc/guided.h) on top of
tests/denoise_ref.py -- test infrastructure.  The same float64 operations in the same order as the device and the host
emulation; the filter's exp may differ from numpy's in the last bit, so a decision may differ where the statistic lies
within rounding of its threshold (`borderline`).

Planes are row-major: c' (..., 3), v' and counts (...).  `crit` is an api.Adaptive; `d` an api.Denoise."""
import numpy as np

from tests import denoise_ref


def filtered(sums, m2, counts, nrm, z, albedo, d):
    """The filter over a buffer state: (c', v') of its last pass, (H, W, 3) and (H, W)."""
    return denoise_ref.denoise(sums, m2, counts, nrm, z, albedo, d, return_variance=True)


def _t2(c, crit):
    """t * t for the remodulated colour c' (..., 3): m' = ((c'_0 + c'_1) + c'_2) / 3, t = rel_tol * m' + abs_tol."""
    with np.errstate(invalid="ignore", over="ignore"):
        m = ((c[..., 0] + c[..., 1]) + c[..., 2]) / 3.0
        t = crit.rel_tol * m + crit.abs_tol
        return t * t


def active(counts, c, v, crit):
    """The whole-image decision: True where a pixel with counts n, denoised colour c' and filtered variance v' takes the
    next entry."""
    with np.errstate(invalid="ignore"):
        converged = np.asarray(v) <= _t2(np.asarray(c), crit)
    return (np.asarray(counts) < crit.min_entries) | ~converged


def borderline(counts, c, v, crit, rel=1e-9):
    """Pixels past min_entries whose v' lies within `rel` (relative) of t * t: where a last-bit difference of exp in the
    filter may flip the decision."""
    t2 = _t2(np.asarray(c), crit)
    with np.errstate(invalid="ignore"):
        near = np.isfinite(t2) & (np.abs(np.asarray(v) - t2) <= rel * np.abs(t2))
    return (np.asarray(counts) >= crit.min_entries) & near


def slot_pixels(width, height, index, count):
    """The row-major pixel of every compact slot of part (index, count) -- tile index + k * count, element j -- or -1
    past a ragged edge (tile.h's tile_pixel)."""
    tiles_x = (width + 15) // 16
    t = np.arange(index, tiles_x * ((height + 7) // 8), count, dtype=np.int64)
    j = np.arange(128, dtype=np.int64)
    warp, lane = j >> 5, j & 31
    x = (t % tiles_x)[:, None] * 16 + (warp & 1) * 8 + (lane & 7)
    y = (t // tiles_x)[:, None] * 8 + (warp >> 1) * 4 + (lane >> 3)
    return np.where((x < width) & (y < height), y * width + x, -1).reshape(-1)


def part_decision(counts, c, v, crit, index, count):
    """The per-slot decision of part (index, count) over row-major planes of shape (H, W[, 3]): (mask (tiles * 128,) bool,
    flags (tiles * 4,) bool -- one per 8x4 warp block with an active slot)."""
    H, W = np.asarray(counts).shape
    p = slot_pixels(W, H, index, count)
    on = active(counts, c, v, crit).reshape(-1)
    mask = np.where(p >= 0, on[np.maximum(p, 0)], False)
    return mask, mask.reshape(-1, 4, 32).any(-1).reshape(-1)
