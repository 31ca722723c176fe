"""numpy restatement of rpt_b200/csrc/select.h -- the per-pixel choice of the filter's pass count from a half-buffer
estimate of each level's error -- on top of tests/halves_ref.py -- test infrastructure.  The same float64 operations in
the same order as the device and the host emulation; the filter's exp may differ from numpy's in the last bit.

Planes are row-major: sums / half / normal / albedo (H, W, 3), m2 / depth / counts (H, W).  `d` is an api.Denoise."""
import numpy as np

from tests import denoise_ref as dr
from tests import halves_ref as href


def m_plane(ik, Uk, i0, u0, albedo, eps_a):
    """m_k per pixel: (((t_0 A_0) A_0 + (t_1 A_1) A_1) + (t_2 A_2) A_2) / 3, t = (D D + 2 (U_k u_0)) - u_0 u_0, D = i_k - i_0."""
    with np.errstate(invalid="ignore", over="ignore"):
        D = ik - i0
        t = (D * D + 2.0 * (Uk * u0)) - u0 * u0
        A = albedo + eps_a
        ta = (t * A) * A
        return ((ta[..., 0] + ta[..., 1]) + ta[..., 2]) / 3.0


def smooth(m):
    """M: m over the 5x5 (1/16, 1/4, 3/8, 1/4, 1/16)^2 taps in the image with a finite m, divided by their weight."""
    H, W = m.shape
    ms, mw = np.zeros((H, W)), np.zeros((H, W))
    for dv in range(-2, 3):
        for du in range(-2, 3):
            mq = dr._shift(m, du, dv, 0.0)
            ok = dr._inside(H, W, du, dv) & dr.finite(mq)
            k = dr.K5[du + 2] * dr.K5[dv + 2]
            ms = ms + np.where(ok, k * np.where(ok, mq, 0.0), 0.0)
            mw = mw + np.where(ok, k, 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return ms / mw


def levels(sums, m2, half, counts, nrm, z, albedo, d):
    """Every level's output and estimate: a list over k = 0 .. d.iterations of (c_k (H, W, 3), m_k (H, W), M_k (H, W)),
    c_0 = S / n and c_k = i_k (a + eps_a)."""
    eps = d.albedo_eps
    i0, v0 = dr.demodulate(sums, m2, counts, albedo, eps)
    u0 = href.u_plane(sums, half, counts, albedo, eps)
    with np.errstate(invalid="ignore", divide="ignore"):
        c0 = sums / np.asarray(counts, np.float64)[..., None]
    m = m_plane(i0, u0, i0, u0, albedo, eps)
    out = [(c0, m, smooth(m))]
    i, v, u = i0, v0, u0
    for k in range(d.iterations):
        i, v, u = href.atrous_pass(i, v, u, nrm, z, albedo, 1 << k, d)
        m = m_plane(i, u, i0, u0, albedo, eps)
        with np.errstate(invalid="ignore", over="ignore"):
            out.append((i * (albedo + eps), m, smooth(m)))
    return out


def select(sums, m2, half, counts, nrm, z, albedo, d):
    """(rgb (H, W, 3), level (H, W) uint8, M at the chosen level (H, W)); d.iterations >= 1."""
    assert d.iterations >= 1
    lv = levels(sums, m2, half, counts, nrm, z, albedo, d)
    rgb, _, best = (np.array(a) for a in lv[0])
    level = np.zeros(best.shape, np.uint8)
    for k, (c, _, M) in enumerate(lv[1:], 1):
        win = M < best
        rgb = np.where(win[..., None], c, rgb)
        best = np.where(win, M, best)
        level = np.where(win, np.uint8(k), level)
    return rgb, level, best


def ties(sums, m2, half, counts, nrm, z, albedo, d, rel=1e-9):
    """Pixels where some level's M lies within `rel` (relative) of the chosen level's, or of the running best it was
    compared with: where exp's last bit may change the choice."""
    lv = levels(sums, m2, half, counts, nrm, z, albedo, d)
    Ms = np.stack([M for _, _, M in lv])
    best = np.fmin.accumulate(np.where(np.isnan(Ms), np.inf, Ms), axis=0)
    near = np.zeros(Ms.shape[1:], bool)
    with np.errstate(invalid="ignore"):
        for k in range(1, Ms.shape[0]):
            near |= np.abs(Ms[k] - best[k - 1]) <= rel * np.maximum(np.abs(best[k - 1]), np.abs(Ms[k]))
    return near
