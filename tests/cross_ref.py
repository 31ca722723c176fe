"""numpy restatement of rpt_b200/csrc/cross.h -- the cross-filtered denoiser with a smoothed selection map -- on top of
tests/halves_ref.py and tests/select_ref.py -- test infrastructure.  The same float64 operations in the same order as
the device and the host emulation; the filter's exp may differ from numpy's in the last bit.

Planes are row-major: sums / half / normal / albedo (H, W, 3), m2 / depth / counts (H, W).  `d` is an api.Denoise."""
import numpy as np

from tests import denoise_ref as dr
from tests import halves_ref as href
from tests import select_ref as sref


def _counts(counts):
    n = np.asarray(counts, dtype=np.uint64)
    nb = n >> np.uint64(1)
    return n.astype(np.float64), (n - nb).astype(np.float64), nb.astype(np.float64), nb == 0


def demodulate(sums, m2, half, counts, albedo, eps_a):
    """(i_A, v_A, i_B, v_B): i_H = (S_H / n_H) / A, v_H = (v n) / n_H; NaN in all four where n_B = 0."""
    dn, dA, dB, none = _counts(counts)
    with np.errstate(divide="ignore", invalid="ignore"):
        vn = dr.mean_variance(counts, m2) * dn
        vA, vB = vn / dA, vn / dB
        A = albedo + eps_a
        sb = half
        sa = sums - sb
        iA = (sa / dA[..., None]) / A
        iB = (sb / dB[..., None]) / A
    iA, iB = np.where(none[..., None], np.nan, iA), np.where(none[..., None], np.nan, iB)
    return iA, np.where(none, np.nan, vA), iB, np.where(none, np.nan, vB)


def _mean_c(x):
    return ((x[..., 0] + x[..., 1]) + x[..., 2]) / 3.0


def m_plane(XA, XB, iA0, iB0, vA, vB, counts, albedo, eps_a):
    """m_k = 0.5 ((m^A - (D n_B) / n) + (m^B - (D n_A) / n)) + ((D n_A) n_B) / (n n)."""
    dn, dA, dB, _ = _counts(counts)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        A = albedo + eps_a
        da, db, de = A * (XA - iB0), A * (XB - iA0), A * (XA - XB)
        mA = _mean_c(da * da) - vB
        mB = _mean_c(db * db) - vA
        D = _mean_c(de * de)
        return 0.5 * ((mA - (D * dB) / dn) + (mB - (D * dA) / dn)) + ((D * dA) * dB) / (dn * dn)


def output(XA, XB, counts, albedo, eps_a):
    """O_k = ((n_A X_A + n_B X_B) / n) A, k >= 1."""
    dn, dA, dB, _ = _counts(counts)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return ((dA[..., None] * XA + dB[..., None] * XB) / dn[..., None]) * (albedo + eps_a)


def levels(sums, m2, half, counts, nrm, z, albedo, d):
    """Every level: a list over k = 0 .. d.iterations of (O_k (H, W, 3), m_k (H, W), M_k (H, W))."""
    eps = d.albedo_eps
    iA0, vA0, iB0, vB0 = demodulate(sums, m2, half, counts, albedo, eps)
    with np.errstate(invalid="ignore", divide="ignore"):
        O0 = sums / np.asarray(counts, np.float64)[..., None]
    m = m_plane(iA0, iB0, iA0, iB0, vA0, vB0, counts, albedo, eps)
    out = [(O0, m, sref.smooth(m))]
    gA, vA, XB, gB, vB, XA = iA0, vA0, iB0, iB0, vB0, iA0
    for k in range(d.iterations):
        # chain A: guide (i_A, v_A) carrying X_B; chain B: guide (i_B, v_B) carrying X_A
        gA2, vA2, XB2 = href.atrous_pass(gA, vA, XB, nrm, z, albedo, 1 << k, d)
        gB2, vB2, XA2 = href.atrous_pass(gB, vB, XA, nrm, z, albedo, 1 << k, d)
        gA, vA, XB, gB, vB, XA = gA2, vA2, XB2, gB2, vB2, XA2
        m = m_plane(XA, XB, iA0, iB0, vA0, vB0, counts, albedo, eps)
        out.append((output(XA, XB, counts, albedo, eps), m, sref.smooth(m)))
    return out


def argmin(Ms):
    """k* from the list of M_k: level 0 starts, a strictly smaller M_k replaces the best (NaN never wins)."""
    best = np.array(Ms[0])
    level = np.zeros(best.shape, np.uint8)
    for k, M in enumerate(Ms[1:], 1):
        win = M < best
        best = np.where(win, M, best)
        level = np.where(win, np.uint8(k), level)
    return level


def beta(level, k):
    """(beta_k, first): the 5x5 binomial share of the in-image taps with k* = k, and whether no tap chose below k."""
    H, W = level.shape
    bs, bw, below = np.zeros((H, W)), np.zeros((H, W)), np.zeros((H, W), bool)
    lv = level.astype(np.int64)
    for dv in range(-2, 3):
        for du in range(-2, 3):
            inside = dr._inside(H, W, du, dv)
            lq = dr._shift(lv, du, dv, -1)
            K = dr.K5[du + 2] * dr.K5[dv + 2]
            bs = bs + np.where(inside & (lq == k), K, 0.0)
            below |= inside & (lq < k)
            bw = bw + np.where(inside, K, 0.0)
    return bs / bw, ~below


def blend(lv, level):
    """(out (H, W, 3), M^ (H, W)) from the levels and k*."""
    H, W = level.shape
    out, Mh = np.zeros((H, W, 3)), np.zeros((H, W))
    for k, (O, _, M) in enumerate(lv):
        b, first = beta(level, k)
        use = b != 0.0
        with np.errstate(invalid="ignore", over="ignore"):
            bO, bM = b[..., None] * O, b * M
            out = np.where(use[..., None], np.where(first[..., None], bO, out + bO), out)
            Mh = np.where(use, np.where(first, bM, Mh + bM), Mh)
    return out, Mh


def cross(sums, m2, half, counts, nrm, z, albedo, d):
    """(rgb (H, W, 3), k* (H, W) uint8, M^ (H, W)); d.iterations >= 1."""
    assert d.iterations >= 1
    lv = levels(sums, m2, half, counts, nrm, z, albedo, d)
    level = argmin([M for _, _, M in lv])
    rgb, Mh = blend(lv, level)
    return rgb, level, Mh


def ties(lv, rel=1e-9):
    """Pixels where some level's M lies within `rel` (relative) of the running best it was compared with: where exp's
    last bit may change k*.  lv: levels()'s list."""
    Ms = np.stack([M for _, _, M in lv])
    best = np.fmin.accumulate(np.where(np.isnan(Ms), np.inf, Ms), axis=0)
    near = np.zeros(Ms.shape[1:], bool)
    with np.errstate(invalid="ignore"):
        for k in range(1, Ms.shape[0]):
            near |= np.abs(Ms[k] - best[k - 1]) <= rel * np.maximum(np.abs(best[k - 1]), np.abs(Ms[k]))
    return near


def dilate(mask, r=2):
    """mask grown by r pixels in x and y: the pixels whose (2r+1)^2 neighbourhood holds a masked pixel."""
    H, W = mask.shape
    out = np.zeros_like(mask)
    for dv in range(-r, r + 1):
        for du in range(-r, r + 1):
            out |= dr._shift(mask, du, dv, False)
    return out
