"""numpy restatement of the history halves of rptb_buffer_reproject and rptb_buffer_reproject_merge (reproject_history,
reproject_merge_halves in rpt_b200/csrc/reproject.h), on top of tests/reproject_ref.py and tests/reproject_merge_ref.py
-- test infrastructure.  The same float64 operations in the same order as the device and the host emulation, so the
results agree to the last bit.  Planes as in tests/reproject_ref.py; half is (..., 3) like sums."""
import numpy as np

from tests import reproject_merge_ref as mref
from tests import reproject_ref as ref


def _taps(dcam, dnrm, dz, df, scam, scounts, ssums, sm2, snrm, sz, sf, prm):
    """reproject_ref.reproject's tap selection: (W, [(valid, w, (cy, cx)) per tap in tap order])."""
    dh, dw = dz.shape
    sh, sw = sz.shape
    px, py, ell, ok = ref.project(dcam, dw, dh, dz, df, scam, sw, sh)
    px, py = np.where(ok, px, 0.0), np.where(ok, py, 0.0)
    x0, y0 = np.floor(px), np.floor(py)
    fx, fy = px - x0, py - y0
    wx, wy = (1.0 - fx, fx), (1.0 - fy, fy)
    surface = df > 0.0
    taps = []
    W = np.zeros((dh, dw))
    for t in range(4):
        w = wx[t & 1] * wy[t >> 1]
        qx, qy = x0.astype(np.int64) + (t & 1), y0.astype(np.int64) + (t >> 1)
        inside = ok & (w > 0.0) & (qx >= 0) & (qy >= 0) & (qx < sw) & (qy < sh)
        cx, cy = np.clip(qx, 0, sw - 1), np.clip(qy, 0, sh - 1)
        n = scounts[cy, cx]
        fq, zq, Nq = sf[cy, cx], sz[cy, cx], snrm[cy, cx]
        with np.errstate(invalid="ignore"):
            surf_ok = (fq > 0.0) & (np.abs(zq - ell) <= prm.depth_tol * ell) & (ref._dot(dnrm, Nq) >= prm.normal_cos)
        valid = inside & (n >= 2) & ref.finite(ssums[cy, cx]).all(-1) & ref.finite(sm2[cy, cx]) & np.where(surface, surf_ok, fq == 0.0)
        w = np.where(valid, w, 0.0)
        W = np.where(valid, W + w, W)
        taps.append((valid, w, (cy, cx)))
    return W, taps


def reproject(dcam, dnrm, dz, df, scam, ssums, sm2, scounts, shalf, snrm, sz, sf, prm):
    """-> (sums, M2, counts, half) of the destination view: reproject_ref.reproject's planes and the history's HALF."""
    out_s, out_m, nh = ref.reproject(dcam, dnrm, dz, df, scam, ssums, sm2, scounts, snrm, sz, sf, prm)
    counts = np.asarray(scounts, np.uint32)
    W, taps = _taps(dcam, dnrm, dz, df, scam, counts, ssums, sm2, snrm, sz, sf, prm)
    has = nh > 0
    dh, dw = nh.shape
    mu, t, w2 = np.zeros((dh, dw, 3)), np.zeros((dh, dw, 3)), np.zeros((dh, dw))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for valid, w, (cy, cx) in taps:
            wh = w / W
            n = counts[cy, cx]
            S, Hq = ssums[cy, cx], shalf[cy, cx]
            dn = n.astype(np.float64)
            nb = n >> np.uint32(1)
            dB, dA = nb.astype(np.float64), (n - nb).astype(np.float64)
            g = np.sqrt((dA * dB) / dn)
            delta = ((S - Hq) / dA[..., None] - Hq / dB[..., None]) * g[..., None]
            v3 = valid[..., None]
            mu = np.where(v3, mu + wh[..., None] * (S / dn[..., None]), mu)
            t = np.where(v3, t + wh[..., None] * delta, t)
            w2 = np.where(valid, w2 + wh * wh, w2)
        nb = nh >> np.uint32(1)
        dB, dA, dhf = nb.astype(np.float64), (nh - nb).astype(np.float64), nh.astype(np.float64)
        k = np.sqrt((dA * dB) / dhf)
        half = dB[..., None] * mu - (t / np.sqrt(w2)[..., None]) * k[..., None]
    return out_s, out_m, nh, np.where(has[..., None], half, 0.0)


def merge(hsums, hm2, hcounts, hhalf, gamma, sums, m2, counts, half):
    """reproject_merge_ref.merge with HALF: an accepted history adds hhalf (fresh count even) or hsums - hhalf (odd) to
    half -> (sums, M2, counts, half, verdict)."""
    s, m, n, verdict = mref.merge(hsums, hm2, hcounts, gamma, sums, m2, counts)
    odd = (np.asarray(counts, np.uint32) & np.uint32(1)) == 1
    add = np.where(odd[..., None], hsums - hhalf, hhalf)
    return s, m, n, np.where((verdict == mref.REUSED)[..., None], half + add, half), verdict


def reproject_merge(dcam, dnrm, dz, df, scam, ssums, sm2, scounts, shalf, snrm, sz, sf, prm, gamma, sums, m2, counts, half):
    """rptb_buffer_reproject_merge on row-major planes of buffers with halves -> merge's (sums, M2, counts, half, verdict)."""
    hs, hm, hn, hh = reproject(dcam, dnrm, dz, df, scam, ssums, sm2, scounts, shalf, snrm, sz, sf, prm)
    return merge(hs, hm, hn, hh, gamma, sums, m2, counts, half)
