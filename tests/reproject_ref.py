"""numpy restatement of rpt_b200/csrc/reproject.h -- test infrastructure.  The same float64 operations in the same order as
the device and the host emulation, so the results agree to the last bit.

Cameras are capi.Camera or api.Camera; planes are row-major: sums / normal (H, W, 3), M2 / counts / depth / hit fraction
(H, W).  `prm` is an api.Reproject."""
import math

import numpy as np

MIN_WEIGHT = 1e-2


def view(cam, width, height):
    """(eye, D, U, R, dc, dim) as reproject_view computes them: Python floats are IEEE doubles, math.tan is the C library's."""
    di, up = [float(v) for v in cam.direction], [float(v) for v in cam.up]
    right = [di[1] * up[2] - di[2] * up[1], di[2] * up[0] - di[0] * up[2], di[0] * up[1] - di[1] * up[0]]
    ln = math.sqrt((right[0] * right[0] + right[1] * right[1]) + right[2] * right[2])
    R = np.array([r / ln for r in right])
    return (np.array([float(v) for v in cam.eye]), np.array(di), np.array(up), R, 1.0 / math.tan(float(cam.fov) / 2.0),
            float(max(width, height)))


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    a, b = np.broadcast_arrays(a, b)
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def finite(x):
    with np.errstate(invalid="ignore"):
        return (x - x) == 0.0


def project(dcam, dw, dh, dz, df, scam, sw, sh):
    """Per destination pixel: (px, py, l, ok) -- the continuous source position, the distance l of the first hit from the
    source eye (+inf for the environment) and whether the pixel lies in front of the source camera and near its image."""
    eye, D, U, R, dc, dim = view(dcam, dw, dh)
    seye, sD, sU, sR, sdc, sdim = view(scam, sw, sh)
    x = np.arange(dw, dtype=np.float64)[None, :]
    y = np.arange(dh, dtype=np.uint64)[:, None]
    xn = ((2.0 * x + 1.0) - float(dw)) / dim
    yn = ((2 * (dh - y) - 1).astype(np.float64) - float(dh)) / dim
    xn, yn = np.broadcast_arrays(xn, yn)
    r = (dc * D + xn[..., None] * R) + yn[..., None] * U
    rl = np.sqrt(_dot(r, r))
    u = r / rl[..., None]
    surface = df > 0.0
    with np.errstate(invalid="ignore", over="ignore"):
        v = np.where(surface[..., None], (eye + np.where(surface, dz, 0.0)[..., None] * u) - seye, u)
        ell = np.where(surface, np.sqrt(_dot(v, v)), np.inf)
    a = sdc * sD
    bc = _cross(sR, sU)
    det = _dot(a, bc)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        alpha = _dot(v, bc) / det
        beta = _dot(a, _cross(v, sU)) / det
        gamma = _dot(a, _cross(sR, v)) / det
        xs, ys = beta / alpha, gamma / alpha
        px = (xs * sdim + float(sw - 1)) / 2.0
        py = (float(sh - 1) - ys * sdim) / 2.0
        ok = (alpha > 0.0) & (px > -1.0) & (px < float(sw)) & (py > -1.0) & (py < float(sh))
    return px, py, ell, ok


def reproject(dcam, dnrm, dz, df, scam, ssums, sm2, scounts, snrm, sz, sf, prm):
    """-> (sums (dh, dw, 3), M2 (dh, dw), counts (dh, dw) uint32) of the destination view."""
    dh, dw = dz.shape
    sh, sw = sz.shape
    px, py, ell, ok = project(dcam, dw, dh, dz, df, scam, sw, sh)
    px, py = np.where(ok, px, 0.0), np.where(ok, py, 0.0)
    x0, y0 = np.floor(px), np.floor(py)
    fx, fy = px - x0, py - y0
    wx, wy = (1.0 - fx, fx), (1.0 - fy, fy)
    surface = df > 0.0
    counts = np.asarray(scounts, np.uint32)
    taps = []
    W = np.zeros((dh, dw))
    nmin = np.full((dh, dw), 0xFFFFFFFF, np.uint64)
    for t in range(4):
        w = wx[t & 1] * wy[t >> 1]
        qx, qy = x0.astype(np.int64) + (t & 1), y0.astype(np.int64) + (t >> 1)
        inside = ok & (w > 0.0) & (qx >= 0) & (qy >= 0) & (qx < sw) & (qy < sh)
        cx, cy = np.clip(qx, 0, sw - 1), np.clip(qy, 0, sh - 1)
        n = counts[cy, cx]
        S, M = ssums[cy, cx], sm2[cy, cx]
        fq, zq, Nq = sf[cy, cx], sz[cy, cx], snrm[cy, cx]
        with np.errstate(invalid="ignore"):
            surf_ok = (fq > 0.0) & (np.abs(zq - ell) <= prm.depth_tol * ell) & (_dot(dnrm, Nq) >= prm.normal_cos)
        valid = inside & (n >= 2) & finite(S).all(-1) & finite(M) & np.where(surface, surf_ok, fq == 0.0)
        w = np.where(valid, w, 0.0)
        W = np.where(valid, W + w, W)
        nmin = np.where(valid, np.minimum(nmin, n), nmin)
        taps.append((valid, w, S, M, n))
    has = W >= MIN_WEIGHT
    mu = np.zeros((dh, dw, 3))
    s2 = np.zeros((dh, dw))
    with np.errstate(invalid="ignore", divide="ignore"):
        for valid, w, S, M, n in taps:
            wh = w / W
            dn = n.astype(np.float64)
            mu = np.where(valid[..., None], mu + wh[..., None] * (S / dn[..., None]), mu)
            s2 = np.where(valid, s2 + wh * (M / (n.astype(np.uint64) - 1).astype(np.float64)), s2)
    nh = np.where(has, np.minimum(np.uint64(prm.max_history), nmin), 0).astype(np.uint32)
    dhf = nh.astype(np.float64)
    out_s = np.where(has[..., None], mu * dhf[..., None], 0.0)
    out_m = np.where(has, s2 * (nh.astype(np.int64) - 1).astype(np.float64), 0.0)
    return out_s, out_m, nh
