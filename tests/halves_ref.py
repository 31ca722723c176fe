"""numpy restatement of rpt_b200/csrc/halves.h -- the error estimate of the denoised image from two half buffers -- and of
the guided criterion on it (rptb_sample_into_guided_error), on top of tests/denoise_ref.py -- test infrastructure.  The
same float64 operations in the same order as the device and the host emulation; the filter's exp may differ from numpy's
in the last bit.

Planes are row-major: sums / half / normal / albedo (H, W, 3), m2 / depth / counts (H, W).  `d` is an api.Denoise, `crit`
an api.Adaptive."""
import numpy as np

from tests import denoise_ref as dr
from tests import guided_ref


def u_plane(sums, half, counts, albedo, eps_a):
    """u per pixel and channel: ((S_A / n_A - S_B / n_B) * sqrt(n_A n_B) / n) / (a + eps_a); NaN where n_B = 0."""
    n = np.asarray(counts, dtype=np.uint64)
    nb = n >> np.uint64(1)
    na = n - nb
    dA, dB, dn = na.astype(np.float64)[..., None], nb.astype(np.float64)[..., None], n.astype(np.float64)[..., None]
    with np.errstate(divide="ignore", invalid="ignore"):
        f = np.sqrt(dA * dB) / dn
        sb = half
        sa = sums - sb
        u = ((sa / dA - sb / dB) * f) / (albedo + eps_a)
    return np.where((nb == 0)[..., None], np.nan, u)


def atrous_pass(i, v, u, nrm, z, albedo, h, d):
    """One pass with step h: (i', v', u').  i' and v' are denoise_ref.atrous_pass's; u' is u filtered with the same
    weights over the taps whose u is finite, and a pixel whose own i or v is not finite keeps its u."""
    H, W = v.shape
    own_ok = dr.finite(i).all(-1) & dr.finite(v)
    gs, gw = np.zeros((H, W)), np.zeros((H, W))
    for dv in (-1, 0, 1):
        for du in (-1, 0, 1):
            inside = dr._inside(H, W, du, dv)
            vq = dr._shift(v, du, dv, 0.0)
            ok = inside & dr.finite(vq)
            k = dr.K3[du + 1] * dr.K3[dv + 1]
            gs = gs + np.where(ok, k * np.where(ok, vq, 0.0), 0.0)
            gw = gw + np.where(ok, k, 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        g = np.minimum(v, gs / gw)
    np_zero = (nrm == 0.0).all(-1)
    zp_inf = ~dr.finite(z)
    gx, gy = dr.grad(z)
    eps_z = dr.EPS_Z * z
    A = albedo + d.albedo_eps
    lp = dr.lum(i * A)
    with np.errstate(invalid="ignore"):
        lden = d.sigma_luminance * np.sqrt(g) + dr.EPS_L
    sw, sww, swu = np.zeros((H, W)), np.zeros((H, W)), np.zeros((H, W))
    s, su = np.zeros((H, W, 3)), np.zeros((H, W, 3))
    for dv in range(-2, 3):
        for du in range(-2, 3):
            dx, dy = du * h, dv * h
            inside = dr._inside(H, W, dx, dy)
            iq = dr._shift(i, dx, dy, 0.0)
            vq = dr._shift(v, dx, dy, 0.0)
            uq = dr._shift(u, dx, dy, 0.0)
            K = dr.K5[du + 2] * dr.K5[dv + 2]
            if du == 0 and dv == 0:
                w = np.full((H, W), K)
                ok = inside
            else:
                ok = inside & dr.finite(iq).all(-1) & dr.finite(vq)
                nq = dr._shift(nrm, dx, dy, 0.0)
                with np.errstate(invalid="ignore"):
                    c = (nrm[..., 0] * nq[..., 0] + nrm[..., 1] * nq[..., 1]) + nrm[..., 2] * nq[..., 2]
                wn = np.where(np_zero & (nq == 0.0).all(-1), 1.0, dr.powu(np.where(c > 0.0, c, 0.0), d.sigma_normal))
                zq = dr._shift(z, dx, dy, 0.0)
                zq_inf = ~dr.finite(zq)
                with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
                    plane = np.minimum(np.abs(gx * float(-dx) + gy * float(-dy)),
                                       np.abs(dr._shift(gx, dx, dy, 0.0) * float(-dx) + dr._shift(gy, dx, dy, 0.0) * float(-dy)))
                    wz = np.exp(-(np.abs(z - zq) / (d.sigma_depth * plane + eps_z)))
                    wz = np.where(zp_inf | zq_inf, np.where(zp_inf & zq_inf, 1.0, 0.0), wz)
                    wl = np.exp(-(np.abs(lp - dr.lum(iq * A)) / lden))
                    w = ((K * wn) * wz) * wl
            w = np.where(ok, w, 0.0)
            iq = np.where(ok[..., None], iq, 0.0)
            vq = np.where(ok, vq, 0.0)
            sw = sw + w
            sww = sww + (w * w) * vq
            s = s + w[..., None] * iq
            uok = ok & dr.finite(uq).all(-1)
            wu = np.where(uok, w, 0.0)
            swu = swu + wu
            su = su + wu[..., None] * np.where(uok[..., None], uq, 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        out_i = s / sw[..., None]
        out_v = sww / (sw * sw)
        out_u = su / swu[..., None]
    out_i = np.where(own_ok[..., None], out_i, i)
    out_v = np.where(own_ok, out_v, v)
    out_u = np.where(own_ok[..., None], out_u, u)
    return out_i, out_v, out_u


def e_plane(U, albedo, eps_a):
    """e: the channel mean of the remodulated U squared."""
    with np.errstate(invalid="ignore", over="ignore"):
        r = U * (albedo + eps_a)
        return ((r[..., 0] * r[..., 0] + r[..., 1] * r[..., 1]) + r[..., 2] * r[..., 2]) / 3.0


def smooth(e):
    """E: e over the 3x3 (1/4, 1/2, 1/4)^2 taps in the image with a finite e, divided by the sum of their weights."""
    H, W = e.shape
    es, ew = np.zeros((H, W)), np.zeros((H, W))
    for dv in (-1, 0, 1):
        for du in (-1, 0, 1):
            eq = dr._shift(e, du, dv, 0.0)
            ok = dr._inside(H, W, du, dv) & dr.finite(eq)
            k = dr.K3[du + 1] * dr.K3[dv + 1]
            es = es + np.where(ok, k * np.where(ok, eq, 0.0), 0.0)
            ew = ew + np.where(ok, k, 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return es / ew


def error(sums, m2, half, counts, nrm, z, albedo, d):
    """The filter with the estimate over a buffer state: (c' (H, W, 3), v' (H, W), E (H, W)); d.iterations >= 1."""
    assert d.iterations >= 1
    i, v = dr.demodulate(sums, m2, counts, albedo, d.albedo_eps)
    u = u_plane(sums, half, counts, albedo, d.albedo_eps)
    for k in range(d.iterations):
        i, v, u = atrous_pass(i, v, u, nrm, z, albedo, 1 << k, d)
    return i * (albedo + d.albedo_eps), v, smooth(e_plane(u, albedo, d.albedo_eps))


def active(counts, c, E, crit):
    """The guided-error decision: guided_ref.active with E in place of v'."""
    return guided_ref.active(counts, c, E, crit)


def borderline(counts, c, E, crit, rel=1e-9):
    return guided_ref.borderline(counts, c, E, crit, rel)


def odd_sums(entries):
    """HALF rebuilt from a pixel's entries in order: entries is a list of (npix, 3) renders with, for each, the (npix,)
    bool of the pixels that took it; the entry a pixel takes at its count k goes into HALF iff k is odd.  Summed in entry
    order, as the accumulate adds it."""
    npix = entries[0][0].shape[0] if entries else 0
    half, k = np.zeros((npix, 3)), np.zeros(npix, np.int64)
    for x, took in entries:
        odd = took & (k % 2 == 1)
        half = np.where(odd[:, None], half + x, half)
        k = k + took
    return half
