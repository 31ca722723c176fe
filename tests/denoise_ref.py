"""numpy restatement of rpt_b200/csrc/denoise.h -- test infrastructure.  The same float64 operations in the same order as
the device and the host emulation, so the results agree to the last bit except where exp differs from numpy's.

Planes are row-major: colour / normal / albedo (H, W, 3), variance / depth / counts (H, W).  `d` is an api.Denoise."""
import numpy as np

K5 = (1.0 / 16.0, 1.0 / 4.0, 3.0 / 8.0, 1.0 / 4.0, 1.0 / 16.0)
K3 = (0.25, 0.5, 0.25)
EPS_Z = 1e-3
EPS_L = 1e-10


def lum(c):
    return (0.2126 * c[..., 0] + 0.7152 * c[..., 1]) + 0.0722 * c[..., 2]


def powu(x, e):
    r, b = np.ones_like(x), x.copy()
    while e:
        if e & 1:
            r = r * b
        e >>= 1
        if e:
            b = b * b
    return r


def finite(x):
    with np.errstate(invalid="ignore"):
        return (x - x) == 0.0


def features_resolve(hits, sn, sz, sa, rays):
    """Per-pixel feature sums -> (N, z, a, hit fraction)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        length = np.sqrt((sn[..., 0] * sn[..., 0] + sn[..., 1] * sn[..., 1]) + sn[..., 2] * sn[..., 2])
        n = np.where((length > 0.0)[..., None], sn / length[..., None], 0.0)
        z = np.where(hits > 0.0, sz / hits, np.inf)
    miss = rays - hits
    a = (sa + miss[..., None]) / rays
    return n, z, a, hits / rays


def mean_variance(counts, m2):
    dn = np.asarray(counts, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return m2 / (((dn - 1.0) * dn) * 3.0)


def demodulate(sums, m2, counts, albedo, eps_a):
    dn = np.asarray(counts, dtype=np.float64)[..., None]
    a = albedo + eps_a
    with np.errstate(divide="ignore", invalid="ignore"):
        i = (sums / dn) / a
        v = mean_variance(counts, m2)
    return i, v


def _shift(x, dx, dy, fill):
    """out[y, x] = x[y + dy, x + dx], `fill` outside."""
    H, W = x.shape[:2]
    out = np.full_like(x, fill)
    ys, yd = (slice(dy, H), slice(0, H - dy)) if dy >= 0 else (slice(0, H + dy), slice(-dy, H))
    xs, xd = (slice(dx, W), slice(0, W - dx)) if dx >= 0 else (slice(0, W + dx), slice(-dx, W))
    if ys.start < ys.stop and xs.start < xs.stop and yd.start < yd.stop and xd.start < xd.stop:
        out[yd, xd] = x[ys, xs]
    return out


def _inside(H, W, dx, dy):
    ys, xs = np.arange(H)[:, None] + dy, np.arange(W)[None, :] + dx
    return (ys >= 0) & (ys < H) & (xs >= 0) & (xs < W)


def _grad1(zm, has_m, z, zp, has_p):
    with np.errstate(invalid="ignore"):
        b, f = z - zm, zp - z
    ok_b, ok_f = has_m & finite(b), has_p & finite(f)
    both = np.where(np.abs(f) < np.abs(b), f, b)
    return np.where(ok_b & ok_f, both, np.where(ok_b, b, np.where(ok_f, f, 0.0)))


def grad(z):
    H, W = z.shape
    gx = _grad1(_shift(z, -1, 0, 0.0), _inside(H, W, -1, 0), z, _shift(z, 1, 0, 0.0), _inside(H, W, 1, 0))
    gy = _grad1(_shift(z, 0, -1, 0.0), _inside(H, W, 0, -1), z, _shift(z, 0, 1, 0.0), _inside(H, W, 0, 1))
    return gx, gy


def atrous_pass(i, v, nrm, z, albedo, h, d):
    """One pass with step h: (i', v')."""
    H, W = v.shape
    own_ok = finite(i).all(-1) & finite(v)
    gs, gw = np.zeros((H, W)), np.zeros((H, W))
    for dv in (-1, 0, 1):
        for du in (-1, 0, 1):
            inside = _inside(H, W, du, dv)
            vq = _shift(v, du, dv, 0.0)
            ok = inside & finite(vq)
            k = K3[du + 1] * K3[dv + 1]
            gs = gs + np.where(ok, k * np.where(ok, vq, 0.0), 0.0)
            gw = gw + np.where(ok, k, 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        g = np.minimum(v, gs / gw)
    np_zero = (nrm == 0.0).all(-1)
    zp_inf = ~finite(z)
    gx, gy = grad(z)
    eps_z = EPS_Z * z
    A = albedo + d.albedo_eps
    lp = lum(i * A)
    with np.errstate(invalid="ignore"):
        lden = d.sigma_luminance * np.sqrt(g) + EPS_L
    sw, sww = np.zeros((H, W)), np.zeros((H, W))
    s = np.zeros((H, W, 3))
    for dv in range(-2, 3):
        for du in range(-2, 3):
            dx, dy = du * h, dv * h
            inside = _inside(H, W, dx, dy)
            iq = _shift(i, dx, dy, 0.0)
            vq = _shift(v, dx, dy, 0.0)
            K = K5[du + 2] * K5[dv + 2]
            if du == 0 and dv == 0:
                w = np.full((H, W), K)
                ok = inside
            else:
                ok = inside & finite(iq).all(-1) & finite(vq)
                nq = _shift(nrm, dx, dy, 0.0)
                with np.errstate(invalid="ignore"):
                    c = (nrm[..., 0] * nq[..., 0] + nrm[..., 1] * nq[..., 1]) + nrm[..., 2] * nq[..., 2]
                wn = np.where(np_zero & (nq == 0.0).all(-1), 1.0, powu(np.where(c > 0.0, c, 0.0), d.sigma_normal))
                zq = _shift(z, dx, dy, 0.0)
                zq_inf = ~finite(zq)
                with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
                    plane = np.minimum(np.abs(gx * float(-dx) + gy * float(-dy)),
                                       np.abs(_shift(gx, dx, dy, 0.0) * float(-dx) + _shift(gy, dx, dy, 0.0) * float(-dy)))
                    wz = np.exp(-(np.abs(z - zq) / (d.sigma_depth * plane + eps_z)))
                    wz = np.where(zp_inf | zq_inf, np.where(zp_inf & zq_inf, 1.0, 0.0), wz)
                    wl = np.exp(-(np.abs(lp - lum(iq * A)) / lden))
                    w = ((K * wn) * wz) * wl
            w = np.where(ok, w, 0.0)
            iq = np.where(ok[..., None], iq, 0.0)
            vq = np.where(ok, vq, 0.0)
            sw = sw + w
            sww = sww + (w * w) * vq
            s = s + w[..., None] * iq
    with np.errstate(invalid="ignore", divide="ignore"):
        out_i = s / sw[..., None]
        out_v = sww / (sw * sw)
    out_i = np.where(own_ok[..., None], out_i, i)
    out_v = np.where(own_ok, out_v, v)
    return out_i, out_v


def denoise(sums, m2, counts, nrm, z, albedo, d, return_variance=False):
    """The whole filter: c' (H, W, 3) (and the final demodulated variance)."""
    counts = np.asarray(counts, dtype=np.float64)
    if d.iterations == 0:
        return sums / counts[..., None]
    i, v = demodulate(sums, m2, counts, albedo, d.albedo_eps)
    for k in range(d.iterations):
        i, v = atrous_pass(i, v, nrm, z, albedo, 1 << k, d)
    out = i * (albedo + d.albedo_eps)
    return (out, v) if return_variance else out


# ---- the feature pass, from closest-hit queries ------------------------------------------------------------------
def camera_rays(cam, width, height, iterations, seed, first_sample=0):
    """The render's camera rays (features.cuh / camera.cuh) in f64, per pixel (row-major) and sample: (npix, iterations, 6).
    `cam` is a capi.Camera; the draws are tests/trace_ref.py's Philox stream for (seed, pixel, sample)."""
    import math

    from tests import trace_ref as tr

    d = 1.0 / math.tan(cam.fov / 2.0)
    di, up = tuple(cam.direction), tuple(cam.up)
    right = (di[1] * up[2] - di[2] * up[1], di[2] * up[0] - di[0] * up[2], di[0] * up[1] - di[1] * up[0])
    ln = math.sqrt(right[0] * right[0] + right[1] * right[1] + right[2] * right[2])
    cright = (right[0] / ln, right[1] / ln, right[2] / ln)
    eye = tuple(cam.eye)
    dim = float(max(width, height))
    out = np.empty((width * height, iterations, 6))
    for y in range(height):
        for x in range(width):
            pix = y * width + x
            xn = (float(2 * x + 1) - float(width)) / dim
            yn = (float(2 * (height - y) - 1) - float(height)) / dim
            for i in range(iterations):
                rng = tr.Rng(seed, pix, first_sample + i)
                dx = rng.gen_range(-1.0 / dim, 1.0 / dim)
                dy = rng.gen_range(-1.0 / dim, 1.0 / dim)
                cx, cy = xn + dx, yn + dy
                origin = eye
                new_dir = tr.add(tr.add(tr.mul(di, d), tr.mul(cright, cx)), tr.mul(up, cy))
                if cam.aperture > 0.0:
                    focal = tr.add(origin, tr.mul(tr.normalize(new_dir), cam.focal_distance))
                    ax, ay = rng.unit_disc()
                    origin = tr.add(origin, tr.mul(tr.add(tr.mul(cright, ax), tr.mul(up, ay)), cam.aperture))
                    new_dir = tr.sub(focal, origin)
                out[pix, i, :3] = origin
                out[pix, i, 3:] = tr.normalize(new_dir)
    return out


def feature_sums(rays, t, obj, nrm, colors):
    """The sums rptb_buffer_add_features keeps, from the closest hits of `rays` ((npix, iters, 6); t, obj, nrm flattened
    the same way) and the colour of each object's material: (normal (npix, 3), albedo (npix, 3), hits (npix,),
    depth (npix,)), added in sample order."""
    npix, iters = rays.shape[:2]
    t, obj, nrm = t.reshape(npix, iters), obj.reshape(npix, iters), nrm.reshape(npix, iters, 3)
    sn, sa, h, sz = np.zeros((npix, 3)), np.zeros((npix, 3)), np.zeros(npix), np.zeros(npix)
    for i in range(iters):
        hit = obj[:, i] >= 0
        n = nrm[:, i]
        rd = rays[:, i, 3:]
        facing = (n[:, 0] * rd[:, 0] + n[:, 1] * rd[:, 1]) + n[:, 2] * rd[:, 2]
        n = np.where((facing > 0.0)[:, None], -n, n)
        col = colors[np.where(hit, obj[:, i], 0)]
        h = np.where(hit, h + 1.0, h)
        sn = np.where(hit[:, None], sn + n, sn)
        sz = np.where(hit, sz + t[:, i], sz)
        sa = np.where(hit[:, None], sa + col, sa)
    return sn, sa, h, sz


def object_colors(flat):
    """The colour of every flattened object's material, (nobjects, 3)."""
    d = flat.desc
    return np.array([[d.materials[d.objects[k].material].color[c] for c in range(3)] for k in range(d.nobjects)])
