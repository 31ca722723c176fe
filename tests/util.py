"""Helpers shared by the tests: an independent numpy restatement of the BSDF / pdf
formulas (second implementation, used to validate the oracle), ray generators, and
image-comparison metrics."""
import math

import numpy as np


def normalize(v):
    v = np.asarray(v, dtype=np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def random_unit(rng, n):
    return normalize(rng.normal(size=(n, 3)))


# ---- independent restatement of src/material.rs:125-210 (vectorised over wi) -------------
def bsdf_ref(color, index, roughness, metallic, transparent, n, wo, wi):
    color = np.asarray(color, dtype=np.float64)
    n, wo, wi = (np.asarray(a, dtype=np.float64) for a in (n, wo, wi))
    ndwi = (n * wi).sum(-1)
    ndwo = (n * wo).sum(-1)
    wi_out = ~np.signbit(ndwi)
    wo_out = ~np.signbit(ndwo)
    m2 = roughness * roughness
    f0s = ((index - 1.0) / (index + 1.0)) ** 2
    f0 = f0s * (1.0 - metallic) + color * metallic
    out = np.zeros(wi.shape)
    with np.errstate(all="ignore"):
        # same side
        h = normalize(wi + wo)
        wodh = (wo * h).sum(-1)
        ndh = (n * h).sum(-1)
        nh2 = ndh**2
        d = np.exp((nh2 - 1.0) / (m2 * nh2)) / (m2 * math.pi * nh2 * nh2)
        tir = (~wi_out) & (np.sqrt(1.0 - wodh * wodh) * index > 1.0)
        f = f0[None, :] + (1.0 - f0[None, :]) * ((1.0 - wodh) ** 5)[:, None]
        f = np.where(tir[:, None], 1.0, f)
        g = np.minimum(1.0, 2.0 * np.minimum(ndwi * ndh, ndwo * ndh) / wodh)
        spec = d[:, None] * f * g[:, None] / (4.0 * ndwo * ndwi)[:, None]
        same = spec if transparent else spec + (1.0 - f) * color[None, :] / math.pi
        # opposite sides
        eta = np.where(wo_out, index, 1.0 / index)
        h2 = normalize(wi * eta[:, None] + wo)
        widh = (wi * h2).sum(-1)
        wodh2 = (wo * h2).sum(-1)
        ndh2 = (n * h2).sum(-1)
        nh22 = ndh2**2
        d2 = np.exp((nh22 - 1.0) / (m2 * nh22)) / (m2 * math.pi * nh22 * nh22)
        f2 = f0[None, :] + (1.0 - f0[None, :]) * ((1.0 - np.abs(widh)) ** 5)[:, None]
        g2 = np.minimum(1.0, 2.0 * np.minimum(np.abs(ndwi * ndh2), np.abs(ndwo * ndh2)) / np.abs(wodh2))
        btdf = (np.abs(widh * wodh2 / (ndwi * ndwo)) * d2 * g2 / (eta * widh + wodh2) ** 2)[:, None] * (1.0 - f2)
        opp = btdf * color[None, :]
    side = wi_out == wo_out
    out = np.where(side[:, None], same, opp)
    if not transparent:
        out = np.where((wi_out & wo_out)[:, None], out, 0.0)
    return out


# ---- independent restatement of the pdf of src/material.rs:290-312 ------------------------
def pdf_ref(color, index, roughness, metallic, transparent, n, wo, wi):
    color = np.asarray(color, dtype=np.float64)
    n, wo, wi = (np.asarray(a, dtype=np.float64) for a in (n, wo, wi))
    m2 = roughness * roughness
    f0 = ((index - 1.0) / (index + 1.0)) ** 2
    f = 0.8 * ((1.0 - metallic) * f0 + metallic * color.mean()) + 0.2
    wodn = (wo * n).sum(-1)
    eta = np.where(wodn > 0.0, index, 1.0 / index)

    def p_h(h):
        c = np.abs((h * n).sum(-1))
        s = np.sqrt(1.0 - c * c)
        return np.exp(-((s / c) ** 2) / m2) / (math.pi * m2 * c**3)

    with np.errstate(all="ignore"):
        h = normalize(wi + wo)
        p = f * p_h(h) / (4.0 * np.abs((h * wo).sum(-1)))
        widn = (wi * n).sum(-1)
        if not transparent:
            p = p + (1.0 - f) * np.maximum(widn, 0.0) / math.pi
        else:
            h2 = normalize(wi * eta[:, None] + wo)
            hwo = (h2 * wo).sum(-1)
            hwi = (h2 * wi).sum(-1)
            t = (1.0 - f) * p_h(h2) * np.abs(hwo) / (eta * hwi + hwo) ** 2
            p = p + np.where(np.signbit(wodn) != np.signbit(widn), t, 0.0)
    return p


def camera_rays(camera, n, rng, spread=0.7, jitter=0.0):
    """Rays from the camera eye fanned over the field of view (mostly hitting the scene)."""
    right = np.cross(camera.direction, camera.up)
    right = right / np.linalg.norm(right)
    d = (camera.direction[None, :] / math.tan(camera.fov / 2.0) + rng.uniform(-1, 1, (n, 1)) * right[None, :]
         + rng.uniform(-spread, spread, (n, 1)) * camera.up[None, :])
    d = normalize(d)
    o = np.tile(camera.eye, (n, 1)) + rng.normal(0.0, jitter, (n, 3))
    return np.concatenate([o, d], axis=1)


def interior_rays(lo, hi, n, rng):
    """Random rays starting inside a box -- exercises inside hits and all directions."""
    o = rng.uniform(lo, hi, (n, 3))
    return np.concatenate([o, random_unit(rng, n)], axis=1)


def rmse(a, b):
    return float(np.sqrt(np.mean((np.asarray(a) - np.asarray(b)) ** 2)))


REPEATED_DEVICES = "RPTB_ALLOW_REPEATED_DEVICES"


def replica_lists(gpu_ok):
    """Device lists for the tests that must give the same bits for every replica count.  A repeated device is a replica
    of its own (under RPTB_ALLOW_REPEATED_DEVICES=1, which the caller sets with monkeypatch.setenv), so one GPU runs every
    multi-part path; with two or more GPUs the lists also cross devices, and [0, 1, 0, 1] mixes same-device and
    cross-device copies in one buffer."""
    lists = [[0], [0, 0], [0, 0, 0], [0] * 5, [0] * 8]
    if gpu_ok >= 2:
        lists += [[0, 1], [0, 1, 0, 1], list(range(min(gpu_ok, 8)))]
    return lists


def golden_config(name):
    """The scene behind each committed fixture of tests/golden (tools/make_golden.py builds it the same way)."""
    from rpt_b200 import scenes
    if name == "glass":
        return scenes.glass_scene(256, 128)
    if name == "fractal_spheres":
        return scenes.fractal_spheres_scene(4)
    if name == "fractal_teapots":
        return scenes.fractal_teapots_scene(3)
    if name == "monomial_glass":
        return scenes.monomial_glass_scene(128, 64)
    return scenes.CONFIGS[name]()


# ---- SURVEY 8(d) parity criterion at full size -----------------------------------------------------------------
class Moments:
    """Per-pixel, per-channel mean and variance-of-the-mean of a render delivered as equally weighted batches --
    the reference's own mechanism: Renderer::iterative_render appends one entry per pixel per `sample()` call and
    Buffer::variance reads the spread of those entries (src/renderer.rs:103-115, src/buffer.rs:59-73)."""

    def __init__(self, npix):
        self.n = 0
        self.s1 = np.zeros((npix, 3))
        self.s2 = np.zeros((npix, 3))

    def add(self, batch):
        self.n += 1
        self.s1 += batch
        self.s2 += batch * batch

    @property
    def mean(self):
        return self.s1 / self.n

    @property
    def var_of_mean(self):
        n = self.n
        s2 = np.maximum(self.s2 - self.s1 * self.s1 / n, 0.0) / (n - 1)  # unbiased sample variance of the batches
        return s2 / n


def z_outlier_fraction(a: "Moments", b: "Moments", z_limit=4.0):
    """Fraction of pixels where some channel has |mu_a - mu_b| / sqrt(var_a/N + var_b/N) beyond z_limit.  With few
    batches the statistic is Student-t, not normal: it is mapped through Welch's degrees of freedom to the normal
    quantile with the same tail probability, so `z_limit` keeps its meaning for any batch count.  A rounding floor
    (1e-5 relative) keeps pixels that are constant on both sides (environment, 0 variance) from dividing by 0."""
    from scipy import stats as sps

    d = a.mean - b.mean
    va, vb = a.var_of_mean, b.var_of_mean
    floor = (1e-5 * np.maximum(np.maximum(np.abs(a.mean), np.abs(b.mean)), 1e-3)) ** 2
    v = va + vb + floor
    t = np.abs(d) / np.sqrt(v)
    with np.errstate(divide="ignore", invalid="ignore"):
        dof = v * v / (va * va / (a.n - 1) + vb * vb / (b.n - 1) + 1e-300)
    dof = np.clip(np.nan_to_num(dof, nan=1e9, posinf=1e9), 1.0, 1e9)
    p = 2.0 * sps.t.sf(t, dof)
    p_limit = 2.0 * sps.norm.sf(z_limit)
    bad = (p < p_limit).any(axis=1)
    return float(bad.mean()), t
