"""numpy restatement of the history test of rptb_buffer_reproject_merge (reproject_merge in rpt_b200/csrc/reproject.h) --
test infrastructure.  The same float64 operations in the same order as the device and the host emulation, so the
results agree to the last bit.  Planes as in tests/reproject_ref.py: sums (..., 3), M2 and counts (...)."""
import numpy as np

from tests import reproject_ref

NONE, REUSED, REJECTED = 0, 1, 2


def merge(hsums, hm2, hcounts, gamma, sums, m2, counts):
    """The history (hsums, hm2, hcounts) merged into the fresh state (sums, m2, counts) where the test accepts it ->
    (sums, M2, counts, verdict), verdict NONE (no history, or fewer than 2 fresh entries), REUSED or REJECTED."""
    hn, fn = np.asarray(hcounts, np.uint32), np.asarray(counts, np.uint32)
    dnh, dnf = hn.astype(np.float64), fn.astype(np.float64)
    test = (hn > 0) & (fn >= 2)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        d = hsums / dnh[..., None] - sums / dnf[..., None]
        d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        v = m2 / ((fn.astype(np.int64) - 1).astype(np.float64) * dnf) + hm2 / ((hn.astype(np.int64) - 1).astype(np.float64) * dnh)
        rejected = test & (d2 > (gamma * gamma) * v)
        n = (fn.astype(np.uint64) + hn).astype(np.uint32)
        m_acc = (m2 + hm2) + d2 * ((dnf * dnh) / n.astype(np.float64))
    accepted = test & ~rejected
    out_s = np.where(accepted[..., None], sums + hsums, sums)
    out_m = np.where(accepted, m_acc, m2)
    out_n = np.where(accepted, n, fn).astype(np.uint32)
    verdict = np.where(accepted, REUSED, np.where(rejected, REJECTED, NONE)).astype(np.int32)
    return out_s, out_m, out_n, verdict


def reproject_merge(dcam, dnrm, dz, df, scam, ssums, sm2, scounts, snrm, sz, sf, prm, gamma, sums, m2, counts):
    """rptb_buffer_reproject_merge on row-major planes: reproject_ref.reproject's history of every destination pixel,
    merged into its fresh (sums, m2, counts) -> merge's (sums, M2, counts, verdict)."""
    hs, hm, hn = reproject_ref.reproject(dcam, dnrm, dz, df, scam, ssums, sm2, scounts, snrm, sz, sf, prm)
    return merge(hs, hm, hn, gamma, sums, m2, counts)
