"""numpy fp64 restatement of the precision / recall / density / coverage definition (fadtk_b200.fad.calc_prdc).

Test infrastructure only.  The fp16 rows are taken as exact reals.  Distances come from the expanded form
|a|^2 + |b|^2 - 2 a.b in row blocks (as kad_oracle._pair_blocks), so that no m x n matrix is formed.  Unlike
kad_oracle, the rows are not centred: every fp16 value times 2^24 is an integer, and the expansion is done in exact
integer parts (_blocks), so q has no cancellation to control and is a function of the two rows alone.  That matters
here because the metrics are strict comparisons, and exact ties are common: duplicate rows, and an eval row equal to
a baseline row whose distance is some other row's radius.  An fp64 expansion, centred or not, would break such ties
by its rounding residue.  prdc_direct is the definition written as a plain double loop on differences: the oracle's
own check.

decision_bounds brackets what any computation of q within a known error can give.  The GPU path (csrc/prdc.cuh)
computes q on rows shifted by s = the fp16-rounded mean of X, y^ = z - s, as

    q^ = fp32(|y^_a|^2 + |y^_b|^2 - 2 y^_a . y^_b),   q^ := 0 when q^ <= 2^-14 (|y^_a|^2 + |y^_b|^2)

so, with S = |y^_a|^2 + |y^_b|^2:
  * the accumulator's rounding (three fp16 products per column, chunked fp32 sums; worst case at d = 1024 about
    2e-5 S, kad.cuh), the fp32 norms (2^-24 S) and the dropped lo.lo product (2^-23 S) give |q^ - q| <= 2.1e-5 S
    < 2^-15 S away from the flush;
  * the flush sets q^ = 0 only when the computed value is <= 2^-14 S, so there the true q <= 2^-14 S + 2^-15 S;
  * hence |q^ - q| <= 2^-14 S + 2^-15 S < 2^-13 S = tau S with tau = 2^-13, twice kQResolution.
A decision q < thr of the GPU can then differ from the exact one only when |q - thr| <= delta_ab = tau S: such a
decision is ambiguous.  With tau = 0 no decision is ambiguous and the bounds are the exact counts.
"""
from __future__ import annotations

import numpy as np

BLOCK = 512
TAU = 2.0 ** -13


def _parts(a: np.ndarray):
    """fp16 [r, d] -> (H, L, |.|^2 parts): a * 2^24 = H 2^20 + L exactly (integers, |H| <= 2^20, 0 <= L < 2^20), and
    per row sum H^2, 2 sum H L, sum L^2 (exact: every partial sum is an integer below 2^53 for d <= 2048)"""
    n = a.astype(np.float64) * 2.0 ** 24
    h = np.floor(n / 2.0 ** 20)
    lo = n - h * 2.0 ** 20
    return h, lo, ((h * h).sum(1), 2.0 * (h * lo).sum(1), (lo * lo).sum(1))


def _blocks(a: np.ndarray, b: np.ndarray, block: int = BLOCK):
    """(i0, i1, q) for row blocks of a against all of b: q fp64 [i1 - i0, len(b)] = |a_i - b_j|^2.  The three integer
    parts of 2^48 q are exact (fp64 GEMMs of integers whose sums stay below 2^53), and q is a fixed rounding of them:
    a function of the two rows alone, so equal real distances (duplicates, an eval row equal to a baseline row) give
    equal q, and q = 0 exactly for equal rows."""
    ha, la, (n1a, n2a, n3a) = _parts(a)
    hb, lb, (n1b, n2b, n3b) = _parts(b)
    for i0 in range(0, a.shape[0], block):
        i1 = min(a.shape[0], i0 + block)
        h, lo = ha[i0:i1], la[i0:i1]
        t1 = n1a[i0:i1, None] + n1b[None, :] - 2.0 * (h @ hb.T)
        t2 = n2a[i0:i1, None] + n2b[None, :] - 2.0 * (h @ lb.T + lo @ hb.T)
        t3 = n3a[i0:i1, None] + n3b[None, :] - 2.0 * (lo @ lb.T)
        yield i0, i1, (t1 * 2.0 ** 40 + t2 * 2.0 ** 20 + t3) * 2.0 ** -48


def _kth_other(q: np.ndarray, i0: int, k: int) -> np.ndarray:
    """per row r of the block (row i0 + r of the set): the k-th smallest q over the other rows (self excluded by index)"""
    q = q.copy()
    r = np.arange(q.shape[0])
    q[r, i0 + r] = np.inf
    return np.partition(q, k - 1, axis=1)[:, k - 1]


def radii_sq(x: np.ndarray, y: np.ndarray, k: int) -> np.ndarray:
    """fp64 [m + n]: r_i^2 (k-th nearest other row of X), then s_j^2 (within Y)"""
    out = []
    for a in (x, y):
        for i0, _, q in _blocks(a, a):
            out.append(_kth_other(q, i0, k))
    return np.concatenate(out)


def counts(x: np.ndarray, y: np.ndarray, radii: np.ndarray):
    """radii fp64 [m + n] (r^2 then s^2) -> (inside int64 [n], flags uint8 [m]) with exact strict comparisons"""
    (lo_in, _), (lo_cov, _), (lo_rec, _) = _bounds(x, y, radii, 0.0)
    return lo_in, (lo_cov.astype(np.uint8) | (lo_rec.astype(np.uint8) << 1))


def metrics(inside: np.ndarray, flags: np.ndarray, k: int) -> tuple[float, float, float, float]:
    """(precision, recall, density, coverage) from the counts"""
    n, m = inside.shape[0], flags.shape[0]
    return (np.count_nonzero(inside) / n, np.count_nonzero(flags & 2) / m, float(inside.sum()) / (k * n),
            np.count_nonzero(flags & 1) / m)


def prdc(x: np.ndarray, y: np.ndarray, k: int = 5) -> tuple[float, float, float, float]:
    """(precision, recall, density, coverage) by the block oracle"""
    return metrics(*counts(x, y, radii_sq(x, y, k)), k)


def prdc_direct(x: np.ndarray, y: np.ndarray, k: int = 5):
    """The definition as a plain double loop on differences -> (radii [m + n], inside, flags, (p, r, d, c))"""
    x, y = x.astype(np.float64), y.astype(np.float64)
    m, n = x.shape[0], y.shape[0]
    q = lambda a, b: float(((a - b) ** 2).sum())  # noqa: E731
    r2 = [sorted(q(x[i], x[j]) for j in range(m) if j != i)[k - 1] for i in range(m)]
    s2 = [sorted(q(y[i], y[j]) for j in range(n) if j != i)[k - 1] for i in range(n)]
    inside = np.array([sum(q(x[i], y[j]) < r2[i] for i in range(m)) for j in range(n)], dtype=np.int64)
    cov = [any(q(x[i], y[j]) < r2[i] for j in range(n)) for i in range(m)]
    rec = [any(q(x[i], y[j]) < s2[j] for j in range(n)) for i in range(m)]
    flags = np.array([int(c) | (int(r) << 1) for c, r in zip(cov, rec)], dtype=np.uint8)
    return np.array(r2 + s2), inside, flags, metrics(inside, flags, k)


def _shifted_norms(x: np.ndarray, y: np.ndarray):
    """|z - s|^2 per row (fp64), s = the fp16-rounded mean of X (the GPU's shift)"""
    s = x.astype(np.float64).mean(0).astype(np.float16).astype(np.float64)
    return (((x.astype(np.float64) - s) ** 2).sum(1), ((y.astype(np.float64) - s) ** 2).sum(1))


def _bounds(x, y, radii, tau):
    m = x.shape[0]
    r2, s2 = np.asarray(radii[:m], np.float64), np.asarray(radii[m:], np.float64)
    nx, ny = _shifted_norms(x, y)
    n = y.shape[0]
    in_lo, in_hi = np.zeros(n, np.int64), np.zeros(n, np.int64)
    cov_lo, cov_hi = np.zeros(m, bool), np.zeros(m, bool)
    rec_lo, rec_hi = np.zeros(m, bool), np.zeros(m, bool)
    for i0, i1, q in _blocks(x, y):
        delta = tau * (nx[i0:i1, None] + ny[None, :])
        ball_r, ball_s = r2[i0:i1, None], s2[None, :]
        r_lo = q < ball_r - delta
        r_hi = (q < ball_r) | ((delta > 0) & (q <= ball_r + delta))
        s_lo = q < ball_s - delta
        s_hi = (q < ball_s) | ((delta > 0) & (q <= ball_s + delta))
        in_lo += r_lo.sum(0)
        in_hi += r_hi.sum(0)
        cov_lo[i0:i1], cov_hi[i0:i1] = r_lo.any(1), r_hi.any(1)
        rec_lo[i0:i1], rec_hi[i0:i1] = s_lo.any(1), s_hi.any(1)
    return (in_lo, in_hi), (cov_lo, cov_hi), (rec_lo, rec_hi)


def decision_bounds(x: np.ndarray, y: np.ndarray, radii: np.ndarray, tau: float = TAU) -> dict:
    """For thresholds radii [m + n] (r^2 then s^2, e.g. the GPU's fp32 values): every ambiguous decision (|q - thr| <=
    delta_ab = tau (|y^_a|^2 + |y^_b|^2), module docstring) taken false, and taken true.  -> {"inside": (lo, hi) int64
    [n], "covered": (lo, hi) bool [m], "recalled": (lo, hi) bool [m]}; lo <= hi, and lo == hi wherever no decision of
    that output is ambiguous."""
    inside, covered, recalled = _bounds(x, y, radii, tau)
    return {"inside": inside, "covered": covered, "recalled": recalled}


def radii_bounds(x: np.ndarray, y: np.ndarray, k: int, tau: float = TAU):
    """(lo, hi) fp64 [m + n]: per row the k-th smallest of q - delta and of q + delta over the other rows of its set, the
    range any q^ with |q^ - q| <= delta puts the k-th smallest in"""
    nx, ny = _shifted_norms(x, y)
    lo, hi = [], []
    for a, na in ((x, nx), (y, ny)):
        for i0, i1, q in _blocks(a, a):
            delta = tau * (na[i0:i1, None] + na[None, :])
            lo.append(_kth_other(q - delta, i0, k))
            hi.append(_kth_other(q + delta, i0, k))
    return np.concatenate(lo), np.concatenate(hi)
