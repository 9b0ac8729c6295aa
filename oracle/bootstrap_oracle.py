"""numpy fp64 restatement of the bootstrap confidence intervals of FAD and KAD (fadtk_b200.fad.calc_fad_bootstrap,
calc_kad_bootstrap).

Test infrastructure only.  The draw rule is restated in wrapping uint64 arithmetic, so the multiplicities are compared
bit for bit.  FAD: the multiplicity-weighted sums of fad_test_oracle's unit records, finalised by its statistics() and
scored by fad_oracle's Frechet distance.  KAD: exact fp64 kernel values (kad_test_oracle.kernel_matrix); the GPU rounds
each one to fp16 once, and error_scale() gives the expected size of what that does to S_yy(b).  Meant for eval sets of
up to a few thousand rows (the kernel matrix is held whole).
"""
from __future__ import annotations

import numpy as np

from . import fad_oracle as fo
from .fad_test_oracle import records, statistics
from .kad_test_oracle import kernel_matrix, mix64

_M32 = np.uint64(0xFFFFFFFF)


def draws(n_units: int, resamples: int, seed: int) -> np.ndarray:
    """int64 [B + 1, F]: the unit picked by draw t of resample b, floor(mix64(mix64(seed + b) ^ t) F / 2^64), the high
    word of the 128-bit product (row 0: every unit once, in order)"""
    F = n_units
    out = np.empty((resamples + 1, F), dtype=np.int64)
    out[0] = np.arange(F)
    t = np.arange(F, dtype=np.uint64)
    f = np.uint64(F)
    with np.errstate(over="ignore"):
        for b in range(1, resamples + 1):
            key = mix64(mix64(np.uint64((seed + b) & 0xFFFFFFFFFFFFFFFF)) ^ t)
            hi, lo = key >> np.uint64(32), key & _M32
            out[b] = ((hi * f + ((lo * f) >> np.uint64(32))) >> np.uint64(32)).astype(np.int64)
    return out


def counts(n_units: int, resamples: int, seed: int) -> np.ndarray:
    """int64 [B + 1, F]: the multiplicity of each unit in each resample"""
    dr = draws(n_units, resamples, seed)
    return np.stack([np.bincount(row, minlength=n_units) for row in dr])


def materialise(units: list, w: np.ndarray) -> np.ndarray:
    """the rows of one resample: unit u's rows w[u] times, units in order"""
    return np.concatenate([np.concatenate([units[u]] * int(w[u])) for u in range(len(units)) if w[u] > 0])


def weighted_sums(rec: np.ndarray, cnt: np.ndarray) -> np.ndarray:
    """fp64 [B + 1, R]: per resample the multiplicity-weighted sum of the unit records"""
    return cnt.astype(np.float64) @ rec


def fad(mu_x, cov_x, units: list, resamples: int, seed: int, shift: np.ndarray) -> dict:
    """Every resample of the units: counts, weighted record sums, (n, mu, cov) and the FAD against (mu_x, cov_x)"""
    cnt = counts(len(units), resamples, seed)
    sums = weighted_sums(records(units, shift), cnt)
    out = np.empty(resamples + 1)
    stats = []
    for b in range(resamples + 1):
        st = statistics(sums[b], shift)
        stats.append(st)
        out[b] = fo.frechet_distance(np.asarray(mu_x, np.float64), cov_x, st[1], st[2])
    return {"counts": cnt, "sums": sums, "stats": stats, "fad": out}


def unit_rows(units: list) -> np.ndarray:
    """int64 [n]: the unit of each row"""
    return np.repeat(np.arange(len(units)), [u.shape[0] for u in units])


def kad_sums(k_yy: np.ndarray, sizes: np.ndarray, cnt: np.ndarray, g_units: np.ndarray) -> np.ndarray:
    """fp64 [B + 1, 3] = (n_b, S_yy(b), S_xy(b)); k_yy the zero-diagonal kernel matrix of the eval rows, sizes the rows
    of each unit, g_units per unit the kernel sum against the baseline rows"""
    v = np.repeat(cnt.astype(np.float64), sizes, axis=1)
    w = cnt.astype(np.float64)
    quad = 0.5 * np.einsum("bi,ij,bj->b", v, k_yy, v)
    self_pairs = (w * (w - 1.0) * 0.5) @ sizes.astype(np.float64)
    return np.stack([w @ sizes.astype(np.float64), quad + self_pairs, w @ g_units], axis=1)


def error_scale(k_yy: np.ndarray, sizes: np.ndarray, cnt: np.ndarray) -> np.ndarray:
    """e_b of S_yy(b): 2^-11 sqrt(sum_{i<j} (v_i v_j)^2 K_ij^2) (the fp16 rounding of every kernel value) plus
    2^-20 sum_{i<j} v_i v_j K_ij (the fp32 terms)"""
    v = np.repeat(cnt.astype(np.float64), sizes, axis=1)
    sq = 0.5 * np.einsum("bi,ij,bj->b", v * v, k_yy * k_yy, v * v)
    lin = 0.5 * np.einsum("bi,ij,bj->b", v, k_yy, v)
    return 2.0 ** -11 * np.sqrt(sq) + 2.0 ** -20 * lin


def kad(x: np.ndarray, units: list, sigma: float, resamples: int, seed: int, s_xx=None) -> dict:
    """Every resample of the units against the fixed x: sums, KAD replicates and the error scale of S_yy"""
    m = x.shape[0]
    y = np.concatenate(units)
    sizes = np.array([u.shape[0] for u in units], dtype=np.int64)
    kall = kernel_matrix(np.concatenate([x, y]), sigma)
    g = kall[:m, m:].sum(0)
    g_units = np.add.reduceat(g, np.concatenate([[0], np.cumsum(sizes)[:-1]]))
    s_xx = 0.5 * kall[:m, :m].sum() if s_xx is None else s_xx
    cnt = counts(len(units), resamples, seed)
    s = kad_sums(kall[m:, m:], sizes, cnt, g_units)
    return {"counts": cnt, "sums": s, "g_units": g_units, "s_xx": s_xx, "kad": statistic(s_xx, s, m),
            "err": error_scale(kall[m:, m:], sizes, cnt)}


def statistic(s_xx: float, s: np.ndarray, m: int) -> np.ndarray:
    """KAD_b = 1000 (2 S_xx / (m (m - 1)) + 2 S_yy(b) / (n_b (n_b - 1)) - 2 S_xy(b) / (m n_b))"""
    n = s[:, 0]
    return 1000.0 * (2.0 * s_xx / (m * (m - 1.0)) + 2.0 * s[:, 1] / (n * (n - 1.0)) - 2.0 * s[:, 2] / (float(m) * n))


def interval(theta: np.ndarray, level: float, method: str):
    """(ci_low, ci_high, standard_error, bias) of the replicates theta[1:] about the observed theta[0]"""
    rep, obs = theta[1:], theta[0]
    q_lo, q_hi = np.quantile(rep, [(1.0 - level) / 2.0, (1.0 + level) / 2.0])
    lo, hi = (q_lo, q_hi) if method == "percentile" else (2.0 * obs - q_hi, 2.0 * obs - q_lo)
    return float(lo), float(hi), float(np.std(rep, ddof=1)), float(np.mean(rep) - obs)
