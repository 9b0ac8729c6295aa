"""numpy fp64 restatement of the permutation tests of KAD (fadtk_b200.fad.calc_kad_test, calc_kad_comparison).

Test infrastructure only.  The label rule is restated in uint64 arithmetic (wrapping, as the device computes it), so the
labels are compared bit for bit.  Kernel values are exact fp64 here; the GPU rounds each one to fp16 once, and
error_scale() gives the expected size of what that rounding does to each labelling's statistic.  Meant for pools of up
to a few thousand rows (the kernel matrix is held whole).
"""
from __future__ import annotations

import numpy as np

from .kad_oracle import _centred

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def mix64(x: np.ndarray) -> np.ndarray:
    """splitmix64's finaliser on uint64 (pair_mix64 in csrc/pair_tile.cuh), vectorised"""
    with np.errstate(over="ignore"):
        x = np.asarray(x, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def labels(n: int, a: int, permutations: int, seed: int) -> np.ndarray:
    """bool [B + 1, n]: labelling 0 marks rows 0 .. a - 1; labelling b marks the a rows with the smallest
    (mix64(mix64(seed + b) ^ i), i)"""
    out = np.zeros((permutations + 1, n), dtype=bool)
    out[0, :a] = True
    i = np.arange(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        for b in range(1, permutations + 1):
            base = mix64(np.uint64((seed + b) & 0xFFFFFFFFFFFFFFFF))
            keys = mix64(base ^ i)
            out[b, np.lexsort((i, keys))[:a]] = True
    return out


def pack_bits(lab: np.ndarray) -> np.ndarray:
    """bool [L, n] -> uint32 [L, 4 ceil(n / 128)]: bit i & 31 of word i >> 5 (fad_perm_labels' layout)"""
    L, n = lab.shape
    words = 4 * ((n + 127) // 128)
    padded = np.zeros((L, words * 32), dtype=np.uint64)
    padded[:, :n] = lab
    w = padded.reshape(L, words, 32) << np.arange(32, dtype=np.uint64)
    return w.sum(axis=2).astype(np.uint32)


def kernel_matrix(z: np.ndarray, sigma: float) -> np.ndarray:
    """K [n, n] fp64 with zero diagonal: exp(-|z_i - z_j|^2 / (2 sigma^2)) of the fp16 rows as exact reals"""
    (zc,) = _centred(z)
    nz = (zc * zc).sum(1)
    q = np.maximum(nz[:, None] + nz[None, :] - 2.0 * (zc @ zc.T), 0.0)
    k = np.exp(-q / (2.0 * sigma * sigma))
    np.fill_diagonal(k, 0.0)
    return k


def class_sums(k: np.ndarray, lab: np.ndarray) -> np.ndarray:
    """fp64 [L, 3]: (S_aa, S_bb, S_ab) of each labelling over the pairs i < j of the symmetric, zero-diagonal k"""
    w = lab.astype(np.float64)
    kw = w @ k
    total = 0.5 * k.sum()
    s_aa = 0.5 * np.einsum("bi,bi->b", kw, w)
    s_ab = np.einsum("bi,bi->b", kw, 1.0 - w)
    return np.stack([s_aa, total - s_aa - s_ab, s_ab], axis=1)


def _test_coefs(a: int, b: int):
    return 1000.0 * 2.0 / (a * (a - 1.0)), 1000.0 * 2.0 / (b * (b - 1.0)), -1000.0 * 2.0 / (float(a) * b)


def test_statistics(s: np.ndarray, a: int, b: int) -> np.ndarray:
    """KAD of each labelling from its sums (calc_kad_test's statistic)"""
    caa, cbb, cab = _test_coefs(a, b)
    return caa * s[:, 0] + cbb * s[:, 1] + cab * s[:, 2]


def comparison_statistics(s: np.ndarray, s_xa: np.ndarray, s_xb: np.ndarray, m: int, na: int, nb: int) -> np.ndarray:
    """KAD(X, A_l) - KAD(X, B_l) of each labelling (calc_kad_comparison's statistic)"""
    return 1000.0 * (2.0 * s[:, 0] / (na * (na - 1.0)) - 2.0 * s[:, 1] / (nb * (nb - 1.0))
                     - 2.0 * s_xa / (float(m) * na) + 2.0 * s_xb / (float(m) * nb))


def error_scale(k: np.ndarray, lab: np.ndarray, coefs) -> np.ndarray:
    """e_b per labelling: 2^-11 sqrt(sum coef_ij^2 K_ij^2), the size of the fp16 rounding of every kernel value, plus
    2^-20 sum |coef_ij| K_ij for the fp32 terms (q, ex2, the fp32 sums).  coefs = (c_aa, c_bb, c_ab)."""
    c = np.asarray(coefs, dtype=np.float64)
    sq = class_sums(k * k, lab)
    lin = class_sums(k, lab)
    return 2.0 ** -11 * np.sqrt(sq @ (c * c)) + 2.0 ** -20 * (lin @ np.abs(c))


def p_value(null: np.ndarray, observed: float) -> float:
    return (1.0 + float(np.count_nonzero(null >= observed))) / (null.shape[0] + 1.0)


def kad_test(x: np.ndarray, y: np.ndarray, sigma: float, permutations: int, seed: int) -> dict:
    """Every labelling of the pool [x; y]: sums, statistics, error scales, p-value"""
    m, n = x.shape[0], y.shape[0]
    k = kernel_matrix(np.concatenate([x, y]), sigma)
    lab = labels(m + n, m, permutations, seed)
    s = class_sums(k, lab)
    stats = test_statistics(s, m, n)
    return {"labels": lab, "sums": s, "stats": stats, "err": error_scale(k, lab, _test_coefs(m, n)),
            "p_value": p_value(stats[1:], stats[0])}


def kad_comparison(x: np.ndarray, ya: np.ndarray, yb: np.ndarray, sigma: float, permutations: int, seed: int) -> dict:
    """Every labelling of the pool [ya; yb] against the fixed x: sums, differences, error scales, two-sided p-value"""
    m, na, nb = x.shape[0], ya.shape[0], yb.shape[0]
    z = np.concatenate([x, ya, yb])
    kall = kernel_matrix(z, sigma)
    g = kall[:m, m:].sum(0)
    k = kall[m:, m:]
    lab = labels(na + nb, na, permutations, seed)
    s = class_sums(k, lab)
    s_xa = lab.astype(np.float64) @ g
    s_xb = g.sum() - s_xa
    diff = comparison_statistics(s, s_xa, s_xb, m, na, nb)
    coefs = (1000.0 * 2.0 / (na * (na - 1.0)), -1000.0 * 2.0 / (nb * (nb - 1.0)), 0.0)
    return {"labels": lab, "sums": s, "stats": diff, "err": error_scale(k, lab, coefs),
            "p_value": p_value(np.abs(diff[1:]), abs(float(diff[0])))}
