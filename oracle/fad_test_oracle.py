"""numpy fp64 restatement of the permutation test of the FAD difference (fadtk_b200.fad.calc_fad_comparison).

Test infrastructure only.  Units are files; a unit record is [n | sum y | upper triangle of sum y y^T] with y = x - s
(csrc/stats.cuh), here in fp64 from the fp16 rows.  The labels are kad_test_oracle.labels over units, and the Frechet
distance is fad_oracle's arithmetic (the reference's eigen-decomposition route).
"""
from __future__ import annotations

import numpy as np

from . import fad_oracle as fo
from .kad_test_oracle import labels


def record_len(d: int) -> int:
    return 1 + d + d * (d + 1) // 2


def records(units: list, shift: np.ndarray) -> np.ndarray:
    """fp64 [F, R(d)]: the record of each unit (fp16 [rows, d] arrays) about the shift (fp16 [d])"""
    d = shift.shape[0]
    iu = np.triu_indices(d)
    out = np.empty((len(units), record_len(d)))
    for u, rows in enumerate(units):
        y = rows.astype(np.float64) - shift.astype(np.float64)
        out[u, 0] = rows.shape[0]
        out[u, 1:1 + d] = y.sum(0)
        out[u, 1 + d:] = (y.T @ y)[iu]
    return out


def statistics(rec: np.ndarray, shift: np.ndarray):
    """(n, mu [d], cov [d, d]) of one (summed) record: the exact fp64 mean and the ddof = 1 covariance"""
    d = shift.shape[0]
    n = rec[0]
    sy = rec[1:1 + d]
    upper = np.zeros((d, d))
    upper[np.triu_indices(d)] = rec[1 + d:]
    g = upper + np.triu(upper, 1).T
    return n, shift.astype(np.float64) + sy / n, (g - np.outer(sy, sy) / n) / (n - 1.0)


def union_statistics(units: list):
    """(mu, cov) of the concatenated rows, straight from the rows (the check of the record path)"""
    rows = np.concatenate(units).astype(np.float64)
    return rows.mean(0), np.cov(rows, rowvar=False)


def labelled_sums(rec: np.ndarray, lab: np.ndarray) -> np.ndarray:
    """fp64 [L, 2, R]: per labelling the sum of the records of the marked units and of the others"""
    w = lab.astype(np.float64)
    return np.stack([w @ rec, (1.0 - w) @ rec], axis=1)


def pool_shift(units: list) -> np.ndarray:
    """fp16 mean of all rows of the pool (the device's pair_shift_kernel)"""
    return np.concatenate(units).astype(np.float64).mean(0).astype(np.float16)


def p_value(diff: np.ndarray) -> float:
    """two-sided: (1 + #{b >= 1 : |D_b| >= |D_0|}) / (B + 1)"""
    return (1.0 + float(np.count_nonzero(np.abs(diff[1:]) >= abs(diff[0])))) / diff.shape[0]


def comparison(mu_x, cov_x, units_a: list, units_b: list, permutations: int, seed: int, shift=None) -> dict:
    """Every labelling of the pool units_a + units_b: FAD of both sides, the differences and the two-sided p-value"""
    units = list(units_a) + list(units_b)
    shift = pool_shift(units) if shift is None else shift
    lab = labels(len(units), len(units_a), permutations, seed)
    sums = labelled_sums(records(units, shift), lab)
    fad = np.empty((permutations + 1, 2))
    trace = np.empty((permutations + 1, 2))
    for b in range(permutations + 1):
        for side in range(2):
            _, mu, cov = statistics(sums[b, side], shift)
            fad[b, side] = fo.frechet_distance(np.asarray(mu_x, np.float64), cov_x, mu, cov)
            trace[b, side] = np.trace(cov)
    diff = fad[:, 0] - fad[:, 1]
    return {"labels": lab, "sums": sums, "shift": shift, "fad": fad, "trace": trace, "stats": diff,
            "p_value": p_value(diff)}
