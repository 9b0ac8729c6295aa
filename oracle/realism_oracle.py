"""numpy fp64 restatement of the per-sample realism and nearest-baseline-row definition (fadtk_b200.fad.calc_realism).

Test infrastructure only.  The fp16 rows are taken as exact reals, and q comes from prdc_oracle._blocks: exact integer
parts rounded once, a function of the two rows alone, so equal real distances give equal q and equal rows give q = 0.
The radii are prdc_oracle's k-th smallest other-row distances, the threshold is numpy.median of them in fp64.
realism_direct is the definition written as a plain double loop on differences: the oracle's own check.

realism_bounds brackets what the GPU can return from its own pruned radii r~^2 (fp32, exact inputs) when its q^ lies
within delta = tau (|y^_a|^2 + |y^_b|^2) of the exact q (prdc_oracle's module docstring):
  * realism^2 in [max r~^2 / (q + delta), max r~^2 / max(q - delta, 0)] over the rows with r~^2 > 0 (+inf at the upper
    end where q - delta <= 0: the flush of a small q^ to 0 gives +inf), widened by one fp32 rounding each for the
    quotient and the square root;
  * the nearest index is one of {i : q_i - delta_i <= min_l (q_l + delta_l)}, and its nearest_sq lies within delta_i of
    its exact q_i.
"""
from __future__ import annotations

import numpy as np

from . import prdc_oracle as po

TAU = po.TAU
U32 = 2.0 ** -24          # fp32 unit roundoff


def x_radii_sq(x: np.ndarray, k: int) -> np.ndarray:
    """fp64 [m]: r_i^2, the k-th smallest q from x_i to the other rows of X"""
    return np.concatenate([po._kth_other(q, i0, k) for i0, _, q in po._blocks(x, x)])


def threshold(radii_sq: np.ndarray) -> float:
    """T = numpy.median of the radii in fp64"""
    return float(np.median(np.asarray(radii_sq, dtype=np.float64)))


def pruned(radii_sq: np.ndarray, t: float) -> np.ndarray:
    """r~^2 = r^2 where r^2 <= T, else 0"""
    r = np.asarray(radii_sq, dtype=np.float64)
    return np.where(r <= t, r, 0.0)


def _ratio(kept: np.ndarray, q: np.ndarray) -> np.ndarray:
    """kept[:, None] / q where kept > 0 (+inf where q = 0), 0 where kept = 0"""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(kept[:, None] > 0, kept[:, None] / q, 0.0)


def realism(x: np.ndarray, y: np.ndarray, k: int = 3):
    """-> (kept fp64 [m], realism fp64 [n], nearest int64 [n], nearest_sq fp64 [n], T) by the block oracle"""
    kept_all = x_radii_sq(x, k)
    t = threshold(kept_all)
    kept = pruned(kept_all, t)
    n = y.shape[0]
    best = np.zeros(n)
    nq, ni = np.full(n, np.inf), np.full(n, -1, np.int64)
    for i0, i1, q in po._blocks(x, y):
        best = np.maximum(best, _ratio(kept[i0:i1], q).max(0))
        a = q.argmin(0)                                   # first minimum: the smallest index in the block
        qa = q[a, np.arange(n)]
        better = qa < nq                                  # strict: an earlier block keeps a tie
        nq[better], ni[better] = qa[better], i0 + a[better]
    return kept, np.sqrt(best), ni, nq, t


def realism_direct(x: np.ndarray, y: np.ndarray, k: int = 3):
    """The definition as a plain double loop on differences -> (kept, realism, nearest, nearest_sq, T)"""
    x, y = x.astype(np.float64), y.astype(np.float64)
    m, n = x.shape[0], y.shape[0]
    q = lambda a, b: float(((a - b) ** 2).sum())  # noqa: E731
    r2 = [sorted(q(x[i], x[j]) for j in range(m) if j != i)[k - 1] for i in range(m)]
    t = float(np.median(np.array(r2, dtype=np.float64)))
    kept = [r if r <= t else 0.0 for r in r2]
    real, near, near_sq = [], [], []
    for j in range(n):
        d = [q(x[i], y[j]) for i in range(m)]
        vals = [kept[i] / d[i] if d[i] > 0 else np.inf for i in range(m) if kept[i] > 0]
        real.append(np.sqrt(max(vals)) if vals else 0.0)
        i_min = min(range(m), key=lambda i: (d[i], i))
        near.append(i_min)
        near_sq.append(d[i_min])
    return np.array(kept), np.array(real), np.array(near, dtype=np.int64), np.array(near_sq), t


def realism_bounds(x: np.ndarray, y: np.ndarray, kept_radii_sq: np.ndarray, nearest: np.ndarray | None = None,
                   tau: float = TAU) -> dict:
    """From the GPU's pruned radii kept_radii_sq [m] -> per eval row {"lo", "hi": the realism bracket, "bound":
    min_l (q_l + delta_l), "count": the number of nearest candidates, "only": the candidate when there is one, else -1};
    with the GPU's nearest [n] also {"cand": nearest_j is a candidate, "q", "delta": the exact q and delta of the pair
    (nearest_j, j)}."""
    kept = np.asarray(kept_radii_sq, dtype=np.float64)
    nx, ny = po._shifted_norms(x, y)
    n = y.shape[0]
    lo2, hi2, bound = np.zeros(n), np.zeros(n), np.full(n, np.inf)
    for i0, i1, q in po._blocks(x, y):
        delta = tau * (nx[i0:i1, None] + ny[None, :])
        lo2 = np.maximum(lo2, _ratio(kept[i0:i1], q + delta).max(0))
        hi2 = np.maximum(hi2, _ratio(kept[i0:i1], np.maximum(q - delta, 0.0)).max(0))
        bound = np.minimum(bound, (q + delta).min(0))
    count, only = np.zeros(n, np.int64), np.full(n, -1, np.int64)
    out = {}
    if nearest is not None:
        nearest = np.asarray(nearest, dtype=np.int64)
        out = {"q": np.full(n, np.nan), "delta": np.full(n, np.nan)}
    for i0, i1, q in po._blocks(x, y):
        delta = tau * (nx[i0:i1, None] + ny[None, :])
        c = q - delta <= bound[None, :]
        count += c.sum(0)
        only = np.where(c.any(0), i0 + c.argmax(0), only)
        if nearest is not None:
            j = np.flatnonzero((nearest >= i0) & (nearest < i1))
            out["q"][j] = q[nearest[j] - i0, j]
            out["delta"][j] = delta[nearest[j] - i0, j]
    only[count != 1] = -1
    out.update(lo=np.sqrt(lo2 * (1 - U32)) * (1 - U32), hi=np.sqrt(hi2 * (1 + U32)) * (1 + U32), bound=bound,
               count=count, only=only)
    if nearest is not None:
        out["cand"] = out["q"] - out["delta"] <= bound
    return out
