"""numpy fp64 restatement of the k nearest distinct baseline groups (fadtk_b200.fad.calc_nearest, fad_nearest).

Test infrastructure only.  The fp16 rows are taken as exact reals, and q comes from prdc_oracle._blocks: exact integer
parts rounded once, a function of the two rows alone, so equal real distances give equal q and equal rows give q = 0.
For eval row y_j the baseline rows are ordered by the key (q(x_i, y_j), i); each group (a contiguous row range given by
offsets; every row its own group without them) is represented by its smallest key, and the k groups with the smallest
representative keys are the result, ascending, each as (row, q); -1 / +inf fill the slots past the last non-empty
group.  nearest_direct is the definition written as a plain double loop on differences: the oracle's own check.

nearest_bounds checks what the GPU returns when its q^ lies within delta = tau (|y^_a|^2 + |y^_b|^2) of the exact q
(prdc_oracle's module docstring).  With L_g = min_{i in g} (q_i - delta_i) and U_g = min_{i in g} (q_i + delta_i), the
interval the GPU's representative q of group g lies in:
  * every returned row lies in its group, its q^ within delta of the exact q, and it is a candidate for the group's
    minimum (q_i - delta_i <= U_g);
  * the returned groups are distinct, their q^ ascending, and there are min(k, non-empty groups) of them;
  * no group left out is certainly closer than a returned one: U_h >= L_g for every left-out h and returned g;
  * where no comparison is ambiguous (each of the oracle's first k groups has one candidate row, and U of each of the
    first k groups lies below L of every group after it), the list equals the oracle's.
"""
from __future__ import annotations

import numpy as np

from . import prdc_oracle as po

TAU = po.TAU


def groups_of(m: int, offsets=None) -> np.ndarray:
    """int64 [m]: the group of each baseline row (every row its own group without offsets)"""
    if offsets is None:
        return np.arange(m, dtype=np.int64)
    off = np.asarray(offsets, dtype=np.int64)
    return np.searchsorted(off, np.arange(m), side="right") - 1


def _q(x: np.ndarray, y: np.ndarray) -> np.ndarray:
    """exact q [m, n] from prdc_oracle's blocks"""
    return np.concatenate([q for _, _, q in po._blocks(x, y)])


def _top(qj: np.ndarray, gid: np.ndarray, k: int):
    """one eval row's exact q [m] -> (rows [k], q [k]) of its k nearest groups"""
    order = np.lexsort((np.arange(qj.shape[0]), qj))
    _, first = np.unique(gid[order], return_index=True)
    pick = order[np.sort(first)[:k]]
    rows, qs = np.full(k, -1, np.int64), np.full(k, np.inf)
    rows[:pick.size], qs[:pick.size] = pick, qj[pick]
    return rows, qs


def nearest(x: np.ndarray, y: np.ndarray, k: int, offsets=None):
    """-> (rows int64 [n, k], q fp64 [n, k]) by the block oracle"""
    gid = groups_of(x.shape[0], offsets)
    q = _q(x, y)
    out = [_top(q[:, j], gid, k) for j in range(y.shape[0])]
    return np.array([o[0] for o in out]).reshape(-1, k), np.array([o[1] for o in out]).reshape(-1, k)


def nearest_direct(x: np.ndarray, y: np.ndarray, k: int, offsets=None):
    """The definition as a plain double loop on differences -> (rows, q)"""
    x, y = x.astype(np.float64), y.astype(np.float64)
    m, n = x.shape[0], y.shape[0]
    gid = groups_of(m, offsets)
    rows, qs = np.full((n, k), -1, np.int64), np.full((n, k), np.inf)
    for j in range(n):
        d = [float(((x[i] - y[j]) ** 2).sum()) for i in range(m)]
        best = {}
        for i in sorted(range(m), key=lambda i: (d[i], i)):
            best.setdefault(int(gid[i]), i)
        ranked = sorted(best.values(), key=lambda i: (d[i], i))[:k]
        for r, i in enumerate(ranked):
            rows[j, r], qs[j, r] = i, d[i]
    return rows, qs


def nearest_bounds(x: np.ndarray, y: np.ndarray, rows: np.ndarray, q_gpu: np.ndarray, k: int, offsets=None,
                   tau: float = TAU) -> dict:
    """Checks of the GPU's rows / q_gpu [n, k] (module docstring) -> per eval row booleans {"rows": every returned row
    is in range, within delta and a candidate for its group's minimum; "order": distinct groups, ascending q^, the
    right count, empty slots last; "missing": no left-out group certainly closer; "clear": no comparison ambiguous;
    "equal": the list equals the oracle's}, and the oracle's own lists ("want_rows", "want_q")."""
    m, n = x.shape[0], y.shape[0]
    rows = np.asarray(rows, dtype=np.int64)
    q_gpu = np.asarray(q_gpu, dtype=np.float64)
    gid = groups_of(m, offsets)
    q = _q(x, y)
    nx, ny = po._shifted_norms(x, y)
    delta = tau * (nx[:, None] + ny[None, :])
    starts = np.flatnonzero(np.r_[True, gid[1:] != gid[:-1]])       # the non-empty groups, in order
    ng = starts.size
    lo_g = np.minimum.reduceat(q - delta, starts, axis=0)          # [groups, n]
    hi_g = np.minimum.reduceat(q + delta, starts, axis=0)
    slot_of = np.full(int(gid[-1]) + 1, -1, np.int64)
    slot_of[gid[starts]] = np.arange(ng)
    want_rows, want_q = nearest(x, y, k, offsets)
    out = {key: np.ones(n, bool) for key in ("rows", "order", "missing", "clear", "equal")}
    for j in range(n):
        live = rows[j] >= 0
        r = rows[j][live]
        if not ((r < m).all() and np.array_equal(live, np.arange(k) < min(k, ng))):
            out["rows"][j] = out["order"][j] = False
            continue
        s = slot_of[gid[r]]
        out["rows"][j] = bool((np.abs(q_gpu[j][live] - q[r, j]) <= delta[r, j]).all() and
                              (q[r, j] - delta[r, j] <= hi_g[s, j]).all())
        out["order"][j] = bool(np.unique(s).size == s.size and (np.diff(q_gpu[j][live]) >= 0).all() and
                               np.isinf(q_gpu[j][~live]).all())
        left = np.setdiff1d(np.arange(ng), s)
        out["missing"][j] = bool(left.size == 0 or hi_g[left, j].min() >= lo_g[s, j].max())
        # the oracle's order of the groups: ambiguous if a first-k group has two candidate rows, or one of them may
        # swap with any group after it
        ws = slot_of[gid[want_rows[j][want_rows[j] >= 0]]]
        rest = np.ones(ng, bool)
        clear = True
        for t, g in enumerate(ws):
            rest[g] = False
            a, b = starts[g], starts[g + 1] if g + 1 < ng else m
            if ((q[a:b, j] - delta[a:b, j]) <= hi_g[g, j]).sum() != 1:
                clear = False
            if rest.any() and hi_g[g, j] >= lo_g[rest, j].min():
                clear = False
        out["clear"][j] = clear
        out["equal"][j] = bool(np.array_equal(rows[j], want_rows[j]))
    out.update(want_rows=want_rows, want_q=want_q)
    return out
