"""The nearest-groups block oracle (oracle/nearest_oracle.py) against the definition written as a double loop
(nearest_direct), on small sets that reach every rule: one-row groups, groups of several rows, empty groups, fewer
non-empty groups than k, equidistant rows and duplicate rows; and nearest_bounds accepting the oracle's own lists."""
import numpy as np
import pytest

from oracle import nearest_oracle as no


def _rows(m, d, seed, offset=0.0):
    return (offset + np.random.default_rng(seed).standard_normal((m, d))).astype(np.float16)


def _agree(x, y, k, offsets=None):
    rows, q = no.nearest(x, y, k, offsets)
    drows, dq = no.nearest_direct(x, y, k, offsets)
    assert np.array_equal(rows, drows)
    assert np.array_equal(np.isinf(q), np.isinf(dq))
    assert np.allclose(q[np.isfinite(q)], dq[np.isfinite(dq)], rtol=1e-14, atol=0)
    return rows, q


@pytest.mark.parametrize("m,n,k,offsets", [(9, 7, 3, None), (1, 4, 1, None), (5, 3, 16, None),
                                           (12, 6, 2, [0, 4, 4, 9, 12]), (20, 5, 16, [0, 10, 20]),
                                           (7, 4, 3, [0, 0, 7, 7]), (30, 9, 5, list(range(0, 31, 3)))])
def test_block_oracle_is_the_definition(m, n, k, offsets):
    x, y = _rows(m, 12, m), _rows(n, 12, 100 + n, 0.2)
    rows, q = _agree(x, y, k, offsets)
    gid = no.groups_of(m, offsets)
    live = rows >= 0
    groups = len(set(gid.tolist()))
    assert (live.sum(1) == min(k, groups)).all() and np.isinf(q[~live]).all()
    for j in range(n):                                     # distinct groups, ascending, each at its group's minimum
        r = rows[j][live[j]]
        assert len(set(gid[r].tolist())) == r.size and (np.diff(q[j][live[j]]) >= 0).all()


def test_equidistant_rows_go_to_the_smallest_index_and_groups_to_their_first_row():
    x = np.zeros((6, 8), np.float16)
    x[:, 0] = [5.0, 1.0, -1.0, 1.0, 9.0, -1.0]            # rows 1, 2, 3, 5 at distance 1 from the origin
    y = np.zeros((1, 8), np.float16)
    rows, q = _agree(x, y, 3)
    assert rows[0].tolist() == [1, 2, 3] and q[0].tolist() == [1.0, 1.0, 1.0]
    rows, q = _agree(x, y, 3, [0, 2, 4, 6])               # groups {0, 1}, {2, 3}, {4, 5}
    assert rows[0].tolist() == [1, 2, 5] and q[0].tolist() == [1.0, 1.0, 1.0]


def test_duplicates_are_one_group_per_group():
    """a baseline file of repeated frames counts once; the next file is the second group"""
    x = np.concatenate([np.repeat(_rows(1, 8, 1), 5, 0), _rows(4, 8, 2, 3.0)])
    y = x[:1].copy()
    rows, q = _agree(x, y, 4, [0, 5, 9])
    assert rows[0, 0] == 0 and q[0, 0] == 0.0 and 5 <= rows[0, 1] < 9 and (rows[0, 2:] == -1).all()


def test_bounds_accept_the_oracles_own_lists():
    x, y = _rows(300, 16, 2), _rows(40, 16, 3, 0.1)
    y[4] = x[9]
    off = [0, 7, 7, 50, 120, 121, 300]
    for offsets in (None, off):
        for k in (1, 5, 16):
            rows, q = no.nearest(x, y, k, offsets)
            for tau in (0.0, no.TAU):
                b = no.nearest_bounds(x, y, rows, q, k, offsets, tau=tau)
                for key in ("rows", "order", "missing", "equal"):
                    assert b[key].all(), (offsets is None, k, tau, key)
                if tau == 0.0:
                    assert b["clear"].all()
    rows, q = no.nearest(x, y, 3, off)
    bad = rows.copy()
    bad[:, [0, 1]] = bad[:, [1, 0]]                       # out of order
    assert not no.nearest_bounds(x, y, bad, q[:, [1, 0, 2]], 3, off)["order"].all()
    far = rows.copy()
    far[:, 0] = rows[:, 2]                                # a repeated group
    assert not no.nearest_bounds(x, y, far, q, 3, off)["order"].all()
