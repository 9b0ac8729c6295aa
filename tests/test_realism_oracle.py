"""The realism block oracle (oracle/realism_oracle.py) against the definition written as a double loop
(realism_direct), on small sets that reach every rule: the median for odd and even m, duplicate rows, an eval row equal
to a kept baseline row, an eval row inside only a pruned ball, and equidistant baseline rows."""
import numpy as np
import pytest

from oracle import realism_oracle as ro


def _rows(m, d, seed, offset=0.0):
    return (offset + np.random.default_rng(seed).standard_normal((m, d))).astype(np.float16)


def _agree(x, y, k):
    kept, real, near, near_sq, t = ro.realism(x, y, k)
    dk, dr, dn, dq, dt = ro.realism_direct(x, y, k)
    assert t == dt
    assert np.array_equal(kept, dk)
    assert np.array_equal(near, dn)
    assert np.allclose(near_sq, dq, rtol=1e-14, atol=0)
    assert np.array_equal(np.isinf(real), np.isinf(dr))
    assert np.allclose(real[np.isfinite(real)], dr[np.isfinite(dr)], rtol=1e-14, atol=0)
    return kept, real, near, near_sq, t


@pytest.mark.parametrize("m,n,k", [(9, 7, 3), (10, 7, 3), (4, 1, 3), (17, 12, 1), (20, 5, 16)])
def test_block_oracle_is_the_definition(m, n, k):
    x, y = _rows(m, 12, m), _rows(n, 12, 100 + n, 0.2)
    kept, real, _, _, t = _agree(x, y, k)
    r = ro.x_radii_sq(x, k)
    s = np.sort(r)
    assert t == (s[m // 2] if m % 2 else (s[m // 2 - 1] + s[m // 2]) / 2)
    assert np.array_equal(kept, np.where(r <= t, r, 0.0))
    assert (kept > 0).sum() >= (m + 1) // 2 - (r == 0).sum()


def test_even_median_is_the_fp64_mean():
    """two middle radii whose fp32 mean rounds: T is the fp64 value, as numpy.median of the float64 radii"""
    x = np.zeros((4, 8), np.float16)
    x[1, 0], x[2, 0], x[3, 0] = 2.0 ** -13, 5.0, 6.0      # radii 2^-26, 2^-26, 1, 1
    r = ro.x_radii_sq(x, 1)
    t = ro.threshold(r)
    s = np.sort(r)
    assert t == (s[1] + s[2]) / 2 and t != float(np.float32((np.float32(s[1]) + np.float32(s[2])) / np.float32(2)))


def test_duplicates_copy_and_pruned_ball():
    """k exact copies of a baseline row give r = 0 (kept, contributing nothing); an eval row equal to a kept baseline
    row has realism +inf and nearest_sq 0; an eval row inside only a pruned (large) ball has realism < 1"""
    k, d = 3, 8
    rng = np.random.default_rng(4)
    x = (rng.standard_normal((21, d)) * 0.1).astype(np.float16)
    x[:4] = x[0]                                          # four copies: each has 3 neighbours at 0
    x[20] = 40.0                                          # far away: the largest radius, pruned
    r = ro.x_radii_sq(x, k)
    c = int(np.flatnonzero((r > 0) & (r <= ro.threshold(r)))[0])
    y = np.zeros((3, d), np.float16)
    y[0] = x[c]
    y[1] = 40.0
    y[1, 0] = 41.0                                        # distance 1 from x[20], far from the rest
    y[2] = (rng.standard_normal(d) * 0.1).astype(np.float16)
    kept, real, near, near_sq, t = _agree(x, y, k)
    assert (kept[:4] == 0).all() and kept[20] == 0 and kept[c] > 0
    assert np.isinf(real[0]) and near[0] == c and near_sq[0] == 0.0
    assert near[1] == 20 and near_sq[1] < r[20] and real[1] < 1.0
    assert np.isfinite(real[2])


def test_equidistant_baseline_rows_go_to_the_smallest_index():
    x = np.zeros((6, 8), np.float16)
    x[:, 0] = [5.0, 1.0, -1.0, 1.0, 9.0, -1.0]           # rows 1, 2, 3, 5 at distance 1 from the origin
    y = np.zeros((1, 8), np.float16)
    _, _, near, near_sq, _ = _agree(x, y, 1)
    assert near[0] == 1 and near_sq[0] == 1.0


def test_every_radius_zero_gives_realism_zero_and_bounds_hold():
    """all kept radii 0: realism is 0; the bounds built with tau = 0 from the oracle's own radii are its exact values"""
    x = np.zeros((5, 8), np.float16)
    y = _rows(3, 8, 1)
    kept, real, near, near_sq, t = _agree(x, y, 2)
    assert t == 0.0 and not real.any()
    x, y = _rows(40, 16, 2), _rows(30, 16, 3, 0.1)
    y[4] = x[9]
    kept, real, near, near_sq, t = ro.realism(x, y, 3)
    b = ro.realism_bounds(x, y, kept, near, tau=0.0)
    assert ((b["lo"] <= real) & (real <= b["hi"])).all()
    assert b["cand"].all() and np.array_equal(b["q"], near_sq)
    assert np.array_equal(b["only"][b["count"] == 1], near[b["count"] == 1])
    b = ro.realism_bounds(x, y, kept, near)
    assert ((b["lo"] <= real) & (real <= b["hi"])).all() and b["cand"].all()
