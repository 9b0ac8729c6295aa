"""The precision / recall / density / coverage oracle (oracle/prdc_oracle.py) without a GPU: the block oracle against
the definition written as a double loop (duplicates, k = 1 and k = 16 included), its radii against scikit-learn's
nearest neighbours, the X = Y identities, and decision_bounds at tau = 0."""
import numpy as np
import pytest

from oracle import prdc_oracle as po


def _rows(m, d, seed, offset=0.0, scale=1.0):
    return (offset + scale * np.random.default_rng(seed).standard_normal((m, d))).astype(np.float16)


def _with_duplicates(m, d, seed):
    """m rows of which a block repeats one row 6 times and one row appears twice"""
    x = _rows(m, d, seed, 3.0)
    x[1:7] = x[0]
    x[9] = x[8]
    return x


@pytest.mark.parametrize("k", [1, 3, 5, 16])
@pytest.mark.parametrize("dup", [False, True])
def test_block_oracle_equals_double_loop(k, dup):
    m, n, d = 40, 33, 12
    x = _with_duplicates(m, d, 1) if dup else _rows(m, d, 1, 3.0)
    y = _rows(n, d, 2, 3.2, 1.1)
    if dup:
        y[0] = x[0]                                    # an eval row on a duplicated baseline row (r = 0 when k <= 6)
        y[1] = x[20]                                   # and on an ordinary one
    r_d, in_d, fl_d, met_d = po.prdc_direct(x, y, k)
    r = po.radii_sq(x, y, k)
    assert np.allclose(r, r_d, rtol=1e-9, atol=0)
    if dup:
        assert (r[:7] == 0).all() == (k <= 6) and (r[8:10] == 0).all() == (k == 1)
    inside, flags = po.counts(x, y, r_d)
    assert np.array_equal(inside, in_d) and np.array_equal(flags, fl_d)
    assert np.allclose(po.prdc(x, y, k), met_d, rtol=1e-12, atol=0)


def test_radii_equal_sklearn_nearest_neighbours():
    neighbors = pytest.importorskip("sklearn.neighbors")
    x, y = _rows(300, 24, 3), _rows(200, 24, 4, 0.5)
    for k in (1, 5, 16):
        r = po.radii_sq(x, y, k)
        for a, got in ((x, r[:300]), (y, r[300:])):
            nn = neighbors.NearestNeighbors(n_neighbors=k + 1).fit(a.astype(np.float64))
            dist = nn.kneighbors(a.astype(np.float64))[0][:, -1]
            assert np.allclose(np.sqrt(got), dist, rtol=1e-9, atol=1e-9)


def test_identical_sets_are_perfect():
    x = _rows(150, 16, 5)
    p, r, _, c = po.prdc(x, x.copy(), 5)
    assert (p, r, c) == (1.0, 1.0, 1.0)


@pytest.mark.parametrize("dup", [False, True])
def test_decision_bounds_collapse_at_tau_zero(dup):
    x = _with_duplicates(60, 10, 6) if dup else _rows(60, 10, 6)
    y = _rows(50, 10, 7, 0.2)
    y[0] = x[0]
    radii = po.radii_sq(x, y, 3)
    inside, flags = po.counts(x, y, radii)
    b = po.decision_bounds(x, y, radii, tau=0.0)
    assert np.array_equal(b["inside"][0], inside) and np.array_equal(b["inside"][1], inside)
    for key, bit in (("covered", 1), ("recalled", 2)):
        assert np.array_equal(b[key][0], (flags & bit) > 0) and np.array_equal(b[key][1], (flags & bit) > 0)
    wide = po.decision_bounds(x, y, radii)                     # the default tau only widens them
    assert (wide["inside"][0] <= inside).all() and (inside <= wide["inside"][1]).all()


def test_radii_bounds_bracket_the_radii():
    x, y = _rows(80, 16, 8, 20.0), _rows(70, 16, 9, 20.0)
    r = po.radii_sq(x, y, 4)
    lo, hi = po.radii_bounds(x, y, 4)
    assert (lo <= r).all() and (r <= hi).all() and (lo < hi).all()
    lo0, hi0 = po.radii_bounds(x, y, 4, tau=0.0)
    assert np.array_equal(lo0, r) and np.array_equal(hi0, r)
