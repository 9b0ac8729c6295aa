"""The FAD comparison oracle (oracle/fad_test_oracle.py) against direct per-labelling statistics, its calibration over
200 same-distribution draws (the share of p <= 0.05 in the binomial 99.9 % interval), and its power on a planted
shift."""
import numpy as np
from scipy import stats as sst

from oracle import fad_oracle as fo
from oracle import fad_test_oracle as fto


def _units(rng, count, rows, d, shift=0.0, scale=1.0):
    return [(shift + scale * rng.standard_normal((rows if np.isscalar(rows) else rows[i], d))).astype(np.float16)
            for i in range(count)]


def _baseline(rng, d):
    x = rng.standard_normal((400, d)).astype(np.float16)
    mu, cov = fo.embd_statistics(x)
    return mu.astype(np.float64), cov


def test_records_and_sums_against_direct_union_statistics():
    rng = np.random.default_rng(0)
    d = 8
    units = _units(rng, 7, [1, 3, 5, 2, 1, 4, 6], d, shift=2.0)
    shift = fto.pool_shift(units)
    rec = fto.records(units, shift)
    assert rec.shape == (7, fto.record_len(d)) and list(rec[:, 0]) == [1, 3, 5, 2, 1, 4, 6]
    lab = fto.labels(7, 3, 5, 11)
    sums = fto.labelled_sums(rec, lab)
    for b in range(6):
        for side, mask in ((0, lab[b]), (1, ~lab[b])):
            chosen = [u for u, m in zip(units, mask) if m]
            n, mu, cov = fto.statistics(sums[b, side], shift)
            mu_w, cov_w = fto.union_statistics(chosen)
            assert n == sum(u.shape[0] for u in chosen)
            assert np.allclose(mu, mu_w, rtol=1e-12, atol=1e-12)
            assert np.allclose(cov, cov_w, rtol=1e-10, atol=1e-12)


def test_comparison_against_direct_fad():
    rng = np.random.default_rng(1)
    d = 16
    mu_x, cov_x = _baseline(rng, d)
    a, b = _units(rng, 6, 5, d, shift=0.3), _units(rng, 5, 4, d)
    r = fto.comparison(mu_x, cov_x, a, b, 4, 9)
    pool = a + b
    for i in range(5):
        lab = r["labels"][i]
        fa = fo.frechet_distance(mu_x, cov_x, *fto.union_statistics([u for u, m in zip(pool, lab) if m]))
        fb = fo.frechet_distance(mu_x, cov_x, *fto.union_statistics([u for u, m in zip(pool, lab) if not m]))
        assert np.isclose(r["stats"][i], fa - fb, rtol=1e-7, atol=1e-9)
    assert r["p_value"] == (1 + np.count_nonzero(np.abs(r["stats"][1:]) >= abs(r["stats"][0]))) / 5


def test_calibration():
    trials, B, d = 200, 199, 16
    hits = 0
    for t in range(trials):
        rng = np.random.default_rng(2000 + t)
        mu_x, cov_x = _baseline(rng, d)
        a, b = _units(rng, 40, 5, d), _units(rng, 40, 5, d)
        hits += fto.comparison(mu_x, cov_x, a, b, B, t)["p_value"] <= 0.05
    lo, hi = sst.binom.interval(0.999, trials, 0.05)
    assert lo <= hits <= hi, (hits, lo, hi)


def test_planted_shift_gives_the_smallest_p():
    rng = np.random.default_rng(3)
    d = 16
    mu_x, cov_x = _baseline(rng, d)
    a, b = _units(rng, 30, 5, d, shift=0.8), _units(rng, 30, 5, d)
    assert fto.comparison(mu_x, cov_x, a, b, 99, 1)["p_value"] == 1.0 / 100.0
