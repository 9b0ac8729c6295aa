"""The bootstrap oracle (oracle/bootstrap_oracle.py): the multiplicities against a pure-Python-integer restatement of
the draw rule, the multiplicity route against materialising each resample with np.repeat (FAD statistics and the KAD
sums, self-copy pairs included), and the interval formulas on hand-made replicates."""
import numpy as np
import pytest

from oracle import bootstrap_oracle as bo
from oracle import fad_test_oracle as fto
from oracle import kad_test_oracle as kto

_M = (1 << 64) - 1


def _mix(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & _M
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M
    return x ^ (x >> 31)


def _counts_python(F: int, B: int, seed: int) -> list:
    out = [[1] * F]
    for b in range(1, B + 1):
        row = [0] * F
        base = _mix((seed + b) & _M)
        for t in range(F):
            row[(_mix(base ^ t) * F) >> 64] += 1
        out.append(row)
    return out


@pytest.mark.parametrize("F,B,seed", [(2, 30, 0), (3, 20, 7), (65, 9, 2 ** 64 - 3), (1000, 3, 12345)])
def test_counts_match_integer_restatement(F, B, seed):
    got = bo.counts(F, B, seed)
    assert got.tolist() == _counts_python(F, B, seed)
    assert np.all(got.sum(1) == F) and np.all(got[0] == 1)


def test_counts_cover_units_evenly():
    c = bo.counts(50, 400, 1)
    assert abs(c[1:].mean() - 1.0) < 1e-12                         # every row sums to F
    assert 0.3 < (c[1:] == 0).mean() < 0.44                       # about (1 - 1/F)^F of the units are left out


def _units(rng, lens, d, shift=0.0):
    return [(shift + rng.standard_normal((n, d))).astype(np.float16) for n in lens]


def test_fad_multiplicities_equal_materialised_resamples():
    rng = np.random.default_rng(0)
    d = 8
    units = _units(rng, [1, 3, 5, 2, 1, 4, 6, 2], d, 1.5)
    shift = fto.pool_shift(units)
    mu_x, cov_x = np.zeros(d), np.eye(d)
    r = bo.fad(mu_x, cov_x, units, 12, 3, shift)
    for b in range(13):
        rows = bo.materialise(units, r["counts"][b])
        n, mu, cov = r["stats"][b]
        y = rows.astype(np.float64)
        assert n == rows.shape[0]
        assert np.allclose(mu, y.mean(0), rtol=1e-12, atol=1e-12 * np.abs(y).max())
        assert np.allclose(cov, np.cov(y, rowvar=False), rtol=1e-12, atol=1e-12 * np.abs(np.cov(y, rowvar=False)).max())
    assert r["fad"].shape == (13,) and np.isfinite(r["fad"]).all()


def test_kad_multiplicities_equal_materialised_resamples():
    rng = np.random.default_rng(1)
    d = 6
    x = rng.standard_normal((30, d)).astype(np.float16)
    units = _units(rng, [2, 1, 4, 3, 1, 5], d, 0.3)
    sigma = 2.5
    r = bo.kad(x, units, sigma, 15, 4)
    m = x.shape[0]
    for b in range(16):
        y = bo.materialise(units, r["counts"][b])
        k = kto.kernel_matrix(np.concatenate([x, y]), sigma)
        n = y.shape[0]
        s_yy = np.triu(k[m:, m:], 1).sum()                        # copies of one row: K = 1 off the diagonal
        s_xy = k[:m, m:].sum()
        assert r["sums"][b, 0] == n
        assert abs(r["sums"][b, 1] - s_yy) <= 1e-12 * s_yy
        assert abs(r["sums"][b, 2] - s_xy) <= 1e-12 * s_xy
        direct = 1000.0 * (2.0 * r["s_xx"] / (m * (m - 1.0)) + 2.0 * s_yy / (n * (n - 1.0)) - 2.0 * s_xy / (m * n))
        assert abs(r["kad"][b] - direct) <= 1e-10 * max(1.0, abs(direct))
    assert np.all(r["err"] > 0)


def test_intervals_on_hand_made_replicates():
    theta = np.array([2.0, 1.0, 2.0, 3.0, 4.0, 5.0])
    lo, hi, se, bias = bo.interval(theta, 0.5, "percentile")
    assert (lo, hi) == (2.0, 4.0)                                 # the 25 % and 75 % linear quantiles of 1 .. 5
    assert se == pytest.approx(np.sqrt(2.5), rel=1e-15) and bias == 1.0
    lo, hi, _, _ = bo.interval(theta, 0.5, "basic")
    assert (lo, hi) == (0.0, 2.0)                                 # (2 * 2 - 4, 2 * 2 - 2)
    lo, hi, _, _ = bo.interval(np.array([0.0, 1.0, 2.0]), 0.9, "percentile")
    assert lo == pytest.approx(1.05) and hi == pytest.approx(1.95)
