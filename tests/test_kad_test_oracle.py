"""The permutation-test oracle (oracle/kad_test_oracle.py) against a direct O(B N^2) restatement, and the calibration
of both tests: over 200 same-distribution draws, the share of p <= 0.05 lies in the binomial 99.9 % interval."""
import numpy as np
import pytest
from scipy import stats as sst

from oracle import kad_oracle as ko
from oracle import kad_test_oracle as kto


def _mix64_scalar(x: int) -> int:
    m = (1 << 64) - 1
    x = (x + 0x9E3779B97F4A7C15) & m
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & m
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & m
    return x ^ (x >> 31)


def test_label_rule_restated_in_python_integers():
    n, a, B, seed = 97, 40, 6, 2 ** 64 - 3
    lab = kto.labels(n, a, B, seed)
    assert lab[0].tolist() == [True] * a + [False] * (n - a)
    for b in range(1, B + 1):
        base = _mix64_scalar((seed + b) % 2 ** 64)
        order = sorted(range(n), key=lambda i: (_mix64_scalar(base ^ i), i))
        want = np.zeros(n, dtype=bool)
        want[order[:a]] = True
        assert np.array_equal(lab[b], want)


def test_pack_bits_layout():
    lab = np.zeros((2, 130), dtype=bool)
    lab[0, [0, 31, 32, 129]] = True
    w = kto.pack_bits(lab)
    assert w.shape == (2, 8) and w.dtype == np.uint32
    assert w[0, 0] == 0x80000001 and w[0, 1] == 1 and w[0, 4] == 2 and not w[1].any()


def test_sums_and_statistics_against_direct_loops():
    rng = np.random.default_rng(0)
    x = (3.0 + rng.standard_normal((23, 8))).astype(np.float16)
    y = (3.2 + rng.standard_normal((19, 8))).astype(np.float16)
    sigma = ko.bandwidth(x)
    r = kto.kad_test(x, y, sigma, 5, 1)
    z = np.concatenate([x, y]).astype(np.float64)
    N, m, n = 42, 23, 19
    for b in range(6):
        lab = r["labels"][b]
        s = np.zeros(3)
        for i in range(N):
            for j in range(i + 1, N):
                k = np.exp(-np.sum((z[i] - z[j]) ** 2) / (2 * sigma * sigma))
                s[0 if lab[i] and lab[j] else 1 if not (lab[i] or lab[j]) else 2] += k
        assert np.allclose(r["sums"][b], s, rtol=1e-12)
        want = 1000 * (2 * s[0] / (m * (m - 1)) + 2 * s[1] / (n * (n - 1)) - 2 * s[2] / (m * n))
        assert np.isclose(r["stats"][b], want, rtol=1e-9, atol=1e-12)
    assert r["p_value"] == (1 + np.count_nonzero(r["stats"][1:] >= r["stats"][0])) / 6


def test_comparison_against_direct_kad():
    rng = np.random.default_rng(1)
    x = rng.standard_normal((30, 8)).astype(np.float16)
    a = (0.3 + rng.standard_normal((12, 8))).astype(np.float16)
    b = rng.standard_normal((15, 8)).astype(np.float16)
    sigma = ko.bandwidth(x)
    r = kto.kad_comparison(x, a, b, sigma, 4, 9)
    pool = np.concatenate([a, b])

    def kad(y):
        xx = np.concatenate([x, y]).astype(np.float64)
        k = kto.kernel_matrix(xx, sigma)
        m, n = x.shape[0], y.shape[0]
        return 1000 * (k[:m, :m].sum() / (m * (m - 1)) + k[m:, m:].sum() / (n * (n - 1)) - 2 * k[:m, m:].sum() / (m * n))

    for i in range(5):
        lab = r["labels"][i]
        assert np.isclose(r["stats"][i], kad(pool[lab]) - kad(pool[~lab]), rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("which", ["test", "comparison"])
def test_calibration(which):
    trials, B, d = 200, 199, 16
    hits = 0
    for t in range(trials):
        rng = np.random.default_rng(1000 + t)
        if which == "test":
            x, y = (rng.standard_normal((300, d)).astype(np.float16), rng.standard_normal((300, d)).astype(np.float16))
            p = kto.kad_test(x, y, ko.bandwidth(x), B, t)["p_value"]
        else:
            x, a, b = (rng.standard_normal((r, d)).astype(np.float16) for r in (200, 300, 300))
            p = kto.kad_comparison(x, a, b, ko.bandwidth(x), B, t)["p_value"]
        hits += p <= 0.05
    lo, hi = sst.binom.interval(0.999, trials, 0.05)
    assert lo <= hits <= hi, (which, hits, lo, hi)
