"""numpy fp64 restatement of the Kernel Audio Distance definition (fadtk_b200.fad.calc_kernel_audio_distance).

Test infrastructure only.  The fp16 rows are taken as exact reals and centred on their fp64 mean before the expanded
distance GEMM |a|^2 + |b|^2 - 2 a.b, which then has no offset to cancel (the GPU path controls that cancellation
differently: a shared fp16 shift and an fp16 hi/lo split).  Work is done in row blocks to bound memory; the bandwidth
uses np.median over the condensed distances, so it is meant for up to a few thousand baseline rows.
"""
from __future__ import annotations

import numpy as np

BLOCK = 2048


def _pair_blocks(a: np.ndarray, b: np.ndarray, upper: bool, block: int = BLOCK):
    """Yields the squared distances of a-block x b-block (fp64, clamped at 0); upper: only pairs i < j of a == b."""
    na, nb = (a * a).sum(1), (b * b).sum(1)
    for i0 in range(0, a.shape[0], block):
        i1 = min(a.shape[0], i0 + block)
        for j0 in range(i0 if upper else 0, b.shape[0], block):
            j1 = min(b.shape[0], j0 + block)
            q = np.maximum(na[i0:i1, None] + nb[None, j0:j1] - 2.0 * (a[i0:i1] @ b[j0:j1].T), 0.0)
            if upper:
                q = q[np.arange(i0, i1)[:, None] < np.arange(j0, j1)[None, :]]
            yield q.ravel()


def _centred(x: np.ndarray, *others: np.ndarray):
    mu = x.astype(np.float64).mean(0)
    return [a.astype(np.float64) - mu for a in (x, *others)]


def pair_sq_distances(x: np.ndarray) -> np.ndarray:
    """Condensed squared distances {|x_i - x_j|^2 : i < j} (fp64)."""
    (xc,) = _centred(x)
    return np.concatenate(list(_pair_blocks(xc, xc, True)))


def middle_sq(x: np.ndarray) -> tuple[float, float]:
    """The two middle squared distances of the baseline pairs (equal when their number is odd)."""
    q = np.sort(pair_sq_distances(x))
    p = q.shape[0]
    return float(q[(p - 1) // 2]), float(q[p // 2])


def bandwidth(x: np.ndarray) -> float:
    """sigma = np.median of the pairwise distances of x."""
    return float(np.median(np.sqrt(pair_sq_distances(x))))


def kernel_sums(x: np.ndarray, y: np.ndarray, sigma: float) -> tuple[float, float, float]:
    """S_xx (i < j), S_yy (i < j), S_xy (all pairs) of exp(-|a - b|^2 / (2 sigma^2))."""
    xc, yc = _centred(x, y)
    c = 1.0 / (2.0 * sigma * sigma)

    def total(a, b, upper):
        return float(sum(np.exp(-q * c).sum() for q in _pair_blocks(a, b, upper)))
    return total(xc, xc, True), total(yc, yc, True), total(xc, yc, False)


def mmd2_unbiased(s_xx: float, s_yy: float, s_xy: float, m: int, n: int) -> float:
    return 2.0 * s_xx / (m * (m - 1.0)) + 2.0 * s_yy / (n * (n - 1.0)) - 2.0 * s_xy / (float(m) * n)


def kad(x: np.ndarray, y: np.ndarray) -> tuple[float, float]:
    """-> (KAD = 1000 MMD^2_u, sigma)."""
    sigma = bandwidth(x)
    return 1000.0 * mmd2_unbiased(*kernel_sums(x, y, sigma), x.shape[0], y.shape[0]), sigma


def kad_direct(x: np.ndarray, y: np.ndarray) -> tuple[float, float]:
    """The definition as a plain double loop over pairs (differences, no expansion): the oracle's own check."""
    x, y = x.astype(np.float64), y.astype(np.float64)
    m, n = x.shape[0], y.shape[0]
    dist = [float(np.sqrt(((x[i] - x[j]) ** 2).sum())) for i in range(m) for j in range(i + 1, m)]
    sigma = float(np.median(dist))
    k = lambda a, b: float(np.exp(-((a - b) ** 2).sum() / (2.0 * sigma * sigma)))  # noqa: E731
    s_xx = sum(k(x[i], x[j]) for i in range(m) for j in range(i + 1, m))
    s_yy = sum(k(y[i], y[j]) for i in range(n) for j in range(i + 1, n))
    s_xy = sum(k(x[i], y[j]) for i in range(m) for j in range(n))
    return 1000.0 * mmd2_unbiased(s_xx, s_yy, s_xy, m, n), sigma
