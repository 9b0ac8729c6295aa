"""Pin the CPU oracle (oracle/fad_oracle.py) to outputs of the REAL reference functions.

tests/golden/*.npz were produced by oracle/make_golden.py, which imports fadtk/fad.py and
fadtk/utils.py unchanged from the reference checkout.  Bit-level agreement is expected wherever the
oracle performs the same numpy/LAPACK calls; 1e-12 relative elsewhere.
"""
import numpy as np
import pytest

from oracle import fad_oracle as fo
from oracle.make_golden import spectrum_cov


def test_frechet_real_fma_pop_statistics(golden_dir):
    g = np.load(golden_dir / "frechet_fma_pop_128.npz")
    got = fo.frechet_distance(g["mu1"], g["cov1"], g["mu2"], g["cov2"])
    assert got == pytest.approx(float(g["fad"]), rel=1e-12)
    # SURVEY.md section 8c known answer computed from the reference at survey time
    assert got == pytest.approx(4420.894217705201, rel=1e-12)


@pytest.mark.parametrize("i", [0, 1, 2])
def test_frechet_ill_conditioned_real_spectra(golden_dir, i):
    g = np.load(golden_dir / "frechet_spectra.npz")
    c1 = spectrum_cov(g[f"evals1_{i}"], 100 + i)
    c2 = spectrum_cov(g[f"evals2_{i}"], 200 + i)
    got = fo.frechet_distance(g[f"mu1_{i}"], c1, g[f"mu2_{i}"], c2)
    assert got == pytest.approx(float(g[f"fad_{i}"]), rel=1e-9)


def test_statistics_and_online_merge(golden_dir):
    g = np.load(golden_dir / "stats_cases.npz")
    cat, sizes = g["cat"], g["sizes"]
    mu, cov = fo.embd_statistics(cat)
    assert mu.dtype == np.float16 == g["mu_cat"].dtype          # fad.py:48 dtype quirk
    assert np.array_equal(mu, g["mu_cat"])
    assert np.allclose(cov, g["cov_cat"], rtol=1e-13, atol=0)
    files = np.split(cat, np.cumsum(sizes)[:-1])
    mu_o, cov_o = fo.online_statistics(files)
    assert np.allclose(mu_o, g["mu_online"], rtol=1e-14, atol=1e-15)
    assert np.allclose(cov_o, g["cov_online"], rtol=1e-12, atol=1e-14)
    # utils.py:16 - a single-frame file poisons the covariance with NaN
    assert bool(g["cov_with_single_frame_file_is_nan"])
    with np.errstate(all="ignore"):
        _, cov_nan = fo.online_statistics(files + [files[0][:1]])
    assert np.isnan(cov_nan).all()


def test_statistics_need_two_rows():
    with pytest.raises(AssertionError):
        fo.embd_statistics(np.zeros((1, 8), np.float16))


def test_fad_inf_reproduces_reference_rng_stream(golden_dir):
    g = np.load(golden_dir / "inf_case.npz")
    mu_b, cov_b = fo.embd_statistics(g["base"])
    np.random.seed(0)
    res = fo.score_inf(mu_b, cov_b, g["eval"], steps=int(g["steps"]), min_n=int(g["min_n"]))
    assert np.array_equal(np.array(res.points)[:, 0], g["points"][:, 0])
    assert np.allclose(np.array(res.points)[:, 1], g["points"][:, 1], rtol=1e-10)
    assert res.score == pytest.approx(float(g["score"]), rel=1e-9)
    assert res.slope == pytest.approx(float(g["slope"]), rel=1e-9)
    assert res.r2 == pytest.approx(float(g["r2"]), rel=1e-9)


def test_per_song_scores_and_order(golden_dir):
    g = np.load(golden_dir / "indiv_case.npz")
    songs = [(k + ".wav", g[k]) for k in sorted(g.files) if k.startswith("song")]
    got = fo.score_individual(g["mu_base"], g["cov_base"], songs)
    assert [n for n, _ in got] == list(g["names"])              # single-frame song dropped
    assert np.allclose([s for _, s in got], g["scores"], rtol=1e-10)


def test_identity_and_gram_form_properties():
    rng = np.random.default_rng(0)
    x = rng.normal(size=(500, 32))
    mu, cov = x.mean(0), np.cov(x, rowvar=False)
    assert abs(fo.frechet_distance(mu, cov, mu, cov)) < 1e-8 * np.trace(cov)
    # rank-deficient eval set: tr sqrt(C1 C2) equals the n x n Gram form (SURVEY.md section 7)
    y = rng.normal(size=(10, 32))
    cy = np.cov(y, rowvar=False)
    yc = y - y.mean(0)
    gram = yc @ cov @ yc.T / (y.shape[0] - 1)
    want = np.sqrt(np.clip(np.linalg.eigvalsh(gram), 0, None)).sum()
    assert fo.trace_sqrt_product(cov, cy) == pytest.approx(want, rel=1e-6)
