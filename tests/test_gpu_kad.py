"""Kernel Audio Distance on the H100 (csrc/kad.cuh) against the fp64 numpy oracle (oracle/kad_oracle.py), on the
same fp16 rows: the three kernel sums at a fixed bandwidth (2e-6 relative), the two middle squared distances (1e-5
relative), KAD for distinct sets (1e-4 relative) and for same-distribution sets (|dMMD^2_u| <= 1e-6), reproducibility,
tile / set boundaries, and the directory command line."""
import csv

import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import synth
from oracle import kad_oracle as ko

pytestmark = pytest.mark.gpu


def encodec_like(rows, d, seed, shift=0.0, spread=1.8):
    """rows with a large common offset (|mu| ~ 64 per dimension), spread ~1.8, rounded to fp16"""
    mu = np.random.default_rng(1234 + d).choice([-1.0, 1.0], d) * np.random.default_rng(99 + d).uniform(48, 80, d)
    rng = np.random.default_rng(seed)
    return (mu + shift + spread * rng.standard_normal((rows, d))).astype(np.float16)


def clap_like(rows, d, seed, tilt=0.0):
    """L2-normalised rows (CLAP embeddings), rounded to fp16"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((rows, d)) + 0.3
    x[:, 0] += tilt
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float16)


DATA = {"encodec": encodec_like, "clap": clap_like}


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _gpu_sums(engine, x, y, sigma):
    z = _dev(np.concatenate([x, y]))
    return engine.kad_sums(z, x.shape[0], torch.tensor([sigma], dtype=torch.float64, device="cuda")).cpu().numpy()


def _fixed_sigma(x):
    return float(np.sqrt(ko.middle_sq(x[:600])[0]))


def _check_sums(engine, x, y, sigma=None):
    sigma = _fixed_sigma(x) if sigma is None else sigma
    got = _gpu_sums(engine, x, y, sigma)
    want = np.array(ko.kernel_sums(x, y, sigma))
    rel = np.abs(got - want) / np.abs(want)
    assert (rel <= 2e-6).all(), (got, want, rel)


@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("m,n,d", [(2, 2, 128), (127, 129, 128), (1000, 777, 512), (3001, 2049, 768), (640, 700, 1024),
                                   (500, 600, 384), (16001, 16383, 128)])
def test_sums_at_fixed_sigma(engine, kind, m, n, d):
    gen = DATA[kind]
    _check_sums(engine, gen(m, d, 1), gen(n, d, 2))


@pytest.mark.parametrize("m,n", [(200, 183), (200, 184), (200, 185), (128, 129), (130, 2), (2, 130)])
def test_sums_tile_and_set_boundaries(engine, m, n):
    """m + n = 384 - 1, 384, 384 + 1 with the X/Y boundary inside a tile; the boundary on a tile edge; a set of two rows
    at either end; d = 136 (zero-filled columns in the last k box)"""
    _check_sums(engine, encodec_like(m, 136, 3), encodec_like(n, 136, 4, shift=0.3))


@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("m", [101, 102, 2, 3, 300])
def test_median_odd_and_even_pair_counts(engine, kind, m):
    """m = 101: 5050 pairs (even, two middle values); 102: 5151 (odd); 2: one pair; 3: three"""
    x = DATA[kind](m, 128, 5)
    got = engine.kad_median_sq(_dev(x)).cpu().numpy()
    want = np.array(ko.middle_sq(x))
    assert (np.abs(got - want) <= 1e-5 * want).all(), (got, want)
    if (m * (m - 1) // 2) % 2:
        assert got[0] == got[1]


def test_median_with_exact_ties(engine):
    """30 distinct rows, each twice: every distance occurs four times, and 30 pairs are 0"""
    x = np.repeat(encodec_like(30, 128, 6), 2, axis=0)
    got = engine.kad_median_sq(_dev(x)).cpu().numpy()
    want = np.array(ko.middle_sq(x))
    assert (np.abs(got - want) <= 1e-5 * want).all(), (got, want)
    ties = np.tile(encodec_like(1, 128, 7), (9, 1))                   # all 36 pairs identical
    assert (engine.kad_median_sq(_dev(ties)).cpu().numpy() == 0.0).all()


def test_zero_bandwidth_raises(engine):
    """more than half of the baseline pairs are identical rows (e.g. silent clips): sigma = 0"""
    x = np.concatenate([np.zeros((50, 128), np.float16), clap_like(10, 128, 8)])
    with pytest.raises(ValueError, match="bandwidth is 0"):
        fk.calc_kernel_audio_distance(x, clap_like(20, 128, 9))


@pytest.mark.parametrize("kind", sorted(DATA))
def test_kad_distinct_sets(engine, kind):
    gen = DATA[kind]
    x = gen(1500, 128, 10)
    y = gen(1200, 128, 11, 0.4) if kind == "encodec" else gen(1200, 128, 11, 3.0)
    got = fk.calc_kernel_audio_distance(x, y)
    want, sigma = ko.kad(x, y)
    assert got.n_baseline == 1500 and got.n_eval == 1200
    assert abs(got.bandwidth - sigma) <= 1e-5 * sigma
    assert want > 1.0 and abs(got.score - want) <= 1e-4 * abs(want), (got, want)


@pytest.mark.parametrize("kind", sorted(DATA))
def test_kad_same_distribution(engine, kind):
    gen = DATA[kind]
    x, y = gen(1400, 256, 12), gen(1300, 256, 13)
    got = fk.calc_kernel_audio_distance(_dev(x), _dev(y))          # torch input too
    want, _ = ko.kad(x, y)
    assert abs(got.score - want) <= 1e-3, (got, want)               # |dMMD^2_u| <= 1e-6


def test_results_are_bitwise_reproducible(engine):
    x, y = encodec_like(3001, 128, 14), encodec_like(2500, 128, 15, 0.2)
    z = _dev(np.concatenate([x, y]))
    sigma = torch.tensor([_fixed_sigma(x)], dtype=torch.float64, device="cuda")
    a, b = engine.kad_sums(z, 3001, sigma), engine.kad_sums(z, 3001, sigma)
    assert torch.equal(a, b)
    ma, mb = engine.kad_median_sq(z[:3001]), engine.kad_median_sq(z[:3001])
    assert torch.equal(ma, mb)


def test_width_not_a_multiple_of_8_is_padded(engine):
    x, y = clap_like(700, 100, 16), clap_like(650, 100, 17, 0.5)
    got = fk.calc_kernel_audio_distance(x, y)
    want, sigma = ko.kad(x, y)
    assert abs(got.bandwidth - sigma) <= 1e-5 * sigma
    assert abs(got.score - want) <= 1e-4 * abs(want), (got, want)


def test_directory_command_line(engine, tmp_path, capsys):
    """FADTK_SYNTHETIC VGGish over synthetic clips: python -m fadtk_b200.kad embeds both directories, prints the score
    and appends the CSV row, which equals score_kad on the cached embeddings and the oracle"""
    from fadtk_b200 import kad as kad_cli
    for kind in ("base", "eval"):
        (tmp_path / kind).mkdir()
        for i in range(4):
            synth.write_wav(tmp_path / kind / f"clip{i}.wav",
                            synth.musiclike_clip(i, 4.0, 16000, baseline=(kind == "base")), 16000)
    out = tmp_path / "kad.csv"
    argv = ["vggish", str(tmp_path / "base"), str(tmp_path / "eval"), str(out), "-w", "2"]
    assert kad_cli.main(argv) == 0
    assert "The KAD vggish score between" in capsys.readouterr().out
    rows = list(csv.reader(out.open()))
    assert rows[0] == kad_cli.CSV_HEADER.strip().split(",") and len(rows) == 2
    row = dict(zip(rows[0], rows[1]))
    ml = fk.VGGishModel()
    res = fk.FrechetAudioDistance(ml, load_model=False).score_kad(tmp_path / "base", tmp_path / "eval")
    assert float(row["kad"]) == res.score and float(row["bandwidth"]) == res.bandwidth
    assert int(row["n_baseline"]) == res.n_baseline and int(row["n_eval"]) == res.n_eval
    load = lambda k: np.concatenate([np.load(f) for f in sorted((tmp_path / k / "embeddings" / "vggish").glob("*.npy"))])  # noqa: E731
    want, sigma = ko.kad(load("base"), load("eval"))
    assert abs(res.bandwidth - sigma) <= 1e-5 * sigma
    assert abs(res.score - want) <= 1e-4 * abs(want) + 1e-3, (res, want)
    assert kad_cli.main(argv) == 0 and len(list(csv.reader(out.open()))) == 3      # appended, header once
