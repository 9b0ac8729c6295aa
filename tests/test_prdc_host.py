"""Precision, recall, density and coverage without a GPU (the device calls replaced by the oracle): the argument errors
of calc_prdc and of ``python -m fadtk_b200.prdc``, the zero-padding of the width, the refusal of statistics, and the
csv header check and append."""
import csv

import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native, fad as fad_mod, kad as kad_cli, prdc as prdc_cli
from oracle import prdc_oracle as po


def _rows(m, d, seed, offset=0.0):
    return (offset + np.random.default_rng(seed).standard_normal((m, d))).astype(np.float16)


class _OracleEngine:
    """Stands in for _native.Engine: the two PRDC passes computed by the oracle on the host."""
    torch_device = torch.device("cpu")

    def __init__(self):
        self.widths = []

    def knn_radii_sq(self, z, m, k):
        zn = z.numpy()
        self.widths.append(zn.copy())
        return torch.from_numpy(po.radii_sq(zn[:m], zn[m:], k))       # fp64: exact ties stay ties

    def prdc_counts(self, z, m, radii_sq):
        zn = z.numpy()
        inside, flags = po.counts(zn[:m], zn[m:], radii_sq.numpy())
        return torch.from_numpy(inside.astype(np.int32)), torch.from_numpy(flags)


@pytest.fixture
def oracle_engine(monkeypatch):
    eng = _OracleEngine()
    monkeypatch.setattr(_native, "engine", lambda *a, **k: eng)
    return eng


@pytest.mark.parametrize("m,n,k", [(5, 9, 5), (9, 5, 5), (1, 2, 1), (2, 1, 1), (16, 30, 16)])
def test_too_few_rows(oracle_engine, m, n, k):
    with pytest.raises(ValueError, match="more than k"):
        fk.calc_prdc(_rows(m, 8, 1), _rows(n, 8, 2), k=k)
    assert not oracle_engine.widths


@pytest.mark.parametrize("k", [0, 17, -1, 2.0, True, "5", None])
def test_bad_k(oracle_engine, k):
    with pytest.raises(ValueError, match="integer k in \\[1, 16\\]"):
        fk.calc_prdc(_rows(30, 8, 1), _rows(30, 8, 2), k=k)
    assert not oracle_engine.widths


def test_bad_inputs(oracle_engine):
    with pytest.raises(ValueError, match="PRDC needs fp16"):
        fk.calc_prdc(_rows(20, 8, 5).astype(np.float32), _rows(20, 8, 6))
    with pytest.raises(ValueError, match="widths differ"):
        fk.calc_prdc(_rows(20, 8, 5), _rows(20, 16, 6))
    with pytest.raises(ValueError, match=r"\[rows, d\]"):
        fk.calc_prdc(_rows(20, 8, 5)[None], _rows(20, 8, 6))
    assert not oracle_engine.widths


def test_width_is_zero_padded_to_a_multiple_of_8(oracle_engine):
    x, y = _rows(60, 100, 7), _rows(50, 100, 8, 0.3)
    x[1] = x[0]
    y[0] = x[5]
    got = fk.calc_prdc(x, y, k=3)
    assert oracle_engine.widths[0].shape == (110, 104) and not oracle_engine.widths[0][:, 100:].any()
    assert tuple(got[:4]) == pytest.approx(po.prdc(x, y, 3), abs=0, rel=1e-15)
    assert (got.k, got.n_baseline, got.n_eval) == (3, 60, 50)
    _, inside, flags, want = po.prdc_direct(x, y, 3)
    assert tuple(got[:4]) == pytest.approx(want, abs=0, rel=1e-15)


def test_identical_sets(oracle_engine):
    x = _rows(40, 16, 9)
    got = fk.calc_prdc(x, torch.from_numpy(x.copy()), k=5)
    assert (got.precision, got.recall, got.coverage) == (1.0, 1.0, 1.0)


# ------------------------------------------------------------------------------------------------ command line
class _ML:
    name = "vggish"


@pytest.fixture
def cli(monkeypatch, tmp_path):
    monkeypatch.setattr(prdc_cli, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(prdc_cli, "_embed_directories", lambda *a: pytest.fail("embedding started before the checks"))
    (tmp_path / "base").mkdir()
    (tmp_path / "eval").mkdir()
    return tmp_path


def test_cli_refuses_statistics(cli, monkeypatch):
    npz = cli / "base.npz"
    np.savez(npz, **{"vggish.mu": np.zeros(128), "vggish.cov": np.eye(128)})
    for argv in (["vggish", str(npz), str(cli / "eval")], ["vggish", str(cli / "base"), str(npz)]):
        with pytest.raises(ValueError, match="PRDC needs embeddings, not \\(mu, C\\) statistics"):
            prdc_cli.main(argv)
    with pytest.raises(ValueError, match="not a directory"):
        prdc_cli.main(["vggish", "fma_pop", str(cli / "eval")])
    stats = cli / "stats"
    stats.mkdir()
    np.savez(stats / "fma_pop.npz", **{"vggish.mu": np.zeros(128), "vggish.cov": np.eye(128)})
    monkeypatch.setenv("FADTK_STATS_DIR", str(stats))
    with pytest.raises(ValueError, match="not \\(mu, C\\) statistics"):
        prdc_cli.main(["vggish", "fma_pop", str(cli / "eval")])


@pytest.mark.parametrize("k", ["0", "17"])
def test_cli_refuses_k(cli, k):
    with pytest.raises(ValueError, match="k in \\[1, 16\\]"):
        prdc_cli.main(["vggish", str(cli / "base"), str(cli / "eval"), "-k", k])


def test_cli_refuses_a_csv_with_another_header(cli):
    out = cli / "scores.csv"
    out.write_text(kad_cli.CSV_HEADER)
    with pytest.raises(ValueError, match="header.*PRDC results"):
        prdc_cli.main(["vggish", str(cli / "base"), str(cli / "eval"), str(out)])
    assert out.read_text() == kad_cli.CSV_HEADER


def test_cli_writes_the_header_once_and_appends(cli, monkeypatch, oracle_engine, capsys):
    """embedding skipped (the caches are written here): a new file gets the header, a second run appends"""
    monkeypatch.setattr(prdc_cli, "_embed_directories", lambda *a: None)
    monkeypatch.setattr(fad_mod.FrechetAudioDistance, "__init__",
                        lambda self, ml, audio_load_worker=8, load_model=True: setattr(self, "ml", ml)
                        or setattr(self, "audio_load_worker", audio_load_worker))
    sets = {"base": _rows(40, 24, 11), "eval": _rows(30, 24, 12, 0.2)}
    for name, emb in sets.items():
        (cli / name / "embeddings" / "vggish").mkdir(parents=True)
        np.save(cli / name / "embeddings" / "vggish" / "a.npy", emb[:25])
        np.save(cli / name / "embeddings" / "vggish" / "b.npy", emb[25:])
    out = cli / "sub" / "prdc.csv"
    argv = ["vggish", str(cli / "base"), str(cli / "eval"), str(out), "-k", "4", "-w", "1"]
    assert prdc_cli.main(argv) == 0
    assert "precision" in capsys.readouterr().out
    assert prdc_cli.main(argv) == 0
    rows = list(csv.reader(out.open()))
    assert rows[0] == prdc_cli.CSV_HEADER.strip().split(",") and len(rows) == 3
    row = dict(zip(rows[0], rows[1]))
    want = po.prdc(sets["base"], sets["eval"], 4)
    got = tuple(float(row[c]) for c in ("precision", "recall", "density", "coverage"))
    assert got == pytest.approx(want, abs=0, rel=1e-15)
    assert (row["k"], row["n_baseline"], row["n_eval"]) == ("4", "40", "30")


def test_score_prdc_refuses_statistics(tmp_path):
    fad = fad_mod.FrechetAudioDistance.__new__(fad_mod.FrechetAudioDistance)
    fad.ml, fad.audio_load_worker = _ML(), 1
    npz = tmp_path / "s.npz"
    np.savez(npz, a=np.zeros(1))
    with pytest.raises(ValueError, match="PRDC needs embeddings"):
        fad.score_prdc(npz, tmp_path)
    with pytest.raises(ValueError, match="no vggish embeddings"):
        fad.score_prdc(tmp_path, tmp_path)
