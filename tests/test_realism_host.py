"""Per-sample realism without a GPU (the device call replaced by the oracle): the argument errors of calc_realism and of
``python -m fadtk_b200.realism``, the zero-padding of the width, the threshold-0 refusal, and the per-file table of
score_realism_individual: header, sort order, nearest baseline file and path rules."""
import csv

import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native, fad as fad_mod, realism as realism_cli
from oracle import realism_oracle as ro


def _rows(m, d, seed, offset=0.0):
    return (offset + np.random.default_rng(seed).standard_normal((m, d))).astype(np.float16)


class _OracleEngine:
    """Stands in for _native.Engine: fad_realism computed by the oracle on the host."""
    torch_device = torch.device("cpu")

    def __init__(self):
        self.calls = []

    def realism(self, z, m, k):
        zn = z.numpy()
        self.calls.append(zn.copy())
        kept, real, near, near_sq, t = ro.realism(zn[:m], zn[m:], k)
        return (torch.from_numpy(kept.astype(np.float32)), torch.from_numpy(real.astype(np.float32)),
                torch.from_numpy(near.astype(np.int32)), torch.from_numpy(near_sq.astype(np.float32)), t)


@pytest.fixture
def oracle_engine(monkeypatch):
    eng = _OracleEngine()
    monkeypatch.setattr(_native, "engine", lambda *a, **k: eng)
    return eng


@pytest.mark.parametrize("m,n,k", [(3, 9, 3), (1, 2, 1), (16, 30, 16), (10, 0, 3)])
def test_too_few_rows(oracle_engine, m, n, k):
    with pytest.raises(ValueError, match="more than k baseline rows and at least one eval row"):
        fk.calc_realism(_rows(m, 8, 1), _rows(n, 8, 2), k=k)
    assert not oracle_engine.calls


@pytest.mark.parametrize("k", [0, 17, -1, 2.0, True, "3", None])
def test_bad_k(oracle_engine, k):
    with pytest.raises(ValueError, match="realism needs an integer k in \\[1, 16\\]"):
        fk.calc_realism(_rows(30, 8, 1), _rows(30, 8, 2), k=k)
    assert not oracle_engine.calls


def test_bad_inputs(oracle_engine):
    with pytest.raises(ValueError, match="realism needs fp16"):
        fk.calc_realism(_rows(20, 8, 5).astype(np.float32), _rows(20, 8, 6))
    with pytest.raises(ValueError, match="widths differ"):
        fk.calc_realism(_rows(20, 8, 5), _rows(20, 16, 6))
    with pytest.raises(ValueError, match=r"\[rows, d\]"):
        fk.calc_realism(_rows(20, 8, 5)[None], _rows(20, 8, 6))
    assert not oracle_engine.calls


def test_width_is_zero_padded_and_results_are_the_oracle(oracle_engine):
    x, y = _rows(60, 100, 7), _rows(50, 100, 8, 0.3)
    y[3] = x[11]
    got = fk.calc_realism(x, y)
    assert oracle_engine.calls[0].shape == (110, 104) and not oracle_engine.calls[0][:, 100:].any()
    kept, real, near, near_sq, t = ro.realism(x, y, 3)
    assert (got.k, got.n_baseline, got.n_eval, got.threshold_sq) == (3, 60, 50, t)
    assert got.realism.dtype == np.float32 and got.nearest.dtype == np.int64 and got.nearest_distance.dtype == np.float32
    assert np.array_equal(got.realism, real.astype(np.float32)) and np.array_equal(got.nearest, near)
    assert np.array_equal(got.nearest_distance, np.sqrt(near_sq.astype(np.float32)))
    assert got.nearest[3] == 11 and got.nearest_distance[3] == 0


def test_threshold_zero_is_refused(oracle_engine):
    x = np.zeros((9, 8), np.float16)
    x[8] = 1.0
    with pytest.raises(ValueError, match="threshold is 0"):
        fk.calc_realism(x, _rows(4, 8, 1), k=3)


# ------------------------------------------------------------------------------------------------ command line
class _ML:
    name = "vggish"


@pytest.fixture
def cli(monkeypatch, tmp_path):
    monkeypatch.setattr(realism_cli, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(realism_cli, "_embed_directories", lambda *a: pytest.fail("embedding started before the checks"))
    (tmp_path / "base").mkdir()
    (tmp_path / "eval").mkdir()
    return tmp_path


def test_cli_parses_the_arguments():
    ap = realism_cli._parser("fadtk_b200.realism", realism_cli._REALISM_ARGS, {"vggish": _ML()})
    a = ap.parse_args(["vggish", "b", "e"])
    assert (a.k, a.csv, a.workers) == (3, None, 8)
    a = ap.parse_args(["vggish", "b", "e", "t.csv", "-k", "5", "-w", "2"])
    assert (a.model, a.baseline, a.eval, a.csv, a.k, a.workers) == ("vggish", "b", "e", "t.csv", 5, 2)


@pytest.mark.parametrize("k", ["0", "17"])
def test_cli_refuses_k(cli, k):
    with pytest.raises(ValueError, match="k in \\[1, 16\\]"):
        realism_cli.main(["vggish", str(cli / "base"), str(cli / "eval"), "-k", k])


def test_cli_refuses_statistics_and_missing_directories(cli):
    npz = cli / "base.npz"
    np.savez(npz, **{"vggish.mu": np.zeros(128), "vggish.cov": np.eye(128)})
    for argv in (["vggish", str(npz), str(cli / "eval")], ["vggish", str(cli / "base"), str(npz)]):
        with pytest.raises(ValueError, match="realism needs embeddings, not \\(mu, C\\) statistics"):
            realism_cli.main(argv)
    npz.unlink()
    with pytest.raises(ValueError, match="not a directory"):
        realism_cli.main(["vggish", str(cli / "base"), str(cli / "nowhere")])


def _caches(root, sets):
    """sets: {dir: {stem: rows}} -> the audio stand-ins and their embedding caches"""
    for name, files in sets.items():
        emb = root / name / "embeddings" / "vggish"
        emb.mkdir(parents=True, exist_ok=True)
        for stem, rows in files.items():
            (root / name / f"{stem}.wav").write_bytes(b"")
            np.save(emb / f"{stem}.npy", rows)


@pytest.fixture
def scored(cli, monkeypatch, oracle_engine):
    monkeypatch.setattr(realism_cli, "_embed_directories", lambda *a: None)
    monkeypatch.setattr(fad_mod.FrechetAudioDistance, "__init__",
                        lambda self, ml, audio_load_worker=8, load_model=True: setattr(self, "ml", ml)
                        or setattr(self, "audio_load_worker", audio_load_worker))
    base = _rows(50, 24, 11)
    ev = {"copy": np.concatenate([_rows(3, 24, 1, 0.1), base[37:38]]),     # a frame copies baseline row 37 (b.npy)
          "far": _rows(6, 24, 2, 4.0), "near": _rows(5, 24, 3, 0.05), "x,y": _rows(4, 24, 4, 0.05),
          "empty": np.zeros((0, 24), np.float16), "wide": _rows(3, 16, 5)}
    _caches(cli, {"base": {"a": base[:30], "b": base[30:]}, "eval": ev})
    return cli, base, ev


def test_cli_writes_the_per_file_table(scored):
    root, base, ev = scored
    out = root / "sub" / "realism.csv"
    assert realism_cli.main(["vggish", str(root / "base"), str(root / "eval"), str(out), "-k", "4", "-w", "1"]) == 0
    rows = list(csv.reader(out.open()))
    assert rows[0] == ["file", "realism_median", "realism_min", "nearest_baseline", "nearest_distance", "n_eval"]
    table = {r[0]: dict(zip(rows[0], r)) for r in rows[1:]}
    names = [str(root / "eval" / f"{s}.wav") for s in ("copy", "far", "near", "x_y")]
    assert sorted(table) == sorted(names)            # the empty and the narrow cache are dropped, the comma replaced
    med = [float(r[1]) for r in rows[1:]]
    assert med == sorted(med) and rows[1][0] == names[1]     # least realistic first
    kept = ["copy", "far", "near", "x,y"]
    y = np.concatenate([ev[k] for k in kept])
    _, real, near, near_sq, _ = ro.realism(base, y, 4)
    off = np.cumsum([0] + [ev[k].shape[0] for k in kept])
    for i, k in enumerate(kept):
        r = table[names[i]]
        a, b = off[i], off[i + 1]
        rr = real[a:b].astype(np.float32).astype(np.float64)
        j = a + int(np.argmin(np.sqrt(near_sq[a:b].astype(np.float32))))
        want = root / "base" / "embeddings" / "vggish" / ("a.npy" if near[j] < 30 else "b.npy")
        assert (float(r["realism_median"]), float(r["realism_min"])) == (float(np.median(rr)), float(rr.min()))
        assert (r["nearest_baseline"], int(r["n_eval"])) == (str(want), b - a)
    assert table[names[0]]["nearest_baseline"].endswith("b.npy") and float(table[names[0]]["nearest_distance"]) == 0.0


def test_existing_table_is_returned_untouched_and_str_names_go_under_data(scored, monkeypatch):
    root, base, _ = scored
    monkeypatch.chdir(root)
    fad = fad_mod.FrechetAudioDistance(_ML(), audio_load_worker=1)
    got = fad.score_realism_individual(root / "base", root / "eval", "t.csv")
    assert got == fad_mod.Path("data") / "realism-individual" / "vggish" / "t.csv" and got.is_file()
    got.write_text("kept\n")
    assert fad.score_realism_individual(root / "base", root / "eval", "t.csv") == got and got.read_text() == "kept\n"
    with pytest.raises(ValueError, match="k in \\[1, 16\\]"):
        fad.score_realism_individual(root / "base", root / "eval", "u.csv", k=0)
    _caches(root, {"tiny": {"a": base[:5]}})
    with pytest.raises(ValueError, match="more than k baseline rows"):
        fad.score_realism_individual(root / "tiny", root / "eval", "u.csv", k=5)
    assert not (root / "data" / "realism-individual" / "vggish" / "u.csv").exists()
