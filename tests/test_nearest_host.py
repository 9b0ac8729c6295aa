"""The k nearest baseline groups without a GPU (the device call replaced by the oracle): the argument errors of
calc_nearest and of ``python -m fadtk_b200.nearest``, the zero-padding of the width, groups against rows, fewer groups
than k, empty groups, and the per-file table of score_nearest_individual: the merge of the rows' lists, header, order
and path rules."""
import csv

import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native, fad as fad_mod, nearest as nearest_cli
from oracle import nearest_oracle as no


def _rows(m, d, seed, offset=0.0):
    return (offset + np.random.default_rng(seed).standard_normal((m, d))).astype(np.float16)


class _OracleEngine:
    """Stands in for _native.Engine: fad_nearest computed by the oracle on the host."""
    torch_device = torch.device("cpu")

    def __init__(self):
        self.calls = []

    def nearest(self, z, m, k, offsets=None):
        zn = z.numpy()
        off = None if offsets is None else offsets.numpy()
        self.calls.append((zn.copy(), off))
        rows, q = no.nearest(zn[:m], zn[m:], k, off)
        return torch.from_numpy(rows.astype(np.int32)), torch.from_numpy(q.astype(np.float32))


@pytest.fixture
def oracle_engine(monkeypatch):
    eng = _OracleEngine()
    monkeypatch.setattr(_native, "engine", lambda *a, **k: eng)
    return eng


@pytest.mark.parametrize("m,n", [(0, 3), (3, 0)])
def test_too_few_rows(oracle_engine, m, n):
    with pytest.raises(ValueError, match="at least one baseline row and one eval row"):
        fk.calc_nearest(_rows(m, 8, 1), _rows(n, 8, 2))
    with pytest.raises(ValueError, match="at least one baseline row and one eval row"):
        fk.calc_nearest([_rows(m, 8, 1), _rows(0, 8, 3)], _rows(n, 8, 2))
    with pytest.raises(ValueError, match="at least one baseline group"):
        fk.calc_nearest([], _rows(3, 8, 2))
    assert not oracle_engine.calls


@pytest.mark.parametrize("k", [0, 17, -1, 2.0, True, "3", None])
def test_bad_k(oracle_engine, k):
    with pytest.raises(ValueError, match="nearest needs an integer k in \\[1, 16\\]"):
        fk.calc_nearest(_rows(30, 8, 1), _rows(30, 8, 2), k=k)
    assert not oracle_engine.calls


def test_bad_inputs(oracle_engine):
    with pytest.raises(ValueError, match="nearest needs fp16"):
        fk.calc_nearest(_rows(20, 8, 5).astype(np.float32), _rows(20, 8, 6))
    with pytest.raises(ValueError, match="nearest needs fp16"):
        fk.calc_nearest([_rows(20, 8, 5), _rows(3, 8, 5).astype(np.float32)], _rows(20, 8, 6))
    with pytest.raises(ValueError, match="widths differ"):
        fk.calc_nearest(_rows(20, 8, 5), _rows(20, 16, 6))
    with pytest.raises(ValueError, match="widths differ"):
        fk.calc_nearest([_rows(20, 16, 5), _rows(20, 8, 5)], _rows(20, 16, 6))
    with pytest.raises(ValueError, match=r"\[rows, d\]"):
        fk.calc_nearest(_rows(20, 8, 5)[None], _rows(20, 8, 6))
    assert not oracle_engine.calls


def test_width_is_zero_padded_and_rows_are_their_own_groups(oracle_engine):
    x, y = _rows(60, 100, 7), _rows(50, 100, 8, 0.3)
    y[3] = x[11]
    got = fk.calc_nearest(x, y)
    z, off = oracle_engine.calls[0]
    assert z.shape == (110, 104) and not z[:, 100:].any() and off is None
    rows, q = no.nearest(x, y, 5)
    assert (got.k, got.n_baseline, got.n_eval) == (5, 60, 50)
    assert got.rows.dtype == np.int64 and got.groups.dtype == np.int64 and got.distance.dtype == np.float32
    assert got.rows.shape == (50, 5) and np.array_equal(got.rows, rows) and np.array_equal(got.groups, rows)
    assert np.array_equal(got.distance, np.sqrt(q.astype(np.float32)))
    assert got.rows[3, 0] == 11 and got.distance[3, 0] == 0


def test_groups_fewer_than_k_and_empty_groups(oracle_engine):
    x = _rows(40, 16, 9)
    parts = [x[:10], x[10:10], x[10:25], np.zeros((0, 16), np.float16), x[25:]]
    y = np.concatenate([x[12:13], _rows(6, 16, 10, 0.2)])
    got = fk.calc_nearest(parts, y, k=6)
    z, off = oracle_engine.calls[0]
    assert off.tolist() == [0, 10, 10, 25, 25, 40] and z.shape == (47, 16)
    assert got.rows.shape == (7, 6)
    live = got.rows >= 0
    assert (live.sum(1) == 3).all() and (got.groups[~live] == -1).all() and np.isinf(got.distance[~live]).all()
    assert set(got.groups[0, :3].tolist()) == {0, 2, 4} and got.rows[0, 0] == 12 and got.groups[0, 0] == 2
    want = np.searchsorted(off, got.rows[live], side="right") - 1
    assert np.array_equal(got.groups[live], want)
    rows, q = no.nearest(x, y, 6, off)
    assert np.array_equal(got.rows, rows)
    one = fk.calc_nearest(x, y, k=6)                       # rows as groups: six distinct rows, not three groups
    assert (one.rows >= 0).all() and np.array_equal(one.rows[:, 0], np.where(live[:, 0], got.rows[:, 0], -1))


# ------------------------------------------------------------------------------------------------ command line
class _ML:
    name = "vggish"


@pytest.fixture
def cli(monkeypatch, tmp_path):
    monkeypatch.setattr(nearest_cli, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(nearest_cli, "_embed_directories", lambda *a: pytest.fail("embedding started before the checks"))
    (tmp_path / "base").mkdir()
    (tmp_path / "eval").mkdir()
    return tmp_path


def test_cli_parses_the_arguments():
    ap = nearest_cli._parser("fadtk_b200.nearest", nearest_cli._NEAREST_ARGS, {"vggish": _ML()})
    a = ap.parse_args(["vggish", "b", "e"])
    assert (a.k, a.csv, a.workers) == (5, None, 8)
    a = ap.parse_args(["vggish", "b", "e", "t.csv", "-k", "3", "-w", "2"])
    assert (a.model, a.baseline, a.eval, a.csv, a.k, a.workers) == ("vggish", "b", "e", "t.csv", 3, 2)


@pytest.mark.parametrize("k", ["0", "17"])
def test_cli_refuses_k(cli, k):
    with pytest.raises(ValueError, match="k in \\[1, 16\\]"):
        nearest_cli.main(["vggish", str(cli / "base"), str(cli / "eval"), "-k", k])


def test_cli_refuses_statistics_and_missing_directories(cli):
    npz = cli / "base.npz"
    np.savez(npz, **{"vggish.mu": np.zeros(128), "vggish.cov": np.eye(128)})
    for argv in (["vggish", str(npz), str(cli / "eval")], ["vggish", str(cli / "base"), str(npz)]):
        with pytest.raises(ValueError, match="nearest needs embeddings, not \\(mu, C\\) statistics"):
            nearest_cli.main(argv)
    npz.unlink()
    with pytest.raises(ValueError, match="not a directory"):
        nearest_cli.main(["vggish", str(cli / "base"), str(cli / "nowhere")])


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
    monkeypatch.setattr(nearest_cli, "_embed_directories", lambda *a: None)
    monkeypatch.setattr(fad_mod.FrechetAudioDistance, "__init__",
                        lambda self, ml, audio_load_worker=8, load_model=True: setattr(self, "ml", ml)
                        or setattr(self, "audio_load_worker", audio_load_worker))
    base = _rows(60, 24, 11)
    ev = {"copy": np.concatenate([_rows(3, 24, 1, 0.1), base[37:40]]),    # frames 3..5 copy rows 7..9 of c.npy
          "far": _rows(6, 24, 2, 4.0), "near": _rows(5, 24, 3, 0.05), "x,y": _rows(4, 24, 4, 0.05),
          "empty": np.zeros((0, 24), np.float16), "wide": _rows(3, 16, 5)}
    _caches(cli, {"base": {"a": base[:20], "b": base[20:20], "c": base[30:60], "d": base[20:30]}, "eval": ev})
    return cli, base, ev


def _want(base_parts, ev, kept, k):
    """the per-file table from the oracle: rows of every kept eval file merged per file by brute force"""
    x = np.concatenate(base_parts)
    off = np.cumsum([0] + [p.shape[0] for p in base_parts])
    gid = no.groups_of(x.shape[0], off)
    out = {}
    for name in kept:
        y = ev[name]
        q = no._q(x, y)                                     # [m, rows]
        best = {}
        for i in range(x.shape[0]):
            for j in range(y.shape[0]):
                key = (q[i, j], j, i)
                g = int(gid[i])
                if g not in best or key < best[g]:
                    best[g] = key
        ranked = sorted((v, g) for g, v in best.items())[:k]
        out[name] = [(g, j, i - off[g], float(np.sqrt(np.float32(qq)))) for (qq, j, i), g in ranked]
    return out


def test_cli_writes_the_per_file_table(scored):
    root, base, ev = scored
    out = root / "sub" / "nearest.csv"
    assert nearest_cli.main(["vggish", str(root / "base"), str(root / "eval"), str(out), "-k", "2", "-w", "1"]) == 0
    rows = list(csv.reader(out.open()))
    assert rows[0] == ["file", "rank", "nearest_baseline", "distance", "eval_row", "baseline_row", "n_eval"]
    names = {s: str(root / "eval" / f"{s.replace(',', '_')}.wav") for s in ("copy", "far", "near", "x,y")}
    files = [r[0] for r in rows[1:]]
    assert sorted(set(files)) == sorted(names.values())  # the empty and the narrow cache dropped, the comma replaced
    assert all(files.count(f) == 2 for f in names.values())
    first = [float(r[3]) for r in rows[1:] if r[1] == "1"]
    assert first == sorted(first) and rows[1][0] == names["copy"] and float(rows[1][3]) == 0.0   # closest first
    emb = root / "base" / "embeddings" / "vggish"
    parts = [base[:20], base[20:20], base[30:60], base[20:30]]
    want = _want(parts, ev, list(names), 2)
    for s, f in names.items():
        got = [r for r in rows[1:] if r[0] == f]
        assert [int(r[1]) for r in got] == [1, 2]
        for r, (g, j, i, dist) in zip(got, want[s]):
            assert r[2] == str(emb / f"{'abcd'[g]}.npy") and float(r[3]) == dist
            assert (int(r[4]), int(r[5]), int(r[6])) == (j, i, ev[s].shape[0])
    copy = [r for r in rows[1:] if r[0] == names["copy"]][0]
    assert copy[2].endswith("c.npy") and (copy[4], copy[5]) == ("3", "7")


def test_existing_table_is_returned_untouched_and_str_names_go_under_data(scored, monkeypatch):
    root, base, _ = scored
    monkeypatch.chdir(root)
    fad = fad_mod.FrechetAudioDistance(_ML(), audio_load_worker=1)
    got = fad.score_nearest_individual(root / "base", root / "eval", "t.csv")
    assert got == fad_mod.Path("data") / "nearest-individual" / "vggish" / "t.csv" and got.is_file()
    lines = got.read_text().splitlines()
    assert len(lines) == 1 + 4 * 3                         # k = 5, but three non-empty baseline files
    got.write_text("kept\n")
    assert fad.score_nearest_individual(root / "base", root / "eval", "t.csv") == got and got.read_text() == "kept\n"
    with pytest.raises(ValueError, match="k in \\[1, 16\\]"):
        fad.score_nearest_individual(root / "base", root / "eval", "u.csv", k=0)
    _caches(root, {"void": {"a": base[:0]}})
    with pytest.raises(ValueError, match="at least one baseline row"):
        fad.score_nearest_individual(root / "void", root / "eval", "u.csv")
    assert not (root / "data" / "nearest-individual" / "vggish" / "u.csv").exists()
