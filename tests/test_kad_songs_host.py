"""Per-song Kernel Audio Distance without a GPU: the fp64 per-song sums (song_kernel_sums, used by the GPU tests too)
against the definition written as a double loop, the argument errors of calc_kernel_audio_distance_songs and of
``python -m fadtk_b200.kad --indiv``, and the per-file table of score_kad_individual (sorting, naming, dropped files),
with the device calls replaced by the oracle."""
import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native, fad as fad_mod, kad as kad_cli
from oracle import kad_oracle as ko


def song_kernel_sums(x, songs, sigma):
    """fp64 S_xx (i < j) of x and, per song y_k, (S_yy,k (i < j), S_xy,k (all pairs)) of exp(-|a - b|^2 / (2 sigma^2));
    every set centred on the mean of x, as kad_oracle.kernel_sums does for one eval set."""
    xc, *ycs = ko._centred(x, *songs)
    c = 1.0 / (2.0 * sigma * sigma)

    def total(a, b, upper):
        return float(sum(np.exp(-q * c).sum() for q in ko._pair_blocks(a, b, upper)))
    return total(xc, xc, True), [(total(y, y, True), total(xc, y, False)) for y in ycs]


def _rows(m, d, seed, offset=0.0):
    return (offset + np.random.default_rng(seed).standard_normal((m, d))).astype(np.float16)


@pytest.mark.parametrize("m", [2, 5, 6])
def test_song_sums_match_double_loop_per_song(m):
    x = _rows(m, 16, 1, 30.0)
    songs = [_rows(n, 16, 10 + n, 30.4) for n in (2, 3, 5)]
    sigma = ko.bandwidth(x)
    s_xx, per_song = song_kernel_sums(x, songs, sigma)
    for y, (s_yy, s_xy) in zip(songs, per_song):
        want, sigma_d = ko.kad_direct(x, y)
        assert abs(sigma - sigma_d) <= 1e-12 * sigma_d
        got = 1000.0 * ko.mmd2_unbiased(s_xx, s_yy, s_xy, m, y.shape[0])
        assert abs(got - want) <= 1e-9 * max(1.0, abs(want)), (got, want)


def test_song_sums_of_empty_and_single_row_songs():
    x = _rows(4, 8, 2)
    s_xx, per_song = song_kernel_sums(x, [_rows(0, 8, 3), _rows(1, 8, 4)], 1.5)
    assert s_xx == ko.kernel_sums(x, _rows(2, 8, 5), 1.5)[0]
    assert per_song[0] == (0.0, 0.0)
    assert per_song[1][0] == 0.0 and per_song[1][1] > 0.0


def test_bad_inputs():
    x = _rows(4, 8, 5)
    with pytest.raises(ValueError, match="fp16"):
        fk.calc_kernel_audio_distance_songs(x.astype(np.float32), [_rows(4, 8, 6)])
    with pytest.raises(ValueError, match="fp16"):
        fk.calc_kernel_audio_distance_songs(x, [_rows(4, 8, 6), _rows(4, 8, 7).astype(np.float32)])
    with pytest.raises(ValueError, match="widths differ"):
        fk.calc_kernel_audio_distance_songs(x, [_rows(4, 8, 6), _rows(4, 16, 7)])
    with pytest.raises(ValueError, match=r"\[rows, d\]"):
        fk.calc_kernel_audio_distance_songs(x, [_rows(4, 8, 6)[None]])
    for m in (0, 1):
        with pytest.raises(ValueError, match="at least two"):
            fk.calc_kernel_audio_distance_songs(_rows(m, 8, 5), [_rows(4, 8, 6)])


class _OracleEngine:
    """Stands in for _native.Engine: the KAD stages computed by the oracle on the host."""
    torch_device = torch.device("cpu")

    def __init__(self):
        self.widths = []

    def kad_median_sq(self, x):
        self.widths.append(x.shape[1])
        return torch.tensor(ko.middle_sq(x.numpy()), dtype=torch.float64)

    def kad_song_sums(self, z, m, offsets, sigma):
        zn, off = z.numpy(), offsets.numpy()
        s_xx, per_song = song_kernel_sums(zn[:m], [zn[m + a:m + b] for a, b in zip(off[:-1], off[1:])], float(sigma[0]))
        return torch.tensor([s_xx] + [v for pair in per_song for v in pair], dtype=torch.float64)


@pytest.fixture
def oracle_engine(monkeypatch):
    eng = _OracleEngine()
    monkeypatch.setattr(_native, "engine", lambda *a, **k: eng)
    return eng


def test_songs_match_the_whole_set_definition(oracle_engine):
    """each song's result is the KAD of (baseline, song); short songs are NaN; the width is zero-padded to 104"""
    x = _rows(30, 100, 7)
    songs = [_rows(n, 100, 20 + n, 0.2) for n in (5, 0, 2, 1, 9)]
    got = fk.calc_kernel_audio_distance_songs(x, songs)
    assert oracle_engine.widths == [104]
    assert [r.n_eval for r in got] == [5, 0, 2, 1, 9] and all(r.n_baseline == 30 for r in got)
    for y, r in zip(songs, got):
        if y.shape[0] < 2:
            assert np.isnan(r.score)
            continue
        want, sigma = ko.kad(x, y)
        assert abs(r.bandwidth - sigma) <= 1e-12 * sigma and abs(r.score - want) <= 1e-9 * abs(want), (r, want)
    assert fk.calc_kernel_audio_distance_songs(x, []) == []


class _ML:
    name = "vggish"


def _fad():
    fad = fad_mod.FrechetAudioDistance.__new__(fad_mod.FrechetAudioDistance)
    fad.ml, fad.audio_load_worker = _ML(), 1
    return fad


def _cache(directory, stem, arr):
    emb = directory / "embeddings" / "vggish"
    emb.mkdir(parents=True, exist_ok=True)
    np.save(emb / f"{stem}.npy", arr)


def test_score_kad_individual_table(oracle_engine, tmp_path, monkeypatch):
    """rows file,score sorted by |score| under data/kad-individual/<model>/, commas in names replaced, no header;
    missing, non-fp16 and one-row caches dropped; a second call returns the table untouched"""
    monkeypatch.chdir(tmp_path)
    base, ev = tmp_path / "base", tmp_path / "eval"
    base.mkdir()
    ev.mkdir()
    x = _rows(40, 16, 30)
    _cache(base, "b0", x[:25])
    _cache(base, "b1", x[25:])
    songs = {"far": _rows(6, 16, 31, 1.0), "near": _rows(7, 16, 32), "mid,dle": _rows(5, 16, 33, 0.5),
             "short": _rows(1, 16, 34), "f32": _rows(4, 16, 35).astype(np.float32)}
    for stem, y in songs.items():
        (ev / f"{stem}.wav").write_bytes(b"")
        _cache(ev, stem, y)
    (ev / "uncached.wav").write_bytes(b"")
    out = _fad().score_kad_individual(base, ev, "t.csv")
    assert out.resolve() == tmp_path / "data" / "kad-individual" / "vggish" / "t.csv"
    rows = [line.rsplit(",", 1) for line in out.read_text().split("\n")]
    want = {str(ev / f"{k}.wav").replace(",", "_"): ko.kad(x, songs[k])[0] for k in ("far", "near", "mid,dle")}
    assert [r[0] for r in rows] == sorted(want, key=lambda k: abs(want[k]))
    for name, score in rows:
        assert abs(float(score) - want[name]) <= 1e-9 * abs(want[name])
    before = out.read_text()
    _cache(ev, "near", _rows(7, 16, 36))
    assert _fad().score_kad_individual(base, ev, "t.csv") == out and out.read_text() == before


def test_score_kad_individual_refuses_bad_baselines(oracle_engine, tmp_path):
    ev = tmp_path / "eval"
    ev.mkdir()
    npz = tmp_path / "s.npz"
    np.savez(npz, a=np.zeros(1))
    with pytest.raises(ValueError, match="statistics"):
        _fad().score_kad_individual(npz, ev, tmp_path / "a.csv")
    with pytest.raises(ValueError, match="no vggish embeddings"):
        _fad().score_kad_individual(tmp_path / "eval", ev, tmp_path / "a.csv")
    one = tmp_path / "one"
    _cache(one, "b", _rows(1, 16, 1))
    (ev / "s.wav").write_bytes(b"")
    _cache(ev, "s", _rows(3, 16, 2))
    with pytest.raises(ValueError, match="at least two"):
        _fad().score_kad_individual(one, ev, tmp_path / "a.csv")
    f32 = tmp_path / "f32"
    _cache(f32, "b", _rows(5, 16, 1).astype(np.float32))
    with pytest.raises(ValueError, match="fp16"):
        _fad().score_kad_individual(f32, ev, tmp_path / "a.csv")
    assert not (tmp_path / "a.csv").exists()


@pytest.fixture
def cli(monkeypatch, tmp_path):
    monkeypatch.setattr(kad_cli, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(kad_cli, "_embed_directories", lambda *a: pytest.fail("embedding started before the checks"))
    (tmp_path / "base").mkdir()
    (tmp_path / "eval").mkdir()
    return tmp_path


def test_indiv_cli_refuses_statistics(cli):
    npz = cli / "base.npz"
    np.savez(npz, **{"vggish.mu": np.zeros(128), "vggish.cov": np.eye(128)})
    with pytest.raises(ValueError, match="not \\(mu, C\\) statistics"):
        kad_cli.main(["vggish", str(npz), str(cli / "eval"), "--indiv"])
    with pytest.raises(ValueError, match="not \\(mu, C\\) statistics"):
        kad_cli.main(["vggish", str(cli / "base"), str(npz), "--indiv"])


def test_indiv_cli_keeps_an_existing_table(cli, monkeypatch):
    """the aggregate table's header check does not apply to --indiv, and an existing per-file table is not rewritten"""
    monkeypatch.setattr(kad_cli, "_embed_directories", lambda *a: None)
    out = cli / "table.csv"
    out.write_text("model,baseline,eval,score,inf_r2,time\n")
    assert kad_cli.main(["vggish", str(cli / "base"), str(cli / "eval"), str(out), "--indiv"]) == 0
    assert out.read_text() == "model,baseline,eval,score,inf_r2,time\n"
