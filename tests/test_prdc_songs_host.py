"""Per-song precision, recall, density and coverage without a GPU: the fp64 per-song reference (song_radii, song_counts,
song_bounds, used by the GPU tests too) against the definition written as a double loop on each song; the span cut of
the counts pass (fad_prdc_song_spans, host only); and calc_prdc_songs, score_prdc_individual and
``python -m fadtk_b200.prdc --indiv`` with the device calls replaced by the oracle."""
import csv

import numpy as np
import pytest
import torch
from hypothesis import given, settings, strategies as st

import fadtk_b200 as fk
from fadtk_b200 import _native, fad as fad_mod, prdc as prdc_cli
from oracle import prdc_oracle as po


def _offsets(songs):
    off = np.zeros(len(songs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([s.shape[0] for s in songs])
    return off


def song_radii(x, songs, k):
    """fp64 [m + n_total]: r_i^2 within x, then s_j^2 of every song's rows within that song"""
    m = x.shape[0]
    return np.concatenate([po.radii_sq(x, songs[0], k)[:m]] + [po.radii_sq(x, y, k)[m:] for y in songs])


def _per_song(x, songs, radii):
    m, off = x.shape[0], _offsets(songs)
    for s, y in enumerate(songs):
        yield s, y, np.concatenate([radii[:m], radii[m + off[s]:m + off[s + 1]]])


def song_counts(x, songs, radii):
    """radii [m + n_total] (r^2, then each song's s^2) -> (inside int64 [n_total], song_counts int64 [K, 2]: covered,
    recalled baseline rows per song), exact strict comparisons"""
    inside, per_song = [], np.zeros((len(songs), 2), dtype=np.int64)
    for s, y, r in _per_song(x, songs, radii):
        ins, flags = po.counts(x, y, r)
        inside.append(ins)
        per_song[s] = np.count_nonzero(flags & 1), np.count_nonzero(flags & 2)
    return np.concatenate(inside), per_song


def song_bounds(x, songs, radii, tau=po.TAU):
    """decision_bounds per song: {"inside": (lo, hi) [n_total], "covered" / "recalled": (lo, hi) int64 [K]}"""
    ins_lo, ins_hi = [], []
    cnt = {key: np.zeros((2, len(songs)), dtype=np.int64) for key in ("covered", "recalled")}
    for s, y, r in _per_song(x, songs, radii):
        b = po.decision_bounds(x, y, r, tau)
        ins_lo.append(b["inside"][0])
        ins_hi.append(b["inside"][1])
        for key in cnt:
            cnt[key][:, s] = np.count_nonzero(b[key][0]), np.count_nonzero(b[key][1])
    return {"inside": (np.concatenate(ins_lo), np.concatenate(ins_hi)),
            "covered": tuple(cnt["covered"]), "recalled": tuple(cnt["recalled"])}


def song_metrics(inside, per_song, off, m, k):
    """[(precision, recall, density, coverage)] per song, as calc_prdc_songs assembles them"""
    out = []
    for s in range(len(off) - 1):
        ins, n = inside[off[s]:off[s + 1]], int(off[s + 1] - off[s])
        out.append((float(np.count_nonzero(ins)) / n, float(per_song[s, 1]) / m,
                    float(ins.sum(dtype=np.int64)) / (k * n), float(per_song[s, 0]) / m))
    return out


def _rows(m, d, seed, offset=0.0):
    return (offset + np.random.default_rng(seed).standard_normal((m, d))).astype(np.float16)


@pytest.mark.parametrize("k", [1, 3, 5])
def test_reference_matches_double_loop_per_song(k):
    """every song's radii, counts and metrics == prdc_direct(x, song), with duplicates and an eval row equal to a
    baseline row (exact ties)"""
    x = _rows(14, 8, 1)
    x[1] = x[0]
    songs = [_rows(n, 8, 10 + n, 0.3 * (n % 3)) for n in (k + 1, 7, 12, k + 2)]
    songs[1][0] = x[3]
    songs[2][4] = songs[2][5]
    radii = song_radii(x, songs, k)
    inside, per_song = song_counts(x, songs, radii)
    off = _offsets(songs)
    got = song_metrics(inside, per_song, off, x.shape[0], k)
    for s, y in enumerate(songs):
        r, ins, flags, want = po.prdc_direct(x, y, k)
        assert np.array_equal(radii[:14], r[:14]) and np.array_equal(radii[14 + off[s]:14 + off[s + 1]], r[14:])
        assert np.array_equal(inside[off[s]:off[s + 1]], ins)
        assert tuple(per_song[s]) == (np.count_nonzero(flags & 1), np.count_nonzero(flags & 2))
        assert got[s] == pytest.approx(want, abs=0, rel=1e-15)
    b = song_bounds(x, songs, radii)
    for key, exact in (("inside", inside), ("covered", per_song[:, 0]), ("recalled", per_song[:, 1])):
        lo, hi = b[key]
        assert ((lo <= exact) & (exact <= hi)).all(), key
    b0 = song_bounds(x, songs, radii, tau=0.0)          # no ambiguity: the bounds are the exact counts
    assert np.array_equal(b0["inside"][0], inside) and np.array_equal(b0["inside"][1], inside)
    assert np.array_equal(b0["covered"][0], per_song[:, 0]) and np.array_equal(b0["recalled"][1], per_song[:, 1])


# ------------------------------------------------------------------------------------------------ span cut
def _row_cap(m, n_total):
    tx, ty = -(-m // 128), -(-n_total // 128)
    return 128 * max(4, -(-(tx * ty) // 8192))


def check_spans(lengths, m):
    off = np.zeros(len(lengths) + 1, dtype=np.int64)
    off[1:] = np.cumsum(lengths)
    sp = _native.Engine.prdc_song_spans(off, m)
    cap = _row_cap(m, int(off[-1]))
    assert sp.ndim == 2 and sp.shape[1] == 4 and sp.shape[0] >= 1
    # in order, no song split: span i = songs [first, first + count), rows [off[first], off[first + count])
    assert sp[0, 2] == 0 and sp[-1, 2] + sp[-1, 3] == len(lengths)
    assert (sp[1:, 2] == sp[:-1, 2] + sp[:-1, 3]).all() and (sp[:, 3] >= 1).all()
    assert (sp[:, 0] == off[sp[:, 2]]).all() and (sp[:, 1] == off[sp[:, 2] + sp[:, 3]]).all()
    rows = sp[:, 1] - sp[:, 0]
    assert (sp[:, 3] <= 512).all()
    assert ((rows <= cap) | (sp[:, 3] == 1)).all()          # the row cap, except for a lone oversized song
    # greedy: a span is closed only when the next song would break a cap
    for i in range(len(sp) - 1):
        nxt = lengths[sp[i + 1, 2]]
        assert sp[i, 3] == 512 or rows[i] + nxt > cap, (i, sp[i], nxt, cap)
    return sp


@settings(max_examples=300, deadline=None)
@given(st.lists(st.integers(1, 3000), min_size=1, max_size=300), st.integers(0, 300_000))
def test_spans_partition_the_songs(lengths, m):
    check_spans(lengths, m)


@settings(max_examples=100, deadline=None)
@given(st.integers(1, 4), st.integers(600, 3000))
def test_spans_song_cap(rows, songs):
    """many short songs: spans of 512 songs until the row cap binds"""
    sp = check_spans([rows] * songs, 100_000)
    assert sp[0, 3] == min(512, songs, _row_cap(100_000, rows * songs) // rows)


def test_span_examples():
    sp = check_spans([100_000], 2000)                       # one long song: one span, Tx units of its own
    assert sp.tolist() == [[0, 100_000, 0, 1]]
    sp = check_spans([10, 600, 10, 10], 100)                # cap 512 rows: the 600-row song alone
    assert sp.tolist() == [[0, 10, 0, 1], [10, 610, 1, 1], [610, 630, 2, 2]]


@pytest.mark.parametrize("off,m,msg", [([1, 5], 10, "offsets\\[0\\]"), ([0, 5, 5], 10, "at least one row"),
                                       ([0, 5, 3], 10, "at least one row"), ([0], 10, "n_items"),
                                       ([0, 1 << 30], 10, "too many rows")])
def test_span_rejections(off, m, msg):
    with pytest.raises(_native.NativeError, match=msg):
        _native.Engine.prdc_song_spans(np.array(off, dtype=np.int64), m)


# ------------------------------------------------------------------------------------------------ Python layer
class _OracleEngine:
    """Stands in for _native.Engine: the per-song PRDC passes computed by the reference above on the host."""
    torch_device = torch.device("cpu")

    def __init__(self):
        self.calls = []

    def _split(self, z, m, offsets):
        zn, off = z.numpy(), offsets.numpy()
        return zn[:m], [zn[m + a:m + b] for a, b in zip(off[:-1], off[1:])]

    def knn_song_radii_sq(self, z, m, offsets, k):
        self.calls.append((tuple(z.shape), offsets.numpy().tolist(), k))
        x, songs = self._split(z, m, offsets)
        return torch.from_numpy(song_radii(x, songs, k))          # fp64: exact ties stay ties

    def prdc_song_counts(self, z, m, offsets, radii_sq):
        x, songs = self._split(z, m, offsets)
        inside, per_song = song_counts(x, songs, radii_sq.numpy())
        return torch.from_numpy(inside.astype(np.int32)), torch.from_numpy(per_song.astype(np.int32))

    def knn_radii_sq(self, z, m, k):                             # the whole-set calc_prdc, for comparison
        zn = z.numpy()
        return torch.from_numpy(po.radii_sq(zn[:m], zn[m:], k))

    def prdc_counts(self, z, m, radii_sq):
        zn = z.numpy()
        inside, flags = po.counts(zn[:m], zn[m:], radii_sq.numpy())
        return torch.from_numpy(inside.astype(np.int32)), torch.from_numpy(flags)


@pytest.fixture
def oracle_engine(monkeypatch):
    eng = _OracleEngine()
    monkeypatch.setattr(_native, "engine", lambda *a, **k: eng)
    return eng


def test_songs_equal_calc_prdc_per_song(oracle_engine):
    """each song's result is calc_prdc(baseline, song); songs of at most k rows are NaN and never sent; the width is
    zero-padded to 104"""
    k = 3
    x = _rows(40, 100, 7)
    lengths = [5, 0, 3, 2, 9, 4]
    songs = [_rows(n, 100, 20 + n, 0.2) for n in lengths]
    got = fk.calc_prdc_songs(x, songs, k=k)
    assert len(oracle_engine.calls) == 1
    shape, off, kk = oracle_engine.calls[0]
    assert shape == (40 + 5 + 9 + 4, 104) and off == [0, 5, 14, 18] and kk == k
    assert [r.n_eval for r in got] == lengths and all(r.n_baseline == 40 and r.k == k for r in got)
    for y, r in zip(songs, got):
        if y.shape[0] <= k:
            assert all(np.isnan(v) for v in r[:4])
            continue
        assert r == fk.calc_prdc(x, y, k=k)
    assert fk.calc_prdc_songs(x, [], k=k) == []
    assert all(np.isnan(r.density) for r in fk.calc_prdc_songs(x, [_rows(2, 100, 1)], k=k))
    assert len(oracle_engine.calls) == 1


def test_bad_inputs(oracle_engine):
    x = _rows(10, 8, 5)
    with pytest.raises(ValueError, match="PRDC needs fp16"):
        fk.calc_prdc_songs(x.astype(np.float32), [_rows(6, 8, 6)])
    with pytest.raises(ValueError, match="PRDC needs fp16"):
        fk.calc_prdc_songs(x, [_rows(6, 8, 6), _rows(6, 8, 7).astype(np.float32)])
    with pytest.raises(ValueError, match="widths differ"):
        fk.calc_prdc_songs(x, [_rows(6, 8, 6), _rows(6, 16, 7)])
    with pytest.raises(ValueError, match=r"\[rows, d\]"):
        fk.calc_prdc_songs(x, [_rows(6, 8, 6)[None]])
    for k in (0, 17, 2.0, True):
        with pytest.raises(ValueError, match="integer k in \\[1, 16\\]"):
            fk.calc_prdc_songs(x, [_rows(20, 8, 6)], k=k)
    with pytest.raises(ValueError, match="more than k"):
        fk.calc_prdc_songs(_rows(5, 8, 5), [_rows(20, 8, 6)], k=5)
    assert not oracle_engine.calls


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


def _read_table(path):
    rows = list(csv.reader(path.open()))
    return rows[0], rows[1:]


def test_score_prdc_individual_table(oracle_engine, tmp_path, monkeypatch):
    """header, rows sorted by density (highest first, ties by path) under data/prdc-individual/<model>/, commas in
    names replaced; missing, non-fp16, wrong-width and <= k-row caches dropped; a second call keeps the table"""
    monkeypatch.chdir(tmp_path)
    base, ev = tmp_path / "base", tmp_path / "eval"
    base.mkdir()
    ev.mkdir()
    x = _rows(40, 16, 30)
    _cache(base, "b0", x[:25])
    _cache(base, "b1", x[25:])
    songs = {"far": _rows(6, 16, 31, 3.0), "near": _rows(7, 16, 32), "mid,dle": _rows(5, 16, 33, 0.5),
             "far2": _rows(6, 16, 34, 3.5), "short": _rows(4, 16, 35), "f32": _rows(6, 16, 36).astype(np.float32),
             "wide": _rows(6, 24, 37)}
    for stem, y in songs.items():
        (ev / f"{stem}.wav").write_bytes(b"")
        _cache(ev, stem, y)
    (ev / "uncached.wav").write_bytes(b"")
    out = _fad().score_prdc_individual(base, ev, "t.csv", k=4)
    assert out.resolve() == tmp_path / "data" / "prdc-individual" / "vggish" / "t.csv"
    header, rows = _read_table(out)
    assert header == ["file", "precision", "recall", "density", "coverage", "n_eval"]
    kept = ("far", "near", "mid,dle", "far2")
    want = {str(ev / f"{s}.wav"): fk.calc_prdc(x, songs[s], k=4) for s in kept}
    order = sorted(want, key=lambda f: (-want[f].density, f))
    assert [r[0] for r in rows] == [f.replace(",", "_") for f in order]
    assert want[str(ev / "far.wav")].density == want[str(ev / "far2.wav")].density == 0.0   # a tie, broken by path
    for (name, *vals), f in zip(rows, order):
        w = want[f]
        assert [float(v) for v in vals[:4]] == [w.precision, w.recall, w.density, w.coverage]
        assert int(vals[4]) == w.n_eval
    before = out.read_text()
    _cache(ev, "near", _rows(7, 16, 38))
    assert _fad().score_prdc_individual(base, ev, "t.csv", k=4) == out and out.read_text() == before


def test_score_prdc_individual_refuses_bad_baselines(oracle_engine, tmp_path):
    ev = tmp_path / "eval"
    ev.mkdir()
    (ev / "s.wav").write_bytes(b"")
    _cache(ev, "s", _rows(8, 16, 2))
    npz = tmp_path / "s.npz"
    np.savez(npz, a=np.zeros(1))
    with pytest.raises(ValueError, match="PRDC needs embeddings"):
        _fad().score_prdc_individual(npz, ev, tmp_path / "a.csv")
    (tmp_path / "empty").mkdir()
    with pytest.raises(ValueError, match="no vggish embeddings"):
        _fad().score_prdc_individual(tmp_path / "empty", ev, tmp_path / "a.csv")
    few = tmp_path / "few"
    _cache(few, "b", _rows(5, 16, 1))
    with pytest.raises(ValueError, match="more than k"):
        _fad().score_prdc_individual(few, ev, tmp_path / "a.csv", k=5)
    f32 = tmp_path / "f32"
    _cache(f32, "b", _rows(9, 16, 1).astype(np.float32))
    with pytest.raises(ValueError, match="fp16"):
        _fad().score_prdc_individual(f32, ev, tmp_path / "a.csv")
    with pytest.raises(ValueError, match="integer k"):
        _fad().score_prdc_individual(few, ev, tmp_path / "a.csv", k=0)
    assert not (tmp_path / "a.csv").exists()


@pytest.fixture
def cli(monkeypatch, tmp_path):
    monkeypatch.setattr(prdc_cli, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(prdc_cli, "_embed_directories", lambda *a: pytest.fail("embedding started before the checks"))
    (tmp_path / "base").mkdir()
    (tmp_path / "eval").mkdir()
    return tmp_path


def test_indiv_cli_writes_the_table(cli, monkeypatch, oracle_engine):
    """--indiv: the default table name, k passed through; the aggregate header check does not apply, and an existing
    table is kept"""
    monkeypatch.setattr(prdc_cli, "_embed_directories", lambda *a: None)
    monkeypatch.setattr(fad_mod.FrechetAudioDistance, "__init__",
                        lambda self, ml, audio_load_worker=8, load_model=True: setattr(self, "ml", ml)
                        or setattr(self, "audio_load_worker", audio_load_worker))
    monkeypatch.chdir(cli)
    x = _rows(30, 16, 40)
    _cache(cli / "base", "b", x)
    for i, n in enumerate((6, 3, 8)):
        (cli / "eval" / f"c{i}.wav").write_bytes(b"")
        _cache(cli / "eval", f"c{i}", _rows(n, 16, 41 + i, 0.1 * i))
    argv = ["vggish", str(cli / "base"), str(cli / "eval"), "-k", "3", "--indiv", "-w", "1"]
    assert prdc_cli.main(argv) == 0
    out = cli / "prdc-individual-results.csv"
    header, rows = _read_table(out)
    assert header[0] == "file" and sorted(r[0] for r in rows) == [str(cli / "eval" / f"c{i}.wav") for i in (0, 2)]
    assert oracle_engine.calls[0][2] == 3
    other = cli / "other.csv"
    other.write_text("model,baseline,eval,score,inf_r2,time\n")
    assert prdc_cli.main(argv[:3] + [str(other)] + argv[3:]) == 0
    assert other.read_text() == "model,baseline,eval,score,inf_r2,time\n"
