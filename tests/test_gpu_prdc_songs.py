"""Per-song precision, recall, density and coverage on the H100 (fad_knn_song_radii_sq, fad_prdc_song_counts;
csrc/prdc.cuh PASS 2 and 3) against the fp64 per-song reference (test_prdc_songs_host) and against calc_prdc on each
song.  Every song's pair is evaluated with the operand orientation and chunking calc_prdc(X, Y_k) uses, so the per-song
values must equal calc_prdc's exactly, not within a tolerance: radii bitwise, counts as integers, metrics as floats.
Also: the bounds with oracle radii, shards, reproducibility, rejected calls and the ``--indiv`` command line."""
import csv

import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native, synth
from gpu_checks import Guarded, expect_rejected
from oracle import prdc_oracle as po
from test_gpu_kad import DATA, encodec_like
from test_prdc_songs_host import song_bounds, song_radii

pytestmark = pytest.mark.gpu

# songs that start and end on both sides of 128-row tile edges, a 128-row song, k + 1 rows
LENGTHS = [6, 129, 127, 6, 128, 750, 7, 300, 129, 10, 6]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _songs(kind, lengths, d, seed):
    gen = DATA[kind]
    return [gen(n, d, seed + s, 0.05 * (s % 4)) for s, n in enumerate(lengths)]


def _off(songs):
    off = np.zeros(len(songs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([s.shape[0] for s in songs])
    return off


def _gpu(engine, x, songs, k, radii=None, shards=None):
    """-> (radii [m + n_total], inside [n_total], song_counts [K, 2]) as numpy; radii given: the counts pass alone"""
    z, off = _dev(np.concatenate([x, *songs])), _dev(_off(songs))
    m = x.shape[0]
    if radii is None:
        r = (engine.knn_song_radii_sq(z, m, off, k) if shards is None
             else engine.knn_song_radii_sq_sharded(z, m, off, k, local_shards=shards))
    else:
        r = _dev(radii)
    ins, cnt = (engine.prdc_song_counts(z, m, off, r) if shards is None
                else engine.prdc_song_counts_sharded(z, m, off, r, local_shards=shards))
    return r.cpu().numpy(), ins.cpu().numpy(), cnt.cpu().numpy()


# ------------------------------------------------------------------------------------------------ against fp64
@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("k", [1, 5, 16])
@pytest.mark.parametrize("m,d", [(129, 128), (300, 512), (1000, 768)])
def test_radii_within_bounds(engine, kind, k, m, d):
    """within-song radii in radii_bounds per song; the baseline radii equal fad_knn_radii_sq's X part bitwise"""
    x = DATA[kind](m, d, 1)
    songs = _songs(kind, [max(n, k + 1) for n in LENGTHS], d, 100)
    got, _, _ = _gpu(engine, x, songs, k)
    whole = engine.knn_radii_sq(_dev(np.concatenate([x, songs[0]])), m, k).cpu().numpy()
    assert np.array_equal(got[:m].view(np.uint32), whole[:m].view(np.uint32))
    off = _off(songs)
    for s, y in enumerate(songs):
        lo, hi = po.radii_bounds(x, y, k)
        r = got[m + off[s]:m + off[s + 1]].astype(np.float64)
        bad = np.flatnonzero((r < lo[m:]) | (r > hi[m:]))
        assert bad.size == 0, (s, bad[:5], r[bad[:5]], lo[m:][bad[:5]], hi[m:][bad[:5]])


@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("m,d,k", [(129, 128, 1), (257, 512, 5), (1000, 1024, 16)])
def test_counts_with_oracle_radii(engine, kind, m, d, k):
    """with the fp64 reference's radii (rounded to fp32): inside and the per-song covered / recalled counts within the
    per-song decision bounds, and exact wherever no decision is ambiguous"""
    x = DATA[kind](m, d, 2)
    songs = _songs(kind, [max(n, k + 1) for n in LENGTHS], d, 200)
    radii32 = song_radii(x, songs, k).astype(np.float32)
    _, inside, cnt = _gpu(engine, x, songs, k, radii=radii32)
    b = song_bounds(x, songs, radii32.astype(np.float64))
    for key, got in (("inside", inside), ("covered", cnt[:, 0]), ("recalled", cnt[:, 1])):
        lo, hi = b[key]
        assert ((lo <= got) & (got <= hi)).all(), key
        assert np.array_equal(got[lo == hi], lo[lo == hi]), key


# ------------------------------------------------------------------------------------------------ == calc_prdc
def _equal_per_song(x, songs, k, sample=None):
    res = fk.calc_prdc_songs(x, songs, k=k)
    assert [r.n_eval for r in res] == [s.shape[0] for s in songs]
    for s in (range(len(songs)) if sample is None else sample):
        if songs[s].shape[0] <= k:
            assert np.isnan(res[s].precision)
            continue
        assert res[s] == fk.calc_prdc(x, songs[s], k=k), (s, songs[s].shape[0], res[s])
    return res


@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("k", [1, 5, 16])
def test_equals_calc_prdc_per_song(engine, kind, k):
    """k + 1-row songs, songs straddling tile edges on both sides, a 128-row song, short songs that get NaN"""
    x = DATA[kind](1500, 128, 3)
    songs = _songs(kind, LENGTHS + [k + 1, k, 0, k + 1], 128, 300)
    _equal_per_song(x, songs, k)


@pytest.mark.parametrize("kind", sorted(DATA))
def test_long_songs(engine, kind):
    """a 5 000-row song between short songs sharing its first and last tiles, and a song longer than the span's row
    cap (m = 3 001: 24 X tiles, cap 512 rows) next to songs that fit"""
    x = DATA[kind](3001, 128, 4)
    songs = _songs(kind, [10, 5000, 6, 129, 600, 7, 513, 512], 128, 400)
    _equal_per_song(x, songs, 5)
    off = np.zeros(len(songs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([s.shape[0] for s in songs])
    sp = _native.Engine.prdc_song_spans(off, 3001)
    assert [1, 1] in sp[:, 2:].tolist() and (sp[:, 1] - sp[:, 0]).max() > 512


def test_span_song_cap(engine):
    """24 000 songs of 2 rows with k = 1 against m = 20 000: a row cap of 1 024 rows, so spans of 512 songs; songs
    on both sides of span edges"""
    x = encodec_like(20_000, 128, 5)
    y = encodec_like(48_000, 128, 1000, 0.05)
    songs = [y[2 * s:2 * s + 2] for s in range(24_000)]
    sp = _native.Engine.prdc_song_spans(_off(songs), 20_000)
    assert (sp[:-1, 3] == 512).all() and len(sp) == 47
    _equal_per_song(x, songs, 1, sample=[0, 1, 511, 512, 1023, 1024, 12_287, 12_288, 23_999])


def test_single_song_is_the_whole_set(engine):
    x, y = encodec_like(2500, 256, 6), encodec_like(1800, 256, 7, 0.2)
    assert fk.calc_prdc_songs(x, [y], k=4)[0] == fk.calc_prdc(x, y, k=4)
    radii, inside, cnt = _gpu(engine, x, [y], 4)
    z = _dev(np.concatenate([x, y]))
    want_r = engine.knn_radii_sq(z, 2500, 4)
    want_in, flags = (t.cpu().numpy() for t in engine.prdc_counts(z, 2500, want_r))
    assert np.array_equal(radii.view(np.uint32), want_r.cpu().numpy().view(np.uint32))
    assert np.array_equal(inside, want_in)
    assert cnt.tolist() == [[np.count_nonzero(flags & 1), np.count_nonzero(flags & 2)]]


# ------------------------------------------------------------------------------------------------ shards, repeats
def test_shards_and_repeats_are_bitwise_equal(engine):
    """local_shards 1, 2, 3, 7, 8 and more shards than units give the unsharded outputs; two runs are equal"""
    x = encodec_like(1000, 128, 8)
    songs = _songs("encodec", LENGTHS + [5000, 17], 128, 500)
    want = _gpu(engine, x, songs, 5)
    again = _gpu(engine, x, songs, 5)
    tx, ty = 8, -(-sum(s.shape[0] for s in songs) // 128)
    for a, b in zip(want, again):
        assert np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a, b.view(np.uint32) if b.dtype == np.float32 else b)
    for shards in (1, 2, 3, 7, 8, tx + ty + tx * len(songs) + 3):
        got = _gpu(engine, x, songs, 5, shards=shards)
        assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)), shards
        assert np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2]), shards


# ------------------------------------------------------------------------------------------------ rejections
def test_rejections(engine):
    """bad offsets, a song of at most k rows, k out of range, null and misaligned pointers: NativeError with the
    exact message, nothing launched, nothing written"""
    lib, h = _native.lib(), engine._h
    m, d = 300, 128
    songs = [encodec_like(n, 128, 20 + n) for n in (40, 9, 200)]
    z = _dev(np.concatenate([encodec_like(m, d, 9), *songs]))
    n_total = 249
    good_off = _dev(np.array([0, 40, 49, 249], dtype=np.int64))
    radii_in = engine.knn_song_radii_sq(z, m, good_off, 5)
    torch.cuda.synchronize()

    def ptr(t, kind):
        """the tensor's address, None, or 2 bytes past it (misaligned for 4-byte elements); int32 outputs are float32
        Guarded buffers viewed as int32"""
        return {"ok": t.data_ptr(), "null": None, "odd": t.data_ptr() + 2}[kind]

    def radii_call(off, k=5, zp="ok", rp="ok", n_items=3):
        def call(eng, outs):
            r = Guarded((m + n_total,), torch.float32, "cuda", 64)
            outs.append(r)
            _native._check(lib.fad_knn_song_radii_sq(eng._h, ptr(z, zp), m, _dev(np.array(off, dtype=np.int64)).data_ptr(),
                                                     n_items, d, k, ptr(r.body, rp),
                                                     torch.cuda.current_stream().cuda_stream))
        return call

    def counts_call(off, ip="ok", cp="ok", rp="ok"):
        def call(eng, outs):
            ins = Guarded((n_total,), torch.float32, "cuda", 64)
            cnt = Guarded((3, 2), torch.float32, "cuda", 64)
            outs += [ins, cnt]
            _native._check(lib.fad_prdc_song_counts(eng._h, z.data_ptr(), m,
                                                    _dev(np.array(off, dtype=np.int64)).data_ptr(), len(off) - 1, d,
                                                    ptr(radii_in, rp), ptr(ins.body.view(torch.int32), ip),
                                                    ptr(cnt.body.view(torch.int32), cp),
                                                    torch.cuda.current_stream().cuda_stream))
        return call

    ok = [0, 40, 49, 249]
    cases = [(radii_call([1, 40, 49, 249]), "offsets[0] must be 0"),
             (radii_call([0, 49, 40, 249]), "offsets must be non-decreasing"),
             (radii_call(ok, k=9), "every song needs more than k rows"),
             (radii_call(ok, k=0), "k must be in [1, 16]"),
             (radii_call(ok, k=17), "k must be in [1, 16]"),
             (radii_call(ok, zp="null"), "null argument"),
             (radii_call(ok, rp="null"), "null argument"),
             (radii_call(ok, zp="odd"), "pointers must be aligned (z to 16 bytes, the fp32 and int32 arrays to 4)"),
             (radii_call(ok, rp="odd"), "pointers must be aligned (z to 16 bytes, the fp32 and int32 arrays to 4)"),
             (radii_call([0], n_items=0), "n_items must be >= 1"),
             (counts_call([0, 40, 41, 249]), "every song needs more than k rows"),
             (counts_call([2, 40, 49, 249]), "offsets[0] must be 0"),
             (counts_call(ok, ip="null"), "null argument"),
             (counts_call(ok, cp="null"), "null argument"),
             (counts_call(ok, rp="null"), "null argument"),
             (counts_call(ok, cp="odd"), "pointers must be aligned (z to 16 bytes, the fp32 and int32 arrays to 4)"),
             (counts_call(ok, ip="odd"), "pointers must be aligned (z to 16 bytes, the fp32 and int32 arrays to 4)"),
             (counts_call(ok, rp="odd"), "pointers must be aligned (z to 16 bytes, the fp32 and int32 arrays to 4)")]
    for call, msg in cases:
        expect_rejected(engine, call, msg, [])


# ------------------------------------------------------------------------------------------------ command line
def test_directory_command_line(engine, tmp_path):
    """FADTK_SYNTHETIC VGGish over synthetic clips: --indiv writes the header and one row per file sorted by density,
    each equal to calc_prdc on that file's cache; a file of at most k frames is dropped; a second run keeps the table"""
    from fadtk_b200 import prdc as prdc_cli
    (tmp_path / "base").mkdir()
    (tmp_path / "eval").mkdir()
    for i in range(6):
        synth.write_wav(tmp_path / "base" / f"clip{i}.wav", synth.musiclike_clip(i, 6.0, 16000, baseline=True), 16000)
    for i in range(5):
        synth.write_wav(tmp_path / "eval" / f"clip,{i}.wav", synth.musiclike_clip(i, 4.0 + i, 16000), 16000)
    synth.write_wav(tmp_path / "eval" / "short.wav", synth.musiclike_clip(9, 2.0, 16000), 16000)
    out = tmp_path / "indiv.csv"
    argv = ["vggish", str(tmp_path / "base"), str(tmp_path / "eval"), str(out), "-k", "3", "--indiv", "-w", "2"]
    assert prdc_cli.main(argv) == 0
    emb = lambda k, s: np.load(tmp_path / k / "embeddings" / "vggish" / f"{s}.npy")  # noqa: E731
    assert emb("eval", "short").shape[0] <= 3
    rows = list(csv.reader(out.open()))
    assert rows[0] == ["file", "precision", "recall", "density", "coverage", "n_eval"]
    x = np.concatenate([emb("base", f"clip{i}") for i in range(6)])
    want = {str(tmp_path / "eval" / f"clip_{i}.wav"): fk.calc_prdc(x, emb("eval", f"clip,{i}"), k=3) for i in range(5)}
    assert [r[0] for r in rows[1:]] == sorted(want, key=lambda f: (-want[f].density, f))
    for name, *vals in rows[1:]:
        w = want[name]
        assert [float(v) for v in vals[:4]] == [w.precision, w.recall, w.density, w.coverage] and int(vals[4]) == w.n_eval
    text, mtime = out.read_text(), out.stat().st_mtime_ns
    assert prdc_cli.main(argv) == 0
    assert out.read_text() == text and out.stat().st_mtime_ns == mtime
