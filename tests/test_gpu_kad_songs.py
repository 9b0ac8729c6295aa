"""Per-song Kernel Audio Distance on the H100 (fad_kad_song_sums, csrc/kad.cuh MODE 2) against the fp64 per-song
sums (song_kernel_sums) on the same fp16 rows: S_xx, S_yy,k and S_xy,k at a fixed bandwidth within 2e-6 relative,
with songs that start and end on both sides of 128-row tile edges and one song whose band spans many tiles;
agreement with the whole-set path song by song; user-sized shapes; reproducibility; the ``--indiv`` command line."""
import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import synth
from oracle import kad_oracle as ko
from test_kad_songs_host import song_kernel_sums

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
# song lengths: empty and one-row songs, and songs that start and end on both sides of 128-row tile edges
LENGTHS = [3, 0, 129, 1, 2, 127, 10, 128, 750, 2, 2000, 1, 129, 3, 128, 10]


def _songs(kind, lengths, d, seed):
    gen = DATA[kind]
    step = 0.05 if kind == "encodec" else 0.3
    return [gen(n, d, seed + k, step * (k % 4)) for k, n in enumerate(lengths)]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _fixed_sigma(x):
    return float(np.sqrt(ko.middle_sq(x[:600])[0]))


def _gpu_song_sums(engine, x, songs, sigma):
    off = np.zeros(len(songs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([s.shape[0] for s in songs])
    z = _dev(np.concatenate([x, *songs]))
    out = engine.kad_song_sums(z, x.shape[0], _dev(off), torch.tensor([sigma], dtype=torch.float64, device="cuda"))
    return out.cpu().numpy()


def _check(got, want_xx, want_songs, idx=None):
    idx = range(len(want_songs)) if idx is None else idx
    want = np.array([want_xx] + [v for k in idx for v in want_songs[k]])
    got = np.array([got[0]] + [got[1 + 2 * k + i] for k in idx for i in range(2)])
    rel = np.abs(got - want) / np.where(want == 0.0, 1.0, np.abs(want))
    assert (rel <= 2e-6).all(), (np.argmax(rel), got[np.argmax(rel)], want[np.argmax(rel)], rel.max())


@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("m", [2, 129, 256, 3001])
@pytest.mark.parametrize("d", [128, 512, 768, 1024])
def test_song_sums_match_oracle(engine, kind, m, d):
    x = DATA[kind](m, d, 1)
    songs = _songs(kind, LENGTHS, d, 100)
    sigma = _fixed_sigma(x)
    got = _gpu_song_sums(engine, x, songs, sigma)
    want_xx, want_songs = song_kernel_sums(x, songs, sigma)
    _check(got, want_xx, want_songs)
    for k, s in enumerate(songs):                       # no pair within a song of fewer than two rows, none at all when empty
        if s.shape[0] < 2:
            assert got[1 + 2 * k] == 0.0 and (got[2 + 2 * k] == 0.0) == (s.shape[0] == 0)


@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("m", [129, 3001])
def test_long_song_band(engine, kind, m):
    """a 5000-row song (its band spans 40 tiles) between short songs that share its first and last tiles"""
    x = DATA[kind](m, 128, 2)
    songs = _songs(kind, [10, 5000, 3, 129, 1], 128, 200)
    sigma = _fixed_sigma(x)
    got = _gpu_song_sums(engine, x, songs, sigma)
    _check(got, *song_kernel_sums(x, songs, sigma))


@pytest.mark.parametrize("kind", sorted(DATA))
def test_agrees_with_whole_set_path(engine, kind):
    """KAD_k = calc_kernel_audio_distance(X, Y_k) with the same bandwidth; the S_xy,k of a partition of Y add up to
    fad_kad_sums' S_xy"""
    x = DATA[kind](1500, 128, 3)
    songs = _songs(kind, LENGTHS, 128, 300)
    res = fk.calc_kernel_audio_distance_songs(x, songs)
    assert [r.n_eval for r in res] == LENGTHS
    for y, r in zip(songs, res):
        if y.shape[0] < 2:
            assert np.isnan(r.score)
            continue
        want = fk.calc_kernel_audio_distance(x, y)
        assert r.bandwidth == want.bandwidth and r.n_baseline == want.n_baseline == 1500
        assert abs(r.score - want.score) <= max(1e-4 * abs(want.score), 1e-3), (y.shape[0], r, want)
    sigma = torch.tensor([res[0].bandwidth], dtype=torch.float64, device="cuda")
    whole = engine.kad_sums(_dev(np.concatenate([x, *songs])), 1500, sigma).cpu().numpy()
    parts = _gpu_song_sums(engine, x, songs, res[0].bandwidth)
    assert abs(parts[2::2].sum() - whole[2]) <= 4e-6 * abs(whole[2]), (parts[2::2].sum(), whole[2])


def test_width_not_a_multiple_of_8_is_padded(engine):
    x = clap_like(700, 100, 4)
    songs = [clap_like(n, 100, 40 + n, 0.5) for n in (130, 7, 300)]
    for y, r in zip(songs, fk.calc_kernel_audio_distance_songs(x, songs)):
        want, sigma = ko.kad(x, y)
        assert abs(r.bandwidth - sigma) <= 1e-5 * sigma
        assert abs(r.score - want) <= max(1e-4 * abs(want), 1e-3), (r, want)


def test_user_scale(engine):
    """m = 20 000 (d = 128) against 2 000 songs x 10 rows and against 40 Encodec-like songs x 750 rows; a fixed sample
    of songs checked against the oracle"""
    x = encodec_like(20_000, 128, 5)
    sigma = _fixed_sigma(x)
    short = [encodec_like(10, 128, 1000 + k, 0.02 * (k % 7)) for k in range(2000)]
    long = [encodec_like(750, 128, 5000 + k, 0.05 * (k % 3)) for k in range(40)]
    got_short = _gpu_song_sums(engine, x, short, sigma)
    got_long = _gpu_song_sums(engine, x, long, sigma)
    ks, kl = [0, 1, 12, 13, 500, 1024, 1999], [0, 17, 39]
    want_xx, want = song_kernel_sums(x, [short[k] for k in ks] + [long[k] for k in kl], sigma)
    sample = dict(zip(ks, want[:len(ks)]))
    _check(got_short, want_xx, [sample.get(k, (0.0, 0.0)) for k in range(2000)], ks)
    sample = dict(zip(kl, want[len(ks):]))
    _check(got_long, want_xx, [sample.get(k, (0.0, 0.0)) for k in range(40)], kl)


def test_results_are_bitwise_reproducible(engine):
    x = encodec_like(3001, 128, 6)
    songs = _songs("encodec", LENGTHS + [5000, 17], 128, 400)
    sigma = _fixed_sigma(x)
    a, b = _gpu_song_sums(engine, x, songs, sigma), _gpu_song_sums(engine, x, songs, sigma)
    assert np.array_equal(a, b)


def test_rejections(engine):
    x = encodec_like(10, 128, 7)
    z = _dev(np.concatenate([x, encodec_like(20, 128, 8)]))
    sigma = torch.tensor([1.0], dtype=torch.float64, device="cuda")
    from fadtk_b200._native import NativeError
    for off, msg in (([1, 20], "offsets\\[0\\]"), ([0, 12, 8, 20], "non-decreasing")):
        with pytest.raises(NativeError, match=msg):
            engine.kad_song_sums(z, 10, _dev(np.array(off, dtype=np.int64)), sigma)
    with pytest.raises(NativeError, match="at least two"):
        engine.kad_song_sums(z, 1, _dev(np.array([0, 29], dtype=np.int64)), sigma)


def test_directory_command_line(engine, tmp_path):
    """FADTK_SYNTHETIC VGGish over synthetic clips: --indiv writes one row per file sorted by |score|, equal to
    score_kad_individual and to calc_kernel_audio_distance per file; a one-frame file is dropped; a second run leaves
    the table untouched"""
    from fadtk_b200 import kad as kad_cli
    (tmp_path / "base").mkdir()
    (tmp_path / "eval").mkdir()
    for i in range(4):
        synth.write_wav(tmp_path / "base" / f"clip{i}.wav", synth.musiclike_clip(i, 4.0, 16000, baseline=True), 16000)
    for i in range(5):
        synth.write_wav(tmp_path / "eval" / f"clip,{i}.wav", synth.musiclike_clip(i, 2.0 + i, 16000), 16000)
    synth.write_wav(tmp_path / "eval" / "short.wav", synth.musiclike_clip(9, 1.0, 16000), 16000)
    out = tmp_path / "indiv.csv"
    argv = ["vggish", str(tmp_path / "base"), str(tmp_path / "eval"), str(out), "--indiv", "-w", "2"]
    assert kad_cli.main(argv) == 0
    emb = lambda k, s: np.load(tmp_path / k / "embeddings" / "vggish" / f"{s}.npy")  # noqa: E731
    assert emb("eval", "short").shape[0] == 1
    text = out.read_text()
    rows = [line.rsplit(",", 1) for line in text.split("\n")]
    assert [r[0] for r in rows] == sorted((str(tmp_path / "eval" / f"clip_{i}.wav") for i in range(5)),
                                          key=lambda n: abs(float(dict(rows)[n])))
    again = fk.FrechetAudioDistance(fk.VGGishModel(), load_model=False).score_kad_individual(
        tmp_path / "base", tmp_path / "eval", tmp_path / "again.csv")
    assert again.read_text() == text
    x = np.concatenate([emb("base", f"clip{i}") for i in range(4)])
    for name, score in rows:
        want = fk.calc_kernel_audio_distance(x, emb("eval", "clip," + name.rsplit("_", 1)[1][:-4]))
        assert abs(float(score) - want.score) <= max(1e-4 * abs(want.score), 1e-3), (name, score, want)
    mtime = out.stat().st_mtime_ns
    assert kad_cli.main(argv) == 0
    assert out.read_text() == text and out.stat().st_mtime_ns == mtime
