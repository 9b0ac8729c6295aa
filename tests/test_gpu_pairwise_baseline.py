"""A prepared baseline on the H100 (DESIGN.md 5.15): the radius lists (prdc_tile_kernel<6>), the eval-only passes
(fad_kad_eval_sums, fad_knn_eval_radii_sq, fad_realism_prepared) and the Python layer on top of them, each bitwise
equal to the unprepared call it stands in for, for one and many local shards; KAD against the fp64 oracle; rejected
calls; and a save / load round trip."""
import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native
from gpu_checks import Guarded, expect_rejected
from oracle import kad_oracle as ko
from test_gpu_kad import clap_like, encodec_like

pytestmark = pytest.mark.gpu

SHARDS = [1, 2, 3, 7, 8, 64]          # 64: more shards than units at the small shapes


def gaussian(rows, d, seed, shift=0.0):
    return (shift + np.random.default_rng(seed).standard_normal((rows, d))).astype(np.float16)


def duplicates(rows, d, seed, shift=0.0):
    """every row three times: radii of 0 up to k = 2, and ties everywhere"""
    base = gaussian((rows + 2) // 3, d, seed, shift)
    return np.repeat(base, 3, axis=0)[:rows]


def sigma_ties(rows, d, seed, shift=0.0):
    """rows on a coarse integer grid: many equal pair distances, the two middle ones among them"""
    return (np.random.default_rng(seed).integers(0, 3, (rows, d)) + shift).astype(np.float16)


DATA = {"gauss": gaussian, "encodec": encodec_like, "clap": clap_like, "dup": duplicates, "ties": sigma_ties}


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _padded(a):
    return np.pad(a, ((0, 0), (0, -a.shape[1] % 8)))


def _bits(t):
    a = t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    return a.view(np.uint32 if a.dtype.itemsize == 4 else np.uint64)


def _songs(n_rows, seed):
    """file lengths with one-row and empty files among them, summing to n_rows"""
    rng = np.random.default_rng(seed)
    cuts = np.sort(rng.choice(np.arange(1, n_rows), size=min(6, n_rows - 1), replace=False))
    off = np.concatenate([[0], cuts, [n_rows]]).astype(np.int64)
    return np.insert(off, 2, off[1])   # an empty file


# ------------------------------------------------------------------------------------------------ device entries
@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("m,d", [(17, 8), (300, 128), (1000, 40)])
def test_lists_are_the_radii_at_every_k(engine, kind, m, d):
    x = _padded(DATA[kind](m, d, 1))
    xd = _dev(x)
    lists = engine.knn_lists_sq(xd, 16)
    ref = _dev(np.concatenate([x, x[:17]]))          # 17 eval rows stand in for the absent Y
    for k in range(1, 17):
        r = engine.knn_radii_sq(ref, m, k)[:m]
        assert np.array_equal(_bits(lists[:, k - 1].contiguous()), _bits(r)), (kind, k)
    assert bool((lists[:, 1:] >= lists[:, :-1]).all())
    for s in SHARDS:
        assert np.array_equal(_bits(engine.knn_lists_sq(xd, 16, s)), _bits(lists)), s


@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("m,n,d", [(40, 100, 16), (300, 257, 128), (129, 1000, 512)])
def test_eval_passes_are_bitwise_the_unprepared_ones(engine, kind, m, n, d):
    x, y = DATA[kind](m, d, 2), DATA[kind](n, d, 3, 0.3)
    z = _dev(_padded(np.concatenate([x, y])))
    off = _songs(n, 4)
    offd = _dev(off)
    ymask = np.diff(off) > 5                          # per-song radii need more than k rows per song
    # KAD: fad_kad_eval_sums against fad_kad_song_sums
    sq = engine.kad_median_sq(z[:m]).cpu().numpy()
    sig = torch.tensor([0.5 * (np.sqrt(sq[0]) + np.sqrt(sq[1]))], dtype=torch.float64, device="cuda")
    if sig.item() > 0:
        want = engine.kad_song_sums(z, m, offd, sig)
        one = _dev(np.array([0, n], dtype=np.int64))
        for s in [None] + SHARDS:
            got = engine.kad_eval_sums(z, m, offd, sig, s)
            assert np.array_equal(_bits(got.reshape(-1)), _bits(want[1:])), s
            got1 = engine.kad_eval_sums(z, m, one, sig, s)
            assert np.array_equal(_bits(got1.reshape(-1)), _bits(engine.kad_song_sums(z, m, one, sig)[1:])), s
    # PRDC radii: the Y part of the whole-set and the per-song radii
    k = 5
    whole = engine.knn_radii_sq(z, m, k)[m:]
    kept_off = np.concatenate([[0], np.cumsum(np.diff(off)[ymask])]).astype(np.int64)
    zs = _dev(_padded(np.concatenate([x] + [y[a:b] for a, b, ok in zip(off[:-1], off[1:], ymask) if ok])))
    per_song = engine.knn_song_radii_sq(zs, m, _dev(kept_off), k)[m:]
    for s in [None] + SHARDS:
        assert np.array_equal(_bits(engine.knn_eval_radii_sq(z, m, k, None, s)), _bits(whole)), s
        assert np.array_equal(_bits(engine.knn_eval_radii_sq(zs, m, k, _dev(kept_off), s)), _bits(per_song)), s
    # realism: the tile pass alone on fad_realism's kept radii
    kept, real, near, near_sq, _ = engine.realism(z, m, 3)
    for s in [None] + SHARDS:
        got = engine.realism_prepared(z, m, kept, s)
        for g, w in zip(got, (real, near, near_sq)):
            assert np.array_equal(_bits(g), _bits(w)), s


def test_digest_is_the_row_order_digest(engine):
    x = encodec_like(300, 128, 5)
    a = engine.pair_digest(_dev(x))
    assert a == engine.pair_digest(_dev(x)) and a != engine.pair_digest(_dev(x[::-1]))
    y = x.copy()
    y[123, 45] = np.float16(y[123, 45] + 1)
    assert a != engine.pair_digest(_dev(y))


def test_rejected_calls_launch_and_write_nothing(engine):
    lib = _native.lib()
    m, n, d = 300, 200, 128
    z = _dev(encodec_like(m + n, d, 6))
    zbuf = torch.zeros((m + n) * d + 8, dtype=torch.float16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    lists = Guarded((m, 16), torch.float32, "cuda", 64)
    radii = Guarded((n,), torch.float32, "cuda", 64)
    # fp64 [2] sums and int32 [n] nearest rows: fp32 buffers of the same bytes, sentinel-filled
    sums = Guarded((4,), torch.float32, "cuda", 64)
    reals = [Guarded((n,), torch.float32, "cuda", 64) for _ in range(3)]
    kept = torch.ones(m, dtype=torch.float32, device="cuda")
    sig = torch.ones(1, dtype=torch.float64, device="cuda")
    one = _dev(np.array([0, n], dtype=np.int64))
    bad_off = _dev(np.array([1, n], dtype=np.int64))

    def c(fn, *args, shards=None):
        def run(eng, _):
            f = getattr(lib, fn if shards is None else fn + "_sharded")
            _native._check(f(eng._h, *args, st) if shards is None else f(eng._h, None, shards, *args, st))
        return run

    zp, L, R, S = z.data_ptr(), lists.body.data_ptr(), radii.body.data_ptr(), sums.body.data_ptr()
    rp = [g.body.data_ptr() for g in reals]
    cases = [
        (c("fad_knn_lists_sq", zp, m, d, 0, L), "k must be in [1, 16]"),
        (c("fad_knn_lists_sq", zp, m, d, 17, L), "k must be in [1, 16]"),
        (c("fad_knn_lists_sq", zp, 16, d, 16, L), "PRDC needs more than k rows in each set"),
        (c("fad_knn_lists_sq", zp, m, 124, 16, L), "d must be a positive multiple of 8"),
        (c("fad_knn_lists_sq", zbuf.data_ptr() + 2, m, d, 16, L),
         "pointers must be aligned (z to 16 bytes, the fp32 and int32 arrays to 4)"),
        (c("fad_knn_lists_sq", zp, m, d, 16, lists.buf[65:].data_ptr() - 2),
         "pointers must be aligned (z to 16 bytes, the fp32 and int32 arrays to 4)"),
        (c("fad_knn_lists_sq", zp, m, d, 16, None), "null argument"),
        (c("fad_knn_lists_sq", zp, m, d, 17, L, shards=3), "k must be in [1, 16]"),
        (c("fad_kad_eval_sums", zp, m, one.data_ptr(), 1, d, None, S), "null argument"),
        (c("fad_kad_eval_sums", zp, m, bad_off.data_ptr(), 1, d, sig.data_ptr(), S), "offsets[0] must be 0"),
        (c("fad_kad_eval_sums", zp, 1, one.data_ptr(), 1, d, sig.data_ptr(), S),
         "KAD needs at least two rows in each set"),
        (c("fad_kad_eval_sums", zp, m, one.data_ptr(), 1, 124, sig.data_ptr(), S), "d must be a positive multiple of 8"),
        (c("fad_knn_eval_radii_sq", zp, m, None, n, d, 17, R), "k must be in [1, 16]"),
        (c("fad_knn_eval_radii_sq", zp, m, None, 5, d, 5, R), "PRDC needs more than k rows in each set"),
        (c("fad_knn_eval_radii_sq", zp, 5, None, n, d, 5, R), "PRDC needs more than k rows in each set"),
        (c("fad_knn_eval_radii_sq", zp, m, bad_off.data_ptr(), 1, d, 5, R), "offsets[0] must be 0"),
        (c("fad_knn_eval_radii_sq", zp, m, None, n, d, 5, None), "null argument"),
        (c("fad_realism_prepared", zp, m, 0, d, kept.data_ptr(), *rp),
         "realism needs more than k baseline rows and at least one eval row"),
        (c("fad_realism_prepared", zp, m, n, d, None, *rp), "null argument"),
        (c("fad_realism_prepared", zp, m, n, d, kept.data_ptr(), rp[0], rp[1], None), "null argument"),
        (c("fad_realism_prepared", zp, m, n, 120 + 4, kept.data_ptr(), *rp), "d must be a positive multiple of 8"),
        (c("fad_realism_prepared", zp, m, n, d, kept.data_ptr(), *rp, shards=-1), "local_shards must be >= 0"),
        (c("fad_pair_digest", zbuf.data_ptr() + 2, m, d, S), "pointers must be aligned (z to 16 bytes, out to 8)"),
        (c("fad_pair_digest", zp, m, 12, S), "rows must be >= 0 and d a positive multiple of 8"),
    ]
    for fn, msg in cases:
        expect_rejected(engine, fn, msg, [lists, radii, sums, *reals])


# ------------------------------------------------------------------------------------------------ Python layer
@pytest.mark.parametrize("kind", sorted(DATA))
def test_prepared_results_are_bitwise_the_unprepared_ones(engine, kind):
    m, n, d = 700, 500, 100
    x, y = DATA[kind](m, d, 7), DATA[kind](n, d, 8, 0.3)
    off = _songs(m, 9)
    parts = [x[a:b] for a, b in zip(off[:-1], off[1:])]
    pb = fk.prepare_pairwise_baseline(x, 16, off)
    songs = [y[a:b] for a, b in zip((0, 1, 1, 40, 300), (1, 1, 40, 300, n))]     # one-row and empty songs
    for k in (1, 3, 5, 16):
        assert fk.calc_prdc(pb, y, k) == fk.calc_prdc(x, y, k)
        got, want = fk.calc_prdc_songs(pb, songs, k), fk.calc_prdc_songs(x, songs, k)
        assert np.array_equal(np.array(got, dtype=np.float64), np.array(want, dtype=np.float64), equal_nan=True)
        try:
            want = fk.calc_realism(x, y, k)
        except ValueError:                          # T = 0: more than half of the rows have k duplicates
            with pytest.raises(ValueError, match="threshold is 0"):
                fk.calc_realism(pb, y, k)
            continue
        got = fk.calc_realism(pb, y, k)
        assert got.threshold_sq == want.threshold_sq
        for a in ("realism", "nearest", "nearest_distance"):
            assert np.array_equal(getattr(got, a), getattr(want, a)), (k, a)
        g, w = fk.calc_nearest(pb, y, k), fk.calc_nearest(parts, y, k)
        for a in ("rows", "groups", "distance"):
            assert np.array_equal(getattr(g, a), getattr(w, a)), (k, a)
    if pb.sigma > 0:
        whole = fk.calc_kernel_audio_distance_songs(x, [y])[0]
        assert fk.calc_kernel_audio_distance(pb, y) == whole
        got = fk.calc_kernel_audio_distance_songs(pb, songs)
        want = fk.calc_kernel_audio_distance_songs(x, songs)
        assert np.array_equal(np.array(got, dtype=np.float64), np.array(want, dtype=np.float64), equal_nan=True)
    with pytest.raises(ValueError, match="k_max >= k"):
        fk.calc_prdc(fk.prepare_pairwise_baseline(x, 4), y, 5)


@pytest.mark.parametrize("d", [8, 128, 768, 1024])
def test_prepared_kad_within_the_oracle_bounds(engine, d):
    x, y = encodec_like(1500, d, 11), encodec_like(900, d, 12, 0.2)
    pb = fk.prepare_pairwise_baseline(x)
    got = fk.calc_kernel_audio_distance(pb, y)
    sigma = ko.bandwidth(x)
    assert abs(got.bandwidth - sigma) <= 1e-6 * sigma
    s_xx, s_yy, s_xy = ko.kernel_sums(x, y, got.bandwidth)
    sums = engine.kad_eval_sums(_dev(_padded(np.concatenate([x, y]))), 1500, _dev(np.array([0, 900])),
                                torch.tensor([got.bandwidth], dtype=torch.float64, device="cuda")).cpu().numpy()[0]
    for g, w in ((pb.s_xx, s_xx), (sums[0], s_yy), (sums[1], s_xy)):
        assert abs(g - w) <= 2e-6 * abs(w), (g, w)


def test_save_load_round_trip(engine, tmp_path):
    x = encodec_like(400, 64, 13)
    off = np.array([0, 150, 400], dtype=np.int64)
    pb = fk.prepare_pairwise_baseline(x, 8, off)
    fp = {"files": 2, "bytes": 1}
    pb.save(tmp_path / "p.npz", fp)
    xd = _dev(x)
    back, why = _native.PairwiseBaseline.load(tmp_path / "p.npz", engine, xd, 8, 64, fp, off)
    assert why == "" and back.digest == pb.digest
    assert (back.sigma, back.s_xx, back.k_max) == (pb.sigma, pb.s_xx, pb.k_max)
    assert np.array_equal(_bits(back.lists), _bits(pb.lists))
    y = encodec_like(200, 64, 14, 0.2)
    assert fk.calc_prdc(back, y, 5) == fk.calc_prdc(pb, y, 5)
    assert fk.calc_kernel_audio_distance(back, y) == fk.calc_kernel_audio_distance(pb, y)
    x2 = x.copy()
    x2[7, 3] += np.float16(1)
    assert _native.PairwiseBaseline.load(tmp_path / "p.npz", engine, _dev(x2), 8, 64, fp, off)[0] is None
    assert _native.PairwiseBaseline.load(tmp_path / "p.npz", engine, xd, 9, 64, fp, off)[0] is None
