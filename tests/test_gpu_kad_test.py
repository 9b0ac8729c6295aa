"""Permutation tests of KAD on the H100 (DESIGN.md 5.16): the label bits (kad_perm_label_kernel) bitwise against the
oracle's rule, every labelling's statistic (kad_perm_tile_kernel) within the oracle's fp16 error scale, the p-values,
the Python layer (calc_kad_test, calc_kad_comparison) against the existing KAD calls, reproducibility, local shards, a
prepared baseline, and rejected calls."""
import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native
from gpu_checks import Guarded, expect_rejected
from oracle import kad_oracle as ko
from oracle import kad_test_oracle as kto
from test_gpu_kad import clap_like, encodec_like

pytestmark = pytest.mark.gpu

DATA = {"encodec": encodec_like, "clap": clap_like}


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def check_p_counts(null, observed, ref):
    """The count of null values at or above the observed one, GPU against oracle: every null value farther than
    6 (e_b + e_0) from the observed one in the oracle must fall on the same side on the GPU, so the counts differ by at
    most the number of near ones (always checked; equal counts, hence equal p-values, when none is near)"""
    ref_null, ref_obs = ref["stats"][1:], ref["stats"][0]
    near = np.abs(ref_null - ref_obs) <= 6.0 * (ref["err"][1:] + ref["err"][0])
    got = np.count_nonzero(null >= observed)
    want = np.count_nonzero(ref_null >= ref_obs)
    assert abs(got - want) <= np.count_nonzero(near), (got, want, np.count_nonzero(near))
    assert np.array_equal(null[~near] >= observed, ref_null[~near] >= ref_obs)


def _bits(engine, n, a, B, seed):
    return engine.perm_labels(n, a, B, seed).cpu().numpy().view(np.uint32)


# a on and off word (32) and tile (128) boundaries, n not a multiple of 128; B = 1500 takes two tile passes
@pytest.mark.parametrize("n,a,B,seed", [(4, 2, 1, 0), (300, 128, 63, 5), (301, 32, 63, 2 ** 64 - 1),
                                        (1000, 517, 999, 11), (777, 2, 1500, 3), (2048, 1024, 64, 9),
                                        (129, 127, 200, 1)])
def test_labels_bitwise(engine, n, a, B, seed):
    got = _bits(engine, n, a, B, seed)
    want = kto.pack_bits(kto.labels(n, a, B, seed))
    assert got.shape == want.shape
    assert np.array_equal(got, want)
    assert np.all(np.unpackbits(got.view(np.uint8), axis=1).sum(1) == a)


@pytest.mark.parametrize("data,d,m,n,B", [("encodec", 128, 700, 500, 63), ("clap", 512, 1200, 800, 127),
                                          ("encodec", 136, 333, 257, 999), ("clap", 768, 2000, 2000, 63),
                                          ("encodec", 128, 300, 300, 1500)])
def test_statistics_within_fp16_scale(engine, capsys, data, d, m, n, B):
    x = DATA[data](m, d, 1)
    y = DATA[data](n, d, 2)
    sigma = fk.calc_kernel_audio_distance(x, y).bandwidth
    ref = kto.kad_test(x, y, sigma, B, 7)
    sig = torch.tensor([sigma], dtype=torch.float64, device="cuda")
    s = engine.kad_perm_sums(_dev(np.concatenate([x, y])), m, sig, B, 7).cpu().numpy()
    stats = kto.test_statistics(s, m, n)
    ratio = np.abs(stats - ref["stats"]) / ref["err"]
    null_sd = float(np.std(ref["stats"][1:]))
    with capsys.disabled():
        print(f"\n[kad_test] {data} d={d} m={m} n={n} B={B}: max |err| / e_b = {ratio.max():.3f}, "
              f"max e_b / null sd = {ref['err'].max() / null_sd:.2e}")
    assert ratio.max() <= 6.0
    check_p_counts(stats[1:], stats[0], ref)


def test_calc_kad_test(engine):
    x, y = encodec_like(900, 128, 3), encodec_like(700, 128, 4, shift=0.02)
    r = fk.calc_kad_test(x, y, permutations=199, seed=5)
    k = fk.calc_kernel_audio_distance(x, y)
    assert r.score == k.score and r.bandwidth == k.bandwidth
    assert (r.n_baseline, r.n_eval, r.permutations, r.seed) == (900, 700, 199, 5)
    assert r.null_scores.shape == (199,)
    assert abs(r.observed - k.score) <= 1e-3 * max(1.0, abs(k.score))
    ref = kto.kad_test(x, y, k.bandwidth, 199, 5)
    check_p_counts(r.null_scores, r.observed, ref)
    assert r.p_value == (1.0 + np.count_nonzero(r.null_scores >= r.observed)) / 200.0
    again = fk.calc_kad_test(x, y, permutations=199, seed=5)
    assert again.p_value == r.p_value and np.array_equal(again.null_scores, r.null_scores)
    assert again.observed == r.observed


def test_planted_shift_and_same_distribution(engine):
    x = encodec_like(600, 128, 1)
    shifted = fk.calc_kad_test(x, encodec_like(500, 128, 2, shift=0.5), permutations=99, seed=1)
    assert shifted.p_value == 1.0 / 100.0
    same = fk.calc_kad_test(x, encodec_like(500, 128, 3), permutations=99, seed=1)
    assert same.p_value > 0.01


def test_comparison(engine):
    x = encodec_like(800, 128, 1)
    a, b = encodec_like(300, 128, 2, shift=0.3), encodec_like(400, 128, 3)
    r = fk.calc_kad_comparison(x, a, b, permutations=299, seed=2)
    ra, rb = fk.calc_kernel_audio_distance_songs(x, [a, b])
    assert r.score_a == ra.score and r.score_b == rb.score and r.difference == ra.score - rb.score
    assert (r.n_baseline, r.n_a, r.n_b) == (800, 300, 400)
    ref = kto.kad_comparison(x, a, b, ra.bandwidth, 299, 2)
    diffs = np.concatenate([[0.0], r.null_differences])
    err = np.abs(r.null_differences - ref["stats"][1:]) / ref["err"][1:]
    assert err.max() <= 6.0

    assert r.p_value == 1.0 / 300.0 == ref["p_value"]
    a2 = encodec_like(300, 128, 4)
    same = fk.calc_kad_comparison(x, a2, b, permutations=299, seed=2)
    assert same.p_value > 1.0 / 300.0
    # the two-sided count against the oracle's: only nulls within 6 (e_b + e_0) of the observed value may differ
    ref2 = kto.kad_comparison(x, a2, b, ra.bandwidth, 299, 2)
    assert np.all(np.abs(same.null_differences - ref2["stats"][1:]) <= 6.0 * ref2["err"][1:])
    near = np.abs(np.abs(ref2["stats"][1:]) - abs(ref2["stats"][0])) <= 6.0 * (ref2["err"][1:] + ref2["err"][0])
    got = round(same.p_value * 300) - 1
    want = np.count_nonzero(np.abs(ref2["stats"][1:]) >= abs(ref2["stats"][0]))
    assert abs(got - want) <= np.count_nonzero(near), (got, want)
    assert diffs.shape == (300,)


def test_local_shards_bitwise(engine):
    x, y = encodec_like(1500, 128, 5), encodec_like(1300, 128, 6)
    z = _dev(np.concatenate([x, y]))
    sig = torch.tensor([fk.calc_kernel_audio_distance(x, y).bandwidth], dtype=torch.float64, device="cuda")
    one = engine.kad_perm_sums(z, 1500, sig, 1100, 4)
    for shards in (1, 2, 3, 7, 64):          # 64: more shards than the 11 units
        assert torch.equal(engine.kad_perm_sums_sharded(z, 1500, sig, 1100, 4, shards), one), shards
    assert torch.equal(engine.kad_perm_sums(z, 1500, sig, 1100, 4), one)


def test_prepared_equals_unprepared(engine):
    x, y, y2 = clap_like(700, 512, 8), clap_like(400, 512, 9, tilt=0.1), clap_like(350, 512, 10)
    pb = fk.prepare_pairwise_baseline(x)
    r, rp = fk.calc_kad_test(x, y, 99, 3), fk.calc_kad_test(pb, y, 99, 3)
    assert rp.score == fk.calc_kernel_audio_distance(pb, y).score
    assert rp.p_value == r.p_value and np.array_equal(rp.null_scores, r.null_scores) and rp.observed == r.observed
    c, cp = fk.calc_kad_comparison(x, y, y2, 99, 3), fk.calc_kad_comparison(pb, y, y2, 99, 3)
    assert cp.p_value == c.p_value and np.array_equal(cp.null_differences, c.null_differences)


def test_rejected_calls_launch_and_write_nothing(engine):
    lib = _native.lib()
    N, a, d = 500, 300, 128
    z = _dev(encodec_like(N, d, 6))
    st = torch.cuda.current_stream().cuda_stream
    sig = torch.ones(1, dtype=torch.float64, device="cuda")
    out = Guarded((2 * 3 * 8,), torch.float32, "cuda", 64)        # fp64 [B + 1][3] for B = 7
    bits = Guarded((8 * 16,), torch.float32, "cuda", 64)          # uint32 [B + 1][16]
    v = torch.ones(N, dtype=torch.float64, device="cuda")

    def c(fn, *args, shards=None):
        def run(eng, _):
            f = getattr(lib, fn if shards is None else fn + "_sharded")
            _native._check(f(eng._h, *args, st) if shards is None else f(eng._h, None, shards, *args, st))
        return run

    zp, O, Bp = z.data_ptr(), out.body.data_ptr(), bits.body.data_ptr()
    side = "a permutation test needs at least two rows on each side"
    cases = [
        (c("fad_kad_perm_sums", zp, N, 1, d, sig.data_ptr(), 7, 0, O), "KAD needs at least two rows in each set"),
        (c("fad_kad_perm_sums", zp, N, N - 1, d, sig.data_ptr(), 7, 0, O), "KAD needs at least two rows in each set"),
        (c("fad_kad_perm_sums", zp, N, a, d, sig.data_ptr(), 0, 0, O), "labellings must be in [1, 9999]"),
        (c("fad_kad_perm_sums", zp, N, a, d, sig.data_ptr(), 10000, 0, O), "labellings must be in [1, 9999]"),
        (c("fad_kad_perm_sums", zp, N, a, 124, sig.data_ptr(), 7, 0, O), "d must be a positive multiple of 8"),
        (c("fad_kad_perm_sums", zp, N, a, d, None, 7, 0, O), "null argument"),
        (c("fad_kad_perm_sums", zp, N, a, d, sig.data_ptr(), 7, 0, None), "null argument"),
        (c("fad_kad_perm_sums", zp + 2, N, a, d, sig.data_ptr(), 7, 0, O), "pointers must be 16-byte aligned"),
        (c("fad_kad_perm_sums", zp, N, a, d, sig.data_ptr(), 0, 0, O, shards=3), "labellings must be in [1, 9999]"),
        (c("fad_kad_perm_sums", zp, N, a, d, sig.data_ptr(), 7, 0, O, shards=-1), "local_shards must be >= 0"),
        (c("fad_perm_labels", N, 1, 7, 0, Bp), side),
        (c("fad_perm_labels", N, N - 1, 7, 0, Bp), side),
        (c("fad_perm_labels", N, a, 0, 0, Bp), "labellings must be in [1, 9999]"),
        (c("fad_perm_labels", N, a, 7, 0, None), "null argument"),
        (c("fad_perm_labels", N, a, 7, 0, Bp + 4), "pointers must be 16-byte aligned"),
        (c("fad_perm_dot", Bp, N, 7, None, O), "null argument"),
        (c("fad_perm_dot", Bp, N, 0, v.data_ptr(), O), "labellings must be in [1, 9999]"),
        (c("fad_perm_dot", Bp, 3, 7, v.data_ptr(), O), side),
    ]
    for fn, msg in cases:
        expect_rejected(engine, fn, msg, [out, bits])


def test_launch_counts(engine):
    N, a, d, B = 700, 400, 128, 1100
    z = _dev(encodec_like(N, d, 6))
    sig = torch.ones(1, dtype=torch.float64, device="cuda") * 20.0
    before = engine.launches
    engine.kad_perm_sums(z, a, sig, B, 0)
    # prologue (3), labels, two tile passes each with its reduce, total, dot, finish
    assert engine.launches - before == 3 + 1 + 2 * 2 + 3
    before = engine.launches
    engine.perm_labels(N, a, B, 0)
    assert engine.launches - before == 1


def test_dot_matches_oracle(engine):
    n, a, B = 1000, 400, 300
    v = np.random.default_rng(0).standard_normal(n)
    bits = engine.perm_labels(n, a, B, 21)
    got = engine.perm_dot(bits, _dev(v)).cpu().numpy()
    want = kto.labels(n, a, B, 21).astype(np.float64) @ v
    assert np.allclose(got, want, rtol=1e-12, atol=1e-9)
    assert np.array_equal(got, engine.perm_dot(bits, _dev(v)).cpu().numpy())


def test_directory_command_line(engine, tmp_path, capsys):
    """FADTK_SYNTHETIC VGGish over synthetic clips: python -m fadtk_b200.kad_test embeds the directories, prints the
    score and p-value and appends one csv row, which equals calc_kad_test / calc_kad_comparison on the cached rows;
    --prepared gives the same p-value"""
    import csv
    from fadtk_b200 import kad_test as cli
    from fadtk_b200 import synth
    for kind, n in (("base", 5), ("eval", 4), ("other", 3)):
        (tmp_path / kind).mkdir()
        for i in range(n):
            synth.write_wav(tmp_path / kind / f"clip{i}.wav",
                            synth.musiclike_clip(i + (10 if kind == "other" else 0), 4.0, 16000,
                                                 baseline=(kind == "base")), 16000)
    out = tmp_path / "kt.csv"
    base, ev, other = (str(tmp_path / k) for k in ("base", "eval", "other"))
    assert cli.main(["vggish", base, ev, str(out), "-w", "2", "--permutations", "199", "--seed", "4"]) == 0
    assert "p-value" in capsys.readouterr().out
    assert cli.main(["vggish", base, ev, str(out), "--versus", other, "--permutations", "99"]) == 0
    assert cli.main(["vggish", base, ev, str(out), "--permutations", "199", "--seed", "4", "--prepared"]) == 0
    rows = list(csv.DictReader(out.open()))
    assert out.read_text().splitlines()[0] == cli.CSV_HEADER.strip() and len(rows) == 3
    load = lambda k: np.concatenate([np.load(f) for f in sorted((tmp_path / k / "embeddings" / "vggish").glob("*.npy"))])  # noqa: E731
    x, y, w = load("base"), load("eval"), load("other")
    t = fk.calc_kad_test(x, y, permutations=199, seed=4)
    r = rows[0]
    assert float(r["kad"]) == t.score and float(r["p_value"]) == t.p_value and float(r["bandwidth"]) == t.bandwidth
    assert (int(r["n_baseline"]), int(r["n_eval"]), r["versus"], r["n_versus"]) == (t.n_baseline, t.n_eval, "", "")
    assert (int(r["permutations"]), int(r["seed"])) == (199, 4)
    c = fk.calc_kad_comparison(x, y, w, permutations=99, seed=0)
    r = rows[1]
    assert (float(r["kad"]), float(r["kad_versus"]), float(r["difference"]), float(r["p_value"])) == \
        (c.score_a, c.score_b, c.difference, c.p_value)
    assert (r["versus"], int(r["n_versus"])) == (other, c.n_b)
    assert float(rows[2]["p_value"]) == t.p_value
    assert (tmp_path / "base" / "stats" / "vggish" / "pairwise.npz").is_file()


def test_score_methods_match_the_functions(engine, tmp_path):
    """FrechetAudioDistance.score_kad_test / score_kad_comparison read the caches as score_kad does"""
    rng = np.random.default_rng(3)
    sets = {}
    for kind, files in (("base", 4), ("eval", 3), ("other", 2)):
        (tmp_path / kind / "embeddings" / "vggish").mkdir(parents=True)
        arrs = [(rng.standard_normal((60 + 7 * i, 128)) + (0.2 if kind == "eval" else 0.0)).astype(np.float16)
                for i in range(files)]
        for i, a in enumerate(arrs):
            np.save(tmp_path / kind / "embeddings" / "vggish" / f"f{i}.npy", a)
        sets[kind] = np.concatenate(arrs)
    fad = fk.FrechetAudioDistance(fk.VGGishModel(), load_model=False)
    t = fad.score_kad_test(tmp_path / "base", tmp_path / "eval", permutations=49, seed=2)
    want = fk.calc_kad_test(sets["base"], sets["eval"], permutations=49, seed=2)
    assert t.p_value == want.p_value and t.score == want.score and np.array_equal(t.null_scores, want.null_scores)
    c = fad.score_kad_comparison(tmp_path / "base", tmp_path / "eval", tmp_path / "other", permutations=49, seed=2)
    want = fk.calc_kad_comparison(sets["base"], sets["eval"], sets["other"], permutations=49, seed=2)
    assert c.p_value == want.p_value and np.array_equal(c.null_differences, want.null_differences)
    cp = fad.score_kad_comparison(tmp_path / "base", tmp_path / "eval", tmp_path / "other", permutations=49, seed=2,
                                  prepared=True)
    assert cp.p_value == c.p_value and np.array_equal(cp.null_differences, c.null_differences)
