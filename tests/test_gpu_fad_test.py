"""The permutation test of the FAD difference on the H100 (DESIGN.md 5.17): unit records and labelled sums against the
fp64 oracle, bitwise reproducibility, bitwise invariance to unit chunks and labelling passes, every labelling's FAD
within the batched Frechet bound, the p-value counts, the Python layer against the existing FAD functions, the
directory method and the command line, rejected calls and launch counts."""
import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native
from gpu_checks import Guarded, expect_rejected
from oracle import fad_oracle as fo
from oracle import fad_test_oracle as fto
from oracle import kad_test_oracle as kto

pytestmark = pytest.mark.gpu


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def vggish_like(rows, d, seed, shift=0.0):
    rng = np.random.default_rng(seed)
    mix = np.random.default_rng(77 + d).standard_normal((d, d)) / np.sqrt(d)
    return (shift + 0.5 + rng.standard_normal((rows, d)) @ mix).astype(np.float16)


def clap_like_ill(rows, d, seed, shift=0.0):
    """L2-normalised rows with a spectrum falling over three decades (CLAP-like conditioning)"""
    rng = np.random.default_rng(seed)
    scale = np.logspace(0, -3, d)
    x = rng.standard_normal((rows, d)) * scale + 0.05
    x[:, 0] += shift
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float16)


DATA = {"vggish": vggish_like, "clap": clap_like_ill}


def _files(kind, lens, d, seed, shift=0.0):
    return [DATA[kind](n, d, seed * 1000 + i, shift) for i, n in enumerate(lens)]


def _pool(units):
    offs = np.concatenate([[0], np.cumsum([u.shape[0] for u in units])]).astype(np.int64)
    return _dev(np.concatenate(units)), _dev(offs)


def _baseline(kind, d, seed=99):
    mu, cov = fo.embd_statistics(DATA[kind](4 * d, d, seed))
    return mu.astype(np.float64), cov


@pytest.mark.parametrize("d", [128, 512, 768])
def test_records_match_oracle(engine, d):
    lens = [1, 7, 1, 130, 2, 64, 33, 1, 250]
    units = _files("vggish" if d != 512 else "clap", lens, d, 3)
    shift = fto.pool_shift(units)
    emb, offs = _pool(units)
    got = engine.unit_records(emb, offs, _dev(shift)).cpu().numpy()
    want = fto.records(units, shift)
    absrec = fto.records([np.abs(u.astype(np.float64) - shift.astype(np.float64)) for u in units], np.zeros(d, np.float16))
    assert np.array_equal(got[:, 0], want[:, 0])
    scale = absrec[:, 1:].max(1, keepdims=True)
    assert np.all(np.abs(got[:, 1:] - want[:, 1:]) <= 1e-13 * scale)


def test_sums_bitwise_and_oracle(engine):
    d, B = 128, 150
    units = _files("vggish", [3 + (i * 7) % 11 for i in range(90)], d, 4)
    shift = fto.pool_shift(units)
    emb, offs = _pool(units)
    rec = engine.unit_records(emb, offs, _dev(shift))
    bits = engine.perm_labels(90, 37, B, 5)
    s1 = engine.perm_record_sums(rec, bits, d)
    s2 = engine.perm_record_sums(rec, bits, d)
    assert torch.equal(s1, s2)
    r = rec.cpu().numpy()
    lab = kto.labels(90, 37, B, 5)
    want = fto.labelled_sums(r, lab)
    bound = 1e-14 * fto.labelled_sums(np.abs(r), lab) + 1e-300
    assert np.all(np.abs(s1.cpu().numpy() - want) <= bound)


def _launches(F, d, B, iters=60):
    """fad_frechet_perm's launches (DESIGN.md 5.17): shift (2), labels, then per pass and unit chunk the records
    (once in all when every record fits) and the sums, and per Frechet group the finalise and the chain"""
    R = 1 + d + d * (d + 1) // 2
    pass_ = max(64, min(1024, (2 ** 31 // (16 * R)) // 64 * 64))
    chunk = min(max(64, min(65535, 2 ** 31 // (8 * R)) // 64 * 64), F)
    chunks = -(-F // chunk)
    resident = chunks == 1
    passes = -(-(B + 1) // pass_)
    G = max(1, min(2 ** 31 // (64 * d * d), 32767, 2 * min(pass_, B + 1)))
    groups = sum(-(-2 * min(pass_, B + 1 - l0) // G) for l0 in range(0, B + 1, pass_))
    return 3 + (1 if resident else passes * chunks) + passes * chunks + groups * (7 + 2 * iters), chunks, passes


def test_chunk_and_pass_invariance(engine):
    """1000 one-row units at d = 1024: three unit chunks and two labelling passes, bitwise the stage entries replayed
    over all units at once with the shift the call used"""
    d, F, a, B = 1024, 1000, 480, 200
    launches, chunks, passes = _launches(F, d, B)
    assert chunks >= 3 and passes >= 2
    units = [DATA["clap"](F, d, 8)[i:i + 1] for i in range(F)]
    mu, cov = _baseline("clap", d)
    base = _native.Baseline(engine, mu, cov)
    emb, offs = _pool(units)
    before = engine.launches
    out, shift = base.frechet_perm(emb, offs, a, B, 3)
    assert engine.launches - before == launches
    rec = engine.unit_records(emb, offs, shift)
    sums = engine.perm_record_sums(rec, engine.perm_labels(F, a, B, 3), d)
    del rec
    replay = base.frechet_records(sums, shift)
    assert torch.equal(out, replay)
    o = out.cpu().numpy()
    assert np.all(o[:, 0, 7] == a) and np.all(o[:, 1, 7] == F - a) and np.isfinite(o[:, :, 0]).all()


def _bound(o):
    return 2e-6 * np.abs(o[..., 0]) + 1e-7 * (o[..., 5] + o[..., 6])


@pytest.mark.parametrize("kind,d,B", [("vggish", 128, 63), ("clap", 512, 15), ("vggish", 768, 7)])
def test_every_fad_within_bound_and_p_counts(engine, capsys, kind, d, B):
    mu, cov = _baseline(kind, d)
    # ragged files; at d = 512 more rows per file, so that every side has more rows than d (a full-rank covariance,
    # the regime the batched Frechet bound is held to)
    rng = np.random.default_rng(d)
    lo, hi = (40, 100) if d == 512 else (5, 60)
    la, lb = list(rng.integers(lo, hi, 14)), list(rng.integers(lo, hi, 11))
    ua, ub = _files(kind, la, d, 1, 0.02), _files(kind, lb, d, 2)
    base = _native.Baseline(engine, mu, cov)
    emb, offs = _pool(ua + ub)
    out, shift = base.frechet_perm(emb, offs, len(ua), B, 6)
    o = out.cpu().numpy()
    ref = fto.comparison(mu, cov, ua, ub, B, 6, shift=shift.cpu().numpy())
    # the existing per-set path (Baseline.frechet) on the oracle's statistics of every labelled side: the labelled
    # path must match it within the bound, and the eigen-decomposition route within the bound plus the existing
    # path's own distance from it (the Newton-Schulz chain's accuracy on ill-conditioned covariances)
    ex = np.empty_like(ref["fad"])
    for bb in range(B + 1):
        for side in range(2):
            _, m2, c2 = fto.statistics(ref["sums"][bb, side], ref["shift"])
            ex[bb, side] = base.frechet(_dev(m2), _dev(c2)).cpu().numpy()[0]
    err = np.abs(o[:, :, 0] - ref["fad"])
    chain = np.abs(ex - ref["fad"])
    with capsys.disabled():
        print(f"\n[fad_test] {kind} d={d} B={B}: max |err| / bound = {(err / _bound(o)).max():.3e}, vs the per-set "
              f"path {(np.abs(o[:, :, 0] - ex) / _bound(o)).max():.3e}, per-set path vs eig {(chain / _bound(o)).max():.3e}")
    assert np.all(np.abs(o[:, :, 0] - ex) <= _bound(o))
    assert np.all(err <= _bound(o) + chain)
    # p-value counts: only nulls within the error bounds of the observed difference may fall on the other side
    null, obs = o[1:, 0, 0] - o[1:, 1, 0], o[0, 0, 0] - o[0, 1, 0]
    e = _bound(o).sum(1)
    ref_null, ref_obs = ref["stats"][1:], ref["stats"][0]
    near = np.abs(np.abs(ref_null) - abs(ref_obs)) <= e[1:] + e[0]
    assert np.array_equal((np.abs(null) >= abs(obs))[~near], (np.abs(ref_null) >= abs(ref_obs))[~near])
    got, want = np.count_nonzero(np.abs(null) >= abs(obs)), np.count_nonzero(np.abs(ref_null) >= abs(ref_obs))
    assert abs(got - want) <= np.count_nonzero(near)


def test_calc_fad_comparison_fields_and_plausibility(engine):
    d = 128
    mu, cov = _baseline("vggish", d)
    a = _files("vggish", [20] * 25, d, 11, shift=0.4)
    b = _files("vggish", [20] * 25, d, 12)
    r = fk.calc_fad_comparison((mu, cov), a, b, permutations=99, seed=1)
    sa = fk.calc_frechet_distance(mu, cov, *fk.calc_embd_statistics(np.concatenate(a)))
    sb = fk.calc_frechet_distance(mu, cov, *fk.calc_embd_statistics(np.concatenate(b)))
    assert r.score_a == sa and r.score_b == sb and r.difference == sa - sb
    assert (r.n_units_a, r.n_units_b, r.n_rows_a, r.n_rows_b, r.permutations, r.seed) == (25, 25, 500, 500, 99, 1)
    assert r.null_differences.shape == (99,)
    assert abs(r.observed - r.difference) <= 1e-3 * abs(r.difference)
    assert r.p_value == 1.0 / 100.0
    again = fk.calc_fad_comparison((mu, cov), a, b, permutations=99, seed=1)
    assert again.observed == r.observed and np.array_equal(again.null_differences, r.null_differences)
    same = fk.calc_fad_comparison((mu, cov), _files("vggish", [20] * 25, d, 15), b, permutations=99, seed=1)
    assert same.p_value > 0.01
    rows = fk.calc_fad_comparison((mu, cov), np.concatenate(a[:5]), np.concatenate(b[:5]), permutations=19)
    assert (rows.n_units_a, rows.n_units_b) == (100, 100)


def _cache(root, kind, arrs):
    e = root / kind / "embeddings" / "vggish"
    e.mkdir(parents=True)
    for i, x in enumerate(arrs):
        np.save(e / f"f{i:02d}.npy", x)


def test_directory_method_and_command_line(engine, tmp_path, monkeypatch, capsys):
    import csv
    from fadtk_b200 import fad_test as cli
    d = 128
    sets = {"base": _files("vggish", [40] * 10, d, 21), "eval": _files("vggish", [9, 12, 2, 15, 11, 8], d, 22, 0.1),
            "other": _files("vggish", [10, 14, 9, 13, 12], d, 23)}
    for k, arrs in sets.items():
        _cache(tmp_path, k, arrs)
    fad = fk.FrechetAudioDistance(fk.VGGishModel(), load_model=False)
    base, ev, other = (str(tmp_path / k) for k in ("base", "eval", "other"))
    r = fad.score_fad_comparison(base, ev, other, permutations=49, seed=2)
    mu, cov = fad.load_stats(base)
    want = fk.calc_fad_comparison((mu, cov), sets["eval"], sets["other"], permutations=49, seed=2)
    assert r.score_a == float(fad.score(base, ev)) and r.score_b == float(fad.score(base, other))
    assert r.observed == want.observed and r.p_value == want.p_value
    assert np.array_equal(r.null_differences, want.null_differences) and r.n_units_a == 6
    npz = tmp_path / "base.npz"
    np.savez(npz, **{"vggish.mu": mu, "vggish.cov": cov})
    rz = fad.score_fad_comparison(str(npz), ev, other, permutations=49, seed=2)
    assert rz.p_value == r.p_value and np.array_equal(rz.null_differences, r.null_differences)
    monkeypatch.setattr(cli, "_embed_directories", lambda *a: None)       # the caches are already in place
    out = tmp_path / "ft.csv"
    assert cli.main(["vggish", str(npz), ev, other, str(out), "--permutations", "49", "--seed", "2"]) == 0
    assert "p-value" in capsys.readouterr().out
    row = list(csv.DictReader(out.open()))[0]
    assert out.read_text().splitlines()[0] == cli.CSV_HEADER.strip()
    assert (float(row["fad"]), float(row["fad_versus"]), float(row["observed"]), float(row["p_value"])) == \
        (rz.score_a, rz.score_b, rz.observed, rz.p_value)
    assert (int(row["n_files_eval"]), int(row["n_files_versus"]), int(row["permutations"])) == (6, 5, 49)


def test_rejected_calls_launch_and_write_nothing(engine):
    lib = _native.lib()
    d, F, a = 128, 8, 4
    units = _files("vggish", [3] * F, d, 31)
    emb, offs = _pool(units)
    bad_offs = _dev(np.array([0, 3, 3, 9, 12, 15, 18, 21, 24], np.int64))
    from_one = _dev(np.array([1, 3, 6, 9, 12, 15, 18, 21, 24], np.int64))
    mu, cov = _baseline("vggish", d)
    base = _native.Baseline(engine, mu, cov)
    st = torch.cuda.current_stream().cuda_stream
    out = Guarded((8 * 2 * 8 * 2,), torch.float32, "cuda", 64)            # fp64 [B + 1][2][8] for B = 7
    shift = Guarded((d,), torch.float16, "cuda", 64)
    R = _native.Engine.record_len(d)
    rec = Guarded((F * R * 2,), torch.float32, "cuda", 64)                # fp64 [F][R]
    bits = engine.perm_labels(F, a, 7, 0)
    M, S, C = base.mu.data_ptr(), base.sqrt.data_ptr(), base.scal.data_ptr()
    E, O, O2, SH, Rp = emb.data_ptr(), offs.data_ptr(), out.body.data_ptr(), shift.body.data_ptr(), rec.body.data_ptr()

    def c(fn, *args):
        def run(eng, _):
            _native._check(getattr(lib, fn)(eng._h, *args, st))
        return run

    side = "a permutation test needs at least two units on each side"
    perm = lambda **k: c("fad_frechet_perm", *[k.get(n, v) for n, v in (  # noqa: E731
        ("mu", M), ("sq", S), ("sc", C), ("emb", E), ("offs", O), ("F", F), ("a", a), ("d", d), ("B", 7), ("seed", 0),
        ("iters", 0), ("shift", SH), ("out", O2))])
    cases = [
        (perm(a=1), side), (perm(a=F - 1), side), (perm(B=0), "labellings must be in [1, 9999]"),
        (perm(B=10000), "labellings must be in [1, 9999]"), (perm(d=96), "d must be a positive multiple of 64"),
        (perm(out=None), "null argument"), (perm(mu=None), "null argument"),
        (perm(emb=E + 2), "pointers must be 16-byte aligned"),
        (perm(offs=bad_offs.data_ptr()), "offsets must rise: every unit needs at least one row"),
        (perm(offs=from_one.data_ptr()), "offsets[0] must be 0"),
        (c("fad_unit_records", E, O, F, 96, SH, Rp), "d must be a positive multiple of 64"),
        (c("fad_unit_records", E, bad_offs.data_ptr(), F, d, SH, Rp), "offsets must rise: every unit needs at least one row"),
        (c("fad_perm_record_sums", Rp, F, d, bits.data_ptr(), 0, O2), "labellings must be in [1, 9999]"),
        (c("fad_perm_record_sums", Rp, F, d, None, 7, O2), "null argument"),
        (c("fad_frechet_records", M, S, C, Rp, 0, d, SH, 0, O2), "items must be in [1, 2**30]"),
        (c("fad_frechet_records", M, S, C, Rp, 4, 100, SH, 0, O2), "d must be a positive multiple of 64"),
    ]
    for fn, msg in cases:
        expect_rejected(engine, fn, msg, [out, shift, rec])


def test_launch_count_one_pass(engine):
    d, F, a, B = 128, 20, 9, 100
    units = _files("vggish", [4] * F, d, 41)
    mu, cov = _baseline("vggish", d)
    base = _native.Baseline(engine, mu, cov)
    emb, offs = _pool(units)
    before = engine.launches
    base.frechet_perm(emb, offs, a, B, 0)
    assert engine.launches - before == _launches(F, d, B)[0] == 3 + 1 + 1 + 127
