"""The bootstrap intervals on the H100 (DESIGN.md 5.18): multiplicities bitwise against the oracle's draw rule, the
weighted record sums against the fp64 oracle and bitwise invariant to unit chunks and resample passes, every FAD
replicate within the batched Frechet bound, every KAD replicate within the fp16 error scale, bitwise reproducibility
and prefixes, prepared equal to unprepared, the Python layer, the directory methods and the command line, rejected
calls and launch counts."""
import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native
from gpu_checks import Guarded, expect_rejected
from oracle import bootstrap_oracle as bo
from oracle import fad_oracle as fo
from oracle import fad_test_oracle as fto
from oracle import kad_test_oracle as kto

pytestmark = pytest.mark.gpu
KAD_C = 6.0                        # S_yy(b) within KAD_C e_b of the fp64 oracle (DESIGN.md 5.18 gives the measured ratio)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def vggish_like(rows, d, seed, shift=0.0):
    rng = np.random.default_rng(seed)
    mix = np.random.default_rng(77 + d).standard_normal((d, d)) / np.sqrt(d)
    return (shift + 0.5 + rng.standard_normal((rows, d)) @ mix).astype(np.float16)


def clap_like_ill(rows, d, seed, shift=0.0):
    """L2-normalised rows with a spectrum falling over three decades (CLAP-like conditioning)"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((rows, d)) * np.logspace(0, -3, d) + 0.05
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


@pytest.mark.parametrize("F,B", [(2, 999), (3, 999), (63, 999), (64, 999), (65, 999), (1000, 999), (1000, 1500),
                                 (100000, 999)])
def test_counts_bitwise(engine, F, B):
    got = engine.boot_counts(F, B, 17).cpu().numpy()
    assert np.array_equal(got, bo.counts(F, B, 17))


def test_weighted_record_sums_oracle_and_bitwise(engine):
    d, F, B = 128, 90, 150
    units = _files("vggish", [3 + (i * 7) % 11 for i in range(F)], d, 4)
    shift = fto.pool_shift(units)
    emb, offs = _pool(units)
    rec = engine.unit_records(emb, offs, _dev(shift))
    cnt = engine.boot_counts(F, B, 5)
    s1 = engine.boot_record_sums(rec, cnt, d)
    assert torch.equal(s1, engine.boot_record_sums(rec, cnt, d))
    r = rec.cpu().numpy()
    c = bo.counts(F, B, 5)
    want = bo.weighted_sums(r, c)
    assert np.all(np.abs(s1.cpu().numpy() - want) <= 1e-14 * bo.weighted_sums(np.abs(r), c) + 1e-300)


def _launches(F, d, B, iters=60):
    """fad_frechet_boot's launches (DESIGN.md 5.18): shift (2), then the records (once in all when every record
    fits), per pass and unit chunk the counts and the weighted sums (and the records when they do not fit), and per
    Frechet group the finalise and the chain"""
    R = 1 + d + d * (d + 1) // 2
    pass_ = max(64, min(1024, (2 ** 31 // (8 * R)) // 64 * 64))
    chunk = min(max(64, min(65535, 2 ** 31 // (8 * R)) // 64 * 64), F)
    chunks = -(-F // chunk)
    resident = chunks == 1
    passes = -(-(B + 1) // pass_)
    G = max(1, min(2 ** 31 // (64 * d * d), 32767, min(pass_, B + 1)))
    groups = sum(-(-min(pass_, B + 1 - l0) // G) for l0 in range(0, B + 1, pass_))
    return 2 + (1 if resident else 0) + passes * chunks * (2 if resident else 3) + groups * (7 + 2 * iters), chunks, passes


def test_chunk_and_pass_invariance(engine):
    """1000 one-row units at d = 1024: three unit chunks and two resample passes, bitwise the stage entries replayed
    over all units at once with the shift the call used"""
    d, F, B = 1024, 1000, 600
    launches, chunks, passes = _launches(F, d, B)
    assert chunks >= 3 and passes >= 2
    units = [DATA["clap"](F, d, 8)[i:i + 1] for i in range(F)]
    base = _native.Baseline(engine, *_baseline("clap", d))
    emb, offs = _pool(units)
    before = engine.launches
    out, shift = base.frechet_boot(emb, offs, B, 3)
    assert engine.launches - before == launches
    rec = engine.unit_records(emb, offs, shift)
    sums = engine.boot_record_sums(rec, engine.boot_counts(F, B, 3), d)
    del rec
    assert torch.equal(out, base.frechet_records(sums, shift))
    o = out.cpu().numpy()
    assert np.all(o[:, 7] == F) and np.isfinite(o[:, 0]).all()


def _bound(o):
    return 2e-6 * np.abs(o[..., 0]) + 1e-7 * (o[..., 5] + o[..., 6])


@pytest.mark.parametrize("kind,d,B", [("vggish", 128, 31), ("clap", 512, 7), ("vggish", 768, 7)])
def test_every_fad_replicate_within_bound(engine, capsys, kind, d, B):
    mu, cov = _baseline(kind, d)
    rng = np.random.default_rng(d)
    lo, hi = (40, 100) if d == 512 else (5, 60)
    units = _files(kind, list(rng.integers(lo, hi, 24)), d, 1, 0.02)
    base = _native.Baseline(engine, mu, cov)
    emb, offs = _pool(units)
    out, shift = base.frechet_boot(emb, offs, B, 6)
    o = out.cpu().numpy()
    ref = bo.fad(mu, cov, units, B, 6, shift.cpu().numpy())
    assert np.array_equal(o[:, 7], ref["counts"] @ np.array([u.shape[0] for u in units]))
    ex = np.array([base.frechet(_dev(st[1]), _dev(st[2])).cpu().numpy()[0] for st in ref["stats"]])
    err, chain = np.abs(o[:, 0] - ref["fad"]), np.abs(ex - ref["fad"])
    with capsys.disabled():
        print(f"\n[bootstrap] FAD {kind} d={d} B={B}: max |err| / bound vs the per-set path "
              f"{(np.abs(o[:, 0] - ex) / _bound(o)).max():.3e}, vs eig {(err / _bound(o)).max():.3e}")
    assert np.all(np.abs(o[:, 0] - ex) <= _bound(o))
    assert np.all(err <= _bound(o) + chain)


def _kad_case(kind, d, lens, seed):
    x = DATA[kind](600, d, seed)
    units = _files(kind, lens, d, seed + 1, 0.05)
    return x, units


@pytest.mark.parametrize("kind,d,lens", [("vggish", 128, [10] * 400), ("clap", 512, list(range(1, 61))),
                                         ("vggish", 768, [50] * 30 + [1, 2, 3])])
def test_every_kad_replicate_within_error_scale(engine, capsys, kind, d, lens):
    B = 15
    x, units = _kad_case(kind, d, lens, 3)
    m = x.shape[0]
    sigma = fk.calc_kernel_audio_distance(x, np.concatenate(units)).bandwidth
    z = _dev(np.concatenate([x] + units))
    offs = _dev(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))
    sig = torch.tensor([sigma], dtype=torch.float64, device="cuda")
    g = engine.kad_eval_sums(z, m, offs, sig)[:, 1].contiguous()
    s = engine.kad_boot_sums(z[m:], offs, sig, g, B, 9).cpu().numpy()
    ref = bo.kad(x, units, sigma, B, 9)
    gd = g.cpu().numpy()
    assert np.array_equal(s[:, 0], ref["sums"][:, 0])
    want_xy = ref["counts"].astype(np.float64) @ gd
    assert np.all(np.abs(s[:, 2] - want_xy) <= 1e-12 * np.abs(want_xy))
    ratio = np.abs(s[:, 1] - ref["sums"][:, 1]) / ref["err"]
    with capsys.disabled():
        print(f"\n[bootstrap] KAD {kind} d={d} n={sum(lens)} F={len(lens)}: max |S_yy err| / e_b = {ratio.max():.3f}")
    assert ratio.max() <= KAD_C


def test_determinism_prefix_and_prepared(engine):
    d = 128
    mu, cov = _baseline("vggish", d)
    units = _files("vggish", [3 + i % 7 for i in range(50)], d, 12)
    base = _native.Baseline(engine, mu, cov)
    emb, offs = _pool(units)
    a, _ = base.frechet_boot(emb, offs, 999, 4)
    b, _ = base.frechet_boot(emb, offs, 999, 4)
    c, _ = base.frechet_boot(emb, offs, 1500, 4)
    assert torch.equal(a, b) and torch.equal(a, c[:1000])
    x = vggish_like(300, d, 13)
    r1 = fk.calc_kad_bootstrap(x, units, resamples=999, seed=4)
    r2 = fk.calc_kad_bootstrap(x, units, resamples=1500, seed=4)
    assert np.array_equal(r1.replicates, r2.replicates[:999]) and r1.observed == r2.observed
    pb = fk.prepare_pairwise_baseline(x)
    rp = fk.calc_kad_bootstrap(pb, units, resamples=999, seed=4)
    assert np.array_equal(rp.replicates, r1.replicates) and rp.observed == r1.observed
    y = np.concatenate(units)
    assert r1.score == fk.calc_kernel_audio_distance_songs(x, [y])[0].score
    assert rp.score == fk.calc_kernel_audio_distance_songs(pb, [y])[0].score
    assert rp.bandwidth == r1.bandwidth


def test_calc_fad_bootstrap_fields(engine):
    d = 128
    mu, cov = _baseline("vggish", d)
    units = _files("vggish", [20] * 25, d, 11, shift=0.4)
    r = fk.calc_fad_bootstrap((mu, cov), units, resamples=199, seed=1)
    rows = np.concatenate(units)
    assert r.score == fk.calc_frechet_distance(mu, cov, *fk.calc_embd_statistics(rows))
    assert (r.n_units, r.n_rows, r.resamples, r.seed, r.level, r.method) == (25, 500, 199, 1, 0.95, "percentile")
    assert r.replicates.shape == (199,) and abs(r.observed - r.score) <= 1e-3 * abs(r.score)
    theta = np.concatenate([[r.observed], r.replicates])
    assert (r.ci_low, r.ci_high, r.standard_error, r.bias) == bo.interval(theta, 0.95, "percentile")
    rb = fk.calc_fad_bootstrap((mu, cov), units, resamples=199, seed=1, level=0.8, method="basic")
    assert np.array_equal(rb.replicates, r.replicates)
    assert (rb.ci_low, rb.ci_high) == bo.interval(theta, 0.8, "basic")[:2]
    assert r.ci_low < r.observed + r.bias < r.ci_high and r.standard_error > 0
    per_row = fk.calc_fad_bootstrap((mu, cov), rows[:100], resamples=19)
    assert per_row.n_units == 100


def _cache(root, kind, arrs):
    e = root / kind / "embeddings" / "vggish"
    e.mkdir(parents=True)
    for i, x in enumerate(arrs):
        np.save(e / f"f{i:02d}.npy", x)


def test_directory_methods_and_command_line(engine, tmp_path, monkeypatch, capsys):
    import csv
    from fadtk_b200 import bootstrap as cli
    d = 128
    sets = {"base": _files("vggish", [40] * 10, d, 21), "eval": _files("vggish", [9, 12, 2, 15, 11, 8], d, 22, 0.1)}
    for k, arrs in sets.items():
        _cache(tmp_path, k, arrs)
    fad = fk.FrechetAudioDistance(fk.VGGishModel(), load_model=False)
    base, ev = str(tmp_path / "base"), str(tmp_path / "eval")
    r = fad.score_fad_bootstrap(base, ev, resamples=49, seed=2)
    mu, cov = fad.load_stats(base)
    want = fk.calc_fad_bootstrap((mu, cov), sets["eval"], resamples=49, seed=2)
    assert r.score == float(fad.score(base, ev)) and r.observed == want.observed
    assert np.array_equal(r.replicates, want.replicates) and r.n_units == 6
    k = fad.score_kad_bootstrap(base, ev, resamples=49, seed=2)
    kw = fk.calc_kad_bootstrap(np.concatenate(sets["base"]), sets["eval"], resamples=49, seed=2)
    assert k.score == kw.score and np.array_equal(k.replicates, kw.replicates)
    kp = fad.score_kad_bootstrap(base, ev, resamples=49, seed=2, prepared=True)
    assert np.array_equal(kp.replicates, k.replicates)
    monkeypatch.setattr(cli, "_embed_directories", lambda *a: None)       # the caches are already in place
    out = tmp_path / "boot.csv"
    npz = tmp_path / "stats.npz"          # not base.npz: that would name the base directory's statistics
    np.savez(npz, **{"vggish.mu": mu, "vggish.cov": cov})
    assert cli.main(["fad", "vggish", str(npz), ev, str(out), "--resamples", "49", "--seed", "2"]) == 0
    assert cli.main(["kad", "vggish", base, ev, str(out), "--resamples", "49", "--seed", "2", "--method", "basic",
                     "--level", "0.9"]) == 0
    assert "interval" in capsys.readouterr().out
    assert out.read_text().splitlines()[0] == cli.CSV_HEADER.strip()
    rows = list(csv.DictReader(out.open()))
    assert [row["metric"] for row in rows] == ["fad", "kad"]
    assert (float(rows[0]["score"]), float(rows[0]["ci_low"]), float(rows[0]["ci_high"])) == (r.score, r.ci_low, r.ci_high)
    kb = fk.calc_kad_bootstrap(np.concatenate(sets["base"]), sets["eval"], resamples=49, seed=2, level=0.9,
                               method="basic")
    assert (float(rows[1]["score"]), float(rows[1]["ci_low"]), float(rows[1]["ci_high"])) == (kb.score, kb.ci_low, kb.ci_high)
    assert (rows[1]["method"], float(rows[1]["level"]), int(rows[1]["n_files"]), int(rows[1]["n_rows"])) == \
        ("basic", 0.9, 6, 57)


def test_rejected_calls_launch_and_write_nothing(engine):
    lib = _native.lib()
    d, F, B = 128, 8, 7
    units = _files("vggish", [3] * F, d, 31)
    emb, offs = _pool(units)
    bad_offs = _dev(np.array([0, 3, 3, 9, 12, 15, 18, 21, 24], np.int64))
    from_one = _dev(np.array([1, 3, 6, 9, 12, 15, 18, 21, 24], np.int64))
    base = _native.Baseline(engine, *_baseline("vggish", d))
    st = torch.cuda.current_stream().cuda_stream
    out = Guarded(((B + 1) * 8 * 2,), torch.float32, "cuda", 64)           # fp64 [B + 1][8]
    shift = Guarded((d,), torch.float16, "cuda", 64)
    cnt = Guarded(((B + 1) * F,), torch.float32, "cuda", 64)            # uint32 [B + 1][F]
    R = _native.Engine.record_len(d)
    rec = Guarded((F * R * 2,), torch.float32, "cuda", 64)
    sig = torch.tensor([1.0], dtype=torch.float64, device="cuda")
    g = torch.zeros(F, dtype=torch.float64, device="cuda")
    M, S, C = base.mu.data_ptr(), base.sqrt.data_ptr(), base.scal.data_ptr()
    E, O, O2, SH, Rp, Cn = (emb.data_ptr(), offs.data_ptr(), out.body.data_ptr(), shift.body.data_ptr(),
                            rec.body.data_ptr(), cnt.body.data_ptr())

    def c(fn, *args):
        def run(eng, _):
            _native._check(getattr(lib, fn)(eng._h, *args, st))
        return run

    boot = lambda **k: c("fad_frechet_boot", *[k.get(n, v) for n, v in (  # noqa: E731
        ("mu", M), ("sq", S), ("sc", C), ("emb", E), ("offs", O), ("F", F), ("d", d), ("B", B), ("seed", 0),
        ("iters", 0), ("shift", SH), ("out", O2))])
    kad = lambda **k: c("fad_kad_boot_sums", *[k.get(n, v) for n, v in (  # noqa: E731
        ("y", E), ("offs", O), ("F", F), ("d", d), ("sig", sig.data_ptr()), ("g", g.data_ptr()), ("B", B),
        ("seed", 0), ("out", O2))])
    units_msg = "a bootstrap needs n_units in [2, 2**30]"
    cases = [
        (boot(F=1), units_msg), (boot(B=1), "resamples must be in [2, 9999]"),
        (boot(B=10000), "resamples must be in [2, 9999]"), (boot(d=96), "d must be a positive multiple of 64"),
        (boot(d=2112), "d must be at most 2048"), (boot(out=None), "null argument"), (boot(mu=None), "null argument"),
        (boot(emb=E + 2), "pointers must be 16-byte aligned"),
        (boot(offs=bad_offs.data_ptr()), "offsets must rise: every unit needs at least one row"),
        (boot(offs=from_one.data_ptr()), "offsets[0] must be 0"),
        (kad(F=1), units_msg), (kad(B=1), "resamples must be in [2, 9999]"), (kad(d=12), "d must be a positive multiple of 8"),
        (kad(g=None), "null argument"), (kad(sig=None), "null argument"), (kad(y=E + 2), "pointers must be 16-byte aligned"),
        (kad(offs=bad_offs.data_ptr()), "offsets must rise: every unit needs at least one row"),
        (c("fad_boot_counts", 1, B, 0, Cn), units_msg), (c("fad_boot_counts", F, 10000, 0, Cn), "resamples must be in [2, 9999]"),
        (c("fad_boot_counts", F, B, 0, None), "null argument"),
        (c("fad_boot_record_sums", Rp, F, d, Cn, 1, O2), "resamples must be in [2, 9999]"),
        (c("fad_boot_record_sums", Rp, F, 100, Cn, B, O2), "d must be a positive multiple of 64"),
        (c("fad_boot_record_sums", Rp, F, d, None, B, O2), "null argument"),
    ]
    for fn, msg in cases:
        expect_rejected(engine, fn, msg, [out, shift, cnt, rec])


def test_launch_counts(engine):
    d, F, B = 128, 20, 100
    units = _files("vggish", [4] * F, d, 41)
    base = _native.Baseline(engine, *_baseline("vggish", d))
    emb, offs = _pool(units)
    before = engine.launches
    base.frechet_boot(emb, offs, B, 0)
    assert engine.launches - before == _launches(F, d, B)[0] == 2 + 1 + 2 + 127
    # fad_kad_boot_sums: the pair prologue (3), the unit index, then per pass of up to 1024 resamples the counts, the
    # row weights, the tile pass, the reduction and the unit terms
    sig = torch.tensor([3.0], dtype=torch.float64, device="cuda")
    g = torch.zeros(F, dtype=torch.float64, device="cuda")
    for B, passes in ((100, 1), (1500, 2)):
        before = engine.launches
        engine.kad_boot_sums(emb, offs, sig, g, B, 0)
        assert engine.launches - before == 4 + 5 * passes
