"""Per-sample realism and nearest baseline row on the H100 (fad_realism, prdc_tile_kernel<4>) against the fp64 oracle
(oracle/realism_oracle.py) on the same fp16 rows.  The baseline radii are fad_knn_radii_sq's bitwise, the pruning
follows the median rule exactly on them, and from the GPU's own pruned radii every realism lies within
realism_bounds and every nearest index is a candidate of the oracle (the only one where there is one), its
nearest_sq within delta of the exact q.  Also: duplicates, copies and pruned balls, reproducibility, the split of an
eval set, local shards, rejected arguments, the launch counter, and the directory command line."""
import csv
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native, synth
from gpu_checks import Guarded, expect_rejected
from oracle import realism_oracle as ro
from test_gpu_kad import clap_like, encodec_like
from test_gpu_kad_sharded import SHARDS

pytestmark = pytest.mark.gpu


def gaussian(rows, d, seed, shift=0.0):
    return (shift + np.random.default_rng(seed).standard_normal((rows, d))).astype(np.float16)


DATA = {"gauss": gaussian, "encodec": encodec_like, "clap": clap_like}
SHAPES = [("k+5", 1), (129, 127), (3000, 257), (257, 3000)]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _padded(a):
    return np.pad(a, ((0, 0), (0, -a.shape[1] % 8)))


def _sets(kind, m, n, d, seed=0):
    gen = DATA[kind]
    return gen(m, d, 10 + seed), gen(n, d, 20 + seed, 0.3 if kind != "clap" else 0.5)


def _gpu(engine, x, y, k):
    out = engine.realism(_dev(_padded(np.concatenate([x, y]))), x.shape[0], k)
    return tuple(t.cpu().numpy() for t in out[:4]) + (out[4],)


def _check_radii(engine, x, y, k, kept, t):
    """kept = the median rule applied to fad_knn_radii_sq's first m values (X's radii do not depend on Y, so a Y of
    k + 1 rows stands in where the eval set is too small for fad_knn_radii_sq)"""
    yr = y if y.shape[0] > k else x[:k + 1]
    r = engine.knn_radii_sq(_dev(_padded(np.concatenate([x, yr]))), x.shape[0], k).cpu().numpy()[:x.shape[0]]
    want_t = float(np.median(r.astype(np.float64)))
    assert t == want_t
    assert np.array_equal(kept.view(np.uint32), np.where(r.astype(np.float64) <= want_t, r, np.float32(0)).view(np.uint32))


def _check_bounds(x, y, got, what):
    kept, real, near, near_sq, _ = got
    b = ro.realism_bounds(x, y, kept, near)
    bad = np.flatnonzero(~((b["lo"] <= real) & (real <= b["hi"])))
    assert bad.size == 0, (what, "realism", bad[:5], real[bad[:5]], b["lo"][bad[:5]], b["hi"][bad[:5]])
    assert ((near >= 0) & (near < x.shape[0])).all(), what
    assert b["cand"].all(), (what, "nearest", np.flatnonzero(~b["cand"])[:5])
    assert (np.abs(near_sq.astype(np.float64) - b["q"]) <= b["delta"]).all(), (what, "nearest_sq")
    one = b["count"] == 1
    assert np.array_equal(near[one], b["only"][one]), what


# ------------------------------------------------------------------------------------------------ accuracy
@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("k", [1, 3, 16])
@pytest.mark.parametrize("d", [20, 128, 512, 768, 1024])
def test_within_bounds(engine, kind, k, d):
    """ragged m and n on both sides of the tile edges; d = 20 is zero-padded to 24"""
    for m, n in SHAPES:
        m = k + 5 if m == "k+5" else m
        x, y = _sets(kind, m, n, d)
        got = _gpu(engine, x, y, k)
        _check_radii(engine, x, y, k, got[0], got[4])
        _check_bounds(x, y, got, (m, n))


def test_duplicates_copies_and_pruned_balls(engine):
    """k + 1 silent baseline rows have r = 0 and contribute nothing; an eval row equal to a kept baseline row has
    realism +inf and nearest_sq 0; an eval row next to a far (pruned) baseline row only has realism < 1"""
    k, d = 3, 128
    x = np.concatenate([np.zeros((6, d), np.float16), encodec_like(300, d, 3)])
    x[-1] += np.float16(40.0)                                     # far away: the largest radius
    y = encodec_like(200, d, 4, 0.2)
    y[0] = 0.0
    y[2] = x[-1]
    y[2, :4] += np.float16(0.5)
    got = _gpu(engine, x, y, k)
    kept, real, near, near_sq, t = got
    c = int(np.flatnonzero(kept > 0)[0])
    y[1] = x[c]
    got = _gpu(engine, x, y, k)
    kept, real, near, near_sq, t = got
    assert (kept[:6] == 0).all() and kept[-1] == 0
    assert np.isinf(real[1]) and near[1] == c and near_sq[1] == 0
    assert near[0] == 0 and near_sq[0] == 0 and np.isfinite(real[0])    # the silent rows are nearest, but pruned-to-0
    assert near[2] == x.shape[0] - 1 and real[2] < 1
    _check_bounds(x, y, got, "duplicates")


def test_reproducible_and_split(engine):
    """two calls are bitwise equal; the rows of [Y_1; Y_2; Y_3] get the values of three separate calls"""
    x = encodec_like(3001, 256, 5)
    ys = [encodec_like(n, 256, 6 + i, 0.2) for i, n in enumerate((700, 1, 1300))]
    z = _dev(np.concatenate([x, *ys]))
    a, b = engine.realism(z, 3001, 3), engine.realism(z, 3001, 3)
    assert all(torch.equal(p, q) for p, q in zip(a[:4], b[:4])) and a[4] == b[4]
    off = np.cumsum([0] + [y.shape[0] for y in ys])
    for i, y in enumerate(ys):
        one = engine.realism(_dev(np.concatenate([x, y])), 3001, 3)
        assert torch.equal(one[0], a[0]) and one[4] == a[4]
        for p, q in zip(one[1:4], a[1:4]):
            assert torch.equal(p, q[off[i]:off[i + 1]]), i


@pytest.mark.parametrize("m,n,d", [(4, 1, 128), (129, 127, 512), (3001, 257, 128), (257, 3001, 768)])
def test_local_shards_are_bitwise_equal(engine, m, n, d):
    x, y = _sets("encodec", m, n, d, 3)
    z = _dev(np.concatenate([x, y]))
    want = engine.realism(z, m, 3)
    tx, ty = -(-m // 128), -(-n // 128)
    g = max(4, -(-(tx * ty) // 8192))
    units = max(tx, ty * -(-tx // g))
    for s in SHARDS + [units + 3]:
        got = engine.realism_sharded(z, m, 3, local_shards=s)
        assert all(torch.equal(p, q) for p, q in zip(got[:4], want[:4])) and got[4] == want[4], s


def test_calc_realism(engine):
    x, y = _sets("clap", 900, 1100, 512, 2)
    got = fk.calc_realism(x, y)
    kept, real, near, near_sq, t = _gpu(engine, x, y, 3)
    assert (got.k, got.n_baseline, got.n_eval, got.threshold_sq) == (3, 900, 1100, t)
    assert np.array_equal(got.realism, real) and np.array_equal(got.nearest, near)
    assert np.array_equal(got.nearest_distance, np.sqrt(near_sq))


# ------------------------------------------------------------------------------------------------ rejections
def test_rejected_arguments_launch_and_write_nothing(engine):
    lib = _native.lib()
    m, n, d = 300, 200, 128
    z = _dev(encodec_like(m + n, d, 6))
    zbuf = torch.zeros((m + n) * d + 8, dtype=torch.float16, device="cuda")
    outs = [Guarded((m,), torch.float32, "cuda", 64), Guarded((n,), torch.float32, "cuda", 64),
            Guarded((n,), torch.float32, "cuda", 64), Guarded((n,), torch.float32, "cuda", 64)]
    t = torch.zeros(1, dtype=torch.float64)

    def call(zp=None, mm=m, nn=n, dd=d, k=3, kinds=("ok",) * 4, shards=None):
        def run(eng, _):
            ptrs = [None if o.ptr(kd) is None else o.ptr(kd).data_ptr() for o, kd in zip(outs, kinds)]
            args = (z.data_ptr() if zp is None else zp, mm, nn, dd, k, *ptrs, t.data_ptr(),
                    torch.cuda.current_stream().cuda_stream)
            fn = lib.fad_realism if shards is None else lib.fad_realism_sharded
            _native._check(fn(eng._h, *args) if shards is None else fn(eng._h, None, shards, *args))
        return run

    cases = [(call(k=0), "k must be in [1, 16]"), (call(k=17), "k must be in [1, 16]"),
             (call(mm=3), "realism needs more than k baseline rows and at least one eval row"),
             (call(nn=0), "realism needs more than k baseline rows and at least one eval row"),
             (call(zp=0), "null argument"), (call(kinds=("ok", "null", "ok", "ok")), "null argument"),
             (call(zp=zbuf.data_ptr() + 2), "pointers must be aligned (z to 16 bytes, the fp32 and int32 arrays to 4)"),
             (call(dd=124), "d must be a positive multiple of 8"),
             (call(mm=1 << 30), "too many rows"), (call(k=0, shards=3), "k must be in [1, 16]"),
             (call(shards=-1), "local_shards must be >= 0")]
    for fn, msg in cases:
        expect_rejected(engine, fn, msg, outs)
    assert t.item() == 0.0


_COUNTED = """
import numpy as np, torch
from fadtk_b200 import _native
from test_gpu_kad import encodec_like
from test_gpu_launch_count import counted
engine = _native.engine()
z = torch.from_numpy(np.concatenate([encodec_like(1500, 128, 9), encodec_like(1300, 128, 10, 0.2)])).cuda()
engine.realism(z, 1500, 3)
for fn in (lambda: engine.realism(z, 1500, 3), lambda: engine.realism_sharded(z, 1500, 3, local_shards=3)):
    print(*counted(engine, fn))
"""


def test_launch_counter_is_exact():
    """library kernels seen by torch.profiler == launch-counter delta, in a process of its own"""
    tests = Path(__file__).resolve().parent
    env = dict(os.environ, PYTHONPATH=f"{tests}{os.pathsep}{tests.parent}")
    out = subprocess.run([sys.executable, "-c", _COUNTED], capture_output=True, text=True, cwd=tests.parent, env=env,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    pairs = [tuple(map(int, ln.split())) for ln in out.stdout.split("\n") if ln.strip()]
    assert len(pairs) == 2, out.stdout
    for seen, delta in pairs:
        assert seen == delta > 0, pairs


# ------------------------------------------------------------------------------------------------ command line
def test_directory_command_line(engine, tmp_path):
    """FADTK_SYNTHETIC VGGish over synthetic clips: python -m fadtk_b200.realism embeds both directories and writes the
    per-file table, whose values are calc_realism's on the cached embeddings"""
    from fadtk_b200 import realism as realism_cli
    for kind in ("base", "eval"):
        (tmp_path / kind).mkdir()
        for i in range(4):
            synth.write_wav(tmp_path / kind / f"clip{i}.wav",
                            synth.musiclike_clip(i, 4.0, 16000, baseline=(kind == "base")), 16000)
    out = tmp_path / "realism.csv"
    assert realism_cli.main(["vggish", str(tmp_path / "base"), str(tmp_path / "eval"), str(out), "-w", "2"]) == 0
    rows = list(csv.DictReader(out.open()))
    assert len(rows) == 4 and [float(r["realism_median"]) for r in rows] == sorted(float(r["realism_median"]) for r in rows)
    files = lambda k: sorted((tmp_path / k / "embeddings" / "vggish").glob("*.npy"))  # noqa: E731
    base = [np.load(f) for f in files("base")]
    boff = np.cumsum([0] + [b.shape[0] for b in base])
    for r in rows:
        y = np.load(tmp_path / "eval" / "embeddings" / "vggish" / (Path(r["file"]).stem + ".npy"))
        want = fk.calc_realism(np.concatenate(base), y)
        assert float(r["realism_median"]) == float(np.median(want.realism.astype(np.float64)))
        assert float(r["realism_min"]) == float(want.realism.min())
        j = int(np.argmin(want.nearest_distance))
        assert float(r["nearest_distance"]) == float(want.nearest_distance[j]) and int(r["n_eval"]) == y.shape[0]
        assert r["nearest_baseline"] == str(files("base")[int(np.searchsorted(boff, want.nearest[j], "right")) - 1])
