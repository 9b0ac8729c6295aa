"""The k nearest distinct baseline groups on the H100 (fad_nearest, prdc_tile_kernel<5>) against the fp64 oracle
(oracle/nearest_oracle.py) on the same fp16 rows: every returned row in its group, within delta of the exact q and a
candidate for the group's minimum, the groups distinct and ascending, none left out certainly closer, and the oracle's
list wherever no comparison is ambiguous.  Also: k = 1 without groups is fad_realism's nearest bitwise, planted copies,
reproducibility, the split of an eval set, local shards, rejected arguments, the launch counter, and the directory
command line against calc_nearest and the realism table."""
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
from oracle import nearest_oracle as no
from test_gpu_kad import encodec_like
from test_gpu_kad_sharded import SHARDS
from test_gpu_realism import DATA, _dev, _padded, _sets

pytestmark = pytest.mark.gpu

# (m, n, group sizes): one row each, 10 rows, one group over several tiles and runs, empty groups, fewer groups than k
SHAPES = [(1, 3, None), (129, 127, None), (3000, 257, [10]), (1100, 300, [7, 0, 900, 0, 0, 193]),
          (257, 1200, [1, 0, 255, 1]), (600, 130, [600])]


def _offsets(m, sizes):
    """the offsets of groups of the given sizes, repeated until they cover the m rows (the last one cut at m)"""
    if sizes is None:
        return None
    off = [0]
    while off[-1] < m:
        for s in sizes:
            off.append(min(off[-1] + s, m))
            if off[-1] == m:
                break
    return np.array(off, np.int64)


def _gpu(engine, x, y, k, offsets=None, shards=None):
    z = _dev(_padded(np.concatenate([x, y])))
    off = None if offsets is None else torch.from_numpy(np.asarray(offsets, np.int64)).cuda()
    out = (engine.nearest(z, x.shape[0], k, off) if shards is None
           else engine.nearest_sharded(z, x.shape[0], k, off, local_shards=shards))
    return tuple(t.cpu().numpy() for t in out)


def _check(x, y, k, offsets, got, what):
    rows, q = got
    b = no.nearest_bounds(x, y, rows, q, k, offsets)
    for key in ("rows", "order", "missing"):
        bad = np.flatnonzero(~b[key])
        assert bad.size == 0, (what, key, bad[:5], rows[bad[:3]], b["want_rows"][bad[:3]])
    bad = np.flatnonzero(b["clear"] & ~b["equal"])
    assert bad.size == 0, (what, "equal", bad[:5], rows[bad[:3]], b["want_rows"][bad[:3]])
    return b


# ------------------------------------------------------------------------------------------------ accuracy
@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("k", [1, 5, 16])
@pytest.mark.parametrize("d", [20, 128, 512, 768, 1024])
def test_within_bounds(engine, kind, k, d):
    """ragged m and n on both sides of the tile edges; d = 20 is zero-padded to 24"""
    for m, n, sizes in SHAPES:
        x, y = _sets(kind, m, n, d)
        off = _offsets(m, sizes)
        _check(x, y, k, off, _gpu(engine, x, y, k, off), (m, n, sizes))


def test_k1_without_groups_is_realism_nearest_bitwise(engine):
    for kind, m, n, d in (("encodec", 3001, 1300, 128), ("clap", 700, 129, 512), ("gauss", 5, 1, 24)):
        x, y = _sets(kind, m, n, d, 4)
        z = _dev(np.concatenate([x, y]))
        _, _, near, near_sq, _ = engine.realism(z, m, 3)
        rows, q = engine.nearest(z, m, 1)
        assert torch.equal(rows[:, 0], near) and torch.equal(q[:, 0].view(torch.int32), near_sq.view(torch.int32))


def test_planted_copies_come_first(engine):
    """eval files made of baseline file segments: rank 1 is that baseline file at distance 0, at the right rows"""
    d = 128
    base = [encodec_like(r, d, 30 + i) for i, r in enumerate((40, 75, 10, 300, 55))]
    plant = {"a": (3, 20, 30), "b": (1, 5, 12)}              # eval file -> (baseline file, first row, end row)
    ev = {"a": np.concatenate([encodec_like(4, d, 50, 0.4), base[3][20:30]]),
          "b": np.concatenate([base[1][5:12], encodec_like(9, d, 51, 0.4)]),
          "c": encodec_like(12, d, 52, 0.4)}
    res = fk.calc_nearest(base, np.concatenate(list(ev.values())), k=3)
    off = np.cumsum([0] + [e.shape[0] for e in ev.values()])
    boff = np.cumsum([0] + [b.shape[0] for b in base])
    for s, name in enumerate(ev):
        if name not in plant:
            assert (res.distance[off[s]:off[s + 1], 0] > 0).all()
            continue
        g, r0, r1 = plant[name]
        lo = 4 if name == "a" else 0
        for t in range(r1 - r0):
            j = off[s] + lo + t
            assert res.groups[j, 0] == g and res.distance[j, 0] == 0 and res.rows[j, 0] - boff[g] == r0 + t
            assert len(set(res.groups[j].tolist())) == 3


def test_reproducible_split_and_groups(engine):
    """two calls are bitwise equal; the rows of [Y_1; Y_2; Y_3] get the values of three separate calls"""
    x = encodec_like(3001, 256, 5)
    ys = [encodec_like(n, 256, 6 + i, 0.2) for i, n in enumerate((700, 1, 1300))]
    off = torch.from_numpy(np.r_[0, np.arange(10, 3001, 10), 3001].astype(np.int64)).cuda()
    z = _dev(np.concatenate([x, *ys]))
    for o in (None, off):
        a, b = engine.nearest(z, 3001, 7, o), engine.nearest(z, 3001, 7, o)
        assert all(torch.equal(p, q) for p, q in zip(a, b))
        cut = np.cumsum([0] + [y.shape[0] for y in ys])
        for i, y in enumerate(ys):
            one = engine.nearest(_dev(np.concatenate([x, y])), 3001, 7, o)
            for p, q in zip(one, a):
                assert torch.equal(p, q[cut[i]:cut[i + 1]]), i


@pytest.mark.parametrize("m,n,d,groups", [(4, 1, 128, None), (129, 127, 512, [0, 60, 60, 129]),
                                          (3001, 257, 128, None), (3001, 257, 128, "ten"), (257, 3001, 768, None)])
def test_local_shards_are_bitwise_equal(engine, m, n, d, groups):
    x, y = _sets("encodec", m, n, d, 3)
    if groups == "ten":
        groups = list(range(0, m, 10)) + [m]
    want = _gpu(engine, x, y, 16, groups)
    tx, ty = -(-m // 128), -(-n // 128)
    g = max(4, -(-(tx * ty) // 8192))
    units = ty * -(-tx // g)
    for s in SHARDS + [units + 1]:
        got = _gpu(engine, x, y, 16, groups, shards=s)
        assert all(np.array_equal(p.view(np.uint32), q.view(np.uint32)) for p, q in zip(got, want)), s


def test_calc_nearest(engine):
    x, y = _sets("clap", 900, 1100, 512, 2)
    parts = [x[:300], x[300:300], x[300:]]
    got = fk.calc_nearest(parts, y, k=4)
    rows, q = _gpu(engine, x, y, 4, [0, 300, 300, 900])
    assert (got.k, got.n_baseline, got.n_eval) == (4, 900, 1100)
    assert np.array_equal(got.rows, rows) and np.array_equal(got.distance, np.sqrt(q))
    assert np.array_equal(got.groups, np.where(rows < 0, -1, np.where(rows < 300, 0, 2)))
    assert (got.rows[:, 2:] == -1).all()


# ------------------------------------------------------------------------------------------------ rejections
def test_rejected_arguments_launch_and_write_nothing(engine):
    lib = _native.lib()
    m, n, d, k = 300, 200, 128, 3
    z = _dev(encodec_like(m + n, d, 6))
    zbuf = torch.zeros((m + n) * d + 8, dtype=torch.float16, device="cuda")
    # the int32 rows are guarded as fp32 words: any write changes the sentinel's bits
    outs = [Guarded((n * k,), torch.float32, "cuda", 64), Guarded((n * k,), torch.float32, "cuda", 64)]
    good = torch.tensor([0, 100, 100, 300], dtype=torch.int64, device="cuda")
    dec = torch.tensor([0, 100, 50, 300], dtype=torch.int64, device="cuda")
    short = torch.tensor([0, 100, 299], dtype=torch.int64, device="cuda")
    first = torch.tensor([1, 100, 300], dtype=torch.int64, device="cuda")
    obuf = torch.zeros(8, dtype=torch.int64, device="cuda")

    def call(zp=None, mm=m, nn=n, dd=d, kk=k, off=good, groups=None, kinds=("ok",) * 2, shards=None):
        def run(eng, _):
            ptrs = [None if o.ptr(kd) is None else o.ptr(kd).data_ptr() for o, kd in zip(outs, kinds)]
            op = off if isinstance(off, int) or off is None else off.data_ptr()
            ng = groups if groups is not None else (0 if off is None or isinstance(off, int) else off.numel() - 1)
            args = (z.data_ptr() if zp is None else zp, mm, nn, dd, kk, op, ng, *ptrs,
                    torch.cuda.current_stream().cuda_stream)
            fn = lib.fad_nearest if shards is None else lib.fad_nearest_sharded
            _native._check(fn(eng._h, *args) if shards is None else fn(eng._h, None, shards, *args))
        return run

    aligned = "pointers must be aligned (z to 16 bytes, the fp32 and int32 arrays to 4, the offsets to 8)"
    cases = [(call(kk=0), "k must be in [1, 16]"), (call(kk=17), "k must be in [1, 16]"),
             (call(mm=0), "nearest needs at least one baseline row and one eval row"),
             (call(nn=0), "nearest needs at least one baseline row and one eval row"),
             (call(zp=0), "null argument"), (call(kinds=("ok", "null")), "null argument"),
             (call(zp=zbuf.data_ptr() + 2), aligned), (call(off=obuf.data_ptr() + 4, groups=1), aligned),
             (call(dd=124), "d must be a positive multiple of 8"),
             (call(mm=1 << 30), "too many rows"), (call(groups=0), "n_groups must be >= 1"),
             (call(off=dec), "offsets must be non-decreasing"), (call(off=short), "the last offset must be m"),
             (call(off=first), "offsets[0] must be 0"), (call(kk=0, shards=3), "k must be in [1, 16]"),
             (call(off=dec, shards=2), "offsets must be non-decreasing"),
             (call(shards=-1), "local_shards must be >= 0")]
    for fn, msg in cases:
        expect_rejected(engine, fn, msg, outs)


_COUNTED = """
import numpy as np, torch
from fadtk_b200 import _native
from test_gpu_kad import encodec_like
from test_gpu_launch_count import counted
engine = _native.engine()
z = torch.from_numpy(np.concatenate([encodec_like(1500, 128, 9), encodec_like(1300, 128, 10, 0.2)])).cuda()
off = torch.tensor([0, 700, 700, 1500], dtype=torch.int64, device="cuda")
engine.nearest(z, 1500, 5)
for fn in (lambda: engine.nearest(z, 1500, 5), lambda: engine.nearest(z, 1500, 5, off),
           lambda: engine.nearest_sharded(z, 1500, 5, off, local_shards=3)):
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
    assert len(pairs) == 3, out.stdout
    for seen, delta in pairs:
        assert seen == delta > 0, pairs


# ------------------------------------------------------------------------------------------------ command line
def test_directory_command_line(engine, tmp_path):
    """FADTK_SYNTHETIC VGGish over synthetic clips: python -m fadtk_b200.nearest embeds both directories and writes the
    per-file table, whose values are calc_nearest's on the caches, and whose rank 1 agrees with the realism table"""
    from fadtk_b200 import nearest as nearest_cli, realism as realism_cli
    for kind in ("base", "eval"):
        (tmp_path / kind).mkdir()
        for i in range(4):
            synth.write_wav(tmp_path / kind / f"clip{i}.wav",
                            synth.musiclike_clip(i, 4.0, 16000, baseline=(kind == "base")), 16000)
    out = tmp_path / "nearest.csv"
    assert nearest_cli.main(["vggish", str(tmp_path / "base"), str(tmp_path / "eval"), str(out), "-k", "3",
                             "-w", "2"]) == 0
    rows = list(csv.DictReader(out.open()))
    files = lambda k: sorted((tmp_path / k / "embeddings" / "vggish").glob("*.npy"))  # noqa: E731
    base = [np.load(f) for f in files("base")]
    assert len(rows) == 4 * 3
    first = [float(r["distance"]) for r in rows if r["rank"] == "1"]
    assert first == sorted(first)
    by_file = {}
    for r in rows:
        by_file.setdefault(r["file"], []).append(r)
    for f, rs in by_file.items():
        y = np.load(tmp_path / "eval" / "embeddings" / "vggish" / (Path(f).stem + ".npy"))
        want = fk.calc_nearest(base, y, k=3)
        q = np.square(want.distance.astype(np.float32))
        best = {}
        for j in range(y.shape[0]):
            for t in range(3):
                key = (want.distance[j, t], j, want.rows[j, t])
                g = int(want.groups[j, t])
                if g >= 0 and (g not in best or key < best[g][0]):
                    best[g] = (key, t)
        ranked = sorted(best.items(), key=lambda e: e[1][0])[:3]
        assert [int(r["rank"]) for r in rs] == [1, 2, 3] and q.shape == want.rows.shape
        boff = np.cumsum([0] + [b.shape[0] for b in base])
        for r, (g, ((dist, j, i), _)) in zip(rs, ranked):
            assert r["nearest_baseline"] == str(files("base")[g]) and float(r["distance"]) == float(dist)
            assert (int(r["eval_row"]), int(r["baseline_row"]), int(r["n_eval"])) == (j, i - boff[g], y.shape[0])
    # rank 1 against the realism table of the same directories
    rt = tmp_path / "realism.csv"
    assert realism_cli.main(["vggish", str(tmp_path / "base"), str(tmp_path / "eval"), str(rt), "-w", "2"]) == 0
    for r in csv.DictReader(rt.open()):
        one = by_file[r["file"]][0]
        assert float(one["distance"]) == float(r["nearest_distance"])
        y = np.load(tmp_path / "eval" / "embeddings" / "vggish" / (Path(r["file"]).stem + ".npy"))
        d1 = fk.calc_nearest(base, y, k=1).distance[:, 0]
        if (d1 == d1.min()).sum() == 1:                    # a unique minimum: the same baseline file
            assert one["nearest_baseline"] == r["nearest_baseline"]
