"""Precision, recall, density and coverage on the H100 (csrc/prdc.cuh) against the fp64 oracle (oracle/prdc_oracle.py)
on the same fp16 rows.  The GPU computes q in fp32 within delta = tau (|y^_a|^2 + |y^_b|^2) of the exact value, so:
every radius lies between the k-th smallest of q - delta and of q + delta of its row; with the oracle's radii fed to the
counting pass, every count lies within decision_bounds and equals the exact count wherever no decision is ambiguous;
calc_prdc lies within the bounds built from the GPU's own radii.  Also: duplicates, reproducibility, rejected
arguments, the launch counter, and the directory command line."""
import csv
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native, synth
from fadtk_b200._native import NativeError
from oracle import prdc_oracle as po
from test_gpu_kad import clap_like, encodec_like

pytestmark = pytest.mark.gpu


def gaussian(rows, d, seed, shift=0.0):
    return (shift + np.random.default_rng(seed).standard_normal((rows, d))).astype(np.float16)


DATA = {"gauss": gaussian, "encodec": encodec_like, "clap": clap_like}
SIZES = ["k+1", 127, 128, 129, 257, 3000]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _padded(a):
    return np.pad(a, ((0, 0), (0, -a.shape[1] % 8)))


def _sets(kind, m, n, d, seed=0):
    gen = DATA[kind]
    x = gen(m, d, 10 + seed)
    y = gen(n, d, 20 + seed, 0.3) if kind != "clap" else gen(n, d, 20 + seed, 0.5)
    return x, y


def _gpu_radii(engine, x, y, k):
    return engine.knn_radii_sq(_dev(_padded(np.concatenate([x, y]))), x.shape[0], k).cpu().numpy()


# ------------------------------------------------------------------------------------------------ radii
@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("k", [1, 5, 16])
@pytest.mark.parametrize("d", [20, 128, 512, 768, 1024])
def test_radii_within_bounds(engine, kind, k, d):
    """every m and n of SIZES at least once on each side of the X / Y boundary; d = 20 is zero-padded to 24"""
    sizes = [k + 1 if s == "k+1" else s for s in SIZES]
    for m, n in zip(sizes, sizes[::-1][1:] + sizes[-1:]):
        x, y = _sets(kind, m, n, d)
        got = _gpu_radii(engine, x, y, k).astype(np.float64)
        lo, hi = po.radii_bounds(x, y, k)
        bad = np.flatnonzero((got < lo) | (got > hi))
        assert bad.size == 0, (m, n, bad[:5], got[bad[:5]], lo[bad[:5]], hi[bad[:5]])


# ------------------------------------------------------------------------------------------------ counts
def _check_counts(inside, flags, b):
    lo, hi = b["inside"]
    assert ((lo <= inside) & (inside <= hi)).all()
    assert np.array_equal(inside[lo == hi], lo[lo == hi])
    for key, bit in (("covered", 1), ("recalled", 2)):
        lo, hi = b[key]
        got = (flags & bit) > 0
        assert (lo <= got).all() and (got <= hi).all(), key
        assert np.array_equal(got[lo == hi], lo[lo == hi]), key


@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("m,n,d,k", [(6, 129, 20, 5), (127, 128, 128, 1), (257, 3000, 768, 16), (3000, 257, 512, 5),
                                     (129, 127, 1024, 5), (2, 3, 128, 1)])
def test_counts_with_oracle_radii(engine, kind, m, n, d, k):
    x, y = _sets(kind, m, n, d, 1)
    radii32 = po.radii_sq(x, y, k).astype(np.float32)
    inside, flags = engine.prdc_counts(_dev(_padded(np.concatenate([x, y]))), m, _dev(radii32))
    _check_counts(inside.cpu().numpy(), flags.cpu().numpy(), po.decision_bounds(x, y, radii32.astype(np.float64)))


def _metric_bounds(b, m, n, k):
    (ilo, ihi), (clo, chi), (rlo, rhi) = b["inside"], b["covered"], b["recalled"]
    return {"precision": (np.count_nonzero(ilo) / n, np.count_nonzero(ihi) / n),
            "recall": (np.count_nonzero(rlo) / m, np.count_nonzero(rhi) / m),
            "density": (ilo.sum() / (k * n), ihi.sum() / (k * n)),
            "coverage": (np.count_nonzero(clo) / m, np.count_nonzero(chi) / m)}


@pytest.mark.parametrize("kind,m,n,d,k", [("encodec", 1500, 1200, 768, 5), ("clap", 900, 1100, 512, 3),
                                          ("gauss", 20000, 20000, 128, 5)])
def test_calc_prdc_within_bounds(engine, kind, m, n, d, k):
    """end to end, against the bounds built from the GPU's own radii (20 000 x 20 000: the block oracle's full size)"""
    x, y = _sets(kind, m, n, d, 2)
    got = fk.calc_prdc(x, y, k=k)
    assert (got.k, got.n_baseline, got.n_eval) == (k, m, n)
    b = po.decision_bounds(x, y, _gpu_radii(engine, x, y, k).astype(np.float64))
    for name, (lo, hi) in _metric_bounds(b, m, n, k).items():
        assert lo <= getattr(got, name) <= hi, (name, getattr(got, name), lo, hi)
    exact = po.prdc(x, y, k)
    assert np.allclose(tuple(got[:4]), exact, rtol=0, atol=2e-3), (got, exact)


def test_duplicates(engine):
    """silent baseline rows (more than k copies) have r = 0 and contain nothing, not even an equal eval row; an eval row
    equal to a baseline row with r > 0 is inside that row's ball (q = 0 < r^2)"""
    k, d = 5, 128
    x = np.concatenate([np.zeros((12, d), np.float16), encodec_like(300, d, 3)])
    y = encodec_like(200, d, 4, 0.2)
    y[0] = 0.0
    y[1] = x[100]
    z = _dev(np.concatenate([x, y]))
    radii = engine.knn_radii_sq(z, x.shape[0], k)
    r = radii.cpu().numpy()
    assert (r[:12] == 0).all() and (r[12:312] > 0).all()
    inside, flags = (t.cpu().numpy() for t in engine.prdc_counts(z, x.shape[0], radii))
    assert not (flags[:12] & 1).any()
    assert inside[1] >= 1 and flags[100] & 1
    b = po.decision_bounds(x, y, r.astype(np.float64))
    _check_counts(inside, flags, b)


def test_two_calls_are_bitwise_equal(engine):
    x, y = _sets("encodec", 3001, 2500, 256, 5)
    z = _dev(np.concatenate([x, y]))
    ra, rb = engine.knn_radii_sq(z, 3001, 7), engine.knn_radii_sq(z, 3001, 7)
    assert torch.equal(ra, rb)
    (ia, fa), (ib, fb) = engine.prdc_counts(z, 3001, ra), engine.prdc_counts(z, 3001, ra)
    assert torch.equal(ia, ib) and torch.equal(fa, fb)
    assert fk.calc_prdc(x, y, k=7) == fk.calc_prdc(x, y, k=7)


# ------------------------------------------------------------------------------------------------ rejections
def test_rejected_arguments_launch_and_write_nothing(engine):
    lib, h, st = _native.lib(), engine._h, torch.cuda.current_stream().cuda_stream
    m, n, d = 300, 200, 128
    z = _dev(encodec_like(m + n, d, 6))
    zbuf = torch.zeros((m + n) * d + 8, dtype=torch.float16, device="cuda")
    radii = torch.full((m + n + 1,), 7.0, dtype=torch.float32, device="cuda")
    inside = torch.full((n + 1,), -3, dtype=torch.int32, device="cuda")
    flags = torch.full((m + 1,), 9, dtype=torch.uint8, device="cuda")
    zp, rp, ip, fp = z.data_ptr(), radii.data_ptr(), inside.data_ptr(), flags.data_ptr()
    radii_calls = [((zp, m, n, d, 0, rp), "k must be"), ((zp, m, n, d, 17, rp), "k must be"),
                   ((zp, 5, n, d, 5, rp), "more than k"), ((zp, m, 16, d, 16, rp), "more than k"),
                   ((None, m, n, d, 5, rp), "null"), ((zp, m, n, d, 5, None), "null"),
                   ((zbuf.data_ptr() + 2, m, n, d, 5, rp), "aligned"), ((zp, m, n, d, 5, rp + 2), "aligned"),
                   ((zp, m, n, 124, 5, rp), "multiple of 8"), ((zp, 1 << 30, n, d, 5, rp), "too many rows")]
    count_calls = [((zp, 1, n, d, rp, ip, fp), "more than k"), ((zp, m, 1, d, rp, ip, fp), "more than k"),
                   ((None, m, n, d, rp, ip, fp), "null"), ((zp, m, n, d, None, ip, fp), "null"),
                   ((zp, m, n, d, rp, None, fp), "null"), ((zp, m, n, d, rp, ip, None), "null"),
                   ((zp, m, n, d, rp + 2, ip, fp), "aligned"), ((zp, m, n, d, rp, ip + 2, fp), "aligned"),
                   ((zp, m, n, 20, rp, ip, fp), "multiple of 8"), ((zp, m, 1 << 30, d, rp, ip, fp), "too many rows")]
    before = [t.clone() for t in (radii, inside, flags)]
    torch.cuda.synchronize()
    launches = engine.launches
    for fn, calls in ((lib.fad_knn_radii_sq, radii_calls), (lib.fad_prdc_counts, count_calls)):
        for args, msg in calls:
            assert fn(h, *args, st) != 0
            assert msg in lib.fad_last_error().decode(), (args, lib.fad_last_error())
    torch.cuda.synchronize()
    assert engine.launches == launches
    for t, b in zip((radii, inside, flags), before):
        assert torch.equal(t, b)
    with pytest.raises(NativeError, match="k must be"):
        engine.knn_radii_sq(z, m, 0)


def test_python_argument_errors_need_no_device_work(engine):
    x, y = _sets("gauss", 10, 10, 16)
    for bad in (0, 17, 2.5, True):
        with pytest.raises(ValueError, match="k"):
            fk.calc_prdc(x, y, k=bad)
    with pytest.raises(ValueError, match="more than k"):
        fk.calc_prdc(x, y, k=10)


_COUNTED = """
import numpy as np, torch
from fadtk_b200 import _native
from test_gpu_kad import encodec_like
from test_gpu_launch_count import counted
engine = _native.engine()
z = torch.from_numpy(np.concatenate([encodec_like(1500, 128, 9), encodec_like(1300, 128, 10, 0.2)])).cuda()
radii = engine.knn_radii_sq(z, 1500, 5)
for fn in (lambda: engine.knn_radii_sq(z, 1500, 5), lambda: engine.prdc_counts(z, 1500, radii)):
    print(*counted(engine, fn))
"""


def test_launch_counter_is_exact():
    """library kernels seen by torch.profiler == launch-counter delta, in a process of its own (as the KAD tests do)"""
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
def test_directory_command_line(engine, tmp_path, capsys):
    """FADTK_SYNTHETIC VGGish over synthetic clips: python -m fadtk_b200.prdc embeds both directories, prints the four
    values and appends the CSV row, which equals calc_prdc on the cached embeddings"""
    from fadtk_b200 import prdc as prdc_cli
    for kind in ("base", "eval"):
        (tmp_path / kind).mkdir()
        for i in range(4):
            synth.write_wav(tmp_path / kind / f"clip{i}.wav",
                            synth.musiclike_clip(i, 4.0, 16000, baseline=(kind == "base")), 16000)
    out = tmp_path / "prdc.csv"
    argv = ["vggish", str(tmp_path / "base"), str(tmp_path / "eval"), str(out), "-k", "3", "-w", "2"]
    assert prdc_cli.main(argv) == 0
    assert "The PRDC vggish values (k = 3)" in capsys.readouterr().out
    rows = list(csv.reader(out.open()))
    assert rows[0] == prdc_cli.CSV_HEADER.strip().split(",") and len(rows) == 2
    row = dict(zip(rows[0], rows[1]))
    load = lambda k: np.concatenate([np.load(f) for f in sorted((tmp_path / k / "embeddings" / "vggish").glob("*.npy"))])  # noqa: E731
    want = fk.calc_prdc(load("base"), load("eval"), k=3)
    for name in ("precision", "recall", "density", "coverage"):
        assert float(row[name]) == getattr(want, name), name
    assert (int(row["k"]), int(row["n_baseline"]), int(row["n_eval"])) == (3, want.n_baseline, want.n_eval)
    assert prdc_cli.main(argv) == 0 and len(list(csv.reader(out.open()))) == 3      # appended, header once
