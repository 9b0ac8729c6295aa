"""Sharded precision, recall, density and coverage (fad_knn_radii_sq_sharded, fad_prdc_counts_sharded): the radii and
ball-count work units cut into shards, each shard's radii, column counts and covered / recalled planes in a zero-filled
copy, the copies summed.  On one device (local shards, run one after another) every output must be bitwise equal
(torch.equal) to the unsharded entry's for any shard count, including more shards than units, and including a baseline
row that is covered in two shards and recalled in a third (the flags must be ORed, not added); rejected calls launch
nothing; the launch counter stays exact.  With two visible devices, one engine per device joined in one communicator
from two threads: each rank's output equals one device's bitwise, and ranks whose arguments differ all raise the same
NativeError instead of blocking."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import dist
from fadtk_b200._native import NativeError
from test_gpu_kad import DATA, encodec_like
from test_gpu_kad_sharded import SHARDS, _dev, _on_both, pair  # noqa: F401 - pair is a fixture

pytestmark = pytest.mark.gpu


def _units(m, n):
    """the larger of the two passes' unit counts: Tx + Ty radii units, Tx * cuts counts units"""
    tx, ty = -(-m // 128), -(-n // 128)
    g = max(4, -(-(tx * ty) // 8192))
    return max(tx + ty, tx * -(-ty // g))


def _check_equal(engine, z, m, k, shards):
    """radii, inside and flags of every shard count in `shards` == the unsharded entries' (bitwise)"""
    radii = engine.knn_radii_sq(z, m, k)
    inside, flags = engine.prdc_counts(z, m, radii)
    for s in shards:
        assert torch.equal(engine.knn_radii_sq_sharded(z, m, k, local_shards=s), radii), s
        got_in, got_fl = engine.prdc_counts_sharded(z, m, radii, local_shards=s)
        assert torch.equal(got_in, inside), s
        assert torch.equal(got_fl, flags), s
    return radii, inside, flags


# ------------------------------------------------------------------------------------------ one device
@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("k", [1, 5, 16])
@pytest.mark.parametrize("m,n,d", [("k+1", 129, 128), (127, 129, 256), (129, 128, 512), (128, "k+1", 1024),
                                   (1000, 3001, 768), (3001, 257, 128)])
def test_equal_unsharded(engine, kind, k, m, n, d):
    """the tile edges with Tx != Ty, d = 128 to 1024, up to 24 X tiles and 24 Y tiles"""
    m, n = (k + 1 if v == "k+1" else v for v in (m, n))
    gen = DATA[kind]
    z = _dev(np.concatenate([gen(m, d, 1), gen(n, d, 2)]))
    _check_equal(engine, z, m, k, SHARDS + [_units(m, n) + 3])


def test_duplicates_and_silent_rows(engine):
    """silent baseline rows (r = 0), duplicated eval rows (s = 0) and an eval row equal to a baseline row"""
    k, d = 5, 128
    x = np.concatenate([np.zeros((12, d), np.float16), encodec_like(300, d, 3)])
    y = np.concatenate([encodec_like(200, d, 4, 0.2), np.repeat(encodec_like(3, d, 5, 0.1), 7, axis=0)])
    y[0] = 0.0
    y[1] = x[100]
    radii, _, _ = _check_equal(engine, _dev(np.concatenate([x, y])), x.shape[0], k, SHARDS + [_units(312, 221) + 3])
    r = radii.cpu().numpy()
    assert (r[:12] == 0).all() and (r[-21:] == 0).all()


def _or_trap(k, d=128, m=100, n=4096):
    """x_0 = 0 with k baseline rows at q = 1 (r_0^2 = 1); every other row in a tight cluster at q ~ 37 from x_0, whose
    own radii (~2.5) reach nothing outside it.  Eval: k + 1 copies of a row at q = 0.25 from x_0 in Y columns 0.. (counts
    unit 0) and again in columns 2048.. (unit 4): x_0 is covered from two units, and the copies have s = 0, so they
    recall nothing.  Column 3600 (unit 7) sits at q = 9 from x_0; its k-th neighbour in Y is at q = 9.25 (the copies),
    so it recalls x_0 without covering it.  8 units of 4 column tiles: with 2, 3, 4, 7 or 8 shards the covering units
    fall in two shards and the recalling one in another."""
    rng = np.random.default_rng(7)
    far = 6.0 * np.eye(d)[d - 1]
    x = far + 0.1 * rng.standard_normal((m, d))
    x[0] = 0.0
    x[1:k + 1] = np.eye(d)[1:k + 1]
    y = far + 0.1 * rng.standard_normal((n, d))
    near = 0.5 * np.eye(d)[k + 1]
    y[0:k + 1] = near
    y[2048:2048 + k + 1] = near
    y[3600] = 3.0 * np.eye(d)[k + 2]
    return np.concatenate([x, y]).astype(np.float16), m


@pytest.mark.parametrize("k", [1, 5, 16])
def test_flags_are_ored_over_shards(engine, k):
    z, m = _or_trap(k)
    radii, inside, flags = _check_equal(engine, _dev(z), m, k, [2, 3, 4, 7, 8, 11])
    r = radii.cpu().numpy()
    assert abs(r[0] - 1.0) < 0.02 and abs(r[m + 3600] - 9.25) < 0.05, (r[0], r[m + 3600])
    assert int(flags[0]) == 3                                  # covered and recalled, from three different shards
    assert int(inside[0]) == int(inside[2048]) >= 1 and int(inside[3600]) == 0


def test_rejections_launch_nothing(engine):
    x = encodec_like(300, 128, 7)
    z = _dev(np.concatenate([x, encodec_like(200, 128, 8)]))
    radii = engine.knn_radii_sq(z, 300, 5)
    calls = [lambda s: engine.knn_radii_sq_sharded(z, 300, 5, local_shards=s),
             lambda s: engine.prdc_counts_sharded(z, 300, radii, local_shards=s)]
    assert not engine.has_comm
    for call in calls:
        for s, msg in ((-1, "local_shards must be >= 0"), (0, "no communicator")):
            torch.cuda.synchronize()
            before = engine.launches
            with pytest.raises(NativeError, match=msg):
                call(s)
            torch.cuda.synchronize()
            assert engine.launches == before
    before = engine.launches
    with pytest.raises(NativeError, match="k must be"):              # the plain checks still come first
        engine.knn_radii_sq_sharded(z, 300, 17, local_shards=3)
    with pytest.raises(NativeError, match="more than k"):
        engine.prdc_counts_sharded(z, 1, radii, local_shards=3)
    assert engine.launches == before


_COUNTED = """
import numpy as np, torch
from fadtk_b200 import _native
from test_gpu_kad import encodec_like
from test_gpu_launch_count import counted
engine = _native.engine()
z = torch.from_numpy(np.concatenate([encodec_like(1500, 128, 9), encodec_like(1300, 128, 10, 0.2)])).cuda()
radii = engine.knn_radii_sq(z, 1500, 5)
for fn in (lambda: engine.knn_radii_sq_sharded(z, 1500, 5, local_shards=3),
           lambda: engine.prdc_counts_sharded(z, 1500, radii, local_shards=7),
           lambda: engine.knn_radii_sq_sharded(z, 1500, 5, local_shards=30),      # 30 shards, 23 units
           lambda: engine.prdc_counts_sharded(z, 1500, radii, local_shards=40)):  # 40 shards, 36 units
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
    assert len(pairs) == 4, out.stdout
    for seen, delta in pairs:
        assert seen == delta > 0, pairs


def test_calc_prdc_distributed_at_world_size_one(engine):
    x, y = encodec_like(900, 128, 14), encodec_like(700, 128, 15, 0.2)
    assert dist.world_size() == 1
    assert fk.calc_prdc(x, y, k=4, distributed=True) == fk.calc_prdc(x, y, k=4)


def test_distributed_without_communicator_raises(engine, monkeypatch):
    """world size > 1 without the library's communicator: the RuntimeError names the metric, KAD's word for word"""
    monkeypatch.setattr(dist, "world_size", lambda: 2)
    monkeypatch.setattr(dist, "enable_native_allreduce", lambda eng: False)
    x, y = encodec_like(40, 128, 16), encodec_like(30, 128, 17)
    with pytest.raises(RuntimeError, match="^distributed PRDC runs over the library's own NCCL communicator"):
        fk.calc_prdc(x, y, distributed=True)
    with pytest.raises(RuntimeError) as e:
        fk.calc_kernel_audio_distance(x, y, distributed=True)
    assert str(e.value) == ("distributed KAD runs over the library's own NCCL communicator, which needs torch.distributed "
                            "on the nccl backend and FADTK_NATIVE_ALLREDUCE unset or 1")


# ------------------------------------------------------------------------------------------ two devices
@pytest.mark.parametrize("kind", sorted(DATA))
def test_two_devices_equal_one(pair, kind):  # noqa: F811 - the fixture
    gen = DATA[kind]
    m, d, k = 3001, 512, 5
    z = np.concatenate([gen(m, d, 10), gen(2049, d, 11)])
    one = pair[0]
    with torch.cuda.device(0):
        want_r = one.knn_radii_sq(_dev(z, "cuda:0"), m, k)
        want = [want_r.cpu(), *(t.cpu() for t in one.prdc_counts(_dev(z, "cuda:0"), m, want_r))]

    def run(r, e):
        zz = _dev(z, f"cuda:{r}")
        radii = e.knn_radii_sq_sharded(zz, m, k)
        return [radii.cpu(), *(t.cpu() for t in e.prdc_counts_sharded(zz, m, radii))]
    for r, got in enumerate(_on_both(pair, run)):
        assert not isinstance(got, Exception), got
        for g, w in zip(got, want):
            assert torch.equal(g, w), r


def test_two_devices_disagreement_fails_both(pair):  # noqa: F811 - the fixture
    x, y = encodec_like(700, 128, 12), encodec_like(500, 128, 13)
    z = np.concatenate([x, y])
    z_changed = z.copy()
    z_changed[901] += np.float16(0.5)
    with torch.cuda.device(0):
        radii = pair[0].knn_radii_sq(_dev(z, "cuda:0"), 700, 5).cpu()
    radii_changed = radii.clone()
    radii_changed[1000] = torch.nextafter(radii[1000], torch.tensor(float("inf")))
    # (what the message names, the call of rank r, digest kernels a rank may launch before failing)
    cases = [("(m, n)", lambda r, e: e.knn_radii_sq_sharded(_dev(z, f"cuda:{r}"), 700 if r == 0 else 701, 5), 1),
             ("(k)", lambda r, e: e.knn_radii_sq_sharded(_dev(z, f"cuda:{r}"), 700, 5 if r == 0 else 6), 1),
             ("(z)", lambda r, e: e.knn_radii_sq_sharded(_dev(z if r == 0 else z_changed, f"cuda:{r}"), 700, 5), 1),
             ("(radii)", lambda r, e: e.prdc_counts_sharded(_dev(z, f"cuda:{r}"), 700,
                                                            (radii if r == 0 else radii_changed).to(f"cuda:{r}")), 2)]
    for what, call, digests in cases:
        def run(r, e):
            before = e.launches
            try:
                call(r, e)
            except NativeError as err:
                return str(err), e.launches - before
            return None, e.launches - before
        res = _on_both(pair, run)
        assert all(isinstance(msg, str) for msg, _ in res), (what, res)
        assert res[0][0] == res[1][0] and what in res[0][0], (what, res)
        assert all(n <= digests for _, n in res), (what, res)      # no tile work
    # a rank whose own checks reject the call: both fail with the same message, neither blocks
    def bad(r, e):
        try:
            e.knn_radii_sq_sharded(_dev(z, f"cuda:{r}"), 700, 5 if r == 0 else 17)
        except NativeError as err:
            return str(err)
    res = _on_both(pair, bad)
    assert res[0] == res[1] and "rejected" in res[0], res
    # the communicator still works afterwards
    got = _on_both(pair, lambda r, e: e.knn_radii_sq_sharded(_dev(z, f"cuda:{r}"), 700, 5).cpu())
    assert torch.equal(got[0], got[1]) and torch.equal(got[0], radii)
