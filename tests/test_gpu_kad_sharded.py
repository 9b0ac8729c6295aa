"""Sharded Kernel Audio Distance (fad_kad_*_sharded): the tile work cut into shards of contiguous work units, each
shard's partials or histogram counts in a zero-filled buffer, the buffers summed.  On one device (local shards, run one
after another) every output must be bitwise equal (torch.equal) to the unsharded entry's for any shard count, including
more shards than units; rejected calls launch nothing; the launch counter stays exact.  With two visible devices, one
engine per device joined in one communicator from two threads: each rank's output equals one device's bitwise, and
ranks whose arguments differ all raise the same NativeError instead of blocking."""
import os
import subprocess
import sys
import threading
from pathlib import Path

import numpy as np
import pytest
import torch

from fadtk_b200._native import Engine, NativeError
from test_gpu_kad import DATA, clap_like, encodec_like

pytestmark = pytest.mark.gpu

SHARDS = [1, 2, 3, 7, 8]
LENGTHS = [3, 0, 129, 1, 2, 127, 10, 128, 750, 2, 2000, 1, 129, 3, 128, 10]


def _dev(a, device="cuda"):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def _sigma(x, device="cuda"):
    return torch.tensor([float(np.sqrt(np.median(((x[:200, None].astype(np.float64) - x[None, :200]) ** 2).sum(-1))))],
                        dtype=torch.float64, device=device)


def _pair_units(rows):
    T = -(-rows // 128)
    return (T + 1) // 2


def _shard_counts(units):
    return SHARDS + [units + 3]


# ------------------------------------------------------------------------------------------ one device
@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("m,n,d", [(2, 2, 128), (60, 67, 128), (64, 64, 128), (64, 65, 128), (1000, 777, 512),
                                   (3001, 2049, 768), (640, 700, 1024), (16001, 16383, 128)])
def test_sums_equal_unsharded(engine, kind, m, n, d):
    """N = 127 / 128 / 129 (the tile edges), d = 128 to 1024, up to T = 254 tile rows"""
    gen = DATA[kind]
    x, y = gen(m, d, 1), gen(n, d, 2)
    z = _dev(np.concatenate([x, y]))
    sigma = _sigma(x)
    want = engine.kad_sums(z, m, sigma)
    for s in _shard_counts(_pair_units(m + n)):
        assert torch.equal(engine.kad_sums_sharded(z, m, sigma, local_shards=s), want), s


@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("m,d", [(2, 128), (127, 128), (128, 512), (129, 768), (3001, 1024), (16001, 128)])
def test_median_equal_unsharded(engine, kind, m, d):
    x = _dev(DATA[kind](m, d, 5))
    want = engine.kad_median_sq(x)
    for s in _shard_counts(_pair_units(m)):
        assert torch.equal(engine.kad_median_sq_sharded(x, local_shards=s), want), s


def test_median_ties_and_zero_bandwidth(engine):
    """every distance four times; all pairs identical (sigma = 0, which fad.py turns into a ValueError)"""
    x = _dev(np.repeat(encodec_like(300, 128, 6), 2, axis=0))
    want = engine.kad_median_sq(x)
    ties = _dev(np.concatenate([np.zeros((50, 128), np.float16), clap_like(10, 128, 8)]))
    zero = engine.kad_median_sq(ties)
    assert (zero.cpu().numpy() == 0.0).all()
    for s in SHARDS + [20]:
        assert torch.equal(engine.kad_median_sq_sharded(x, local_shards=s), want), s
        assert torch.equal(engine.kad_median_sq_sharded(ties, local_shards=s), zero), s


def _songs(kind, lengths, d, seed):
    gen = DATA[kind]
    return [gen(n, d, seed + k, 0.05 * (k % 4)) for k, n in enumerate(lengths)]


@pytest.mark.parametrize("kind", sorted(DATA))
@pytest.mark.parametrize("m,lengths,d", [(129, LENGTHS, 128), (3001, LENGTHS, 512), (256, [10, 5000, 3, 129, 1], 128),
                                         (2, [2, 3], 1024), (300, [], 128)])
def test_song_sums_equal_unsharded(engine, kind, m, lengths, d):
    """songs across tile edges, a 5000-row song, n_items = 0"""
    x = DATA[kind](m, d, 3)
    songs = _songs(kind, lengths, d, 100)
    off = np.zeros(len(songs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([s.shape[0] for s in songs])
    z = _dev(np.concatenate([x, *songs])) if songs else _dev(x)
    offsets, sigma = _dev(off), _sigma(x)
    want = engine.kad_song_sums(z, m, offsets, sigma)
    for s in SHARDS + [len(songs) * 8 + 40]:
        assert torch.equal(engine.kad_song_sums_sharded(z, m, offsets, sigma, local_shards=s), want), s


def test_rejections_launch_nothing(engine):
    x = encodec_like(300, 128, 7)
    z = _dev(np.concatenate([x, encodec_like(200, 128, 8)]))
    off, sigma = _dev(np.array([0, 120, 200], dtype=np.int64)), _sigma(x)
    calls = [lambda s: engine.kad_median_sq_sharded(z[:300], local_shards=s),
             lambda s: engine.kad_sums_sharded(z, 300, sigma, local_shards=s),
             lambda s: engine.kad_song_sums_sharded(z, 300, off, sigma, local_shards=s)]
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
    with pytest.raises(NativeError, match="at least two rows"):       # the plain checks still come first
        engine.kad_sums_sharded(z, 1, sigma, local_shards=3)
    assert engine.launches == before


_COUNTED = """
import numpy as np, torch
from fadtk_b200 import _native
from test_gpu_kad_sharded import LENGTHS, _dev, _sigma, _songs, encodec_like
from test_gpu_launch_count import counted
engine = _native.engine()
x = encodec_like(1500, 128, 9)
songs = _songs("encodec", LENGTHS, 128, 200)
off = np.zeros(len(songs) + 1, dtype=np.int64)
off[1:] = np.cumsum([s.shape[0] for s in songs])
z, offsets, sigma = _dev(np.concatenate([x, *songs])), _dev(off), _sigma(x)
for fn in (lambda: engine.kad_median_sq_sharded(z[:1500], local_shards=3),
           lambda: engine.kad_sums_sharded(z, 1500, sigma, local_shards=7),
           lambda: engine.kad_song_sums_sharded(z, 1500, offsets, sigma, local_shards=8),
           lambda: engine.kad_sums_sharded(z, 1500, sigma, local_shards=40)):      # 40 shards, 20 units
    print(*counted(engine, fn))
"""


def test_launch_counter_is_exact():
    """library kernels seen by torch.profiler == launch-counter delta, in a process of its own: profiler sessions of
    this module must not change what later sessions of the suite record"""
    tests = Path(__file__).resolve().parent
    env = dict(os.environ, PYTHONPATH=f"{tests}{os.pathsep}{tests.parent}")
    out = subprocess.run([sys.executable, "-c", _COUNTED], capture_output=True, text=True, cwd=tests.parent, env=env,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    pairs = [tuple(map(int, ln.split())) for ln in out.stdout.split("\n") if ln.strip()]
    assert len(pairs) == 4, out.stdout
    for seen, delta in pairs:
        assert seen == delta > 0, pairs


# ------------------------------------------------------------------------------------------ two devices
def _on_both(engs, fn):
    """fn(rank, engine) on one thread per device -> [result or exception] by rank"""
    out = [None, None]

    def run(r):
        try:
            with torch.cuda.device(r):
                out[r] = fn(r, engs[r])
                torch.cuda.synchronize()
        except Exception as e:          # noqa: BLE001 - returned to the test
            out[r] = e
    threads = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in threads), "a rank is still blocked"
    return out


@pytest.fixture(scope="module")
def pair():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible devices")
    engs = [Engine(r, max_examples=64) for r in range(2)]
    uid = Engine.comm_unique_id()
    res = _on_both(engs, lambda r, e: e.comm_init(uid, r, 2))
    assert res == [None, None], res
    yield engs
    for e in engs:
        e.close()


@pytest.mark.parametrize("kind", sorted(DATA))
def test_two_devices_equal_one(pair, kind):
    gen = DATA[kind]
    m, d = 3001, 512
    x, y = gen(m, d, 10), gen(2049, d, 11)
    songs = _songs(kind, LENGTHS + [5000], d, 300)
    off = np.zeros(len(songs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([s.shape[0] for s in songs])
    zs, z_songs, sig = np.concatenate([x, y]), np.concatenate([x, *songs]), _sigma(x, "cpu")
    one = pair[0]
    with torch.cuda.device(0):
        dev = lambda a: _dev(a, "cuda:0")           # noqa: E731
        want = [one.kad_median_sq(dev(x)).cpu(), one.kad_sums(dev(zs), m, sig.to("cuda:0")).cpu(),
                one.kad_song_sums(dev(z_songs), m, dev(off), sig.to("cuda:0")).cpu()]

    def run(r, e):
        dv = f"cuda:{r}"
        s = sig.to(dv)
        return [e.kad_median_sq_sharded(_dev(x, dv)).cpu(), e.kad_sums_sharded(_dev(zs, dv), m, s).cpu(),
                e.kad_song_sums_sharded(_dev(z_songs, dv), m, _dev(off, dv), s).cpu()]
    for r, got in enumerate(_on_both(pair, run)):
        assert not isinstance(got, Exception), got
        for g, w in zip(got, want):
            assert torch.equal(g, w), r


def test_two_devices_disagreement_fails_both(pair):
    x, y = encodec_like(700, 128, 12), encodec_like(500, 128, 13)
    z = np.concatenate([x, y])
    z_changed = z.copy()
    z_changed[901] += np.float16(0.5)
    sig = _sigma(x, "cpu")
    cases = {"(m, n)": lambda r: (z, 700 if r == 0 else 701), "(z)": lambda r: (z if r == 0 else z_changed, 700)}
    for what, args in cases.items():
        def run(r, e):
            zz, m = args(r)
            before = e.launches
            try:
                e.kad_sums_sharded(_dev(zz, f"cuda:{r}"), m, sig.to(f"cuda:{r}"))
            except NativeError as err:
                return str(err), e.launches - before
            return None, e.launches - before
        res = _on_both(pair, run)
        assert all(isinstance(msg, str) for msg, _ in res), (what, res)
        assert res[0][0] == res[1][0] and what in res[0][0], (what, res)
        assert all(n <= 1 for _, n in res), (what, res)      # at most the digest kernel: no tile work
    # a rank whose own checks reject the call: both fail with the same message, neither blocks
    def bad(r, e):
        try:
            e.kad_median_sq_sharded(_dev(x if r == 0 else x[:1], f"cuda:{r}"))
        except NativeError as err:
            return str(err)
    res = _on_both(pair, bad)
    assert res[0] == res[1] and "rejected" in res[0], res
    # the communicator still works afterwards
    got = _on_both(pair, lambda r, e: e.kad_median_sq_sharded(_dev(x, f"cuda:{r}")).cpu())
    assert torch.equal(got[0], got[1])
