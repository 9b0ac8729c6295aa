"""Host side of the prepared baseline (DESIGN.md 5.15): the saved file's format and atomic write, when a saved
preparation is used and when it is recomputed, the --prepared flags, the prepare command line's argument errors, and
the radius-list definition restated in numpy.  The native passes are stood in for by an fp64 host engine."""
import hashlib
import logging

import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native, fad as fad_mod, kad as kad_cli, nearest as nearest_cli, prdc as prdc_cli
from fadtk_b200 import prepare as prepare_cli, realism as realism_cli


def _rows(rows, d, seed, scale=1.0):
    return (scale * np.random.default_rng(seed).standard_normal((rows, d))).astype(np.float16)


def lists_sq(x: np.ndarray, k: int) -> np.ndarray:
    """per row of x the k smallest |x_i - x_j|^2 over j != i (the self pair excluded by index), ascending, in fp64"""
    a = x.astype(np.float64)
    q = (a * a).sum(1)[:, None] + (a * a).sum(1)[None, :] - 2.0 * a @ a.T
    np.fill_diagonal(q, np.inf)
    return np.sort(np.maximum(q, 0.0), axis=1)[:, :k]


def test_lists_restatement_matches_the_definition():
    x = _rows(40, 8, 1)
    x[5] = x[9] = x[11]                          # duplicates: neighbours at 0, the self pair still excluded
    got = lists_sq(x, 16)
    a = x.astype(np.float64)
    for i in range(40):
        q = sorted(float(((a[i] - a[j]) ** 2).sum()) for j in range(40) if j != i)[:16]
        assert np.allclose(got[i], q, rtol=1e-12, atol=1e-12)
    assert (got[[5, 9, 11], :2] == 0).all() and (got[[5, 9, 11], 2] > 0).all()


class _HostEngine:
    """Stands in for _native.Engine: the preparation's passes in fp64 on the host."""
    torch_device = torch.device("cpu")

    def __init__(self):
        self.prepared = 0

    def pair_digest(self, z):
        return int.from_bytes(hashlib.sha1(z.numpy().tobytes()).digest()[:8], "little")

    def kad_median_sq(self, x):
        a = x.numpy().astype(np.float64)
        q = np.sort(((a[:, None] - a[None]) ** 2).sum(-1)[np.triu_indices(len(a), 1)])
        return torch.tensor([q[(q.size - 1) // 2], q[q.size // 2]], dtype=torch.float64)

    def kad_song_sums(self, x, m, offsets, sigma):
        a = x.numpy().astype(np.float64)
        q = ((a[:, None] - a[None]) ** 2).sum(-1)[np.triu_indices(m, 1)]
        return torch.tensor([np.exp(-q / (2 * float(sigma[0]) ** 2)).sum()], dtype=torch.float64)

    def knn_lists_sq(self, x, k_max, local_shards=None):
        self.prepared += 1
        return torch.from_numpy(lists_sq(x.numpy(), k_max).astype(np.float32))


@pytest.fixture
def host_engine(monkeypatch):
    eng = _HostEngine()
    monkeypatch.setattr(_native, "engine", lambda *a, **k: eng)
    return eng


class _ML:
    name = "vggish"


def _fad():
    f = fad_mod.FrechetAudioDistance.__new__(fad_mod.FrechetAudioDistance)
    f.ml, f.audio_load_worker = _ML(), 1
    return f


def _cache(root, stem, arr):
    emb = root / "embeddings" / "vggish"
    emb.mkdir(parents=True, exist_ok=True)
    np.save(emb / f"{stem}.npy", arr)


def test_prepare_keeps_the_lists_and_checks_its_arguments(host_engine):
    x = _rows(30, 12, 2)
    pb = fk.prepare_pairwise_baseline(x, 6, [0, 10, 10, 30])
    assert (pb.m, pb.d, pb.k_max, tuple(pb.x.shape)) == (30, 12, 6, (30, 16))
    assert np.array_equal(pb.lists.numpy(), lists_sq(np.pad(x, ((0, 0), (0, 4))), 6).astype(np.float32))
    with pytest.raises(ValueError, match="more than k_max rows"):
        fk.prepare_pairwise_baseline(x[:6], 6)
    with pytest.raises(ValueError, match="integer k in \\[1, 16\\]"):
        fk.prepare_pairwise_baseline(x, 17)
    with pytest.raises(ValueError, match="offsets must rise from 0 to m = 30"):
        fk.prepare_pairwise_baseline(x, 6, [0, 20, 10, 30])
    with pytest.raises(ValueError, match="k_max >= k"):
        fk.calc_prdc(pb, x, 7)
    with pytest.raises(ValueError, match="widths differ"):
        fk.calc_realism(pb, _rows(5, 8, 3), 3)


def test_saved_file_format_and_atomic_write(host_engine, tmp_path):
    x = _rows(25, 8, 4)
    pb = fk.prepare_pairwise_baseline(x, 4, [0, 25])
    path = tmp_path / "stats" / "vggish" / "pairwise.npz"
    pb.save(path, {"files": 1})
    assert sorted(p.name for p in path.parent.iterdir()) == ["pairwise.npz"]       # no temporary file left
    with np.load(path) as f:
        assert {"version", "build", "m", "d", "k_max", "digest", "median_sq", "sigma", "s_xx", "lists", "offsets",
                "fingerprint"} <= set(f.files)
        assert (int(f["m"]), int(f["d"]), int(f["k_max"]), f["lists"].shape) == (25, 8, 4, (25, 4))
        assert int(f["digest"]) == pb.digest and str(f["build"]) == _native.build_id()
    back, why = _native.PairwiseBaseline.load(path, host_engine, pb.x, 4, 8, {"files": 1}, [0, 25])
    assert why == "" and np.array_equal(back.lists.numpy(), pb.lists.numpy()) and back.sigma == pb.sigma
    for args, reason in ((({"files": 2}, [0, 25]), "embedding files changed"), (({"files": 1}, None), "offsets differ")):
        assert _native.PairwiseBaseline.load(path, host_engine, pb.x, 4, 8, *args) == (None, f"the {reason}") or \
            reason in _native.PairwiseBaseline.load(path, host_engine, pb.x, 4, 8, *args)[1]
    assert "k_max is 4, below 5" in _native.PairwiseBaseline.load(path, host_engine, pb.x, 5, 8, {"files": 1}, [0, 25])[1]
    with np.load(path) as f:
        st = {k: f[k] for k in f.files}
    for key, val, reason in (("version", np.int64(99), "format version"), ("build", np.array("other"), "another build"),
                             ("lists", st["lists"][:, :2], "wrong shape")):
        np.savez(path, **{**st, key: val})
        assert reason in _native.PairwiseBaseline.load(path, host_engine, pb.x, 2, 8, {"files": 1}, [0, 25])[1]
    path.write_bytes(b"not an npz")
    assert "cannot be read" in _native.PairwiseBaseline.load(path, host_engine, pb.x, 2, 8, {"files": 1}, [0, 25])[1]


def test_saved_preparation_is_reused_until_the_embeddings_change(host_engine, tmp_path, caplog):
    base = tmp_path / "base"
    _cache(base, "a", _rows(20, 8, 5))
    _cache(base, "b", _rows(15, 8, 6))
    f = _fad()
    caplog.set_level(logging.INFO, logger="fadtk_b200")
    pb = f.prepare_pairwise(base, k_max=5)
    assert host_engine.prepared == 1 and np.array_equal(pb.offsets, [0, 20, 35])
    assert (base / "stats" / "vggish" / "pairwise.npz").is_file()
    f.prepare_pairwise(base, k_max=5)
    f.prepare_pairwise(base, k_max=3)                       # a saved k_max above the one asked for serves
    assert host_engine.prepared == 1
    f.prepare_pairwise(base, k_max=8)                       # k_max < k: never trusted
    assert host_engine.prepared == 2
    for change in ("touch", "add", "remove"):
        caplog.clear()
        if change == "touch":
            _cache(base, "a", _rows(20, 8, 5))
        elif change == "add":
            _cache(base, "c", _rows(4, 8, 7))
        else:
            (base / "embeddings" / "vggish" / "c.npy").unlink()
        f.prepare_pairwise(base, k_max=5)
        assert "the embedding files changed, computing" in caplog.text, change
    assert host_engine.prepared == 5


def test_prepared_flags_default_off():
    for mod, table, argv in ((kad_cli, kad_cli._KAD_ARGS, []), (prdc_cli, prdc_cli._PRDC_ARGS, []),
                             (realism_cli, realism_cli._REALISM_ARGS, []), (nearest_cli, nearest_cli._NEAREST_ARGS, [])):
        ap = mod._parser("x", table, {"vggish": _ML()})
        assert ap.parse_args(["vggish", "b", "e", *argv]).prepared is False
        assert ap.parse_args(["vggish", "b", "e", "--prepared"]).prepared is True


@pytest.fixture
def prepare_dirs(monkeypatch, tmp_path):
    monkeypatch.setattr(prepare_cli, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(prepare_cli, "_embed_directories", lambda *a: pytest.fail("embedding started before the checks"))
    (tmp_path / "base").mkdir()
    return tmp_path


def test_prepare_cli_argument_errors(prepare_dirs):
    ap = prepare_cli._parser("fadtk_b200.prepare", prepare_cli._PREPARE_ARGS, {"vggish": _ML()})
    assert ap.parse_args(["vggish", "b"]).k_max == 16 and ap.parse_args(["vggish", "b", "--k-max", "5"]).k_max == 5
    for k in ("0", "17"):
        with pytest.raises(ValueError, match="k_max in \\[1, 16\\]"):
            prepare_cli.main(["vggish", str(prepare_dirs / "base"), "--k-max", k])
    npz = prepare_dirs / "base.npz"
    np.savez(npz, **{"vggish.mu": np.zeros(8), "vggish.cov": np.eye(8)})
    with pytest.raises(ValueError, match="needs embeddings, not \\(mu, C\\) statistics"):
        prepare_cli.main(["vggish", str(npz)])
    with pytest.raises(ValueError, match="not a directory"):
        prepare_cli.main(["vggish", str(prepare_dirs / "nowhere")])
    with pytest.raises(SystemExit):
        prepare_cli.main(["vggish"])
