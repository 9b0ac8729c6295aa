"""Kernel Audio Distance without a GPU: the fp64 oracle against the definition written as a double loop, the argument
errors of calc_kernel_audio_distance and of ``python -m fadtk_b200.kad``, and the zero-padding of the width (with the
device calls replaced by the oracle)."""
import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native, fad as fad_mod, kad as kad_cli
from oracle import kad_oracle as ko


def _rows(m, d, seed, offset=0.0):
    return (offset + np.random.default_rng(seed).standard_normal((m, d))).astype(np.float16)


@pytest.mark.parametrize("m,n", [(5, 4), (6, 7), (2, 2)])        # 10 (even), 15 (odd), 1 baseline pairs
def test_oracle_matches_double_loop(m, n):
    x, y = _rows(m, 16, 1, 30.0), _rows(n, 16, 2, 30.5)
    got, sigma = ko.kad(x, y)
    want, sigma_d = ko.kad_direct(x, y)
    assert abs(sigma - sigma_d) <= 1e-12 * sigma_d
    assert abs(got - want) <= 1e-9 * max(1.0, abs(want)), (got, want)
    d2 = sorted(((x[i].astype(np.float64) - x[j]) ** 2).sum() for i in range(m) for j in range(i + 1, m))
    p = len(d2)
    assert np.allclose(ko.middle_sq(x), (d2[(p - 1) // 2], d2[p // 2]), rtol=1e-12, atol=0)


def test_oracle_with_ties():
    x = np.repeat(_rows(4, 8, 3), 2, axis=0)                     # every distance four times, four zero pairs
    y = _rows(5, 8, 4)
    got, sigma = ko.kad(x, y)
    want, sigma_d = ko.kad_direct(x, y)
    assert abs(sigma - sigma_d) <= 1e-12 * sigma_d and abs(got - want) <= 1e-9 * max(1.0, abs(want))


@pytest.mark.parametrize("m,n", [(1, 5), (5, 1), (0, 3)])
def test_too_few_rows(m, n):
    with pytest.raises(ValueError, match="at least two"):
        fk.calc_kernel_audio_distance(_rows(m, 8, 5), _rows(n, 8, 6))


def test_bad_inputs():
    with pytest.raises(ValueError, match="fp16"):
        fk.calc_kernel_audio_distance(_rows(4, 8, 5).astype(np.float32), _rows(4, 8, 6))
    with pytest.raises(ValueError, match="widths differ"):
        fk.calc_kernel_audio_distance(_rows(4, 8, 5), _rows(4, 16, 6))
    with pytest.raises(ValueError, match=r"\[rows, d\]"):
        fk.calc_kernel_audio_distance(_rows(4, 8, 5)[None], _rows(4, 8, 6))


class _OracleEngine:
    """Stands in for _native.Engine: the two KAD stages computed by the oracle on the host."""
    torch_device = torch.device("cpu")

    def __init__(self):
        self.widths = []

    def kad_median_sq(self, x):
        self.widths.append(x.numpy().copy())
        return torch.tensor(ko.middle_sq(x.numpy()), dtype=torch.float64)

    def kad_sums(self, z, m, sigma):
        zn = z.numpy()
        return torch.tensor(ko.kernel_sums(zn[:m], zn[m:], float(sigma[0])), dtype=torch.float64)


def test_width_is_zero_padded_to_a_multiple_of_8(monkeypatch):
    eng = _OracleEngine()
    monkeypatch.setattr(_native, "engine", lambda *a, **k: eng)
    x, y = _rows(30, 100, 7), _rows(20, 100, 8, 0.3)
    got = fk.calc_kernel_audio_distance(x, y)
    want, sigma = ko.kad(x, y)
    assert eng.widths[0].shape == (30, 104) and not eng.widths[0][:, 100:].any()
    assert abs(got.bandwidth - sigma) <= 1e-12 * sigma and abs(got.score - want) <= 1e-9 * abs(want)
    assert (got.n_baseline, got.n_eval) == (30, 20)


class _ML:
    name = "vggish"


@pytest.fixture
def cli(monkeypatch, tmp_path):
    monkeypatch.setattr(kad_cli, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(kad_cli, "_embed_directories", lambda *a: pytest.fail("embedding started before the checks"))
    (tmp_path / "base").mkdir()
    (tmp_path / "eval").mkdir()
    return tmp_path


def test_cli_refuses_statistics_files(cli):
    npz = cli / "base.npz"
    np.savez(npz, **{"vggish.mu": np.zeros(128), "vggish.cov": np.eye(128)})
    with pytest.raises(ValueError, match="not \\(mu, C\\) statistics"):
        kad_cli.main(["vggish", str(npz), str(cli / "eval")])
    with pytest.raises(ValueError, match="not \\(mu, C\\) statistics"):
        kad_cli.main(["vggish", str(cli / "base"), str(npz)])


def test_cli_refuses_named_statistics(cli, monkeypatch):
    with pytest.raises(ValueError, match="not a directory"):
        kad_cli.main(["vggish", "fma_pop", str(cli / "eval")])
    stats = cli / "stats"
    stats.mkdir()
    np.savez(stats / "fma_pop.npz", **{"vggish.mu": np.zeros(128), "vggish.cov": np.eye(128)})
    monkeypatch.setenv("FADTK_STATS_DIR", str(stats))
    with pytest.raises(ValueError, match="not \\(mu, C\\) statistics"):
        kad_cli.main(["vggish", "fma_pop", str(cli / "eval")])


def test_cli_refuses_a_csv_with_another_header(cli):
    out = cli / "scores.csv"
    out.write_text("model,baseline,eval,score,inf_r2,time\n")
    with pytest.raises(ValueError, match="header"):
        kad_cli.main(["vggish", str(cli / "base"), str(cli / "eval"), str(out)])
    assert out.read_text() == "model,baseline,eval,score,inf_r2,time\n"


def test_score_kad_refuses_statistics(tmp_path):
    fad = fad_mod.FrechetAudioDistance.__new__(fad_mod.FrechetAudioDistance)
    fad.ml, fad.audio_load_worker = _ML(), 1
    npz = tmp_path / "s.npz"
    np.savez(npz, a=np.zeros(1))
    with pytest.raises(ValueError, match="statistics"):
        fad.score_kad(npz, tmp_path)
    with pytest.raises(ValueError, match="no vggish embeddings"):
        fad.score_kad(tmp_path, tmp_path)
