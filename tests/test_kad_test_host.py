"""Host-side logic of the KAD permutation tests: argument checks that raise before any GPU work, and the C ABI
(include/fadtk_b200.h, _native.SIGNATURES) of the new entries."""
import re
from pathlib import Path

import numpy as np
import pytest

import fadtk_b200 as fk
from fadtk_b200 import _native

ROOT = Path(__file__).resolve().parent.parent
ENTRIES = ["fad_perm_labels", "fad_perm_dot", "fad_kad_perm_sums", "fad_kad_perm_sums_sharded"]


def _rows(n, d=16):
    return np.random.default_rng(n).standard_normal((n, d)).astype(np.float16)


@pytest.mark.parametrize("perms", [0, 10000, -1, 2.5, True, "9"])
def test_bad_permutations(perms):
    with pytest.raises(ValueError, match="permutations in"):
        fk.calc_kad_test(_rows(10), _rows(10), permutations=perms)
    with pytest.raises(ValueError, match="permutations in"):
        fk.calc_kad_comparison(_rows(10), _rows(10), _rows(11), permutations=perms)


@pytest.mark.parametrize("seed", [-1, 2 ** 64, 1.0, None])
def test_bad_seed(seed):
    with pytest.raises(ValueError, match="seed in"):
        fk.calc_kad_test(_rows(10), _rows(10), seed=seed)


def test_too_few_rows_and_widths():
    with pytest.raises(ValueError, match="at least two embedding rows"):
        fk.calc_kad_test(_rows(10), _rows(1))
    with pytest.raises(ValueError, match="at least two embedding rows"):
        fk.calc_kad_comparison(_rows(10), _rows(5), _rows(1))
    with pytest.raises(ValueError, match="embedding widths differ"):
        fk.calc_kad_test(_rows(10), _rows(10, 8))
    with pytest.raises(ValueError, match="fp16"):
        fk.calc_kad_comparison(_rows(10), _rows(5).astype(np.float32), _rows(5))


def test_abi_symbols():
    header = (ROOT / "include" / "fadtk_b200.h").read_text()
    for name in ENTRIES:
        assert re.search(rf"\bint {name}\(", header), name
        assert name in _native.SIGNATURES, name
    # argument counts of the declarations match the ctypes signatures
    for name in ENTRIES:
        decl = re.search(rf"\bint {name}\(([^;]*)\);", header, re.S).group(1)
        assert len(decl.split(",")) == len(_native.SIGNATURES[name][1]), name


def test_result_fields():
    assert fk.KADTestResults._fields == ("score", "bandwidth", "p_value", "null_scores", "observed", "permutations",
                                         "seed", "n_baseline", "n_eval")
    assert fk.KADComparisonResults._fields == ("score_a", "score_b", "difference", "p_value", "null_differences",
                                               "bandwidth", "permutations", "seed", "n_baseline", "n_a", "n_b")


class _ML:
    name = "vggish"


@pytest.fixture
def cli(monkeypatch, tmp_path):
    from fadtk_b200 import kad_test
    monkeypatch.setattr(kad_test, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(kad_test, "_embed_directories", lambda *a: pytest.fail("embedding started before the checks"))
    for d in ("base", "eval", "other"):
        (tmp_path / d).mkdir()
    return kad_test, tmp_path


def test_cli_header():
    from fadtk_b200 import kad, kad_test
    assert kad_test.CSV_HEADER == ("model,baseline,eval,versus,kad,kad_versus,difference,p_value,permutations,seed,"
                                   "bandwidth,n_baseline,n_eval,n_versus,time\n")
    assert kad.CSV_HEADER == "model,baseline,eval,kad,bandwidth,n_baseline,n_eval,time\n"


def test_cli_refuses_a_csv_with_another_header(cli):
    mod, root = cli
    out = root / "scores.csv"
    from fadtk_b200 import kad
    out.write_text(kad.CSV_HEADER)
    with pytest.raises(ValueError, match="header"):
        mod.main(["vggish", str(root / "base"), str(root / "eval"), str(out)])
    with pytest.raises(ValueError, match="header"):
        mod.main(["vggish", str(root / "base"), str(root / "eval"), str(out), "--versus", str(root / "other")])
    assert out.read_text() == kad.CSV_HEADER


def test_cli_checks_before_embedding(cli):
    mod, root = cli
    with pytest.raises(ValueError, match="permutations in"):
        mod.main(["vggish", str(root / "base"), str(root / "eval"), "--permutations", "0"])
    with pytest.raises(ValueError, match="seed in"):
        mod.main(["vggish", str(root / "base"), str(root / "eval"), "--seed", "-1"])
    npz = root / "s.npz"
    np.savez(npz, **{"vggish.mu": np.zeros(128), "vggish.cov": np.eye(128)})
    with pytest.raises(ValueError, match="statistics"):
        mod.main(["vggish", str(root / "base"), str(root / "eval"), "--versus", str(npz)])
