"""Host-side logic of the FAD comparison: argument checks that raise before any GPU work, the command line's csv
header and its refusal of another header, and the C ABI (include/fadtk_b200.h, _native.SIGNATURES) of the new
entries."""
import re
from pathlib import Path

import numpy as np
import pytest

import fadtk_b200 as fk
from fadtk_b200 import _native

ROOT = Path(__file__).resolve().parent.parent
ENTRIES = ["fad_unit_records", "fad_perm_record_sums", "fad_frechet_records", "fad_frechet_perm"]


def _files(count, rows=3, d=64, dtype=np.float16):
    rng = np.random.default_rng(count)
    return [rng.standard_normal((rows, d)).astype(dtype) for _ in range(count)]


BASE = (np.zeros(64), np.eye(64))


@pytest.mark.parametrize("perms", [0, 10000, -1, 2.5, True, "9"])
def test_bad_permutations(perms):
    with pytest.raises(ValueError, match="permutations in"):
        fk.calc_fad_comparison(BASE, _files(3), _files(3), permutations=perms)


@pytest.mark.parametrize("seed", [-1, 2 ** 64, 1.0, None])
def test_bad_seed(seed):
    with pytest.raises(ValueError, match="seed in"):
        fk.calc_fad_comparison(BASE, _files(3), _files(3), seed=seed)


def test_bad_baseline_and_units():
    with pytest.raises(ValueError, match=r"\(mu, cov\)"):
        fk.calc_fad_comparison(np.zeros(64), _files(3), _files(3))
    with pytest.raises(ValueError, match="mu \\[d\\], cov \\[d, d\\]"):
        fk.calc_fad_comparison((np.zeros(64), np.eye(32)), _files(3), _files(3))
    with pytest.raises(ValueError, match="multiple of 64"):
        fk.calc_fad_comparison((np.zeros(48), np.eye(48)), _files(3, d=48), _files(3, d=48))
    with pytest.raises(ValueError, match="at least two units"):
        fk.calc_fad_comparison(BASE, _files(1), _files(3))
    with pytest.raises(ValueError, match="at least two units"):
        fk.calc_fad_comparison(BASE, _files(3), _files(1, rows=1)[0])
    with pytest.raises(ValueError, match="fp16"):
        fk.calc_fad_comparison(BASE, _files(3, dtype=np.float32), _files(3))
    with pytest.raises(ValueError, match="baseline's width"):
        fk.calc_fad_comparison(BASE, _files(3), _files(3, d=128))
    with pytest.raises(ValueError, match="at least one row"):
        fk.calc_fad_comparison(BASE, _files(3) + [np.zeros((0, 64), np.float16)], _files(3))


def test_abi_symbols():
    header = (ROOT / "include" / "fadtk_b200.h").read_text()
    for name in ENTRIES:
        assert re.search(rf"\bint {name}\(", header), name
        assert name in _native.SIGNATURES, name
        decl = re.search(rf"\bint {name}\(([^;]*)\);", header, re.S).group(1)
        assert len(decl.split(",")) == len(_native.SIGNATURES[name][1]), name
    assert re.search(r"\blong long fad_record_len\(int d\);", header)


def test_result_fields():
    assert fk.FADComparisonResults._fields == ("score_a", "score_b", "difference", "observed", "p_value",
                                               "null_differences", "permutations", "seed", "n_units_a", "n_units_b",
                                               "n_rows_a", "n_rows_b")


class _ML:
    name = "vggish"


@pytest.fixture
def cli(monkeypatch, tmp_path):
    from fadtk_b200 import fad_test
    monkeypatch.setattr(fad_test, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(fad_test, "_embed_directories", lambda *a: pytest.fail("embedding started before the checks"))
    for d in ("base", "eval", "other"):
        (tmp_path / d).mkdir()
    return fad_test, tmp_path


def test_cli_header():
    from fadtk_b200 import fad_test
    assert fad_test.CSV_HEADER == ("model,baseline,eval,versus,fad,fad_versus,difference,observed,p_value,permutations,"
                                   "seed,n_files_eval,n_files_versus,time\n")


def test_cli_refuses_a_csv_with_another_header(cli):
    mod, root = cli
    out = root / "scores.csv"
    from fadtk_b200 import kad_test
    out.write_text(kad_test.CSV_HEADER)
    with pytest.raises(ValueError, match="header"):
        mod.main(["vggish", str(root / "base"), str(root / "eval"), str(root / "other"), str(out)])
    assert out.read_text() == kad_test.CSV_HEADER


def test_cli_checks_before_embedding(cli):
    mod, root = cli
    dirs = [str(root / k) for k in ("base", "eval", "other")]
    with pytest.raises(ValueError, match="permutations in"):
        mod.main(["vggish", *dirs, "--permutations", "0"])
    with pytest.raises(ValueError, match="seed in"):
        mod.main(["vggish", *dirs, "--seed", "-1"])
    npz = root / "s.npz"
    np.savez(npz, **{"vggish.mu": np.zeros(128), "vggish.cov": np.eye(128)})
    with pytest.raises(ValueError, match="statistics"):
        mod.main(["vggish", dirs[0], dirs[1], str(npz)])
