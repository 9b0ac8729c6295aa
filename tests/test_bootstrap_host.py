"""Host-side logic of the bootstrap intervals: argument checks that raise before any GPU work, the interval formulas
of the Python layer, the command line's arguments, csv header and refusal of another header, and the C ABI of the new
entries (include/fadtk_b200.h, _native.SIGNATURES)."""
import re
from pathlib import Path

import numpy as np
import pytest

import fadtk_b200 as fk
from fadtk_b200 import _native
from fadtk_b200 import fad as fadmod
from oracle import bootstrap_oracle as bo

ROOT = Path(__file__).resolve().parent.parent
ENTRIES = ["fad_boot_counts", "fad_boot_record_sums", "fad_frechet_boot", "fad_kad_boot_sums"]
BASE = (np.zeros(64), np.eye(64))


def _files(count, rows=3, d=64, dtype=np.float16):
    rng = np.random.default_rng(count)
    return [rng.standard_normal((rows, d)).astype(dtype) for _ in range(count)]


@pytest.fixture(autouse=True)
def no_gpu(monkeypatch):
    monkeypatch.setattr(_native, "engine", lambda *a, **k: pytest.fail("GPU work started before the checks"))


@pytest.mark.parametrize("fn", [fk.calc_fad_bootstrap, fk.calc_kad_bootstrap])
@pytest.mark.parametrize("kw,msg", [
    (dict(resamples=1), "resamples in"), (dict(resamples=10000), "resamples in"), (dict(resamples=2.0), "resamples in"),
    (dict(resamples=True), "resamples in"), (dict(seed=-1), "seed in"), (dict(seed=2 ** 64), "seed in"),
    (dict(seed=None), "seed in"), (dict(level=0.0), "level"), (dict(level=1.0), "level"), (dict(level="0.9"), "level"),
    (dict(level=float("nan")), "level"), (dict(method="bca"), "method"),
])
def test_bad_arguments(fn, kw, msg):
    base = BASE if fn is fk.calc_fad_bootstrap else _files(1, rows=20)[0]
    with pytest.raises(ValueError, match=msg):
        fn(base, _files(3), **kw)


def test_bad_fad_baseline_and_units():
    with pytest.raises(ValueError, match=r"\(mu, cov\)"):
        fk.calc_fad_bootstrap(np.zeros(64), _files(3))
    with pytest.raises(ValueError, match="multiple of 64"):
        fk.calc_fad_bootstrap((np.zeros(48), np.eye(48)), _files(3, d=48))
    with pytest.raises(ValueError, match="at least two units"):
        fk.calc_fad_bootstrap(BASE, _files(1))
    with pytest.raises(ValueError, match="at least two units"):
        fk.calc_fad_bootstrap(BASE, _files(1, rows=1)[0])
    with pytest.raises(ValueError, match="fp16"):
        fk.calc_fad_bootstrap(BASE, _files(3, dtype=np.float32))
    with pytest.raises(ValueError, match="baseline's width"):
        fk.calc_fad_bootstrap(BASE, _files(3, d=128))
    with pytest.raises(ValueError, match="at least one row"):
        fk.calc_fad_bootstrap(BASE, _files(3) + [np.zeros((0, 64), np.float16)])


def test_bad_kad_baseline_and_units():
    x = _files(1, rows=20)[0]
    with pytest.raises(ValueError, match="at least two units"):
        fk.calc_kad_bootstrap(x, _files(1))
    with pytest.raises(ValueError, match="at least one row"):
        fk.calc_kad_bootstrap(x, _files(3) + [np.zeros((0, 64), np.float16)])
    with pytest.raises(ValueError, match="fp16"):
        fk.calc_kad_bootstrap(x, _files(3, dtype=np.float32))
    with pytest.raises(ValueError, match="widths differ"):
        fk.calc_kad_bootstrap(x, _files(3, d=128))
    with pytest.raises(ValueError, match="at least two embedding rows"):
        fk.calc_kad_bootstrap(x[:1], _files(3))


@pytest.mark.parametrize("method", ["percentile", "basic"])
def test_interval_matches_oracle(method):
    theta = np.random.default_rng(3).standard_normal(1000) + 4.0
    assert fadmod._boot_interval(theta, 0.9, method) == bo.interval(theta, 0.9, method)


def test_abi_symbols():
    header = (ROOT / "include" / "fadtk_b200.h").read_text()
    for name in ENTRIES:
        assert name in _native.SIGNATURES, name
        decl = re.search(rf"\bint {name}\(([^;]*)\);", header, re.S).group(1)
        assert len(decl.split(",")) == len(_native.SIGNATURES[name][1]), name


def test_result_fields():
    fields = ("score", "observed", "ci_low", "ci_high", "standard_error", "bias", "replicates", "level", "method",
              "resamples", "seed", "n_units", "n_rows")
    assert fk.FADBootstrapResults._fields == fields
    assert fk.KADBootstrapResults._fields == fields + ("bandwidth", "n_baseline")


class _ML:
    name = "vggish"


@pytest.fixture
def cli(monkeypatch, tmp_path):
    from fadtk_b200 import bootstrap
    monkeypatch.setattr(bootstrap, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(bootstrap, "_embed_directories", lambda *a: pytest.fail("embedding started before the checks"))
    for d in ("base", "eval"):
        (tmp_path / d).mkdir()
    return bootstrap, tmp_path


def test_cli_header():
    from fadtk_b200 import bootstrap
    assert bootstrap.CSV_HEADER == ("metric,model,baseline,eval,score,observed,ci_low,ci_high,level,method,"
                                    "standard_error,bias,resamples,seed,n_files,n_rows,time\n")


def test_cli_parses_its_arguments():
    from fadtk_b200 import bootstrap
    from fadtk_b200.cli import _parser
    p = _parser("fadtk_b200.bootstrap", bootstrap._ARGS, {"vggish": _ML()})
    a = p.parse_args(["kad", "vggish", "b", "e", "out.csv", "--resamples", "50", "--seed", "3", "--level", "0.9",
                      "--method", "basic", "--prepared"])
    assert (a.metric, a.baseline, a.eval, a.csv, a.resamples, a.seed, a.level, a.method, a.prepared) == \
        ("kad", "b", "e", "out.csv", 50, 3, 0.9, "basic", True)
    a = p.parse_args(["fad", "vggish", "b", "e"])
    assert (a.csv, a.resamples, a.seed, a.level, a.method, a.prepared) == (None, 999, 0, 0.95, "percentile", False)
    with pytest.raises(SystemExit):
        p.parse_args(["prdc", "vggish", "b", "e"])
    with pytest.raises(SystemExit):
        p.parse_args(["fad", "vggish", "b", "e", "--method", "bca"])


def test_cli_refuses_a_csv_with_another_header(cli):
    mod, root = cli
    out = root / "scores.csv"
    from fadtk_b200 import fad_test
    out.write_text(fad_test.CSV_HEADER)
    with pytest.raises(ValueError, match="header"):
        mod.main(["fad", "vggish", str(root / "base"), str(root / "eval"), str(out)])
    assert out.read_text() == fad_test.CSV_HEADER


def test_cli_checks_before_embedding(cli):
    mod, root = cli
    dirs = [str(root / k) for k in ("base", "eval")]
    with pytest.raises(ValueError, match="resamples in"):
        mod.main(["fad", "vggish", *dirs, "--resamples", "1"])
    with pytest.raises(ValueError, match="level"):
        mod.main(["kad", "vggish", *dirs, "--level", "1.5"])
    with pytest.raises(ValueError, match="kad bootstrap only"):
        mod.main(["fad", "vggish", *dirs, "--prepared"])
    npz = root / "s.npz"
    np.savez(npz, **{"vggish.mu": np.zeros(128), "vggish.cov": np.eye(128)})
    with pytest.raises(ValueError, match="statistics"):
        mod.main(["kad", "vggish", str(npz), dirs[1]])
    with pytest.raises(ValueError, match="statistics"):
        mod.main(["fad", "vggish", dirs[0], str(npz)])
