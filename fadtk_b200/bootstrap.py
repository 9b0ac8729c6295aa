"""``python -m fadtk_b200.bootstrap {fad|kad} <model> <baseline> <eval> [csv] [--resamples 999] [--seed 0]
[--level 0.95] [--method percentile|basic] [--prepared] [-w N] [-s sox]`` - a bootstrap confidence interval of FAD or
KAD over the files of the eval directory, the baseline held fixed (fad.calc_fad_bootstrap, fad.calc_kad_bootstrap).
For fad the baseline is anything ``score`` takes (a directory, an ``.npz`` statistics file or a named set); for kad it
is a directory, and ``--prepared`` scores against its saved pairwise preparation.  Directories without embedding caches
are embedded first; under ``torchrun`` the ranks share the embedding and rank 0 computes.  With ``csv``, one row
``metric,model,baseline,eval,score,observed,ci_low,ci_high,level,method,standard_error,bias,resamples,seed,n_files,
n_rows,time`` is appended; a new file gets the header first, and an existing file with another header is refused.
"""
from __future__ import annotations

import sys
import time

from . import dist
from .cli import _embed_directories, _parser, _registry
from .kad import _append_row, _check_csv

CSV_HEADER = ("metric,model,baseline,eval,score,observed,ci_low,ci_high,level,method,standard_error,bias,resamples,seed,"
              "n_files,n_rows,time\n")
_ARGS = (
    (("metric",), dict(type=str, choices=("fad", "kad"), help="fad or kad")),
    (("model",), dict(type=str, help="embedding model (a registry name)")),
    (("baseline",), dict(type=str, help="baseline: an audio directory (fad also: an .npz statistics file or a named "
                                        "set)")),
    (("eval",), dict(type=str, help="evaluation audio directory; its files are resampled")),
    (("csv",), dict(type=str, nargs="?", help="append the result row here")),
    (("--resamples",), dict(type=int, default=999, help="bootstrap resamples, 2 to 9999 (default 999)")),
    (("--seed",), dict(type=int, default=0, help="seed of the resamples, 0 to 2**64 - 1 (default 0)")),
    (("--level",), dict(type=float, default=0.95, help="confidence level, strictly between 0 and 1 (default 0.95)")),
    (("--method",), dict(type=str, default="percentile", choices=("percentile", "basic"),
                         help="interval: percentile (default) or basic")),
    (("--prepared",), dict(action="store_true", help="kad only: score against the baseline's saved pairwise "
                                                     "preparation (python -m fadtk_b200.prepare)")),
)


def main(argv=None) -> int:
    from .fad import FrechetAudioDistance, _boot_args, kad_embedding_dir, log
    registry = _registry()
    args = _parser("fadtk_b200.bootstrap", _ARGS, registry).parse_args(argv)
    model = registry[args.model]
    _boot_args(args.resamples, args.seed, args.level, args.method, f"a {args.metric.upper()} bootstrap")
    if args.prepared and args.metric != "kad":
        raise ValueError("--prepared is for the kad bootstrap only")
    # before any embedding work: the units are the eval directory's cached files (and KAD needs baseline embeddings)
    kad_embedding_dir(args.eval, model.name, f"the {args.metric.upper()} bootstrap")
    if args.metric == "kad":
        kad_embedding_dir(args.baseline, model.name)
    if args.csv:
        _check_csv(args.csv, CSV_HEADER, "bootstrap")
    dist.init_from_env()
    _embed_directories(model, (args.baseline, args.eval), args.workers)
    if dist.rank() != 0:
        dist.shutdown()
        return 0

    fad = FrechetAudioDistance(model, audio_load_worker=args.workers, load_model=False)
    kw = dict(resamples=args.resamples, seed=args.seed, level=args.level, method=args.method)
    if args.metric == "fad":
        r = fad.score_fad_bootstrap(args.baseline, args.eval, **kw)
    else:
        r = fad.score_kad_bootstrap(args.baseline, args.eval, prepared=args.prepared, **kw)
    if args.csv:
        _append_row(args.csv, (args.metric, model.name, args.baseline, args.eval, r.score, r.observed, r.ci_low,
                               r.ci_high, r.level, r.method, r.standard_error, r.bias, r.resamples, r.seed, r.n_units,
                               r.n_rows, time.time()), CSV_HEADER)
        log.info(f"bootstrap appended to {args.csv}")
    print(f"The {args.metric.upper()} {model.name} score of {args.eval} against {args.baseline} is {r.score}: "
          f"{100 * r.level:g} % {r.method} interval [{r.ci_low}, {r.ci_high}] ({r.resamples} resamples of "
          f"{r.n_units} files)")
    dist.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
