"""``python -m fadtk_b200.prdc <model> <baseline> <eval> [csv] [-k K] [--indiv] [--prepared] [-w N] [-s sox]`` - precision,
recall, density and coverage of an eval directory against a baseline directory (fad.calc_prdc on the cached embeddings).
Directories without embedding caches are embedded first (under ``torchrun`` the embedding is sharded over the ranks as
for ``fadtk``). Under ``torchrun`` every rank then takes its share of the radii and ball-count tiles
(``distributed=True``) when the library's NCCL communicator can be set up, and rank 0 scores alone otherwise; either way
rank 0 alone reports and writes. With ``csv``, one row
``model,baseline,eval,k,precision,recall,density,coverage,n_baseline,n_eval,time`` is appended; a new file gets the
header first, and an existing file with another header is refused rather than mixed. With ``--indiv``, every file of the
eval directory is scored on its own against the baseline (FrechetAudioDistance.score_prdc_individual) and ``csv`` is
that table (default prdc-individual-results.csv).
"""
from __future__ import annotations

import sys
import time
from pathlib import Path

from . import dist
from .cli import _embed_directories, _parser, _registry
from .kad import _append_row, _check_csv

CSV_HEADER = "model,baseline,eval,k,precision,recall,density,coverage,n_baseline,n_eval,time\n"
_PRDC_ARGS = (
    (("model",), dict(type=str, help="embedding model (a registry name)")),
    (("baseline",), dict(type=str, help="baseline audio directory (the real distribution)")),
    (("eval",), dict(type=str, help="evaluation audio directory")),
    (("csv",), dict(type=str, nargs="?", help="append the result row here; with --indiv: where the per-file table "
                                              "goes (default prdc-individual-results.csv)")),
    (("-k",), dict(type=int, default=5, help="nearest neighbour that sets each ball's radius, 1 to 16 (default 5)")),
    (("--indiv",), dict(action="store_true", help="score every evaluation file on its own against the baseline")),
    (("--prepared",), dict(action="store_true", help="score against the baseline's saved pairwise preparation "
                                                     "(python -m fadtk_b200.prepare), built and saved first when it is "
                                                     "missing or stale")),
)


def main(argv=None) -> int:
    from .fad import FrechetAudioDistance, kad_embedding_dir, log
    registry = _registry()
    args = _parser("fadtk_b200.prdc", _PRDC_ARGS, registry).parse_args(argv)
    if not 1 <= args.k <= 16:                       # before any embedding work, like the checks below
        raise ValueError(f"PRDC needs k in [1, 16], not {args.k}")
    model = registry[args.model]
    for p in (args.baseline, args.eval):            # statistics cannot give nearest neighbours
        kad_embedding_dir(p, model.name, "PRDC")
    if args.csv and not args.indiv:
        _check_csv(args.csv, CSV_HEADER, "PRDC")
    dist.init_from_env()
    _embed_directories(model, (args.baseline, args.eval), args.workers)
    from . import _native
    sharded = dist.is_distributed() and dist.enable_native_allreduce(_native.engine())
    if dist.rank() != 0 and not sharded:
        dist.shutdown()
        return 0

    fad = FrechetAudioDistance(model, audio_load_worker=args.workers, load_model=False)
    if args.indiv:
        table = Path(args.csv or "prdc-individual-results.csv")
        fad.score_prdc_individual(args.baseline, args.eval, table, k=args.k, distributed=sharded,
                                  prepared=args.prepared)
        if dist.rank() == 0:
            log.info(f"Individual PRDC values saved to {table}")
        dist.shutdown()
        return 0
    res = fad.score_prdc(args.baseline, args.eval, k=args.k, distributed=sharded, prepared=args.prepared)
    if dist.rank() != 0:
        dist.shutdown()
        return 0
    if args.csv:
        _append_row(args.csv, (model.name, args.baseline, args.eval, res.k, res.precision, res.recall, res.density,
                               res.coverage, res.n_baseline, res.n_eval, time.time()), CSV_HEADER)
        log.info(f"PRDC values appended to {args.csv}")
    print(f"The PRDC {model.name} values (k = {res.k}) of {args.eval} against {args.baseline} are: "
          f"precision {res.precision}, recall {res.recall}, density {res.density}, coverage {res.coverage}")
    dist.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
