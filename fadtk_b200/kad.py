"""``python -m fadtk_b200.kad <model> <baseline> <eval> [csv] [--indiv] [--prepared] [-w N] [-s sox]`` - Kernel Audio
Distance between two audio directories (fad.calc_kernel_audio_distance). Directories without embedding caches are
embedded first (under ``torchrun`` the embedding is sharded over the ranks as for ``fadtk``). Under ``torchrun`` every
rank then takes its share of the pair tiles (``distributed=True``) when the library's NCCL communicator can be set up,
and rank 0 scores alone otherwise; either way rank 0 alone reports and writes. With ``csv``, one row
``model,baseline,eval,kad,bandwidth,n_baseline,n_eval,time`` is appended; a new file gets the header first, and an
existing file with another header is refused rather than mixed. With ``--indiv``, every file of the eval directory is
scored on its own against the baseline (FrechetAudioDistance.score_kad_individual) and ``csv`` is that table (default
kad-individual-results.csv). The ``fadtk`` command line itself is unchanged.
"""
from __future__ import annotations

import sys
import time
from pathlib import Path

from . import dist
from .cli import _embed_directories, _parser, _registry

CSV_HEADER = "model,baseline,eval,kad,bandwidth,n_baseline,n_eval,time\n"
_KAD_ARGS = (
    (("model",), dict(type=str, help="embedding model (a registry name)")),
    (("baseline",), dict(type=str, help="baseline audio directory (its embeddings also set the kernel bandwidth)")),
    (("eval",), dict(type=str, help="evaluation audio directory")),
    (("csv",), dict(type=str, nargs="?", help="append the result row here; with --indiv: where the per-file table "
                                              "goes (default kad-individual-results.csv)")),
    (("--indiv",), dict(action="store_true", help="score every evaluation file on its own against the baseline")),
    (("--prepared",), dict(action="store_true", help="score against the baseline's saved pairwise preparation "
                                                     "(python -m fadtk_b200.prepare), built and saved first when it is "
                                                     "missing or stale")),
)


def _check_csv(csv_path: str, header: str = CSV_HEADER, metric: str = "KAD") -> None:
    """ValueError when csv_path exists with a first line other than header (shared with fadtk_b200.prdc)"""
    out = Path(csv_path)
    if out.is_file():
        with open(out) as f:
            head = f.readline()
        if head and head != header:
            raise ValueError(f"{csv_path} has the header {head.strip()!r}, not {header.strip()!r}: "
                             f"choose another file for {metric} results")


def _append_row(csv_path: str, row, header: str = CSV_HEADER) -> None:
    out = Path(csv_path)
    out.parent.mkdir(parents=True, exist_ok=True)
    if not out.is_file() or out.stat().st_size == 0:
        out.write_text(header)
    with open(out, "a") as f:
        f.write(",".join(str(v) for v in row) + "\n")


def main(argv=None) -> int:
    from .fad import FrechetAudioDistance, kad_embedding_dir, log
    registry = _registry()
    args = _parser("fadtk_b200.kad", _KAD_ARGS, registry).parse_args(argv)
    model = registry[args.model]
    for p in (args.baseline, args.eval):            # before any embedding work: statistics cannot give a KAD
        kad_embedding_dir(p, model.name)
    if args.csv and not args.indiv:
        _check_csv(args.csv)
    dist.init_from_env()
    _embed_directories(model, (args.baseline, args.eval), args.workers)
    from . import _native
    sharded = dist.is_distributed() and dist.enable_native_allreduce(_native.engine())
    if dist.rank() != 0 and not sharded:
        dist.shutdown()
        return 0

    fad = FrechetAudioDistance(model, audio_load_worker=args.workers, load_model=False)
    if args.indiv:
        table = Path(args.csv or "kad-individual-results.csv")
        fad.score_kad_individual(args.baseline, args.eval, table, distributed=sharded, prepared=args.prepared)
        if dist.rank() == 0:
            log.info(f"Individual KAD scores saved to {table}")
        dist.shutdown()
        return 0
    res = fad.score_kad(args.baseline, args.eval, distributed=sharded, prepared=args.prepared)
    if dist.rank() != 0:
        dist.shutdown()
        return 0
    if args.csv:
        _append_row(args.csv, (model.name, args.baseline, args.eval, res.score, res.bandwidth, res.n_baseline,
                               res.n_eval, time.time()))
        log.info(f"KAD score appended to {args.csv}")
    print(f"The KAD {model.name} score between {args.baseline} and {args.eval} is: {res.score} "
          f"(bandwidth {res.bandwidth})")
    dist.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
