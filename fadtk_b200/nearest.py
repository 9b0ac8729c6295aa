"""``python -m fadtk_b200.nearest <model> <baseline> <eval> [csv] [-k K] [--prepared] [-w N] [-s sox]`` - the k baseline
files every file of an eval directory comes closest to, with the distance and the pair of rows where it does: a
memorisation audit (FrechetAudioDistance.score_nearest_individual on the cached embeddings). Directories without
embedding caches are embedded first (under ``torchrun`` the embedding is sharded over the ranks as for ``fadtk``). Under
``torchrun`` every rank then takes its share of the nearest tiles (``distributed=True``) when the library's NCCL
communicator can be set up, and rank 0 scores alone otherwise; either way rank 0 alone writes. ``csv`` is the per-file
table (default nearest-individual-results.csv).
"""
from __future__ import annotations

import sys
from pathlib import Path

from . import dist
from .cli import _embed_directories, _parser, _registry

_NEAREST_ARGS = (
    (("model",), dict(type=str, help="embedding model (a registry name)")),
    (("baseline",), dict(type=str, help="baseline audio directory (the clips that may have been copied)")),
    (("eval",), dict(type=str, help="evaluation audio directory")),
    (("csv",), dict(type=str, nargs="?", help="where the per-file table goes (default nearest-individual-results.csv)")),
    (("-k",), dict(type=int, default=5, help="nearest baseline files per eval file, 1 to 16 (default 5)")),
    (("--prepared",), dict(action="store_true", help="score against the baseline's saved pairwise preparation "
                                                     "(python -m fadtk_b200.prepare), built and saved first when it is "
                                                     "missing or stale")),
)


def main(argv=None) -> int:
    from .fad import FrechetAudioDistance, kad_embedding_dir, log
    registry = _registry()
    args = _parser("fadtk_b200.nearest", _NEAREST_ARGS, registry).parse_args(argv)
    if not 1 <= args.k <= 16:                       # before any embedding work, like the checks below
        raise ValueError(f"nearest needs k in [1, 16], not {args.k}")
    model = registry[args.model]
    for p in (args.baseline, args.eval):            # statistics cannot give nearest neighbours
        kad_embedding_dir(p, model.name, "nearest")
    dist.init_from_env()
    _embed_directories(model, (args.baseline, args.eval), args.workers)
    from . import _native
    sharded = dist.is_distributed() and dist.enable_native_allreduce(_native.engine())
    if dist.rank() != 0 and not sharded:
        dist.shutdown()
        return 0

    fad = FrechetAudioDistance(model, audio_load_worker=args.workers, load_model=False)
    table = Path(args.csv or "nearest-individual-results.csv")
    fad.score_nearest_individual(args.baseline, args.eval, table, k=args.k, distributed=sharded,
                                 prepared=args.prepared)
    if dist.rank() == 0:
        log.info(f"Per-file nearest baseline clips saved to {table}")
    dist.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
