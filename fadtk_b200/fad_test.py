"""``python -m fadtk_b200.fad_test <model> <baseline> <eval> <versus> [csv] [--permutations 999] [--seed 0] [-w N]
[-s sox]`` - is the FAD difference of two systems against one baseline real or noise?  A two-sided permutation test
over the files of the two eval directories (fad.calc_fad_comparison).  The baseline is anything ``score`` takes: a
directory, an ``.npz`` statistics file or a named set.  Directories without embedding caches are embedded first; under
``torchrun`` the ranks share the embedding and rank 0 runs the test.  With ``csv``, one row ``model,baseline,eval,versus,
fad,fad_versus,difference,observed,p_value,permutations,seed,n_files_eval,n_files_versus,time`` is appended; a new file
gets the header first, and an existing file with another header is refused.
"""
from __future__ import annotations

import sys
import time

from . import dist
from .cli import _embed_directories, _parser, _registry
from .kad import _append_row, _check_csv

CSV_HEADER = ("model,baseline,eval,versus,fad,fad_versus,difference,observed,p_value,permutations,seed,n_files_eval,"
              "n_files_versus,time\n")
_ARGS = (
    (("model",), dict(type=str, help="embedding model (a registry name)")),
    (("baseline",), dict(type=str, help="baseline: an audio directory, an .npz statistics file or a named set")),
    (("eval",), dict(type=str, help="evaluation audio directory (system A)")),
    (("versus",), dict(type=str, help="second evaluation audio directory (system B)")),
    (("csv",), dict(type=str, nargs="?", help="append the result row here")),
    (("--permutations",), dict(type=int, default=999, help="random labellings, 1 to 9999 (default 999)")),
    (("--seed",), dict(type=int, default=0, help="seed of the labellings, 0 to 2**64 - 1 (default 0)")),
)


def main(argv=None) -> int:
    from .fad import FrechetAudioDistance, _perm_args, kad_embedding_dir, log
    registry = _registry()
    args = _parser("fadtk_b200.fad_test", _ARGS, registry).parse_args(argv)
    model = registry[args.model]
    _perm_args(args.permutations, args.seed, "a FAD comparison")
    for p in (args.eval, args.versus):              # before any embedding work: the units are the cached files
        kad_embedding_dir(p, model.name, "the FAD comparison")
    if args.csv:
        _check_csv(args.csv, CSV_HEADER, "FAD comparison")
    dist.init_from_env()
    _embed_directories(model, (args.baseline, args.eval, args.versus), args.workers)
    if dist.rank() != 0:
        dist.shutdown()
        return 0

    fad = FrechetAudioDistance(model, audio_load_worker=args.workers, load_model=False)
    r = fad.score_fad_comparison(args.baseline, args.eval, args.versus, permutations=args.permutations, seed=args.seed)
    if args.csv:
        _append_row(args.csv, (model.name, args.baseline, args.eval, args.versus, r.score_a, r.score_b, r.difference,
                               r.observed, r.p_value, r.permutations, r.seed, r.n_units_a, r.n_units_b, time.time()),
                    CSV_HEADER)
        log.info(f"FAD comparison appended to {args.csv}")
    print(f"The FAD {model.name} scores of {args.eval} and {args.versus} against {args.baseline} are {r.score_a} and "
          f"{r.score_b}: difference {r.difference}, p-value {r.p_value} ({r.permutations} permutations over "
          f"{r.n_units_a} + {r.n_units_b} files)")
    dist.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
