"""``python -m fadtk_b200.kad_test <model> <baseline> <eval> [csv] [--versus <eval_b>] [--permutations 999] [--seed 0]
[--prepared] [-w N] [-s sox]`` - permutation p-values of Kernel Audio Distance between audio directories.  Without
``--versus``: can the eval set be told apart from the baseline (fad.calc_kad_test)?  With ``--versus``: is
KAD(baseline, eval) - KAD(baseline, versus) real or noise (fad.calc_kad_comparison, two-sided)?  Directories without
embedding caches are embedded first, and ``torchrun`` splits the work as ``python -m fadtk_b200.kad`` does; rank 0
alone reports and writes.  With ``csv``, one row ``model,baseline,eval,versus,kad,kad_versus,difference,p_value,
permutations,seed,bandwidth,n_baseline,n_eval,n_versus,time`` is appended (the versus fields empty without
``--versus``); a new file gets the header first, and an existing file with another header is refused.
"""
from __future__ import annotations

import sys
import time

from . import dist
from .cli import _embed_directories, _parser, _registry
from .kad import _append_row, _check_csv

CSV_HEADER = ("model,baseline,eval,versus,kad,kad_versus,difference,p_value,permutations,seed,bandwidth,n_baseline,"
              "n_eval,n_versus,time\n")
_ARGS = (
    (("model",), dict(type=str, help="embedding model (a registry name)")),
    (("baseline",), dict(type=str, help="baseline audio directory (its embeddings also set the kernel bandwidth)")),
    (("eval",), dict(type=str, help="evaluation audio directory")),
    (("csv",), dict(type=str, nargs="?", help="append the result row here")),
    (("--versus",), dict(type=str, default=None, help="a second evaluation directory: test the difference of the two "
                                                      "KAD scores against the baseline")),
    (("--permutations",), dict(type=int, default=999, help="random labellings, 1 to 9999 (default 999)")),
    (("--seed",), dict(type=int, default=0, help="seed of the labellings, 0 to 2**64 - 1 (default 0)")),
    (("--prepared",), dict(action="store_true", help="score against the baseline's saved pairwise preparation "
                                                     "(python -m fadtk_b200.prepare), built and saved first when it is "
                                                     "missing or stale")),
)


def main(argv=None) -> int:
    from .fad import FrechetAudioDistance, _perm_args, kad_embedding_dir, log
    registry = _registry()
    args = _parser("fadtk_b200.kad_test", _ARGS, registry).parse_args(argv)
    model = registry[args.model]
    _perm_args(args.permutations, args.seed, "a KAD permutation test")
    dirs = (args.baseline, args.eval) + ((args.versus,) if args.versus else ())
    for p in dirs:                                  # before any embedding work: statistics cannot give a KAD
        kad_embedding_dir(p, model.name)
    if args.csv:
        _check_csv(args.csv, CSV_HEADER, "KAD permutation test")
    dist.init_from_env()
    _embed_directories(model, dirs, args.workers)
    from . import _native
    sharded = dist.is_distributed() and dist.enable_native_allreduce(_native.engine())
    if dist.rank() != 0 and not sharded:
        dist.shutdown()
        return 0

    fad = FrechetAudioDistance(model, audio_load_worker=args.workers, load_model=False)
    kw = dict(permutations=args.permutations, seed=args.seed, distributed=sharded, prepared=args.prepared)
    if args.versus:
        r = fad.score_kad_comparison(args.baseline, args.eval, args.versus, **kw)
        row = (model.name, args.baseline, args.eval, args.versus, r.score_a, r.score_b, r.difference, r.p_value,
               r.permutations, r.seed, r.bandwidth, r.n_baseline, r.n_a, r.n_b, time.time())
        msg = (f"The KAD {model.name} scores of {args.eval} and {args.versus} against {args.baseline} are {r.score_a} "
               f"and {r.score_b}: difference {r.difference}, p-value {r.p_value} ({r.permutations} permutations)")
    else:
        r = fad.score_kad_test(args.baseline, args.eval, **kw)
        row = (model.name, args.baseline, args.eval, "", r.score, "", "", r.p_value, r.permutations, r.seed,
               r.bandwidth, r.n_baseline, r.n_eval, "", time.time())
        msg = (f"The KAD {model.name} score between {args.baseline} and {args.eval} is: {r.score}, p-value {r.p_value} "
               f"({r.permutations} permutations, bandwidth {r.bandwidth})")
    if dist.rank() != 0:
        dist.shutdown()
        return 0
    if args.csv:
        _append_row(args.csv, row, CSV_HEADER)
        log.info(f"KAD permutation test appended to {args.csv}")
    print(msg)
    dist.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
