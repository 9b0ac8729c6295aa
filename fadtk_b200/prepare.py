"""``python -m fadtk_b200.prepare <model> <baseline> [--k-max K] [-w N] [-s sox]`` - prepare a baseline directory for the
pairwise metrics (FrechetAudioDistance.prepare_pairwise): its KAD bandwidth, S_xx and k-NN radius lists, computed once
and saved to ``<baseline>/stats/<model>/pairwise.npz``, so that ``kad``, ``prdc``, ``realism`` and ``nearest`` with
``--prepared`` pay for the eval rows only. A directory without embedding caches is embedded first (under ``torchrun``
sharded over the ranks as for ``fadtk``); under ``torchrun`` every rank then takes its share of the tiles when the
library's NCCL communicator can be set up, and rank 0 prepares alone otherwise; either way rank 0 alone writes. A saved
preparation that is still current is left as it is.
"""
from __future__ import annotations

import sys

from . import dist
from .cli import _embed_directories, _parser, _registry

_PREPARE_ARGS = (
    (("model",), dict(type=str, help="embedding model (a registry name)")),
    (("baseline",), dict(type=str, help="baseline audio directory")),
    (("--k-max",), dict(type=int, default=16, help="the largest k that PRDC and realism may use against it, 1 to 16 "
                                                    "(default 16)")),
)


def main(argv=None) -> int:
    from .fad import FrechetAudioDistance, kad_embedding_dir, log
    registry = _registry()
    args = _parser("fadtk_b200.prepare", _PREPARE_ARGS, registry).parse_args(argv)
    if not 1 <= args.k_max <= 16:                   # before any embedding work, like the check below
        raise ValueError(f"a prepared baseline needs k_max in [1, 16], not {args.k_max}")
    model = registry[args.model]
    kad_embedding_dir(args.baseline, model.name, "a prepared baseline")
    dist.init_from_env()
    _embed_directories(model, (args.baseline,), args.workers)
    from . import _native
    sharded = dist.is_distributed() and dist.enable_native_allreduce(_native.engine())
    if dist.rank() != 0 and not sharded:
        dist.shutdown()
        return 0

    fad = FrechetAudioDistance(model, audio_load_worker=args.workers, load_model=False)
    pb = fad.prepare_pairwise(args.baseline, k_max=args.k_max, distributed=sharded)
    if dist.rank() == 0:
        log.info(f"Pairwise preparation of {args.baseline}: {pb.m} rows, k_max {pb.k_max}, bandwidth {pb.sigma}")
    dist.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
