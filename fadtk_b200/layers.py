"""FAD of every layer of a wav2vec-family checkpoint from one forward pass per file.

fadtk's registry lists each layer of MERT, wav2vec 2.0, HuBERT and WavLM as a model of its own (``MERT-v1-95M-1`` ..
``MERT-v1-95M``) so that users can ask which layer's FAD tracks their listening judgements.  Embedding those names one
by one reads every file, loads the weights and runs the network once per layer; the forward at layer L passes through
every earlier layer on its way.  Here one forward per batch (fad_w2v_forward_taps) writes the caches of every requested
layer, byte-identical to what ``python -m fadtk_b200.embeds -m <name>`` writes, and each layer is then scored by the
ordinary statistics path, with the same ``stats/<name>/`` caches a separate run would use.

    python -m fadtk_b200.layers MERT-v1-95M <baseline dir | .npz | name> <eval dir> [csv] [--layers 1-12] [-w 8]
"""
from __future__ import annotations

import sys
import time
from argparse import ArgumentParser
from pathlib import Path

from . import dist

# checkpoint (the registry name of its last layer, the default) -> the size key model_loader._layer_name names its
# layers by (12 or 24 layers)
CHECKPOINTS = {"MERT-v1-95M": "v1-95M", "w2v2-base": "base", "w2v2-large": "large", "hubert-base": "base",
               "hubert-large": "large", "wavlm-base": "base", "wavlm-base-plus": "base", "wavlm-large": "large"}


def checkpoint_loader(model: str):
    """The registry loader of the checkpoint's last layer; it runs the sweep's forward (the tapped path ignores its layer)."""
    if model not in CHECKPOINTS:
        raise ValueError(f"{model!r} is not a wav2vec-family checkpoint; a layer sweep takes one of {', '.join(CHECKPOINTS)}")
    from .model_loader import get_all_models
    return next(m for m in get_all_models() if m.name == model)


def n_layers(model: str) -> int:
    return int(checkpoint_loader(model).arch["layers"])


def parse_layers(spec, n: int) -> list[int]:
    """``all`` (1..n), a range ``a-b``, a comma list of both, or an iterable of ints -> sorted unique layers in 1..n"""
    if spec is None or (isinstance(spec, str) and spec.strip() == "all"):
        return list(range(1, n + 1))
    out = []
    if isinstance(spec, str):
        for part in spec.split(","):
            a, sep, b = part.strip().partition("-")
            try:
                lo = int(a)
                hi = int(b) if sep else lo
            except ValueError:
                raise ValueError(f"layers {spec!r}: expected 'all', a range a-b or a comma list of layers") from None
            if lo > hi:
                raise ValueError(f"layers {spec!r}: the range {part.strip()} is empty")
            out += range(lo, hi + 1)
    else:
        out = [int(v) for v in spec]
    if not out:
        raise ValueError(f"layers {spec!r}: no layer given")
    bad = sorted({v for v in out if not 1 <= v <= n})
    if bad:
        raise ValueError(f"layers {spec!r}: {', '.join(map(str, bad))} outside 1..{n}")
    return sorted(set(out))


def layer_names(model: str, layers) -> list[str]:
    """the registry names of the checkpoint's layers"""
    from .model_loader import _layer_name
    return [_layer_name(model, CHECKPOINTS[model], k) for k in layers]


def _plan(model: str, layers):
    ml = checkpoint_loader(model)
    layers = parse_layers(layers, int(ml.arch["layers"]))
    return ml, layers, layer_names(model, layers)


def cache_layer_embeddings(dirs_or_files, model: str, layers=None, workers: int = 8):
    """Embed audio directories (or a list of files) for every requested layer of ``model`` in one forward per batch:
    ``<dir>/embeddings/<layer name>/<stem>.npy`` for each layer whose cache is missing.  Weights load once."""
    from .fad_batch import cache_tapped_embedding_files
    ml, layers, names = _plan(model, layers)
    items = [dirs_or_files] if isinstance(dirs_or_files, (str, Path)) else list(dirs_or_files)
    dirs = [p for p in items if Path(p).is_dir()]
    loose = [p for p in items if not Path(p).is_dir()]
    for group in [*dirs, *([loose] if loose else [])]:
        cache_tapped_embedding_files(group, ml, layers, names, workers=workers)
    return names


def _check_statistics_files(paths, names):
    """A statistics .npz (or a packaged statistics name) must hold every requested layer before any audio is embedded."""
    import numpy as np
    from .fad import _named_statistics
    for p in paths:
        f = _named_statistics(p) if isinstance(p, str) else None
        f = Path(f if f is not None else p)
        if f.is_file():
            with np.load(f) as data:
                lack = [n for n in names if f"{n}.mu" not in data or f"{n}.cov" not in data]
            if lack:
                raise ValueError(f"FAD statistics file {f} doesn't contain data for {', '.join(lack)}")


def score_layers(model: str, baseline, eval, layers=None, workers: int = 8) -> list[tuple[str, float]]:
    """FAD between ``baseline`` and ``eval`` (directories, statistics .npz files or packaged statistics names) at every
    requested layer of ``model`` (default: all, 1..layers) -> [(registry name, FAD)] in layer order.  Directories are
    embedded for all layers by one forward per batch; each score is FrechetAudioDistance(<layer>).score(baseline, eval)."""
    from .fad import FrechetAudioDistance
    from .model_loader import get_all_models
    _, layers, names = _plan(model, layers)
    _check_statistics_files((baseline, eval), names)
    cache_layer_embeddings([p for p in (baseline, eval) if Path(p).is_dir()], model, layers, workers)
    registry = {m.name: m for m in get_all_models()}
    return [(n, float(FrechetAudioDistance(registry[n], audio_load_worker=workers, load_model=False).score(baseline, eval)))
            for n in names]


def main(argv=None) -> int:
    """``python -m fadtk_b200.layers CHECKPOINT baseline eval [csv] [--layers SPEC] [-w N]``"""
    from .cli import _append_row
    from .fad import log
    ap = ArgumentParser(prog="fadtk_b200.layers", description="FAD of every layer of a wav2vec-family checkpoint")
    ap.add_argument("model", choices=list(CHECKPOINTS), help="checkpoint (the registry name of its last layer)")
    ap.add_argument("baseline", type=str, help="baseline set: a directory, a statistics .npz, or a built-in statistics name")
    ap.add_argument("eval", type=str, help="evaluation set: a directory or a statistics .npz")
    ap.add_argument("csv", type=str, nargs="?", help="append one result row per layer here")
    ap.add_argument("--layers", type=str, default="all", help="'all' (default: 1..layers), a range a-b or a comma list")
    ap.add_argument("-w", "--workers", type=int, default=8, help="host threads for file I/O and audio conversion")
    args = ap.parse_args(argv)
    try:
        ks = parse_layers(args.layers, n_layers(args.model))
    except ValueError as e:
        ap.error(str(e))
    dist.init_from_env()
    # every rank embeds its shard; the statistics caches are written by rank 0 and read by the others (load_stats)
    result = score_layers(args.model, args.baseline, args.eval, args.layers, args.workers)
    if dist.rank() == 0:
        print(f"{'layer':>5}  {'model':<24} FAD")
        for k, (name, score) in zip(ks, result):
            print(f"{k:>5}  {name:<24} {score}")
        if args.csv:
            for name, score in result:
                _append_row(args.csv, (name, args.baseline, args.eval, score, None, time.time()))
            log.info(f"{len(result)} FAD scores appended to {args.csv}")
    dist.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
