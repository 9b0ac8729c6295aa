"""End to end through FILES on one GPU: .wav directories -> convert cache -> embeddings (.npy) -> statistics -> FAD,
i.e. what `python -m fadtk_b200 vggish <baseline dir> <eval dir>` does (fadtk/__main__.py:39-70), timed as a whole.
Synthetic 10-s clips at the model rate; prints one JSON line.
Usage (on an H100): python benchmarks/file_flow.py [--clips 3000] [--baseline-clips 500] [--workers 16]
"""
import argparse
import json
import shutil
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from fadtk_b200 import _io_native, synth  # noqa: E402
from fadtk_b200.fad import FrechetAudioDistance  # noqa: E402
from fadtk_b200.fad_batch import cache_embedding_files  # noqa: E402
from fadtk_b200.model_loader import VGGishModel  # noqa: E402


def write_set(root: Path, count: int, seed: int, **kw):
    root.mkdir(parents=True, exist_ok=True)
    pcm = synth.musiclike_device(count, 10.0, 16000, seed, torch.device("cuda:0"), **kw).cpu().numpy()
    paths = [root / f"clip{i:06d}.wav" for i in range(count)]
    st = _io_native.wav_write(paths, pcm.reshape(-1), np.arange(count) * pcm.shape[1], np.full(count, pcm.shape[1]), 16000, 16)
    assert not st.any()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=3000)
    ap.add_argument("--baseline-clips", type=int, default=500)
    ap.add_argument("--workers", type=int, default=16)
    ap.add_argument("--dir", default="/tmp/fadtk_file_flow")
    args = ap.parse_args()
    root = Path(args.dir)
    shutil.rmtree(root, ignore_errors=True)
    write_set(root / "eval", args.clips, 1)
    write_set(root / "base", args.baseline_clips, 2, fmax=1500.0, noise=0.08)
    ml = VGGishModel()
    ml.load_model()
    # warm-up on a throw-away directory (CUDA context, workspaces, pinned staging)
    write_set(root / "warm", 64, 3)
    cache_embedding_files(root / "warm", ml, workers=args.workers)
    torch.cuda.synchronize()

    t0 = time.perf_counter()
    cache_embedding_files(root / "base", ml, workers=args.workers)
    t1 = time.perf_counter()
    cache_embedding_files(root / "eval", ml, workers=args.workers)
    t2 = time.perf_counter()
    fad = FrechetAudioDistance(ml, audio_load_worker=args.workers, load_model=False)
    score = fad.score(root / "base", root / "eval")
    t3 = time.perf_counter()
    n = args.clips + args.baseline_clips
    print(json.dumps({
        "workload": f"vggish directory flow: {args.baseline_clips} + {args.clips} x 10 s PCM16 .wav files -> convert cache -> .npy -> stats -> FAD",
        "files": n, "seconds_total": t3 - t0, "files_per_s": n / (t3 - t0), "audio_s_per_s": n * 10.0 / (t3 - t0),
        "embed_eval_files_per_s": args.clips / (t2 - t1), "embed_eval_audio_s_per_s": args.clips * 10.0 / (t2 - t1),
        "stats_and_frechet_s": t3 - t2, "fad": float(score), "workers": args.workers,
        "api": "fadtk_b200.fad_batch.cache_embedding_files + FrechetAudioDistance.score (the fadtk command line's calls)"}))
    shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
