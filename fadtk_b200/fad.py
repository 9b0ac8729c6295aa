"""FAD engine (mirror of fadtk/fad.py): same functions, class, methods, on-disk layout and
error behaviour; the arithmetic runs on the H100 through the C ABI.

    calc_embd_statistics      fad.py:42-48   -> shifted E^T E tensor-core kernel (csrc/stats.cuh)
    calc_frechet_distance     fad.py:51-120  -> Newton-Schulz GEMM chain on the PSD form (csrc/frechet.cuh)
    calc_kernel_audio_distance  (no reference counterpart) -> wgmma pair-tile kernels (csrc/kad.cuh)
    calc_kernel_audio_distance_songs                       -> the same, every song against one baseline in one pass
    calc_prdc                   (no reference counterpart) -> k-NN radii and ball-count tile kernels (csrc/prdc.cuh)
    calc_prdc_songs                                        -> the same, every song against one baseline in one pass
    calc_realism                (no reference counterpart) -> k-NN radii and one max / argmin tile pass (csrc/prdc.cuh)
    calc_nearest                (no reference counterpart) -> one distinct-group top-k tile pass (csrc/prdc.cuh)
    prepare_pairwise_baseline                              -> the baseline-only work of the four above, done once
    calc_kad_test, calc_kad_comparison                     -> permutation p-values of KAD: every labelling in one
                                                              label-product tile pass (csrc/kad.cuh)
    calc_fad_comparison                                    -> permutation p-value of a FAD difference: file records,
                                                              labelled fp64 sums and batched Frechet chains (stats.cuh)
    calc_fad_bootstrap, calc_kad_bootstrap                 -> bootstrap confidence intervals over the eval files:
                                                              seeded multiplicities, weighted record sums (FAD) and a
                                                              weighted label product (KAD)
    FrechetAudioDistance      fad.py:123-395 -> same methods; file <-> GPU staging is batched
"""
from __future__ import annotations

import hashlib
import json
import logging
import os
import threading
import traceback
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import NamedTuple, Union

import numpy as np
import torch

from . import synth
from .model_loader import ModelLoader
from .utils import *  # noqa: F401,F403  (the reference re-exports utils from fad)
from .utils import DeviceStatistics, PathLike, calculate_embd_statistics_online, find_sox_formats, \
    get_cache_embedding_path, statistics_of_arrays

log = logging.getLogger("fadtk_b200")
if not log.handlers:
    _h = logging.StreamHandler()
    _h.setFormatter(logging.Formatter("%(asctime)s %(levelname)s %(message)s", "%H:%M:%S"))
    log.addHandler(_h)
    log.setLevel(os.environ.get("FADTK_LOGLEVEL", "INFO"))

sox_path = os.environ.get('SOX_PATH', 'sox')


_RESAMPLE_LOCK = threading.Lock()
ffmpeg_path = os.environ.get('FFMPEG_PATH', 'ffmpeg')


def decode_container(f: Path):
    """Compressed / non-WAV audio -> (float32 tensor [channels, T], sample rate), DECODE ONLY - mono mix-down and
    resampling stay on the GPU path.  torchaudio.load first (the reference's default branch, fad.py:147); when it has no
    decoder backend (TorchCodec missing), ffmpeg - the tool the reference's other branch shells out to for formats
    SoX cannot read (fad.py:168-176) - unpacks the stream to a float32 WAV at its native rate and channel count."""
    try:
        import torchaudio
        x, sr = torchaudio.load(str(f))
        return x, int(sr)
    except Exception as first:                                  # noqa: BLE001 - any backend failure: try ffmpeg
        import shutil
        import subprocess
        import tempfile
        exe = shutil.which(ffmpeg_path)
        if exe is None:
            raise RuntimeError(f"cannot decode {f}: torchaudio has no working backend ({first}) and ffmpeg "
                               f"('{ffmpeg_path}', $FFMPEG_PATH) is not installed") from first
        with tempfile.TemporaryDirectory() as tmp:
            wav = Path(tmp) / "decoded.wav"
            done = subprocess.run([exe, "-hide_banner", "-loglevel", "error", "-y", "-i", str(f), "-f", "wav",
                                   "-acodec", "pcm_f32le", str(wav)], capture_output=True, text=True)
            if done.returncode != 0 or not wav.exists():
                raise RuntimeError(f"ffmpeg could not decode {f}: {done.stderr.strip()[-500:]}") from first
            x, sr = synth.read_wav_float(wav)
        return torch.from_numpy(x), int(sr)


class FADInfResults(NamedTuple):
    score: float
    slope: float
    r2: float
    points: list[tuple[int, float]]


class KADResults(NamedTuple):
    score: float
    bandwidth: float
    n_baseline: int
    n_eval: int


class KADTestResults(NamedTuple):
    score: float                    # calc_kernel_audio_distance(emb_baseline, emb_eval).score, bitwise
    bandwidth: float
    p_value: float
    null_scores: np.ndarray         # float64 [permutations], KAD of each random labelling
    observed: float                 # KAD of the observed labelling on the permutation path (fp16 kernel values)
    permutations: int
    seed: int
    n_baseline: int
    n_eval: int


class KADComparisonResults(NamedTuple):
    score_a: float                  # calc_kernel_audio_distance_songs(emb_baseline, [emb_a, emb_b]), bitwise
    score_b: float
    difference: float               # score_a - score_b
    p_value: float
    null_differences: np.ndarray    # float64 [permutations]
    bandwidth: float
    permutations: int
    seed: int
    n_baseline: int
    n_a: int
    n_b: int


class FADComparisonResults(NamedTuple):
    score_a: float                  # calc_frechet_distance(mu, cov, *calc_embd_statistics(all rows of A)), bitwise
    score_b: float
    difference: float               # score_a - score_b
    observed: float                 # the difference of the observed labelling on the labelled path
    p_value: float
    null_differences: np.ndarray    # float64 [permutations]
    permutations: int
    seed: int
    n_units_a: int
    n_units_b: int
    n_rows_a: int
    n_rows_b: int


class FADBootstrapResults(NamedTuple):
    score: float                    # calc_frechet_distance(mu, cov, *calc_embd_statistics(all eval rows)), bitwise
    observed: float                 # resample 0 (the observed set) on the weighted path
    ci_low: float
    ci_high: float
    standard_error: float           # std(replicates, ddof=1)
    bias: float                     # mean(replicates) - observed
    replicates: np.ndarray          # float64 [resamples]
    level: float
    method: str                     # "percentile" or "basic"
    resamples: int
    seed: int
    n_units: int
    n_rows: int


class KADBootstrapResults(NamedTuple):
    score: float                    # calc_kernel_audio_distance_songs(emb_baseline, [all eval rows])[0].score, bitwise
    observed: float
    ci_low: float
    ci_high: float
    standard_error: float
    bias: float
    replicates: np.ndarray
    level: float
    method: str
    resamples: int
    seed: int
    n_units: int
    n_rows: int
    bandwidth: float
    n_baseline: int


class PRDCResults(NamedTuple):
    precision: float
    recall: float
    density: float
    coverage: float
    k: int
    n_baseline: int
    n_eval: int


class RealismResults(NamedTuple):
    realism: np.ndarray             # float32 [n]
    nearest: np.ndarray             # int64 [n], rows of the baseline
    nearest_distance: np.ndarray    # float32 [n]
    threshold_sq: float
    k: int
    n_baseline: int
    n_eval: int


class NearestResults(NamedTuple):
    rows: np.ndarray                # int64 [n, k], rows of the baseline, -1 past the last non-empty group
    groups: np.ndarray              # int64 [n, k], the groups of those rows, -1 likewise
    distance: np.ndarray            # float32 [n, k], +inf likewise
    k: int
    n_baseline: int
    n_eval: int


def _kad_rows(a, what: str, metric: str = "KAD"):
    """fp16 [rows, d] numpy array or torch tensor -> contiguous fp16 torch tensor (not moved to a device yet)."""
    t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.asarray(a))
    if t.dtype != torch.float16:
        raise ValueError(f"{metric} needs fp16 embeddings (the cached values); the {what} set is {t.dtype}")
    if t.ndim != 2:
        raise ValueError(f"{metric} needs [rows, d] embeddings; the {what} set has shape {tuple(t.shape)}")
    return t


def calc_kernel_audio_distance(emb_baseline, emb_eval, distributed: bool = False) -> KADResults:
    """Kernel Audio Distance (Chung et al., 2025) between two fp16 embedding sets X [m, d] and Y [n, d], with the fp16
    values taken as exact reals:

        q(a, b) = |a - b|^2,    k(a, b) = exp(-q(a, b) / (2 sigma^2)),
        sigma   = median of {|x_i - x_j| : i < j} (numpy.median: the mean of the two middle distances when
                  m (m - 1) / 2 is even) - from the baseline only, so every eval set scored against one baseline
                  uses the same kernel,
        MMD^2_u = 2/(m(m-1)) sum_{i<j} k(x_i, x_j) + 2/(n(n-1)) sum_{i<j} k(y_i, y_j) - 2/(mn) sum_{i,j} k(x_i, y_j),
        KAD     = 1000 * MMD^2_u   (the paper's scaling; unbiased, so it can be slightly negative; not clamped).

    The pair sums and the bandwidth selection run on the GPU (fad_kad_median_sq, fad_kad_sums); MMD^2_u is assembled
    from the three fp64 sums.  A width that is not a multiple of 8 is zero-padded, which changes no distance.
    Raises ValueError for fewer than two rows on either side, non-fp16 or non-2-D input, mismatched widths, and
    sigma = 0 (more than half of the baseline pairs are identical rows).

    distributed=True under torchrun (world size > 1): a collective call that every rank makes with the same sets.  The
    pair tiles are split over the ranks (fad_kad_*_sharded over the library's NCCL communicator), and every rank gets
    the result, bitwise equal to one GPU's.  The ranks' arguments are compared first; a difference raises NativeError
    on every rank.  RuntimeError when that communicator cannot be set up (gloo backend, FADTK_NATIVE_ALLREDUCE=0).

    emb_baseline may be a PairwiseBaseline (prepare_pairwise_baseline): sigma and S_xx are then the prepared ones, and
    the score is bitwise the one calc_kernel_audio_distance_songs gives for emb_eval as one song (S_xy sums in another
    order than the whole-set pass; DESIGN.md 5.15)."""
    if _is_prepared(emb_baseline):
        y = _kad_rows(emb_eval, "eval")
        if y.shape[0] < 2:
            raise ValueError(f"KAD needs at least two embedding rows in each set (baseline {emb_baseline.m}, "
                             f"eval {y.shape[0]})")
        _prepared_width(emb_baseline, y, "eval")
        return _kad_prepared(emb_baseline, y, np.array([0, y.shape[0]], dtype=np.int64), distributed)[0]
    x, y = _kad_rows(emb_baseline, "baseline"), _kad_rows(emb_eval, "eval")
    m, n = int(x.shape[0]), int(y.shape[0])
    if m < 2 or n < 2:
        raise ValueError(f"KAD needs at least two embedding rows in each set (baseline {m}, eval {n})")
    if x.shape[1] != y.shape[1]:
        raise ValueError(f"embedding widths differ (baseline {x.shape[1]}, eval {y.shape[1]})")
    eng, collective = _kad_engine(distributed)
    z = _kad_device_rows(torch.cat([x, y]), eng)
    sigma = _kad_bandwidth(eng, z, m, collective)
    sig = torch.tensor([sigma], dtype=torch.float64, device=eng.torch_device)
    sums = eng.kad_sums_sharded(z, m, sig) if collective else eng.kad_sums(z, m, sig)
    s_xx, s_yy, s_xy = (float(v) for v in sums.cpu().numpy())
    return KADResults(score=_kad_score(s_xx, s_yy, s_xy, m, n), bandwidth=sigma, n_baseline=m, n_eval=n)


def _kad_engine(distributed: bool, metric: str = "KAD"):
    """-> (this process's engine, whether the KAD (or PRDC) calls are collective over the torchrun group)"""
    from . import _native, dist
    eng = _native.engine()
    if not (distributed and dist.world_size() > 1):
        return eng, False
    if not dist.enable_native_allreduce(eng):
        raise RuntimeError(f"distributed {metric} runs over the library's own NCCL communicator, which needs "
                           "torch.distributed on the nccl backend and FADTK_NATIVE_ALLREDUCE unset or 1")
    return eng, True


def _on_rank0(fn, collective: bool):
    """fn() decided on rank 0 and broadcast, so that every rank of a collective call takes the same branch; a ValueError
    on rank 0 is raised on every rank"""
    if not collective:
        return fn()
    from . import dist
    res = None
    if dist.rank() == 0:
        try:
            res = (True, fn())
        except ValueError as e:
            res = (False, str(e))
    ok, val = dist.broadcast_object(res)
    if not ok:
        raise ValueError(val)
    return val


def _kad_device_rows(z: torch.Tensor, eng) -> torch.Tensor:
    """[rows, d] fp16 -> contiguous on the engine's device, the width zero-padded to a multiple of 8 (no distance
    changes)."""
    z = z.contiguous()
    pad = -z.shape[1] % 8
    if pad:
        z = torch.nn.functional.pad(z, (0, pad))
    return z.to(eng.torch_device, non_blocking=True)


def _kad_bandwidth(eng, z: torch.Tensor, m: int, collective: bool = False) -> float:
    """sigma from the first m rows of z (device): the numpy median of their pairwise distances; ValueError when 0."""
    sq = (eng.kad_median_sq_sharded(z[:m]) if collective else eng.kad_median_sq(z[:m])).cpu().numpy()
    sigma = 0.5 * (float(np.sqrt(sq[0])) + float(np.sqrt(sq[1])))
    if not sigma > 0.0:
        raise ValueError("KAD bandwidth is 0: more than half of the baseline pairs are identical rows")
    return sigma


def _kad_score(s_xx: float, s_yy: float, s_xy: float, m: int, n: int) -> float:
    """1000 * MMD^2_u from the three kernel sums"""
    return 1000.0 * (2.0 * s_xx / (m * (m - 1.0)) + 2.0 * s_yy / (n * (n - 1.0)) - 2.0 * s_xy / (float(m) * n))


def calc_kernel_audio_distance_songs(emb_baseline, songs, distributed: bool = False) -> list[KADResults]:
    """KAD of every song against one baseline: for each fp16 [n_k, d] array in ``songs``, the value
    calc_kernel_audio_distance(emb_baseline, songs[k]) is defined to be (same sigma from the baseline alone, same sums),
    with sigma and the baseline's own pair sum computed once for all songs and every song's sums in one GPU pass
    (fad_kad_song_sums).  A song with fewer than two rows gets score NaN (n_eval still says how many rows it had).
    Raises ValueError like calc_kernel_audio_distance: non-fp16 or non-2-D input, widths that differ from the
    baseline's, fewer than two baseline rows, sigma = 0.  distributed: as for calc_kernel_audio_distance.  emb_baseline
    may be a PairwiseBaseline: the same values, bitwise, without the baseline's own passes."""
    if _is_prepared(emb_baseline):
        ys = [_prepared_width(emb_baseline, _kad_rows(y, f"song {k}"), f"song {k}") for k, y in enumerate(songs)]
        offsets = np.zeros(len(ys) + 1, dtype=np.int64)
        offsets[1:] = np.cumsum([int(y.shape[0]) for y in ys])
        return _kad_prepared(emb_baseline, torch.cat(ys) if ys else None, offsets, distributed)
    x = _kad_rows(emb_baseline, "baseline")
    ys = [_kad_rows(y, f"song {k}") for k, y in enumerate(songs)]
    for k, y in enumerate(ys):
        if y.shape[1] != x.shape[1]:
            raise ValueError(f"embedding widths differ (baseline {x.shape[1]}, song {k} {y.shape[1]})")
    offsets = np.zeros(len(ys) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([int(y.shape[0]) for y in ys])
    return _kad_songs(torch.cat([x, *[y.to(x.device) for y in ys]]), int(x.shape[0]), offsets, distributed)


def _kad_songs(z: torch.Tensor, m: int, offsets: np.ndarray, distributed: bool = False) -> list[KADResults]:
    """z = [X; Y_1; ...] fp16 (host or device), offsets int64 [K + 1] into the rows after X -> one KADResults per song"""
    if m < 2:
        raise ValueError(f"KAD needs at least two embedding rows in each set (baseline {m})")
    eng, collective = _kad_engine(distributed)
    z = _kad_device_rows(z, eng)
    sigma = _kad_bandwidth(eng, z, m, collective)
    dev = eng.torch_device
    args = (z, m, torch.from_numpy(offsets).to(dev), torch.tensor([sigma], dtype=torch.float64, device=dev))
    sums = (eng.kad_song_sums_sharded(*args) if collective else eng.kad_song_sums(*args)).cpu().numpy()
    s_xx = float(sums[0])
    out = []
    for k, n in enumerate(np.diff(offsets).tolist()):
        score = _kad_score(s_xx, float(sums[1 + 2 * k]), float(sums[2 + 2 * k]), m, n) if n >= 2 else float("nan")
        out.append(KADResults(score=score, bandwidth=sigma, n_baseline=m, n_eval=n))
    return out


def _perm_args(permutations, seed, metric: str):
    if isinstance(permutations, bool) or not isinstance(permutations, (int, np.integer)) or not 1 <= permutations <= 9999:
        raise ValueError(f"{metric} needs permutations in [1, 9999] (got {permutations!r})")
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= seed < 2 ** 64:
        raise ValueError(f"{metric} needs an integer seed in [0, 2**64) (got {seed!r})")
    return int(permutations), int(seed)


def _perm_p(null: np.ndarray, observed: float) -> float:
    """(1 + #{null >= observed}) / (B + 1): never 0 (Phipson and Smyth, 2010)"""
    return (1.0 + float(np.count_nonzero(null >= observed))) / (null.shape[0] + 1.0)


def _perm_pool(emb_baseline, pool_parts: list, what: list, metric: str):
    """-> (the pooled sets' fp16 rows, the baseline rows or None when prepared, m, the pooled sets' sizes, the
    PairwiseBaseline or None), with calc_kernel_audio_distance's checks"""
    prepared = emb_baseline if _is_prepared(emb_baseline) else None
    if prepared is not None:
        parts = [_prepared_width(prepared, _kad_rows(y, w, metric), w) for y, w in zip(pool_parts, what)]
        x_rows, m = None, prepared.m
    else:
        x_rows = _kad_rows(emb_baseline, "baseline", metric)
        m = int(x_rows.shape[0])
        parts = [_kad_rows(y, w, metric) for y, w in zip(pool_parts, what)]
        for y, w in zip(parts, what):
            if y.shape[1] != x_rows.shape[1]:
                raise ValueError(f"embedding widths differ (baseline {x_rows.shape[1]}, {w} {y.shape[1]})")
    sizes = [int(y.shape[0]) for y in parts]
    if m < 2 or min(sizes) < 2:
        raise ValueError(f"{metric} needs at least two embedding rows in each set (baseline {m}, "
                         + ", ".join(f"{w} {n}" for w, n in zip(what, sizes)) + ")")
    return parts, x_rows, m, sizes, prepared


def _perm_sums(eng, collective: bool, pool: torch.Tensor, a: int, sigma: float, permutations: int, seed: int):
    sig = torch.tensor([sigma], dtype=torch.float64, device=eng.torch_device)
    if collective:
        return eng.kad_perm_sums_sharded(pool, a, sig, permutations, seed).cpu().numpy()
    return eng.kad_perm_sums(pool, a, sig, permutations, seed).cpu().numpy()


def calc_kad_test(emb_baseline, emb_eval, permutations: int = 999, seed: int = 0,
                  distributed: bool = False) -> KADTestResults:
    """Permutation test of KAD (Gretton et al., 2012): can the eval set be told apart from the baseline at this sample
    size?  The pool [X; Y] (m + n rows) is relabelled `permutations` times (B); labelling b marks the m rows with the
    smallest (pair_mix64(pair_mix64(seed + b) ^ i), i) as the baseline (DESIGN.md 5.16), and KAD is recomputed for each:

        KAD(l) = 1000 * (2 S_aa / (m (m - 1)) + 2 S_bb / (n (n - 1)) - 2 S_ab / (m n)),
        p      = (1 + #{b >= 1 : KAD_b >= KAD_0}) / (B + 1),

    KAD_0 the observed labelling.  sigma is the bandwidth of the observed baseline (as calc_kernel_audio_distance uses
    it), held fixed across labellings: the test is conditional on sigma.  `score` is bitwise calc_kernel_audio_distance's
    value; the rows go to the GPU once and serve both the score and the labellings.

    Precision: every labelling's sums come from one pass over the pair tiles per 1024 labellings (fad_kad_perm_sums),
    with each kernel value rounded to fp16 once.  That moves each labelling's statistic by an amount of the order of
    2^-11 sqrt(sum coef^2 K^2) (oracle/kad_test_oracle.py, error_scale), measured at up to about 0.17 of the null
    distribution's standard deviation on 4 000-row pools.  Null values that close to the observed one can fall either
    side of it, so a p-value near a threshold can move by a few hundredths against an exact fp64 computation; `observed`
    (KAD_0 on the same fp16 path) is what the nulls are compared with.

    emb_baseline may be a PairwiseBaseline: its sigma and rows are used, the p-value and nulls are bitwise the
    unprepared call's, and score is the prepared calc_kernel_audio_distance value.  Raises ValueError as
    calc_kernel_audio_distance does, and for permutations outside [1, 9999] or a seed outside [0, 2**64).
    distributed: as for calc_kernel_audio_distance (the permutation pass is sharded too)."""
    permutations, seed = _perm_args(permutations, seed, "a KAD permutation test")
    parts, x_rows, m, (n,), prepared = _perm_pool(emb_baseline, [emb_eval], ["eval"], "KAD")
    eng, collective = _kad_engine(distributed)
    if prepared is not None:
        yd = _kad_device_rows(parts[0], eng)
        score = _kad_prepared(prepared, yd, np.array([0, n], dtype=np.int64), distributed)[0]
        pool = torch.cat([prepared.x, yd])
    else:
        pool = _kad_device_rows(torch.cat([x_rows, parts[0]]), eng)
        sigma = _kad_bandwidth(eng, pool, m, collective)
        sig = torch.tensor([sigma], dtype=torch.float64, device=eng.torch_device)
        sums = eng.kad_sums_sharded(pool, m, sig) if collective else eng.kad_sums(pool, m, sig)
        s_xx, s_yy, s_xy = (float(v) for v in sums.cpu().numpy())
        score = KADResults(score=_kad_score(s_xx, s_yy, s_xy, m, n), bandwidth=sigma, n_baseline=m, n_eval=n)
    s = _perm_sums(eng, collective, pool, m, score.bandwidth, permutations, seed)
    stats = 1000.0 * (2.0 * s[:, 0] / (m * (m - 1.0)) + 2.0 * s[:, 1] / (n * (n - 1.0)) - 2.0 * s[:, 2] / (float(m) * n))
    return KADTestResults(score=score.score, bandwidth=score.bandwidth, p_value=_perm_p(stats[1:], stats[0]),
                          null_scores=stats[1:].copy(), observed=float(stats[0]), permutations=permutations, seed=seed,
                          n_baseline=m, n_eval=n)


def calc_kad_comparison(emb_baseline, emb_a, emb_b, permutations: int = 999, seed: int = 0,
                        distributed: bool = False) -> KADComparisonResults:
    """Permutation test of the difference of two systems' KAD against one baseline X: is score_a - score_b real or
    noise?  The pool [A; B] (n_a + n_b rows) is relabelled as calc_kad_test relabels [X; Y] (labelling b marks n_a rows
    as system A), X stays put, and

        D(l) = KAD(X, A_l) - KAD(X, B_l)
             = 1000 * (2 S_aa / (n_a (n_a - 1)) - 2 S_bb / (n_b (n_b - 1)) - 2 S_XA / (m n_a) + 2 S_XB / (m n_b)),
        p    = (1 + #{b >= 1 : |D_b| >= |D_0|}) / (B + 1)   (two-sided).

    S_xx cancels, and sigma (from X alone, which is not permuted) is the same for every labelling, so the test is exact.
    S_XA(l) = sum of g_i over the rows l marks, with g_i = sum_x k(x, z_i) taken once per pool row
    (fad_kad_eval_sums with one item per row); S_aa and S_bb come from fad_kad_perm_sums, with each kernel value
    rounded to fp16 once (the precision note of calc_kad_test applies to D_b likewise).  score_a and score_b are
    bitwise calc_kernel_audio_distance_songs(emb_baseline, [emb_a, emb_b]); the rows go to the GPU once.  emb_baseline
    may be a PairwiseBaseline (the p-value and nulls are then bitwise the unprepared call's).  Raises ValueError as
    calc_kad_test does."""
    permutations, seed = _perm_args(permutations, seed, "a KAD comparison")
    parts, x_rows, m, (na, nb), prepared = _perm_pool(emb_baseline, [emb_a, emb_b], ["eval A", "eval B"], "KAD")
    eng, collective = _kad_engine(distributed)
    dev = eng.torch_device
    offsets = np.array([0, na, na + nb], dtype=np.int64)
    if prepared is not None:
        pool = _kad_device_rows(torch.cat(parts), eng)
        ra, rb = _kad_prepared(prepared, pool, offsets, distributed)
        z = torch.cat([prepared.x, pool])
    else:
        z = _kad_device_rows(torch.cat([x_rows, *parts]), eng)
        ra, rb = _kad_songs(z, m, offsets, distributed)
        pool = z[m:]
    n = na + nb
    sig = torch.tensor([ra.bandwidth], dtype=torch.float64, device=dev)
    one_each = torch.arange(n + 1, dtype=torch.int64, device=dev)
    g = eng.kad_eval_sums(z, m, one_each, sig, 0 if collective else None)[:, 1].contiguous()
    s = _perm_sums(eng, collective, pool, na, ra.bandwidth, permutations, seed)
    s_xa = eng.perm_dot(eng.perm_labels(n, na, permutations, seed), g).cpu().numpy()
    s_xb = float(np.sum(g.cpu().numpy())) - s_xa
    diff = 1000.0 * (2.0 * s[:, 0] / (na * (na - 1.0)) - 2.0 * s[:, 1] / (nb * (nb - 1.0))
                     - 2.0 * s_xa / (float(m) * na) + 2.0 * s_xb / (float(m) * nb))
    return KADComparisonResults(score_a=ra.score, score_b=rb.score, difference=ra.score - rb.score,
                                p_value=_perm_p(np.abs(diff[1:]), abs(float(diff[0]))),
                                null_differences=diff[1:].copy(), bandwidth=ra.bandwidth, permutations=permutations,
                                seed=seed, n_baseline=m, n_a=na, n_b=nb)


def _fad_units(emb, what: str, d: int, metric: str = "the FAD comparison") -> list:
    """a list of fp16 [rows, d] arrays (files) or one 2-D fp16 array (one unit per row) -> the list of units"""
    if isinstance(emb, (list, tuple)):
        units = [np.asarray(u) for u in emb]
    else:
        arr = np.asarray(emb)
        if arr.ndim != 2:
            raise ValueError(f"{what} must be a list of 2-D arrays (files) or one 2-D array (rows); got shape {arr.shape}")
        units = [arr[i:i + 1] for i in range(arr.shape[0])]
    for u in units:
        if u.ndim != 2 or u.shape[1] != d:
            raise ValueError(f"every {what} array must be [rows, {d}] (the baseline's width); got shape {u.shape}")
        if u.dtype != np.float16:
            raise ValueError(f"{metric} needs fp16 embeddings; {what} holds {u.dtype}")
        if u.shape[0] == 0:
            raise ValueError(f"every {what} file needs at least one row")
    if len(units) < 2:
        raise ValueError(f"{metric} needs at least two units (files) in {what}; got {len(units)}")
    return units


def calc_fad_comparison(baseline, eval_a, eval_b, permutations: int = 999, seed: int = 0) -> FADComparisonResults:
    """Permutation test of the difference of two systems' FAD against one baseline: is score_a - score_b real or
    noise?  baseline = (mu, cov) (the statistics load_stats returns, fp64 or fp16 mu).  eval_a, eval_b: a list of fp16
    [rows, d] arrays, one per file, or one 2-D fp16 array.  The unit of the test is a file: the pool is the files of A
    followed by those of B, and labelling b marks n_units_a of them (labelling 0: A's own files; b >= 1: the units with
    the smallest (pair_mix64(pair_mix64(seed + b) ^ i), i), DESIGN.md 5.17).  Rows of one file are correlated, so
    files and not rows are exchanged; a single 2-D array is one unit per row, which assumes independent rows.

        D(l) = FAD(X, A_l) - FAD(X, B_l),      p = (1 + #{b >= 1 : |D_b| >= |D_0|}) / (B + 1)   (two-sided),

    A_l (B_l) the union of the rows of the units l marks (does not mark), each with its exact fp64 mean and ddof = 1
    covariance.  The baseline is never permuted, so the test is exact when A's and B's files are exchangeable.

    score_a and score_b are calc_frechet_distance(mu, cov, *calc_embd_statistics(rows)) of all rows of each system,
    the values FAD users see.  `observed` is D_0 on the labelled path, which the nulls are compared with; it can differ
    from score_a - score_b by about 1e-4 relative, because calc_embd_statistics rounds the mean to fp16 (as the
    reference does) and the labelled statistics keep the exact mean.

    Raises ValueError for a baseline that is not (mu [d], cov [d, d]) with d a multiple of 64, arrays that are not fp16
    [rows, d], an empty file, fewer than two units on a side, permutations outside [1, 9999] or a seed outside
    [0, 2**64), before any GPU work."""
    permutations, seed = _perm_args(permutations, seed, "a FAD comparison")
    mu, cov, d = _fad_baseline(baseline, "the FAD comparison")
    units_a, units_b = _fad_units(eval_a, "eval A", d), _fad_units(eval_b, "eval B", d)
    return _fad_comparison(mu, cov, units_a, units_b, None, None, permutations, seed)


def _fad_baseline(baseline, metric: str):
    """(mu, cov) -> (mu, cov, d) as arrays, d a multiple of 64 up to 2048"""
    try:
        mu, cov = baseline
    except (TypeError, ValueError):
        raise ValueError(f"{metric} needs the baseline as (mu, cov)") from None
    mu, cov = np.asarray(mu), np.asarray(cov)
    d = int(mu.shape[0]) if mu.ndim == 1 else -1
    if d <= 0 or cov.shape != (d, d):
        raise ValueError(f"the baseline must be (mu [d], cov [d, d]); got shapes {mu.shape} and {cov.shape}")
    if d % 64 != 0 or d > 2048:
        raise ValueError(f"{metric} needs an embedding width that is a multiple of 64 up to 2048; got {d}")
    return mu, cov, d


def _fad_comparison(mu, cov, units_a: list, units_b: list, score_a, score_b, permutations: int,
                    seed: int) -> FADComparisonResults:
    """calc_fad_comparison on checked units; score_a / score_b None: the array scores"""
    from . import _native
    rows_a, rows_b = np.concatenate(units_a), np.concatenate(units_b)
    if score_a is None:
        score_a = float(calc_frechet_distance(mu, cov, *calc_embd_statistics(rows_a)))
        score_b = float(calc_frechet_distance(mu, cov, *calc_embd_statistics(rows_b)))
    eng = _native.engine()
    dev = eng.torch_device
    base = _native.Baseline(eng, mu, cov)
    sizes = [u.shape[0] for u in units_a + units_b]
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)).to(dev)
    pool = torch.from_numpy(np.concatenate([rows_a, rows_b])).to(dev)
    out, _ = base.frechet_perm(pool, offsets, len(units_a), permutations, seed)
    fad = out[:, :, 0].cpu().numpy()
    if not np.isfinite(fad).all():
        raise ValueError("non-finite covariance statistics (NaN/Inf input)")
    diff = fad[:, 0] - fad[:, 1]
    return FADComparisonResults(score_a=score_a, score_b=score_b, difference=score_a - score_b,
                                observed=float(diff[0]), p_value=_perm_p(np.abs(diff[1:]), abs(float(diff[0]))),
                                null_differences=diff[1:].copy(), permutations=permutations, seed=seed,
                                n_units_a=len(units_a), n_units_b=len(units_b), n_rows_a=int(rows_a.shape[0]),
                                n_rows_b=int(rows_b.shape[0]))


def _boot_args(resamples, seed, level, method, metric: str):
    if isinstance(resamples, bool) or not isinstance(resamples, (int, np.integer)) or not 2 <= resamples <= 9999:
        raise ValueError(f"{metric} needs resamples in [2, 9999] (got {resamples!r})")
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= seed < 2 ** 64:
        raise ValueError(f"{metric} needs an integer seed in [0, 2**64) (got {seed!r})")
    if isinstance(level, bool) or not isinstance(level, (int, float, np.floating)) or not 0.0 < level < 1.0:
        raise ValueError(f"{metric} needs a level strictly between 0 and 1 (got {level!r})")
    if method not in ("percentile", "basic"):
        raise ValueError(f"{metric} needs method 'percentile' or 'basic' (got {method!r})")
    return int(resamples), int(seed), float(level), method


def _boot_interval(theta: np.ndarray, level: float, method: str):
    """theta fp64 [B + 1] (theta[0] the observed set on the same path) -> (ci_low, ci_high, standard_error, bias)"""
    rep, obs = theta[1:], float(theta[0])
    q_lo, q_hi = (float(v) for v in np.quantile(rep, [(1.0 - level) / 2.0, (1.0 + level) / 2.0]))
    lo, hi = (q_lo, q_hi) if method == "percentile" else (2.0 * obs - q_hi, 2.0 * obs - q_lo)
    return lo, hi, float(np.std(rep, ddof=1)), float(np.mean(rep)) - obs


def calc_fad_bootstrap(baseline, eval_units, resamples: int = 999, seed: int = 0, level: float = 0.95,
                       method: str = "percentile") -> FADBootstrapResults:
    """Bootstrap confidence interval of FAD: how precise is this score, given the eval files it was computed from?
    baseline = (mu, cov) (as calc_fad_comparison takes it).  eval_units: a list of fp16 [rows, d] arrays, one per file,
    or one 2-D fp16 array (one unit per row, which assumes independent rows).  Rows of one file are correlated, so whole
    files are resampled: resample b >= 1 draws F files with replacement, draw t picking file
    floor(pair_mix64(pair_mix64(seed + b) ^ t) F / 2^64) (DESIGN.md 5.18), and its replicate is the FAD of the multiset
    of rows, each file's rows as often as the file was drawn, with its exact fp64 mean and ddof = 1 covariance.

    The baseline is held fixed: the interval is the sampling spread of the eval set, conditional on the baseline (an
    .npz baseline has no rows to resample).  With q_lo, q_hi the (1 -+ level) / 2 quantiles of the replicates (numpy's
    default linear method), method "percentile" gives (q_lo, q_hi) and "basic" (2 observed - q_hi, 2 observed - q_lo);
    standard_error = std(replicates, ddof=1), bias = mean(replicates) - observed.  FAD is biased upwards at small n,
    and a resample's duplicate files add about the same bias again, so the percentile interval sits high; `bias` and
    the basic interval are there for that reason.

    score is calc_frechet_distance(mu, cov, *calc_embd_statistics(all rows)), the value FAD users see; `observed` is
    resample 0 (the observed set) on the weighted path, which can differ from score by about 1e-4 relative because
    calc_embd_statistics rounds the mean to fp16.  Raises ValueError for a baseline that is not (mu [d], cov [d, d])
    with d a multiple of 64 up to 2048, arrays that are not fp16 [rows, d], an empty file, fewer than two units,
    resamples outside [2, 9999], a seed outside [0, 2**64), a level outside (0, 1) or another method, before any GPU
    work."""
    resamples, seed, level, method = _boot_args(resamples, seed, level, method, "a FAD bootstrap")
    mu, cov, d = _fad_baseline(baseline, "the FAD bootstrap")
    units = _fad_units(eval_units, "eval", d, "the FAD bootstrap")
    return _fad_bootstrap(mu, cov, units, None, resamples, seed, level, method)


def _fad_bootstrap(mu, cov, units: list, score, resamples: int, seed: int, level: float,
                   method: str) -> FADBootstrapResults:
    """calc_fad_bootstrap on checked units; score None: the array score"""
    from . import _native
    rows = np.concatenate(units)
    if score is None:
        score = float(calc_frechet_distance(mu, cov, *calc_embd_statistics(rows)))
    eng = _native.engine()
    dev = eng.torch_device
    base = _native.Baseline(eng, mu, cov)
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum([u.shape[0] for u in units])]).astype(np.int64)).to(dev)
    out, _ = base.frechet_boot(torch.from_numpy(rows).to(dev), offsets, resamples, seed)
    theta = out[:, 0].cpu().numpy()
    if not np.isfinite(theta).all():
        raise ValueError("non-finite covariance statistics (NaN/Inf input)")
    lo, hi, se, bias = _boot_interval(theta, level, method)
    return FADBootstrapResults(score=score, observed=float(theta[0]), ci_low=lo, ci_high=hi, standard_error=se,
                               bias=bias, replicates=theta[1:].copy(), level=level, method=method, resamples=resamples,
                               seed=seed, n_units=len(units), n_rows=int(rows.shape[0]))


def _kad_units(eval_units) -> list:
    """a list of fp16 [rows, d] arrays or tensors (files) or one 2-D fp16 array (one unit per row) -> fp16 tensors"""
    if isinstance(eval_units, (list, tuple)):
        units = [_kad_rows(u, f"eval file {k}") for k, u in enumerate(eval_units)]
    else:
        y = _kad_rows(eval_units, "eval")
        units = [y[i:i + 1] for i in range(y.shape[0])]
    for u in units:
        if u.shape[0] == 0:
            raise ValueError("every eval file needs at least one row")
        if u.shape[1] != units[0].shape[1]:
            raise ValueError(f"embedding widths differ across the eval files ({units[0].shape[1]}, {u.shape[1]})")
    if len(units) < 2:
        raise ValueError(f"the KAD bootstrap needs at least two units (files) in eval; got {len(units)}")
    return units


def calc_kad_bootstrap(emb_baseline, eval_units, resamples: int = 999, seed: int = 0, level: float = 0.95,
                       method: str = "percentile") -> KADBootstrapResults:
    """Bootstrap confidence interval of KAD over the eval files (units as calc_fad_bootstrap takes them, resampled by
    the same seeded rule).  Row i of a resample carries the multiplicity v_i of its file, n_b = sum v_i, and

        S_yy(b) = sum_{i<j} v_i v_j K_ij + sum_u n_u w_u (w_u - 1) / 2,     S_xy(b) = sum_u w_u G_u,
        KAD_b   = 1000 * (2 S_xx / (m (m - 1)) + 2 S_yy(b) / (n_b (n_b - 1)) - 2 S_xy(b) / (m n_b)),

    the second term of S_yy counting the pairs of two copies of one row (K(y, y) = 1), G_u = sum_{x, i in u} k(x, y_i).
    The baseline X [m, d] (fp16 rows, or a PairwiseBaseline) is held fixed, and so are sigma (X's bandwidth, as
    calc_kernel_audio_distance uses it) and S_xx: the interval is the sampling spread of the eval set, conditional on the
    baseline.  The quadratic form runs on the pair tiles of the eval rows with each kernel value rounded to fp16 once
    and the multiplicities as exact fp16 weights (fad_kad_boot_sums); every other term is an fp64 unit sum.

    Intervals, standard_error and bias as calc_fad_bootstrap (KAD is unbiased, but duplicate rows within a resample
    still shift it).  score is bitwise calc_kernel_audio_distance_songs(emb_baseline, [all eval rows]); `observed` is
    resample 0 on the fp16 path.  A PairwiseBaseline gives replicates bitwise equal to the rows'.  Raises ValueError as
    calc_kad_test does, for fewer than two units or an empty file, and for resamples, seed, level or method as
    calc_fad_bootstrap does, before any GPU work."""
    from . import _native
    resamples, seed, level, method = _boot_args(resamples, seed, level, method, "a KAD bootstrap")
    units = _kad_units(eval_units)
    parts, x_rows, m, (n,), prepared = _perm_pool(emb_baseline, [torch.cat(units)], ["eval"], "KAD")
    sizes = np.array([int(u.shape[0]) for u in units], dtype=np.int64)
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    eng = _native.engine()
    dev = eng.torch_device
    if prepared is not None:
        yd = _kad_device_rows(parts[0], eng)
        r = _kad_prepared(prepared, yd, np.array([0, n], dtype=np.int64))[0]
        score, sigma, s_xx = r.score, prepared.sigma, prepared.s_xx
        z = torch.cat([prepared.x, yd])
    else:
        z = _kad_device_rows(torch.cat([x_rows, parts[0]]), eng)
        sigma = _kad_bandwidth(eng, z, m)
        sig = torch.tensor([sigma], dtype=torch.float64, device=dev)
        sums = eng.kad_song_sums(z, m, torch.tensor([0, n], dtype=torch.int64, device=dev), sig).cpu().numpy()
        s_xx = float(sums[0])
        score = _kad_score(s_xx, float(sums[1]), float(sums[2]), m, n)
    sig = torch.tensor([sigma], dtype=torch.float64, device=dev)
    offs = torch.from_numpy(offsets).to(dev)
    g = eng.kad_eval_sums(z, m, offs, sig)[:, 1].contiguous()
    s = eng.kad_boot_sums(z[m:], offs, sig, g, resamples, seed).cpu().numpy()
    theta = _kad_score(s_xx, s[:, 1], s[:, 2], m, s[:, 0])
    lo, hi, se, bias = _boot_interval(theta, level, method)
    return KADBootstrapResults(score=score, observed=float(theta[0]), ci_low=lo, ci_high=hi, standard_error=se,
                               bias=bias, replicates=theta[1:].copy(), level=level, method=method, resamples=resamples,
                               seed=seed, n_units=len(units), n_rows=n, bandwidth=sigma, n_baseline=m)


def calc_prdc(emb_baseline, emb_eval, k: int = 5, distributed: bool = False) -> PRDCResults:
    """Precision and recall (Kynkaanniemi et al., 2019), density and coverage (Naeem et al., 2020) of an eval set
    Y [n, d] against a baseline X [m, d], both fp16 with the values taken as exact reals, q(a, b) = |a - b|^2:

        r_i = distance from x_i to its k-th nearest other row of X (the self pair excluded by index, so duplicate
              rows are neighbours at distance 0); s_j the same for y_j within Y,
        precision = (1/n) #{j : exists i, q(x_i, y_j) < r_i^2}
        recall    = (1/m) #{i : exists j, q(x_i, y_j) < s_j^2}
        density   = 1/(k n) sum_j #{i : q(x_i, y_j) < r_i^2}
        coverage  = (1/m) #{i : exists j, q(x_i, y_j) < r_i^2}

    All comparisons are strict, so a row with r_i = 0 (at least k exact duplicates, e.g. silent clips) contains
    nothing.  The radii and the ball counts run on the GPU (fad_knn_radii_sq, fad_prdc_counts) without forming a
    distance matrix; the four values are assembled from integer counts.  A width that is not a multiple of 8 is
    zero-padded, which changes no distance.  Raises ValueError for k outside [1, 16], m <= k or n <= k, non-fp16 or
    non-2-D input and mismatched widths.

    distributed=True under torchrun (world size > 1): a collective call that every rank makes with the same sets and k.
    The radii and ball-count tiles are split over the ranks (fad_knn_radii_sq_sharded, fad_prdc_counts_sharded over the
    library's NCCL communicator), and every rank gets the result, bitwise equal to one GPU's.  The ranks' arguments are
    compared first; a difference raises NativeError on every rank.  RuntimeError when that communicator cannot be set
    up, as for calc_kernel_audio_distance.

    emb_baseline may be a PairwiseBaseline with k_max >= k: r_i^2 is then column k - 1 of its radius lists, and the
    results are bitwise the ones the baseline rows give."""
    k = _prdc_k(k)
    if _is_prepared(emb_baseline):
        pb, y = emb_baseline, _kad_rows(emb_eval, "eval", "PRDC")
        _prepared_k(pb, k, "PRDC")
        if y.shape[0] <= k:
            raise ValueError(f"PRDC with k = {k} needs more than k embedding rows in each set (baseline {pb.m}, "
                             f"eval {y.shape[0]})")
        _prepared_width(pb, y, "eval")
        eng, collective = _kad_engine(distributed, "PRDC")
        z = torch.cat([pb.x, _kad_device_rows(y, eng)])
        radii_sq = torch.cat([pb.lists[:, k - 1], eng.knn_eval_radii_sq(z, pb.m, k, None, 0 if collective else None)])
        return _prdc_results(eng, z, pb.m, k, radii_sq, collective)
    x, y = _kad_rows(emb_baseline, "baseline", "PRDC"), _kad_rows(emb_eval, "eval", "PRDC")
    m, n = int(x.shape[0]), int(y.shape[0])
    if m <= k or n <= k:
        raise ValueError(f"PRDC with k = {k} needs more than k embedding rows in each set (baseline {m}, eval {n})")
    if x.shape[1] != y.shape[1]:
        raise ValueError(f"embedding widths differ (baseline {x.shape[1]}, eval {y.shape[1]})")
    eng, collective = _kad_engine(distributed, "PRDC")
    z = _kad_device_rows(torch.cat([x, y]), eng)
    radii_sq = eng.knn_radii_sq_sharded(z, m, k) if collective else eng.knn_radii_sq(z, m, k)
    return _prdc_results(eng, z, m, k, radii_sq, collective)


def _prdc_results(eng, z: torch.Tensor, m: int, k: int, radii_sq: torch.Tensor, collective: bool) -> PRDCResults:
    """the ball counts of z = [X; Y] (device) under radii_sq [m + n] -> PRDCResults"""
    n = int(z.shape[0]) - m
    counts = eng.prdc_counts_sharded(z, m, radii_sq) if collective else eng.prdc_counts(z, m, radii_sq)
    inside, flags = (t.cpu().numpy() for t in counts)
    return PRDCResults(precision=float(np.count_nonzero(inside)) / n,
                       recall=float(np.count_nonzero(flags & 2)) / m,
                       density=float(inside.sum(dtype=np.int64)) / (k * n),
                       coverage=float(np.count_nonzero(flags & 1)) / m,
                       k=k, n_baseline=m, n_eval=n)


def _prdc_k(k, metric: str = "PRDC") -> int:
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= 16:
        raise ValueError(f"{metric} needs an integer k in [1, 16], not {k!r}")
    return int(k)


def calc_realism(emb_baseline, emb_eval, k: int = 3, distributed: bool = False) -> RealismResults:
    """Per-sample realism score (Kynkaanniemi et al., 2019) and nearest baseline row of every row of an eval set
    Y [n, d] against a baseline X [m, d], both fp16 with the values taken as exact reals, q(a, b) = |a - b|^2:

        r_i^2        = the k-NN radius of x_i within X, as calc_prdc defines it (self excluded by index),
        T            = numpy.median of the m values r_i^2 in fp64 (for even m the fp64 mean of the two middle values),
        r~_i^2       = r_i^2 where r_i^2 <= T, 0 otherwise (the half of the balls with the largest radii is dropped),
        realism_j    = sqrt(max_i r~_i^2 / q(x_i, y_j)) over the rows with r~_i^2 > 0: +inf when such a row has
                       q = 0 (y_j copies a kept baseline row), 0 when every r~_i^2 is 0; realism >= 1 means y_j lies in
                       or on the edge of a kept ball,
        nearest_j    = argmin_i q(x_i, y_j) over all rows of X, ties to the smallest i; nearest_distance_j its
                       distance.

    k defaults to the paper's 3.  The authors' code is reported to return the squared ratio with 1e-5 added to q; this
    is the definition above.  realism_j and nearest_j depend on y_j and X alone, so the rows of several eval sets
    scored in one call get the values separate calls give.  The radii and one pass over all (x, y) pairs run on the GPU
    (fad_realism) without forming a distance matrix.  A width that is not a multiple of 8 is zero-padded.  Raises
    ValueError for k outside [1, 16], m <= k, n < 1, non-fp16 or non-2-D input, mismatched widths, and T = 0 (more than
    half of the baseline rows have k exact duplicates).  distributed: as for calc_prdc (fad_realism_sharded).

    emb_baseline may be a PairwiseBaseline with k_max >= k: r_i^2 is then column k - 1 of its radius lists, pruned by
    the same rule, and the results are bitwise the ones the baseline rows give (fad_realism_prepared)."""
    k = _prdc_k(k, "realism")
    if _is_prepared(emb_baseline):
        y = _prepared_width(emb_baseline, _kad_rows(emb_eval, "eval", "realism"), "eval")
        _realism_rows(emb_baseline.m, int(y.shape[0]), k)
        return _realism(y, emb_baseline.m, k, distributed, emb_baseline)
    x, y = _kad_rows(emb_baseline, "baseline", "realism"), _kad_rows(emb_eval, "eval", "realism")
    m, n = int(x.shape[0]), int(y.shape[0])
    _realism_rows(m, n, k)
    if x.shape[1] != y.shape[1]:
        raise ValueError(f"embedding widths differ (baseline {x.shape[1]}, eval {y.shape[1]})")
    return _realism(torch.cat([x, y]), m, k, distributed)


def _realism_rows(m: int, n: int, k: int):
    if m <= k or n < 1:
        raise ValueError(f"realism with k = {k} needs more than k baseline rows and at least one eval row "
                         f"(baseline {m}, eval {n})")


def _realism(z: torch.Tensor, m: int, k: int, distributed: bool = False, prepared=None) -> RealismResults:
    """z = [X; Y] fp16 (host or device) -> RealismResults of the rows after X.  prepared: a PairwiseBaseline of X
    (k_max >= k), and z = Y alone"""
    eng, collective = _kad_engine(distributed, "realism")
    z = _kad_device_rows(z, eng)
    if prepared is not None:
        _prepared_k(prepared, k, "realism")
        z = torch.cat([prepared.x, z])
        kept, t = prepared.kept_radii(k)
        realism, nearest, nearest_sq = eng.realism_prepared(z, m, kept, 0 if collective else None)
    else:
        _, realism, nearest, nearest_sq, t = eng.realism_sharded(z, m, k) if collective else eng.realism(z, m, k)
    if not t > 0.0:
        raise ValueError("realism threshold is 0: more than half of the baseline rows have k exact duplicates")
    return RealismResults(realism=realism.cpu().numpy(), nearest=nearest.cpu().numpy().astype(np.int64),
                          nearest_distance=np.sqrt(nearest_sq.cpu().numpy()), threshold_sq=float(t), k=k,
                          n_baseline=m, n_eval=int(z.shape[0]) - m)


def calc_nearest(emb_baseline, emb_eval, k: int = 5, distributed: bool = False) -> NearestResults:
    """The k nearest distinct baseline groups of every row of an eval set Y [n, d]: a memorisation audit, "which
    baseline clips does this generated frame come closest to, and where".  emb_baseline is one fp16 [m, d] array, each
    row its own group (a plain k-NN), or a list of fp16 [m_g, d] arrays, one group each (e.g. one per baseline file;
    empty arrays are empty groups).  With the fp16 values taken as exact reals and q(a, b) = |a - b|^2, the baseline
    rows are ordered for y_j by the key (q(x_i, y_j), i); each group is represented by its smallest key, and the k groups
    with the smallest representative keys are returned, ascending:

        rows[j, r]     = the baseline row (index into all baseline rows, in order) of the r-th group's smallest key,
        groups[j, r]   = that group,
        distance[j, r] = sqrt(q) of that pair,

    with -1, -1, +inf where fewer than k groups are non-empty.  The nearest rows of an eval frame are mostly
    neighbouring frames of one clip; distinct groups give k different clips instead.  Each row's result depends on that
    row and the baseline alone, so several eval sets scored in one call get the values separate calls give.  With k = 1
    and one array, rows[:, 0] and distance[:, 0] are calc_realism's nearest and nearest_distance.  One GPU pass over all
    (x, y) pairs (fad_nearest) keeps the lists in registers; no distance matrix is formed.  A width that is not a
    multiple of 8 is zero-padded.  Raises ValueError for k outside [1, 16], no baseline or no eval rows, non-fp16 or
    non-2-D input and mismatched widths.  distributed: as for calc_prdc (fad_nearest_sharded).  emb_baseline may be a
    PairwiseBaseline: its resident rows, grouped by its file offsets (each row its own group without them)."""
    k = _prdc_k(k, "nearest")
    if _is_prepared(emb_baseline):
        y = _prepared_width(emb_baseline, _kad_rows(emb_eval, "eval", "nearest"), "eval")
        _nearest_rows(emb_baseline.m, int(y.shape[0]))
        return _nearest(y, emb_baseline.m, k, emb_baseline.offsets, distributed, emb_baseline)[0]
    parts = list(emb_baseline) if isinstance(emb_baseline, (list, tuple)) else [emb_baseline]
    if not parts:
        raise ValueError("nearest needs at least one baseline group")
    xs = [_kad_rows(p, "baseline", "nearest") for p in parts]
    y = _kad_rows(emb_eval, "eval", "nearest")
    for x in xs:
        if x.shape[1] != y.shape[1]:
            raise ValueError(f"embedding widths differ (baseline {x.shape[1]}, eval {y.shape[1]})")
    offsets = None
    if isinstance(emb_baseline, (list, tuple)):
        offsets = np.zeros(len(xs) + 1, dtype=np.int64)
        offsets[1:] = np.cumsum([x.shape[0] for x in xs])
    x = torch.cat(xs) if len(xs) > 1 else xs[0]
    m, n = int(x.shape[0]), int(y.shape[0])
    _nearest_rows(m, n)
    return _nearest(torch.cat([x, y]), m, k, offsets, distributed)[0]


def _nearest_rows(m: int, n: int):
    if m < 1 or n < 1:
        raise ValueError(f"nearest needs at least one baseline row and one eval row (baseline {m}, eval {n})")


def _nearest(z: torch.Tensor, m: int, k: int, offsets, distributed: bool = False, prepared=None):
    """z = [X; Y] fp16 (host or device), offsets int64 [groups + 1] of X or None -> (NearestResults of the rows after
    X, the squared distances fp32 [n, k]).  prepared: a PairwiseBaseline of X, and z = Y alone"""
    eng, collective = _kad_engine(distributed, "nearest")
    z = _kad_device_rows(z, eng)
    if prepared is not None:
        z = torch.cat([prepared.x, z])
    off = None if offsets is None else torch.from_numpy(np.asarray(offsets, dtype=np.int64)).to(eng.torch_device)
    rows, q = eng.nearest_sharded(z, m, k, off) if collective else eng.nearest(z, m, k, off)
    rows, q = rows.cpu().numpy().astype(np.int64), q.cpu().numpy()
    if offsets is None:
        groups = rows.copy()
    else:
        groups = np.where(rows >= 0, np.searchsorted(np.asarray(offsets), rows, side="right") - 1, -1)
    res = NearestResults(rows=rows, groups=groups, distance=np.sqrt(q), k=k, n_baseline=m, n_eval=int(z.shape[0]) - m)
    return res, q


def _file_nearest(groups: np.ndarray, rows: np.ndarray, q: np.ndarray, k: int) -> list:
    """The k nearest groups of a file of eval rows from the rows' lists (groups, rows, q [rows, k]): per group the
    smallest (q, eval row, baseline row) over the file, the groups ranked by that triple -> [(eval row, slot)] of the
    first k.  Merging the rows' lists gives exactly this: a group in the file's top k is in the top k of the row that
    attains its minimum, since every group ahead of it at that row is ahead of it for the file."""
    j, r = np.nonzero(rows >= 0)
    out, seen = [], set()
    for e in np.lexsort((rows[j, r], j, q[j, r])):
        g = int(groups[j[e], r[e]])
        if g not in seen:
            seen.add(g)
            out.append((int(j[e]), int(r[e])))
            if len(out) == k:
                break
    return out


def calc_prdc_songs(emb_baseline, songs, k: int = 5, distributed: bool = False) -> list[PRDCResults]:
    """Precision, recall, density and coverage of every song against one baseline: for each fp16 [n_k, d] array in
    ``songs`` with more than k rows, exactly the values calc_prdc(emb_baseline, songs[k], k) gives - the same r_i, s_j
    the k-NN radius of y_j within its own song, the same fp32 q and strict comparisons, so equal as floats, not merely
    close.  The baseline radii are computed once, and every song's radii and counts in one GPU pass each
    (fad_knn_song_radii_sq, fad_prdc_song_counts).  A song with at most k rows (empty ones included) gets NaN for all
    four values, n_eval still saying how many rows it had, and is never sent to the GPU.  Coverage and recall of a short
    song against a large baseline are small by definition.  Raises ValueError like calc_prdc: k outside [1, 16],
    m <= k, non-fp16 or non-2-D input, widths that differ from the baseline's.  distributed: as for calc_prdc.
    emb_baseline may be a PairwiseBaseline with k_max >= k: the same values, bitwise."""
    k = _prdc_k(k)
    if _is_prepared(emb_baseline):
        ys = [_prepared_width(emb_baseline, _kad_rows(y, f"song {i}", "PRDC"), f"song {i}") for i, y in enumerate(songs)]
        kept = [y for y in ys if y.shape[0] > k]
        return _prdc_songs(torch.cat(kept) if kept else None, emb_baseline.m, [int(y.shape[0]) for y in ys], k,
                           distributed, emb_baseline)
    x = _kad_rows(emb_baseline, "baseline", "PRDC")
    ys = [_kad_rows(y, f"song {i}", "PRDC") for i, y in enumerate(songs)]
    for i, y in enumerate(ys):
        if y.shape[1] != x.shape[1]:
            raise ValueError(f"embedding widths differ (baseline {x.shape[1]}, song {i} {y.shape[1]})")
    kept = [y.to(x.device) for y in ys if y.shape[0] > k]
    return _prdc_songs(torch.cat([x, *kept]), int(x.shape[0]), [int(y.shape[0]) for y in ys], k, distributed)


def _prdc_songs(z: torch.Tensor, m: int, rows: list, k: int, distributed: bool = False,
                prepared=None) -> list[PRDCResults]:
    """z = [X; the songs of more than k rows, in order] fp16 (host or device), rows = the row counts of all songs ->
    one PRDCResults per song (NaN for the songs not in z).  prepared: a PairwiseBaseline of X (k_max >= k), and z the
    songs' rows alone"""
    if prepared is not None:
        _prepared_k(prepared, k, "PRDC")
    if m <= k:
        raise ValueError(f"PRDC with k = {k} needs more than k embedding rows in each set (baseline {m})")
    nan = float("nan")
    out = [PRDCResults(nan, nan, nan, nan, k=k, n_baseline=m, n_eval=n) for n in rows]
    kept = [i for i, n in enumerate(rows) if n > k]
    if not kept:
        return out
    offsets = np.zeros(len(kept) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([rows[i] for i in kept])
    eng, collective = _kad_engine(distributed, "PRDC")
    z = _kad_device_rows(z, eng)
    off = torch.from_numpy(offsets).to(eng.torch_device)
    if prepared is not None:
        z = torch.cat([prepared.x, z])
        radii_sq = torch.cat([prepared.lists[:, k - 1], eng.knn_eval_radii_sq(z, m, k, off, 0 if collective else None)])
    else:
        radii_sq = (eng.knn_song_radii_sq_sharded(z, m, off, k) if collective else eng.knn_song_radii_sq(z, m, off, k))
    counts = (eng.prdc_song_counts_sharded(z, m, off, radii_sq) if collective
              else eng.prdc_song_counts(z, m, off, radii_sq))
    inside, per_song = (t.cpu().numpy() for t in counts)
    for s, i in enumerate(kept):
        ins, n = inside[offsets[s]:offsets[s + 1]], rows[i]
        out[i] = PRDCResults(precision=float(np.count_nonzero(ins)) / n,
                             recall=float(per_song[s, 1]) / m,
                             density=float(ins.sum(dtype=np.int64)) / (k * n),
                             coverage=float(per_song[s, 0]) / m,
                             k=k, n_baseline=m, n_eval=n)
    return out


def prepare_pairwise_baseline(emb_baseline, k_max: int = 16, offsets=None, distributed: bool = False):
    """The baseline-only work of KAD, PRDC, realism and nearest, done once (DESIGN.md 5.15): the fp16 rows X [m, d]
    are moved to the GPU and kept there with their digest, the KAD bandwidth sigma, S_xx, and per row the k_max smallest
    squared distances to the other rows.  The result can be passed wherever these metrics take the baseline rows
    (calc_kernel_audio_distance[_songs], calc_prdc[_songs] and calc_realism for k <= k_max, calc_nearest), which then pay
    for the eval rows only and give the values the rows give (bitwise; KAD: bitwise the per-song value).  offsets: int64
    [files + 1] row offsets of the baseline's files (calc_nearest's groups), or None.  Raises ValueError for k_max
    outside [1, 16], m <= k_max, non-fp16 or non-2-D rows and bad offsets.  distributed: as for calc_prdc, over the
    sharded entries.  FrechetAudioDistance.prepare_pairwise saves it and loads it back."""
    from ._native import PairwiseBaseline
    k_max = _prdc_k(k_max, "a prepared baseline")
    x = _kad_rows(emb_baseline, "baseline", "a prepared baseline")
    m = int(x.shape[0])
    if m <= k_max:
        raise ValueError(f"a prepared baseline with k_max = {k_max} needs more than k_max rows (baseline {m})")
    offsets = _baseline_offsets(offsets, m)
    eng, collective = _kad_engine(distributed, "a prepared baseline")
    return PairwiseBaseline(eng, _kad_device_rows(x, eng), k_max, int(x.shape[1]), offsets, 0 if collective else None)


def _baseline_offsets(offsets, m: int):
    if offsets is None:
        return None
    offsets = np.asarray(offsets, dtype=np.int64)
    if offsets.ndim != 1 or offsets.size < 2 or offsets[0] != 0 or offsets[-1] != m or np.any(np.diff(offsets) < 0):
        raise ValueError(f"baseline offsets must rise from 0 to m = {m}")
    return offsets


def _is_prepared(b) -> bool:
    from ._native import PairwiseBaseline
    return isinstance(b, PairwiseBaseline)


def _prepared_width(pb, y: torch.Tensor, what: str) -> torch.Tensor:
    if y.shape[1] != pb.d:
        raise ValueError(f"embedding widths differ (baseline {pb.d}, {what} {y.shape[1]})")
    return y


def _prepared_k(pb, k: int, metric: str):
    if k > pb.k_max:
        raise ValueError(f"{metric} with k = {k} needs a baseline prepared with k_max >= k (it has {pb.k_max})")


def _kad_prepared(pb, y, offsets: np.ndarray, distributed: bool = False) -> list[KADResults]:
    """KAD of the items of y (fp16 [n_total, d], host or device, or None when n_total = 0; items at offsets [K + 1])
    against a prepared baseline: its sigma and S_xx, then the eval sums alone (fad_kad_eval_sums)"""
    if not pb.sigma > 0.0:
        raise ValueError("KAD bandwidth is 0: more than half of the baseline pairs are identical rows")
    eng, collective = _kad_engine(distributed)
    dev = eng.torch_device
    z = pb.x if y is None or not y.shape[0] else torch.cat([pb.x, _kad_device_rows(y, eng)])
    sig = torch.tensor([pb.sigma], dtype=torch.float64, device=dev)
    sums = eng.kad_eval_sums(z, pb.m, torch.from_numpy(offsets).to(dev), sig, 0 if collective else None).cpu().numpy()
    out = []
    for k, n in enumerate(np.diff(offsets).tolist()):
        score = _kad_score(pb.s_xx, float(sums[k, 0]), float(sums[k, 1]), pb.m, n) if n >= 2 else float("nan")
        out.append(KADResults(score=score, bandwidth=pb.sigma, n_baseline=pb.m, n_eval=n))
    return out


def kad_embedding_dir(path, model_name: str, metric: str = "KAD") -> Path:
    """The embedding cache directory <path>/embeddings/<model> that KAD (and PRDC) reads; ValueError for statistics
    files, named statistics sets and anything else that is not a directory (they hold (mu, C), not embeddings)."""
    named = isinstance(path, str) and _named_statistics(path) is not None
    if named or str(path).endswith(".npz") or Path(path).is_file():
        raise ValueError(f"{metric} needs embeddings, not (mu, C) statistics: '{path}' is a statistics file or set; "
                         "pass the audio directory instead")
    if not Path(path).is_dir():
        raise ValueError(f"{metric} needs a directory of audio or embeddings; '{path}' is not a directory")
    return Path(path) / "embeddings" / model_name


def calc_embd_statistics(embd_lst: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """Mean and covariance matrix of an [n, d] embedding array (fadtk/fad.py:42-48).

    Like numpy in the reference, the mean comes back in the dtype of the input (fp16 embeddings
    give an fp16 mean) and the covariance in float64.
    """
    assert embd_lst.shape[0] >= 2, (f"FAD requires at least two embedding window frames, you have {embd_lst.shape}."
        " (This probably means that your audio is too short)")
    mu, cov = statistics_of_arrays([embd_lst])
    if np.issubdtype(embd_lst.dtype, np.floating):
        mu = mu.astype(embd_lst.dtype)
    return mu, cov


def _frechet_parts(cov1, cov2):
    """-> (tr C1, tr C2, tr sqrt(C1 C2), residual) from the GPU chain."""
    from . import _native
    eng = _native.engine()
    dev = eng.torch_device
    d = cov1.shape[0]
    c1 = torch.from_numpy(np.ascontiguousarray(cov1, dtype=np.float64)).to(dev)
    c2 = torch.from_numpy(np.ascontiguousarray(cov2, dtype=np.float64)).to(dev)
    z = torch.zeros(d, dtype=torch.float64, device=dev)
    out = eng.frechet(z, c1, z, c2).cpu().numpy()
    return out[5], out[6], out[1], out[2]


def calc_frechet_distance(mu1, cov1, mu2, cov2, eps=1e-6):
    """Frechet distance between N(mu1, cov1) and N(mu2, cov2) (fadtk/fad.py:51-120):

        d^2 = ||mu1 - mu2||^2 + Tr(cov1 + cov2 - 2 sqrt(cov1 cov2))

    The reference takes Tr sqrt(cov1 cov2) from an eigen-decomposition of the non-symmetric
    product; here it is the trace of the square root of the similar PSD matrix
    cov1^(1/2) cov2 cov1^(1/2) (same eigenvalues), computed on the GPU.  ``eps`` is accepted for
    signature compatibility: the PSD form has no singular-product failure mode to regularise.
    """
    mu1 = np.atleast_1d(mu1)
    mu2 = np.atleast_1d(mu2)
    cov1 = np.atleast_2d(cov1)
    cov2 = np.atleast_2d(cov2)

    assert mu1.shape == mu2.shape, \
        f'Training and test mean vectors have different lengths ({mu1.shape} vs {mu2.shape})'
    assert cov1.shape == cov2.shape, \
        f'Training and test covariances have different dimensions ({cov1.shape} vs {cov2.shape})'

    diff = mu1 - mu2            # numpy dtype rules as in the reference (fp16 - fp16 stays fp16)
    tr1, tr2, tr_covmean, resid = _frechet_parts(cov1, cov2)
    if not np.isfinite(tr_covmean):
        raise ValueError("non-finite covariance statistics (NaN/Inf input)")
    if resid > 1e-3:
        log.warning(f'Detected high error in matrix square root: residual {resid}')
    return (diff.dot(diff) + tr1 + tr2 - 2 * tr_covmean)


def _device_score(baseline, emb_dev, eng, idx_dev=None):
    """FAD of fp16 device rows (optionally gathered by idx) against a cached Baseline, with the
    reference's calc_embd_statistics semantics: fp16 mean (np.mean dtype rule, fad.py:48), fp64 cov."""
    st = DeviceStatistics(emb_dev.shape[1], eng)
    if idx_dev is None:
        st.add(emb_dev)
    else:
        st.add_gather(emb_dev, idx_dev)
    mu_d, cov_d = st.finalize()
    mu_d = mu_d.to(torch.float16).to(torch.float64)
    out = baseline.frechet(mu_d.contiguous(), cov_d).cpu().numpy()
    if not np.isfinite(out[1]):
        raise ValueError("non-finite covariance statistics (NaN/Inf input)")
    diff = baseline.mu_host - mu_d.cpu().numpy()
    return float(diff.dot(diff) + out[5] + out[6] - 2 * out[1])


def _sorted_npy_files(directory: Path) -> list:
    """sorted(directory.glob('*.npy')) without a pathlib object comparison per sort step (10 000 files: 0.2 s -> 10 ms)"""
    try:
        names = sorted(n for n in os.listdir(directory) if n.endswith(".npy"))
    except OSError:
        names = []
    return [directory / n for n in names]


def _statistics_dirs():
    """Where a baseline NAME such as ``fma_pop`` is looked up (fadtk/fad.py:249-255 reads fadtk/stats/<name>.npz):
    $FADTK_STATS_DIR, this package's stats/ directory, and - when the reference package itself is installed next to
    this one - its fadtk/stats/ directory, so `fadtk vggish fma_pop <dir>` keeps working after the switch."""
    dirs = []
    env = os.environ.get("FADTK_STATS_DIR", "")
    if env:
        dirs.append(Path(env))
    dirs.append(Path(__file__).parent / "stats")
    try:
        import importlib.util
        spec = importlib.util.find_spec("fadtk")
        if spec is not None and spec.submodule_search_locations:
            dirs += [Path(loc) / "stats" for loc in spec.submodule_search_locations]
    except (ImportError, ValueError):
        pass
    return dirs


def _named_statistics(name: str):
    for bp in _statistics_dirs():
        stats = bp / (name.lower() + ".npz")
        if stats.exists():
            return stats
    return None


class FrechetAudioDistance:
    """Same constructor and methods as fadtk.fad.FrechetAudioDistance (fad.py:123-395)."""
    loaded = False

    def __init__(self, ml: ModelLoader, audio_load_worker=8, load_model=True):
        self.ml = ml
        self.audio_load_worker = audio_load_worker
        self.sox_formats = find_sox_formats(sox_path)
        self.device = torch.device('cuda') if torch.cuda.is_available() else torch.device('cpu')
        if load_model:
            self.ml.load_model()
            self.loaded = True
        torch.autograd.set_grad_enabled(False)

    # ------------------------------------------------------------------ audio
    def _converted_path(self, f: Path) -> Path:
        return (f.parent / "convert" / str(self.ml.sr) / f.name).with_suffix(".wav")

    def convert_audio(self, f: Union[str, Path]) -> np.ndarray:
        """Decode -> mono -> model sample rate -> PCM16; cached under <dir>/convert/<sr>/ like
        the reference (fad.py:143-160).  Returns the int16 samples."""
        f = Path(f)
        new = self._converted_path(f)
        if new.exists():
            return synth.read_wav(new)[0]
        new.parent.mkdir(parents=True, exist_ok=True)
        if f.suffix.lower() == ".wav":
            try:
                pcm, sr = synth.read_wav(f)      # int16 [T] or [T, channels]
                x = None
            except Exception:                    # 8/24/32-bit PCM, IEEE float, extensible headers: float path
                x, sr = synth.read_wav_float(f)  # float32 [channels, T], torchaudio.load's normalisation
                x, pcm = torch.from_numpy(x), None
        else:
            x, sr = decode_container(f)          # float32 [channels, T] at the file's own rate
            pcm = None
        if pcm is not None and pcm.ndim == 1 and sr == self.ml.sr:
            out = pcm                            # already mono PCM16 at the model rate: bit-exact copy
        else:
            # mono mix + Kaiser-sinc polyphase resampling + PCM16 quantisation on the GPU
            # (fad_resample; same filter bank as the reference's torchaudio Resample, fad.py:150-160)
            from . import _native
            eng = _native.engine()
            src = torch.from_numpy(np.array(pcm, copy=True)) if pcm is not None else x.to(torch.float32).contiguous()
            with _RESAMPLE_LOCK:                 # a fad_handle is single-threaded; convert_audio runs on worker threads
                out = eng.resample(src.to(eng.torch_device), int(sr), int(self.ml.sr)).cpu().numpy()
        synth.write_wav(new, out, self.ml.sr)
        return out

    def load_audio(self, f: Union[str, Path]):
        self.convert_audio(f)
        return self.ml.load_wav(self._converted_path(Path(f)))

    # ------------------------------------------------------------- embeddings
    def cache_embedding_file(self, audio_dir: Union[str, Path]):
        """Compute the embedding of one audio file and cache it (fad.py:188-201)."""
        cache = get_cache_embedding_path(self.ml.name, audio_dir)
        if cache.exists():
            return
        wav_data = self.load_audio(audio_dir)
        embd = self.ml.get_embedding(wav_data)
        cache.parent.mkdir(parents=True, exist_ok=True)
        np.save(cache, embd)

    def read_embedding_file(self, audio_dir: Union[str, Path]):
        cache = get_cache_embedding_path(self.ml.name, audio_dir)
        assert cache.exists(), f"Embedding file {cache} does not exist, please run cache_embedding_file first."
        return np.load(cache)

    def load_embeddings(self, dir: Union[str, Path], max_count: int = -1, concat: bool = True):
        files = list(Path(dir).glob("*.*"))
        log.info(f"Loading {len(files)} audio files from {dir}...")
        return self._load_embeddings(files, max_count=max_count, concat=concat)

    def _load_embeddings(self, files: list[Path], max_count: int = -1, concat: bool = True):
        if len(files) == 0:
            raise ValueError("No files provided")
        if max_count == -1 and concat:
            from . import _io_native
            caches = [get_cache_embedding_path(self.ml.name, f) for f in files]
            for c in caches:
                assert c.exists(), f"Embedding file {c} does not exist, please run cache_embedding_file first."
            return _io_native.load_embedding_files(caches, self.audio_load_worker)[0]
        if max_count == -1:
            with ThreadPoolExecutor(max(1, self.audio_load_worker)) as ex:
                embd_lst = list(ex.map(self.read_embedding_file, files))
        else:
            total_len = 0
            embd_lst = []
            for f in files:
                embd_lst.append(self.read_embedding_file(f))
                total_len += embd_lst[-1].shape[0]
                if total_len > max_count:
                    break
        if concat:
            return np.concatenate(embd_lst, axis=0)
        return embd_lst, files

    # ------------------------------------------------------------- statistics
    def load_stats(self, path: PathLike):
        """Embedding statistics of a named set, an .npz file or a directory (fad.py:245-290)."""
        if isinstance(path, str):
            named = _named_statistics(path)
            if named is not None:
                path = named
            elif not Path(path).exists() and os.sep not in path and not path.endswith(".npz"):
                log.error(f"'{path}' is neither a path nor a packaged statistics name: no {path.lower()}.npz in "
                          + ", ".join(str(d) for d in _statistics_dirs()) + " (the reference ships fadtk/stats/fma_pop.npz; "
                          "copy it into one of these directories or point $FADTK_STATS_DIR at it)")
        path = Path(path)

        if path.is_file():
            log.info(f"Loading embedding statistics from {path}...")
            with np.load(path) as data:
                if f'{self.ml.name}.mu' not in data or f'{self.ml.name}.cov' not in data:
                    raise ValueError(f"FAD statistics file {path} doesn't contain data for model {self.ml.name}")
                return data[f'{self.ml.name}.mu'], data[f'{self.ml.name}.cov']

        cache_dir = path / "stats" / self.ml.name
        emb_dir = path / "embeddings" / self.ml.name
        # Under torchrun every rank asks for the same statistics: rank 0 alone decides whether the cache is current,
        # computes and writes it (atomically); the others wait at the barrier and then read the finished files -
        # never a half-written mu.npy / cov.npy, never N concurrent writers of the same cache.
        from . import dist
        if dist.is_distributed() and dist.rank() != 0:
            dist.barrier()
            if not (cache_dir / "mu.npy").exists():
                log.error(f"The dataset you want to use ({path}) is not a directory nor a file.")
                exit(1)
            return np.load(cache_dir / "mu.npy"), np.load(cache_dir / "cov.npy")
        try:
            return self._load_or_compute_dir_stats(path, cache_dir, emb_dir)
        finally:
            dist.barrier()

    def _load_or_compute_dir_stats(self, path: Path, cache_dir: Path, emb_dir: Path):
        if (cache_dir / "mu.npy").exists() and (cache_dir / "cov.npy").exists():
            # The reference trusts this cache forever (fad.py:268-274): adding or re-embedding files silently
            # keeps the old statistics.  Caches written here carry a fingerprint of the embedding files they
            # were computed from; a cache without one (written by the reference) is loaded as the reference does.
            if self._stats_cache_is_current(cache_dir, emb_dir):
                log.info(f"Embedding statistics is already cached for {path}, loading...")
                return np.load(cache_dir / "mu.npy"), np.load(cache_dir / "cov.npy")
            log.info(f"Embedding files of {path} changed since the statistics were cached, recomputing...")

        if not path.is_dir():
            log.error(f"The dataset you want to use ({path}) is not a directory nor a file.")
            exit(1)

        log.info(f"Loading embedding files from {path}...")
        mu, cov = calculate_embd_statistics_online(_sorted_npy_files(emb_dir))
        log.info("> Embeddings statistics calculated.")

        cache_dir.mkdir(parents=True, exist_ok=True)
        for name, arr in (("mu.npy", mu), ("cov.npy", cov)):          # write-then-rename: readers never see a partial file
            tmp = cache_dir / (name + f".tmp{os.getpid()}")
            with open(tmp, "wb") as fh:
                np.save(fh, arr)
            os.replace(tmp, cache_dir / name)
        tmp = cache_dir / f"source.json.tmp{os.getpid()}"
        tmp.write_text(json.dumps(self._embedding_fingerprint(emb_dir)))
        os.replace(tmp, cache_dir / "source.json")
        return mu, cov

    @staticmethod
    def _embedding_fingerprint(emb_dir: Path) -> dict:
        """What the cached statistics depend on: the embedding files' names, sizes and newest mtime."""
        try:                                                    # one scandir pass: names and stat results together
            with os.scandir(emb_dir) as it:
                entries = sorted(((e.name, e.stat()) for e in it if e.name.endswith(".npy")), key=lambda p: p[0])
        except OSError:
            entries = []
        names = hashlib.sha1("\n".join(n for n, _ in entries).encode()).hexdigest()
        return {"files": len(entries), "bytes": int(sum(st.st_size for _, st in entries)), "names_sha1": names,
                "newest_mtime_ns": int(max((st.st_mtime_ns for _, st in entries), default=0))}

    @classmethod
    def _stats_cache_is_current(cls, cache_dir: Path, emb_dir: Path) -> bool:
        src = cache_dir / "source.json"
        if not src.exists() or not emb_dir.is_dir():       # reference-written cache, or statistics shipped without embeddings
            return True
        try:
            return json.loads(src.read_text()) == cls._embedding_fingerprint(emb_dir)
        except (OSError, ValueError):
            return False

    # ------------------------------------------------------------------ scores
    def score(self, baseline: PathLike, eval: PathLike):
        """A single FAD score between a baseline and an eval set (fad.py:292-302)."""
        mu_bg, cov_bg = self.load_stats(baseline)
        mu_eval, cov_eval = self.load_stats(eval)
        return calc_frechet_distance(mu_bg, cov_bg, mu_eval, cov_eval)

    def prepare_pairwise(self, baseline_dir: PathLike, k_max: int = 16, distributed: bool = False):
        """The PairwiseBaseline (prepare_pairwise_baseline) of the cached embeddings of baseline_dir, grouped by file:
        loaded from <baseline_dir>/stats/<model>/pairwise.npz when that file was written by this build for these
        embedding files (the fingerprint statistics caches keep in source.json) and these rows (their digest) with
        k_max at least the one asked for; otherwise computed and saved there atomically, with one log line that says
        why.  distributed=True under torchrun: a collective call; rank 0 decides and writes, every rank computes its
        share."""
        k_max = _prdc_k(k_max, "a prepared baseline")
        collective = distributed and _kad_engine(True, "a prepared baseline")[1]
        x, _, base_offs = self._baseline_rows(baseline_dir, "a prepared baseline", collective)
        return self._prepared(baseline_dir, x, base_offs, k_max, distributed, k_max)

    def _baseline_rows(self, baseline_dir: PathLike, metric: str, collective: bool):
        """-> (x, files, offsets): the baseline's fp16 rows, its cache files and their int64 row offsets in x"""
        from . import _io_native
        files = _on_rank0(lambda: _sorted_npy_files(kad_embedding_dir(baseline_dir, self.ml.name, metric)), collective)
        if not files:
            raise ValueError(f"no {self.ml.name} embeddings cached under {baseline_dir}: embed the baseline directory first")
        x, offs = _io_native.load_embedding_files(files, self.audio_load_worker)
        if x.dtype != np.float16:
            raise ValueError(f"{metric} needs fp16 embedding caches; {baseline_dir} holds {x.dtype}")
        return x, files, offs

    def _prepared(self, baseline_dir: PathLike, x: np.ndarray, base_offs: np.ndarray, k: int, distributed: bool,
                  k_max: "int | None" = None):
        """prepare_pairwise over rows already read (x, base_offs), good for k: a saved preparation with k_max >= k, else
        a new one with k_max (default max(k, min(16, m - 1)), so that one preparation serves every k a metric allows)"""
        from . import dist
        from ._native import PairwiseBaseline
        eng, collective = _kad_engine(distributed, "a prepared baseline")
        path = Path(baseline_dir) / "stats" / self.ml.name / "pairwise.npz"
        emb_dir = Path(baseline_dir) / "embeddings" / self.ml.name
        fingerprint = self._embedding_fingerprint(emb_dir)
        xd = _kad_device_rows(torch.from_numpy(x), eng)
        pb, why = PairwiseBaseline.load(path, eng, xd, k, int(x.shape[1]), fingerprint, base_offs)
        # every rank takes rank 0's branch: a collective preparation needs all of them
        if _on_rank0(lambda: pb is not None, collective):
            if pb is None:
                raise ValueError(f"the saved preparation {path} cannot be read on every rank ({why})")
            log.info(f"Pairwise baseline preparation loaded from {path}")
            return pb
        if not collective or dist.rank() == 0:
            log.info(f"Pairwise baseline preparation of {baseline_dir}: {why}, computing...")
        k_max = k_max or max(k, min(16, int(x.shape[0]) - 1))
        pb = prepare_pairwise_baseline(x, k_max, base_offs, distributed)
        if not collective or dist.rank() == 0:
            pb.save(path, fingerprint)
        return pb

    def score_kad(self, baseline_dir: PathLike, eval_dir: PathLike, distributed: bool = False,
                  prepared: bool = False) -> KADResults:
        """Kernel Audio Distance between the cached embeddings of two directories (calc_kernel_audio_distance): all rows
        of all <dir>/embeddings/<model>/*.npy in sorted file order, the files the directory statistics read.
        distributed=True under torchrun: a collective call; rank 0 lists the files, every rank reads them and takes its
        share of the pair tiles, and every rank gets the result.  prepared=True: against prepare_pairwise(baseline_dir),
        loaded or built and saved (bitwise the per-song value of the eval set as one song)."""
        x, y = self._cached_sets(baseline_dir, eval_dir, "KAD", distributed)
        if prepared:
            x = self._prepared(baseline_dir, x, self._cached_offsets(baseline_dir, "KAD", distributed), 1, distributed)
        return calc_kernel_audio_distance(x, y, distributed=distributed)

    def score_kad_test(self, baseline_dir: PathLike, eval_dir: PathLike, permutations: int = 999, seed: int = 0,
                       distributed: bool = False, prepared: bool = False) -> KADTestResults:
        """Permutation test of KAD (calc_kad_test) between the cached embeddings of two directories, read as score_kad
        reads them; distributed and prepared as there (prepared: the p-value and nulls are bitwise the unprepared
        ones, score is score_kad's prepared value)."""
        permutations, seed = _perm_args(permutations, seed, "a KAD permutation test")
        x, y = self._cached_sets(baseline_dir, eval_dir, "KAD", distributed)
        if prepared:
            x = self._prepared(baseline_dir, x, self._cached_offsets(baseline_dir, "KAD", distributed), 1, distributed)
        return calc_kad_test(x, y, permutations, seed, distributed=distributed)

    def score_kad_comparison(self, baseline_dir: PathLike, eval_dir: PathLike, versus_dir: PathLike,
                             permutations: int = 999, seed: int = 0, distributed: bool = False,
                             prepared: bool = False) -> KADComparisonResults:
        """Permutation test of KAD(baseline, eval) - KAD(baseline, versus) (calc_kad_comparison) over the cached
        embeddings of three directories, read as score_kad reads them; distributed and prepared as for score_kad."""
        permutations, seed = _perm_args(permutations, seed, "a KAD comparison")
        x, a, b = self._cached_sets(baseline_dir, eval_dir, "KAD", distributed, versus_dir)
        if prepared:
            x = self._prepared(baseline_dir, x, self._cached_offsets(baseline_dir, "KAD", distributed), 1, distributed)
        return calc_kad_comparison(x, a, b, permutations, seed, distributed=distributed)

    def score_fad_comparison(self, baseline: PathLike, eval_dir: PathLike, versus_dir: PathLike,
                             permutations: int = 999, seed: int = 0) -> FADComparisonResults:
        """Permutation test of score(baseline, eval_dir) - score(baseline, versus_dir) (calc_fad_comparison).  baseline
        is anything load_stats takes (a directory, an .npz file or a named set); the units are the sorted cache files
        <dir>/embeddings/<model>/*.npy that each eval directory's statistics read, empty files dropped.  score_a and
        score_b are self.score's values, so a directory score refuses fails here the same way."""
        permutations, seed = _perm_args(permutations, seed, "a FAD comparison")
        score_a = float(self.score(baseline, eval_dir))
        score_b = float(self.score(baseline, versus_dir))
        mu, cov = self.load_stats(baseline)
        d = int(np.asarray(mu).shape[0])
        units = []
        for p, what in ((eval_dir, "eval A"), (versus_dir, "eval B")):
            arrs = [np.load(f) for f in _sorted_npy_files(Path(p) / "embeddings" / self.ml.name)]
            units.append(_fad_units([a for a in arrs if a.shape[0] > 0], what, d))
        return _fad_comparison(mu, cov, units[0], units[1], score_a, score_b, permutations, seed)

    def score_fad_bootstrap(self, baseline: PathLike, eval_dir: PathLike, resamples: int = 999, seed: int = 0,
                            level: float = 0.95, method: str = "percentile") -> FADBootstrapResults:
        """Bootstrap confidence interval of score(baseline, eval_dir) (calc_fad_bootstrap), conditional on the baseline.
        baseline is anything load_stats takes (a directory, an .npz file or a named set); the units are the sorted
        cache files <eval_dir>/embeddings/<model>/*.npy, empty files dropped.  score is self.score's value."""
        resamples, seed, level, method = _boot_args(resamples, seed, level, method, "a FAD bootstrap")
        score = float(self.score(baseline, eval_dir))
        mu, cov = self.load_stats(baseline)
        d = int(np.asarray(mu).shape[0])
        arrs = [np.load(f) for f in _sorted_npy_files(Path(eval_dir) / "embeddings" / self.ml.name)]
        units = _fad_units([a for a in arrs if a.shape[0] > 0], "eval", d, "the FAD bootstrap")
        return _fad_bootstrap(mu, cov, units, score, resamples, seed, level, method)

    def score_kad_bootstrap(self, baseline_dir: PathLike, eval_dir: PathLike, resamples: int = 999, seed: int = 0,
                            level: float = 0.95, method: str = "percentile", prepared: bool = False) -> KADBootstrapResults:
        """Bootstrap confidence interval of KAD (calc_kad_bootstrap) between the cached embeddings of two directories,
        read as score_kad reads them; the units are the eval directory's sorted cache files, empty files dropped.
        prepared: against the baseline's saved pairwise preparation, with replicates bitwise the unprepared ones."""
        resamples, seed, level, method = _boot_args(resamples, seed, level, method, "a KAD bootstrap")
        x, _ = self._cached_sets(baseline_dir, eval_dir, "KAD", False)
        if prepared:
            x = self._prepared(baseline_dir, x, self._cached_offsets(baseline_dir, "KAD", False), 1, False)
        arrs = [np.load(f) for f in _sorted_npy_files(kad_embedding_dir(eval_dir, self.ml.name))]
        return calc_kad_bootstrap(x, [a for a in arrs if a.shape[0] > 0], resamples, seed, level, method)

    def _cached_offsets(self, baseline_dir: PathLike, metric: str, distributed: bool) -> np.ndarray:
        """the int64 row offsets of the baseline's cache files, from their headers"""
        from . import _io_native
        collective = distributed and _kad_engine(True, metric)[1]
        files = _on_rank0(lambda: _sorted_npy_files(kad_embedding_dir(baseline_dir, self.ml.name, metric)), collective)
        rows = _io_native.npy_probe(files, self.audio_load_worker)[0]
        offs = np.zeros(len(files) + 1, dtype=np.int64)
        offs[1:] = np.cumsum(rows)
        return offs

    def score_prdc(self, baseline_dir: PathLike, eval_dir: PathLike, k: int = 5, distributed: bool = False,
                   prepared: bool = False) -> PRDCResults:
        """Precision, recall, density and coverage (calc_prdc) of the cached embeddings of eval_dir against those of
        baseline_dir, read as score_kad reads them: all rows of all <dir>/embeddings/<model>/*.npy in sorted file
        order.  Statistics files and names are refused.  distributed=True under torchrun: a collective call; rank 0
        lists the files, every rank reads them and takes its share of the radii and ball-count tiles, and every rank
        gets the result.  prepared=True: against prepare_pairwise(baseline_dir) (bitwise the same values)."""
        x, y = self._cached_sets(baseline_dir, eval_dir, "PRDC", distributed)
        if prepared:
            x = self._prepared(baseline_dir, x, self._cached_offsets(baseline_dir, "PRDC", distributed), _prdc_k(k),
                               distributed)
        return calc_prdc(x, y, k=k, distributed=distributed)

    def _cached_sets(self, baseline_dir: PathLike, eval_dir: PathLike, metric: str, distributed: bool,
                     versus_dir: "PathLike | None" = None) -> list:
        """The fp16 embeddings of the two directories that score_kad and score_prdc score (and of versus_dir, when given,
        third), for `metric` (named in the errors).  Collective under distributed=True: rank 0 lists the files, every
        rank reads them."""
        from . import _io_native
        collective = distributed and _kad_engine(True, metric)[1]
        sets = []
        dirs = (("baseline", baseline_dir), ("eval", eval_dir)) + ((("versus", versus_dir),) if versus_dir is not None else ())
        for what, p in dirs:
            files = _on_rank0(lambda: _sorted_npy_files(kad_embedding_dir(p, self.ml.name, metric)), collective)
            if not files:
                raise ValueError(f"no {self.ml.name} embeddings cached under {p}: embed the {what} directory first")
            emb, _ = _io_native.load_embedding_files(files, self.audio_load_worker)
            if emb.dtype != np.float16:
                raise ValueError(f"{metric} needs fp16 embedding caches; {p} holds {emb.dtype}")
            sets.append(emb)
        return sets

    def score_kad_individual(self, baseline_dir: PathLike, eval_dir: PathLike, csv_name: Union[Path, str],
                             distributed: bool = False, prepared: bool = False) -> Path:
        """KAD of every file in eval_dir against the embeddings of baseline_dir (calc_kernel_audio_distance_songs: the
        bandwidth and the baseline's pair sum once, every song's sums in one GPU pass), written as score_individual
        writes FAD: rows ``file,score`` sorted by |score|, commas in names replaced, no header; a str csv_name goes
        under data/kad-individual/<model>/, and an existing table is returned untouched.  Files whose cache is
        missing, unreadable or not an fp16 [rows, d] array of the baseline's width, and files with fewer than two
        embedding rows, are logged and dropped.  distributed=True under torchrun: a collective call; rank 0 lists the
        directories and decides whether the table exists, every rank reads the caches and takes its share of the pair
        tiles, and rank 0 alone logs the dropped files and writes the table.  prepared=True: against
        prepare_pairwise(baseline_dir), loaded or built and saved; the same table."""
        csv = Path(csv_name)
        if isinstance(csv_name, str):
            csv = Path('data') / 'kad-individual' / self.ml.name / csv_name
        collective = distributed and _kad_engine(True)[1]
        from . import dist
        writer = not collective or dist.rank() == 0
        if _on_rank0(csv.exists, collective):
            if writer:
                log.info(f"CSV file {csv} already exists, exiting...")
            return csv

        x, host, offs, names, _, base_offs = self._individual_sets(baseline_dir, eval_dir, "KAD", 2,
                                                                   "at least two embedding rows", collective, writer)
        pairs = []
        if names and prepared:
            pb = self._prepared(baseline_dir, x, base_offs, 1, distributed)
            res = _kad_prepared(pb, host[x.shape[0]:], offs, distributed)
            pairs = [(f, r.score) for f, r in zip(names, res) if f is not None]
        elif names:
            res = _kad_songs(host, x.shape[0], offs, distributed)
            pairs = [(f, r.score) for f, r in zip(names, res) if f is not None]

        if not writer:
            return csv
        pairs = sorted(pairs, key=lambda x: np.abs(x[1]))
        csv.parent.mkdir(parents=True, exist_ok=True)
        csv.write_text("\n".join([",".join([str(x).replace(',', '_') for x in row]) for row in pairs]))
        return csv

    def score_prdc_individual(self, baseline_dir: PathLike, eval_dir: PathLike, csv_name: Union[Path, str],
                              k: int = 5, distributed: bool = False, prepared: bool = False) -> Path:
        """Precision, recall, density and coverage of every file in eval_dir against the embeddings of baseline_dir
        (calc_prdc_songs: the baseline radii once, every file's radii and counts in one GPU pass each).  The table has
        the header ``file,precision,recall,density,coverage,n_eval`` and one row per file, sorted by density, highest
        (most baseline-like) first, ties by path; commas in names are replaced.  A str csv_name goes under
        data/prdc-individual/<model>/, and an existing table is returned untouched.  Files whose cache is missing,
        unreadable or not an fp16 [rows, d] array of the baseline's width, and files with at most k embedding rows,
        are logged and dropped.  distributed=True under torchrun: as for score_kad_individual, over the radii and
        ball-count tiles.  prepared=True: as for score_kad_individual; the same table."""
        k = _prdc_k(k)
        csv = Path(csv_name)
        if isinstance(csv_name, str):
            csv = Path('data') / 'prdc-individual' / self.ml.name / csv_name
        collective = distributed and _kad_engine(True, "PRDC")[1]
        from . import dist
        writer = not collective or dist.rank() == 0
        if _on_rank0(csv.exists, collective):
            if writer:
                log.info(f"CSV file {csv} already exists, exiting...")
            return csv

        x, host, offs, names, _, base_offs = self._individual_sets(baseline_dir, eval_dir, "PRDC", k + 1,
                                                                   f"more than k = {k} embedding rows", collective, writer)
        rows = []
        if names:
            pb = self._prepared(baseline_dir, x, base_offs, k, distributed) if prepared and x.shape[0] > k else None
            res = _prdc_songs(host if pb is None else host[x.shape[0]:], x.shape[0], np.diff(offs).tolist(), k,
                              distributed, pb)
            rows = [(f, r) for f, r in zip(names, res) if f is not None]
        elif x.shape[0] <= k:
            raise ValueError(f"PRDC with k = {k} needs more than k embedding rows in each set (baseline {x.shape[0]})")

        if not writer:
            return csv
        rows.sort(key=lambda t: (-t[1].density, str(t[0])))
        csv.parent.mkdir(parents=True, exist_ok=True)
        lines = ["file,precision,recall,density,coverage,n_eval"]
        lines += [",".join([str(f).replace(',', '_'), *(str(v) for v in (r.precision, r.recall, r.density, r.coverage,
                                                                              r.n_eval))]) for f, r in rows]
        csv.write_text("\n".join(lines) + "\n")
        return csv

    def score_realism_individual(self, baseline_dir: PathLike, eval_dir: PathLike, csv_name: Union[Path, str],
                                 k: int = 3, distributed: bool = False, prepared: bool = False) -> Path:
        """Realism and nearest baseline clip of every file in eval_dir against the embeddings of baseline_dir: one
        calc_realism call over the rows of all files (a row's values depend on that row and the baseline alone).  The
        table has the header ``file,realism_median,realism_min,nearest_baseline,nearest_distance,n_eval`` and one row
        per file: the median and the least realism of its rows, the baseline embedding cache that holds the nearest
        baseline row of its nearest row, and that distance.  Rows are sorted by realism_median, least realistic first,
        ties by path; commas in names are replaced.  A str csv_name goes under data/realism-individual/<model>/, and an
        existing table is returned untouched.  Files whose cache is missing, unreadable, not an fp16 [rows, d] array of
        the baseline's width, or empty are logged and dropped.  distributed=True under torchrun: as for
        score_kad_individual, over the radii and realism tiles.  prepared=True: as for score_kad_individual; the same
        table."""
        k = _prdc_k(k, "realism")
        csv = Path(csv_name)
        if isinstance(csv_name, str):
            csv = Path('data') / 'realism-individual' / self.ml.name / csv_name
        collective = distributed and _kad_engine(True, "realism")[1]
        from . import dist
        writer = not collective or dist.rank() == 0
        if _on_rank0(csv.exists, collective):
            if writer:
                log.info(f"CSV file {csv} already exists, exiting...")
            return csv

        x, host, offs, names, base_files, base_offs = self._individual_sets(
            baseline_dir, eval_dir, "realism", 1, "at least one embedding row", collective, writer)
        _realism_rows(x.shape[0], 1, k)
        rows = []
        if names:
            pb = self._prepared(baseline_dir, x, base_offs, k, distributed) if prepared else None
            res = _realism(host if pb is None else host[x.shape[0]:], x.shape[0], k, distributed, pb)
            for s, f in enumerate(names):
                if f is None:
                    continue
                a, b = int(offs[s]), int(offs[s + 1])
                real = res.realism[a:b].astype(np.float64)
                j = a + int(np.argmin(res.nearest_distance[a:b]))
                base = base_files[int(np.searchsorted(base_offs, res.nearest[j], side="right")) - 1]
                rows.append((f, float(np.median(real)), float(real.min()), base, float(res.nearest_distance[j]), b - a))

        if not writer:
            return csv
        rows.sort(key=lambda t: (t[1], str(t[0])))
        csv.parent.mkdir(parents=True, exist_ok=True)
        lines = ["file,realism_median,realism_min,nearest_baseline,nearest_distance,n_eval"]
        lines += [",".join(str(v).replace(',', '_') for v in row) for row in rows]
        csv.write_text("\n".join(lines) + "\n")
        return csv

    def score_nearest_individual(self, baseline_dir: PathLike, eval_dir: PathLike, csv_name: Union[Path, str],
                                 k: int = 5, distributed: bool = False, prepared: bool = False) -> Path:
        """The k baseline files every file of eval_dir comes closest to: a memorisation audit.  One calc_nearest call
        over the rows of all eval files, with each baseline embedding cache one group; then per eval file, per baseline
        file, the smallest (distance, eval row, baseline row) over the file's rows, and the first k baseline files in
        that order.  The table has the header ``file,rank,nearest_baseline,distance,eval_row,baseline_row,n_eval`` and
        one line per (file, rank): the baseline cache, the distance and the pair of rows (each within its own file)
        where the two come closest.  Files are sorted by their rank-1 distance, closest (most copy-like) first, ties by
        path; commas in names are replaced.  A str csv_name goes under data/nearest-individual/<model>/, and an
        existing table is returned untouched.  Files whose cache is missing, unreadable, not an fp16 [rows, d] array
        of the baseline's width, or empty are logged and dropped.  distributed=True under torchrun: as for
        score_kad_individual, over the nearest tiles.  prepared=True: as for score_kad_individual (nearest reuses the
        resident rows alone); the same table."""
        k = _prdc_k(k, "nearest")
        csv = Path(csv_name)
        if isinstance(csv_name, str):
            csv = Path('data') / 'nearest-individual' / self.ml.name / csv_name
        collective = distributed and _kad_engine(True, "nearest")[1]
        from . import dist
        writer = not collective or dist.rank() == 0
        if _on_rank0(csv.exists, collective):
            if writer:
                log.info(f"CSV file {csv} already exists, exiting...")
            return csv

        x, host, offs, names, base_files, base_offs = self._individual_sets(
            baseline_dir, eval_dir, "nearest", 1, "at least one embedding row", collective, writer)
        _nearest_rows(x.shape[0], 1)
        tables = []
        if names:
            pb = self._prepared(baseline_dir, x, base_offs, 1, distributed) if prepared else None
            res, q = _nearest(host if pb is None else host[x.shape[0]:], x.shape[0], k, base_offs, distributed, pb)
            for s, f in enumerate(names):
                if f is None:
                    continue
                a, b = int(offs[s]), int(offs[s + 1])
                lines = []
                for rank, (j, r) in enumerate(_file_nearest(res.groups[a:b], res.rows[a:b], q[a:b], k)):
                    g, i = int(res.groups[a + j, r]), int(res.rows[a + j, r])
                    lines.append((rank + 1, base_files[g], float(res.distance[a + j, r]), j, i - int(base_offs[g]), b - a))
                tables.append((f, lines))

        if not writer:
            return csv
        tables.sort(key=lambda t: (t[1][0][2], str(t[0])))
        csv.parent.mkdir(parents=True, exist_ok=True)
        lines = ["file,rank,nearest_baseline,distance,eval_row,baseline_row,n_eval"]
        lines += [",".join(str(v).replace(',', '_') for v in (f, *row)) for f, rows in tables for row in rows]
        csv.write_text("\n".join(lines) + "\n")
        return csv

    def _individual_sets(self, baseline_dir: PathLike, eval_dir: PathLike, metric: str, min_rows: int, need: str,
                         collective: bool, writer: bool):
        """The embeddings the score_*_individual methods score -> (x, host, offs, names, base_files, base_offs): x the
        baseline's fp16 rows; host = [x; the kept files' rows] fp16 (pinned when there is a GPU), offs their int64
        offsets after x, names[k] the file of kept song k, or None when its cache could not be read (its rows are
        zeros: score it and drop it); base_files the baseline's cache files, base_offs their int64 row offsets in x.  A
        file is kept when its cache is an fp16 [rows, d] array of the baseline's width with at least min_rows rows
        (`need` says so in the log); the others are logged (by the writer) and dropped.
        Collective: rank 0 lists the directories, every rank reads the caches."""
        from . import _io_native
        files = _on_rank0(lambda: _sorted_npy_files(kad_embedding_dir(baseline_dir, self.ml.name, metric)), collective)
        if not files:
            raise ValueError(f"no {self.ml.name} embeddings cached under {baseline_dir}: embed the baseline directory first")
        x, base_offs = _io_native.load_embedding_files(files, self.audio_load_worker)
        if x.dtype != np.float16:
            raise ValueError(f"{metric} needs fp16 embedding caches; {baseline_dir} holds {x.dtype}")
        kad_embedding_dir(eval_dir, self.ml.name, metric)
        m, d = x.shape

        def _report(f, msg):
            if writer:
                log.error(f"An error occurred calculating individual {metric} using model {self.ml.name} on file {f}")
                log.error(msg)

        # fp16 caches read natively in one pass (libfadtk_io.so) into one pinned buffer after the baseline rows
        all_files = _on_rank0(lambda: sorted(Path(eval_dir).glob("*.*")), collective)
        caches = [get_cache_embedding_path(self.ml.name, f) for f in all_files]
        n_rows, cols, ndim, dt, st = _io_native.npy_probe(caches, self.audio_load_worker)
        keep = []
        for i, f in enumerate(all_files):
            if st[i] != _io_native.OK:
                _report(f, f"cannot read the embedding cache {caches[i]} (status {int(st[i])})")
            elif dt[i] != 2 or ndim[i] != 2:
                _report(f, f"{metric} needs an fp16 [rows, d] embedding cache; {caches[i]} is not one")
            elif cols[i] != d:
                _report(f, f"embedding widths differ (baseline {d}, {caches[i]} {int(cols[i])})")
            elif n_rows[i] < min_rows:
                _report(f, f"{metric} needs {need}, {caches[i]} has {int(n_rows[i])}"
                           " (This probably means that your audio is too short)")
            else:
                keep.append(i)
        if not keep:
            return x, None, None, [], files, base_offs
        rows = n_rows[keep]
        offs = np.zeros(len(keep) + 1, dtype=np.int64)
        offs[1:] = np.cumsum(rows)
        host = torch.empty((m + int(offs[-1]), d), dtype=torch.float16, pin_memory=torch.cuda.is_available())
        host[:m] = torch.from_numpy(x)
        _, st = _io_native.npy_read_f16([caches[i] for i in keep], rows, d, host[m:].numpy(), offs,
                                        self.audio_load_worker)
        for k in np.nonzero(st != _io_native.OK)[0]:     # vanished / rewritten since the probe: dropped by the caller
            _report(all_files[keep[k]], f"cannot read {caches[keep[k]]} (status {int(st[k])})")
            host[m + offs[k]:m + offs[k + 1]] = 0.0
        return (x, host, offs, [all_files[i] if st[k] == _io_native.OK else None for k, i in enumerate(keep)], files,
                base_offs)

    def score_inf(self, baseline: PathLike, eval_files: list[Path], steps: int = 25, min_n=500, raw: bool = False):
        """FAD for growing sample counts and the FAD-inf extrapolation (fad.py:304-351).

        The bootstrap indices come from the host's global numpy RNG exactly as in the reference
        (``np.random.choice(N, n, replace=True)``, fad.py:333) so a seeded run reproduces it; the
        gather, statistics and Frechet chain of every step run on the GPU.
        """
        log.info(f"Calculating FAD-inf for {self.ml.name}...")
        mu_base, cov_base = self.load_stats(baseline)
        if all([Path(f).suffix == '.npy' for f in eval_files]):
            from . import _io_native
            embeds, _ = _io_native.load_embedding_files(eval_files, self.audio_load_worker)
        else:
            embeds = self._load_embeddings(eval_files, concat=True)

        max_n = len(embeds)
        ns = [int(n) for n in np.linspace(min_n, max_n, steps)]

        from . import _native
        eng = _native.engine()
        fp16_rows = embeds.dtype == np.float16
        if fp16_rows:      # baseline sqrt computed once, every bootstrap step stays on the device
            base = _native.Baseline(eng, mu_base, cov_base)
            base.mu_host = np.asarray(mu_base, dtype=np.float64)
            emb_dev = torch.from_numpy(np.ascontiguousarray(embeds)).to(eng.torch_device)

        # Multi-GPU: the bootstrap sizes are independent.  Rank 0 owns the host RNG stream (so a seeded run
        # reproduces the reference's np.random.choice sequence, fad.py:333) and broadcasts every index
        # array; step i is evaluated by rank i mod world and the points are gathered.
        from . import dist
        world, me = dist.world_size(), dist.rank()
        results = []
        for step, n in enumerate(ns):
            indices = np.random.choice(embeds.shape[0], size=n, replace=True) if me == 0 else np.empty(n, dtype=np.int64)
            indices = dist.broadcast_int64(indices)
            if step % world != me:
                continue
            if fp16_rows:
                fad_score = _device_score(base, emb_dev, eng, torch.from_numpy(indices).to(eng.torch_device))
            else:
                mu_eval, cov_eval = calc_embd_statistics(embeds[indices])
                fad_score = calc_frechet_distance(mu_base, cov_base, mu_eval, cov_eval)
            results.append([n, fad_score])
        if world > 1:
            results = sorted((p for part in dist.allgather_objects(results) for p in part), key=lambda p: p[0])

        ys = np.array(results)
        xs = 1 / np.array(ns)
        slope, intercept = np.polyfit(xs, ys[:, 1], 1)
        r2 = 1 - np.sum((ys[:, 1] - (slope * xs + intercept)) ** 2) / np.sum((ys[:, 1] - np.mean(ys[:, 1])) ** 2)
        return FADInfResults(score=intercept, slope=slope, r2=r2, points=results)

    def score_individual(self, baseline: PathLike, eval_dir: PathLike, csv_name: Union[Path, str]) -> Path:
        """FAD of every file in eval_dir against the baseline, written to a csv sorted by |score|
        (fad.py:353-395).  Files whose statistics fail are logged and dropped, as in the reference."""
        csv = Path(csv_name)
        if isinstance(csv_name, str):
            csv = Path('data') / f'fad-individual' / self.ml.name / csv_name
        if csv.exists():
            log.info(f"CSV file {csv} already exists, exiting...")
            return csv

        mu, cov = self.load_stats(baseline)
        from . import _native
        eng = _native.engine()
        base = _native.Baseline(eng, mu, cov)          # C1^(1/2) once, reused for every song
        base.mu_host = np.asarray(mu, dtype=np.float64)

        def _report(f, e):
            log.error(f"An error occurred calculating individual FAD using model {self.ml.name} on file {f}")
            log.error(e)

        def _find_z_helper(f, embd):
            try:                                           # non-fp16 caches: the generic per-item path
                mu_eval, cov_eval = calc_embd_statistics(embd)
                return calc_frechet_distance(mu, cov, mu_eval, cov_eval)
            except Exception as e:
                traceback.print_exc()
                _report(f, e)

        from . import dist
        all_files = sorted(Path(eval_dir).glob("*.*"))
        _files = list(dist.shard(all_files))               # multi-GPU: songs are independent, shard them
        scores: list = [None] * len(_files)
        # fp16 caches (what the reference writes, model_loader.py:47-48): one ragged batch, every song's
        # statistics and Frechet chain in lock-step on the device (fad_frechet_batched)
        # read natively in one pass (libfadtk_io.so) into one pinned buffer; anything else goes file by file
        from . import _io_native
        d = len(mu)
        caches = [get_cache_embedding_path(self.ml.name, f) for f in _files]
        n_rows, cols, ndim, dt, st = _io_native.npy_probe(caches, self.audio_load_worker)
        fast = (st == _io_native.OK) & (dt == 2) & (ndim == 2) & (cols == d)
        batch_idx = [int(i) for i in np.nonzero(fast)[0]]
        for i in np.nonzero(~fast)[0]:
            f = _files[i]
            try:
                embd = self.read_embedding_file(f)
            except Exception as e:
                traceback.print_exc()
                _report(f, e)
                continue
            scores[i] = _find_z_helper(f, embd)
        if batch_idx:
            rows = n_rows[batch_idx]
            offs = np.zeros(len(batch_idx) + 1, dtype=np.int64)
            offs[1:] = np.cumsum(rows)
            host = torch.empty((max(1, int(offs[-1])), d), dtype=torch.float16, pin_memory=torch.cuda.is_available())
            _, st = _io_native.npy_read_f16([caches[i] for i in batch_idx], rows, d, host.numpy(), offs, self.audio_load_worker)
            for k in np.nonzero(st != _io_native.OK)[0]:       # vanished / rewritten since the probe: an empty item, reported below
                _report(_files[batch_idx[k]], OSError(f"cannot read {caches[batch_idx[k]]} (status {int(st[k])})"))
                host[offs[k]:offs[k + 1]] = float("nan")
            flat = host[:int(offs[-1])].to(eng.torch_device, non_blocking=True)
            out = base.frechet_batched(flat, torch.from_numpy(offs).to(eng.torch_device)).cpu().numpy()
            for k, i in enumerate(batch_idx):
                n_k, fad_k = int(out[k, 7]), float(out[k, 0])
                if st[k] != _io_native.OK:
                    continue
                if n_k < 2:
                    _report(_files[i], AssertionError(
                        f"FAD requires at least two embedding window frames, you have {(int(rows[k]), d)}."
                        " (This probably means that your audio is too short)"))
                elif not np.isfinite(fad_k):
                    _report(_files[i], ValueError("non-finite covariance statistics (NaN/Inf input)"))
                else:
                    scores[i] = fad_k

        pairs = [p for p in zip(_files, scores) if p[1] is not None]
        if dist.is_distributed():
            pairs = [p for part in dist.allgather_objects(pairs) for p in part]
            if dist.rank() != 0:
                return csv                                 # rank 0 writes the file
        pairs = sorted(pairs, key=lambda x: np.abs(x[1]))
        csv.parent.mkdir(parents=True, exist_ok=True)
        csv.write_text("\n".join([",".join([str(x).replace(',', '_') for x in row]) for row in pairs]))
        return csv
