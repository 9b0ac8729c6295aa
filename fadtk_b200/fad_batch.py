"""Batch embedding driver (mirror of fadtk/fad_batch.py:15-48).

The reference shards the file list over ``workers`` spawn processes, each loading its own copy
of the model on cuda:0 and looping file by file at batch size one - three filesystem round trips
per clip through Python (SURVEY.md section 8 a4).  Here one process owns one GPU and the host
side is batched too: the PCM16 payloads of a whole chunk of files are read by native threads
straight into ONE pinned buffer (libfadtk_io.so, include/fadtk_b200_io.h), packed into large
batches for the sm_90a forward, and the convert cache and the fp16 ``.npy`` embedding cache
are written back by the same native threads - byte-compatible with what the reference writes.
Files the native reader cannot take as they are (other sample rates, multi-channel, non-PCM16,
other containers) go through FrechetAudioDistance.convert_audio (GPU resampler) on ``workers``
host threads.  Under torchrun (one rank per GPU) the file list is sharded across ranks the way
the reference shards it across processes.
"""
from __future__ import annotations

import os
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import Union

import numpy as np
import torch

from . import _io_native, dist
from .fad import FrechetAudioDistance, log
from .model_loader import ModelLoader

# clips per GPU launch sequence: bounded by audio seconds so ragged sets keep batches even
_BATCH_AUDIO_SECONDS = 4096.0
# files decoded ahead per round of host I/O, bounded both by count and by samples: the pinned staging buffer of a
# chunk never exceeds 512 MB unless a single file does (1600 x 10 s x 16 kHz; 5-minute songs at 48 kHz: 18 per chunk)
_CHUNK_FILES = 2048
_CHUNK_SAMPLES = 256 * 1024 * 1024


def _batches(files, lengths_s, limit_s):
    cur, tot = [], 0.0
    for f, s in zip(files, lengths_s):
        if cur and tot + s > limit_s:
            yield cur
            cur, tot = [], 0.0
        cur.append(f)
        tot += s
    if cur:
        yield cur


def _derived_paths(files, model: str, sr: int):
    """(embedding cache path, convert cache path) of every file as plain strings - the same names as
    utils.get_cache_embedding_path / FrechetAudioDistance._converted_path, without a dozen pathlib objects per file."""
    emb, conv = [], []
    for f in files:
        parent, name = os.path.split(os.fspath(f))
        stem = os.path.splitext(name)[0]
        emb.append(os.path.join(parent, "embeddings", model, stem + ".npy"))
        conv.append(os.path.join(parent, "convert", str(sr), stem + ".wav"))
    return emb, conv


def _names_in(directory) -> set:
    try:
        return set(os.listdir(directory))
    except OSError:
        return set()


_staging = [None, None]
# samples of one pinned staging slot, allocated ONCE at first use (cudaHostAlloc runs at a few GB/s: growing the buffer call
# by call put two 0.1 s allocations inside every directory pass); a chunk never holds more than _CHUNK_SAMPLES samples
# unless a single file does.  $FADTK_STAGING_MB bounds the two slots (default 2 x 512 MB of pinned host memory).
_STAGING_SAMPLES = min(_CHUNK_SAMPLES, max(1, int(os.environ.get("FADTK_STAGING_MB", "512"))) * 512 * 1024)


def _host_buffer(n_samples: int, slot: int) -> np.ndarray:
    """int16 staging buffer of one of the two chunk slots (chunk k+1 is read while chunk k is embedded; a slot is
    reused only after its chunk has been consumed); pinned when a GPU is present so the H2D copy is a straight DMA."""
    if _staging[slot] is None or _staging[slot].numel() < n_samples:
        _staging[slot] = torch.empty(max(1, n_samples, _STAGING_SAMPLES), dtype=torch.int16, pin_memory=torch.cuda.is_available())
    return _staging[slot].numpy()[:max(1, n_samples)]


def _plan_chunks(files, ml: ModelLoader, workers: int):
    """Consecutive runs of ``files`` holding at most _CHUNK_FILES files and (as far as the WAV headers tell)
    _CHUNK_SAMPLES samples; other containers are budgeted as one minute at the model rate."""
    srcs = [os.fspath(f) for f in files]
    _, _, frames, st = _io_native.wav_probe(srcs, workers)
    frames = np.where(st == _io_native.OK, frames, 60 * ml.sr)
    chunks, cur, tot = [], [], 0
    for f, n in zip(files, frames):
        if cur and (len(cur) >= _CHUNK_FILES or tot + int(n) > _CHUNK_SAMPLES):
            chunks.append(cur)
            cur, tot = [], 0
        cur.append(f)
        tot += int(n)
    if cur:
        chunks.append(cur)
    return chunks


def _read_native(part, ml: ModelLoader, workers: int, slot: int):
    """int16 mono clips at ml.sr for the files of ``part`` the native reader can take as they are (None for the
    others), filling the convert cache on the way.  Touches no GPU state: safe to run ahead on another thread."""
    _, conv = _derived_paths(part, ml.name, ml.sr)
    have = {d: _names_in(d) for d in {os.path.dirname(c) for c in conv}}
    cached = np.array([os.path.basename(c) in have[os.path.dirname(c)] for c in conv], dtype=bool)
    # candidates for the native reader: the convert cache when it exists, else a .wav source
    src = [c if ok else os.fspath(f) for f, c, ok in zip(part, conv, cached)]
    is_wav = np.array([s.lower().endswith(".wav") for s in src], dtype=bool)
    sr, ch, fr, st = _io_native.wav_probe(src, workers)
    fast = is_wav & (st == _io_native.OK) & (ch == 1) & (sr == ml.sr)
    clips = [None] * len(part)
    idx = np.nonzero(fast)[0]
    if len(idx):
        buf = _host_buffer(int(fr[idx].sum()), slot)
        off, st2 = _io_native.wav_read([src[i] for i in idx], fr[idx], ch[idx], buf, threads=workers)
        ok = st2 == _io_native.OK
        for j, i in enumerate(idx):
            if ok[j]:
                clips[i] = buf[off[j]:off[j + 1]]
        # The reference always leaves <dir>/convert/<sr>/<stem>.wav behind (fad.py:143-160).  A source that already
        # is mono PCM16 at the model rate IS that file: hard-link it (no second copy of the payload on disk, no
        # write traffic); where links are not possible (other filesystem, no permission) write it out.
        new = [j for j, i in enumerate(idx) if ok[j] and not cached[i]]
        if new:
            for d in {os.path.dirname(conv[idx[j]]) for j in new}:
                os.makedirs(d, exist_ok=True)
            copy = []
            for j in new:
                try:
                    os.link(src[idx[j]], conv[idx[j]])
                except OSError:
                    copy.append(j)
            if copy:
                stw = _io_native.wav_write([conv[idx[j]] for j in copy], buf, off[copy], fr[idx[copy]], ml.sr, workers)
                for j in np.nonzero(stw != _io_native.OK)[0]:
                    # the convert cache is only a memo of the decode step: a file that cannot be written costs a re-read
                    # next time, it must not abort the rest of the directory
                    log.error(f"cannot write {conv[idx[copy[j]]]} (status {int(stw[j])}); continuing without the convert cache entry")
    return clips


def _convert_rest(part, clips, fad: FrechetAudioDistance, pool: ThreadPoolExecutor):
    """Everything the native reader left: decode / mix down / resample per file (convert_audio: decoding and file
    I/O on the pool's threads, the GPU resampler serialised inside)."""
    rest = [i for i in range(len(part)) if clips[i] is None]
    if rest:
        for i, pcm in zip(rest, pool.map(fad.convert_audio, [part[i] for i in rest])):
            clips[i] = pcm
    return clips


def _save_embeddings(ml: ModelLoader, group, flat: np.ndarray, rows, workers: int, name: str = None, keep=None):
    """``<dir>/embeddings/<name>/<stem>.npy`` (default name: the model's) for every file of ``group`` (fp16
    [n_frames, d], as np.save writes it): file i = the next rows[i] rows of ``flat``.  ``keep`` (bool per file):
    only those files are written."""
    paths, _ = _derived_paths(group, ml.name if name is None else name, ml.sr)
    sel = np.arange(len(group)) if keep is None else np.nonzero(np.asarray(keep, dtype=bool))[0]
    for d in {os.path.dirname(paths[i]) for i in sel}:
        os.makedirs(d, exist_ok=True)
    rows = np.asarray(rows, dtype=np.int64)
    off = np.zeros(len(rows) + 1, dtype=np.int64)
    off[1:] = np.cumsum(rows)
    if flat.dtype == np.float16 and flat.ndim == 2:
        st = _io_native.npy_write_f16([paths[i] for i in sel], np.ascontiguousarray(flat), off[sel], rows[sel], workers)
        for k in np.nonzero(st != _io_native.OK)[0]:
            # the reference writes file by file and a failing np.save stops only that worker's loop (fad_batch.py:20-22);
            # here one bad path must not lose the embeddings of the other files of the batch: report it and go on - the
            # file stays without a cache entry and is picked up again by the next run
            log.error(f"cannot write {paths[sel[k]]} (status {int(st[k])}); the other files of the batch were written")
    else:                                                      # a plugin returning another dtype / rank: numpy decides the format
        for i in sel:
            np.save(paths[i], flat[off[i]:off[i + 1]])


def _save_outputs(ml: ModelLoader, names, group, flats, rows, missing, workers: int):
    """every output j of a batch to the caches of names[j], only where that cache is missing (missing[file][j])"""
    for j, (name, flat) in enumerate(zip(names, flats)):
        _save_embeddings(ml, group, flat, rows, workers, name=name, keep=[missing[f][j] for f in group])


def cache_embedding_files(files: Union[list[Path], str, Path], ml: ModelLoader, workers: int = 8, **kwargs):
    """Get embeddings for all audio files in a directory (or list) and cache them as
    ``<dir>/embeddings/<model>/<stem>.npy`` (fp16 [n_frames, d]), skipping files already done.

    Same signature as the reference; ``kwargs`` are forwarded to FrechetAudioDistance.
    """
    def embed(clips):
        flat, rows = ml.embed_pcm_batch_flat(clips)
        return [flat], rows
    _cache_outputs(files, ml, [ml.name], embed, workers, **kwargs)


def cache_tapped_embedding_files(files: Union[list[Path], str, Path], ml: ModelLoader, taps, names, workers: int = 8,
                                 **kwargs):
    """Several layers of one forward per file: hidden_states[taps[t]] cached as ``<dir>/embeddings/<names[t]>/<stem>.npy``,
    byte-identical to what cache_embedding_files writes with the loader of names[t].  ``ml`` is a loader with a tapped
    path (model_loader.Wav2VecFamilyModel.embed_pcm_batch_flat_taps).  A file is embedded when any of its caches is
    missing, and only the missing ones are written: an existing cache keeps its bytes and its mtime, which the
    statistics caches' fingerprints depend on."""
    taps = [int(t) for t in taps]
    names = list(names)
    if len(taps) != len(names) or not taps:
        raise ValueError("one registry name per tap")

    def embed(clips):
        flat, rows = ml.embed_pcm_batch_flat_taps(clips, taps)
        return list(flat), rows
    _cache_outputs(files, ml, names, embed, workers, **kwargs)


def _cache_outputs(files, ml: ModelLoader, names, embed, workers: int, **kwargs):
    """The directory flow: embed(clips) -> (one flat array per output, rows per clip) for every file that lacks the
    cache of any of ``names``; output j goes to the caches of names[j] that are missing."""
    if isinstance(files, (str, Path)):
        files = list(Path(files).glob('*.*'))

    files = [Path(f) for f in files]
    missing = None
    if dist.rank() == 0:
        miss = np.zeros((len(files), len(names)), dtype=bool)
        for j, name in enumerate(names):
            emb_paths, _ = _derived_paths(files, name, ml.sr)
            done = {d: _names_in(d) for d in {os.path.dirname(p) for p in emb_paths}}
            miss[:, j] = [os.path.basename(p) not in done[os.path.dirname(p)] for p in emb_paths]
        missing = {f: tuple(bool(v) for v in m) for f, m in zip(files, miss) if m.any()}
        files = sorted(f for f, m in zip(files, miss) if m.any())
    # ONE listing decides what is left to do: rank 0 filters the already-embedded files and every rank shards that
    # same list (a rank that lists the directory after another has started writing would see a different set)
    files, missing = dist.broadcast_object((files, missing))
    if len(files) == 0:
        log.info("All files already have embeddings, skipping.")
        return

    files = list(dist.shard(files))
    log.info(f"[Frechet Audio Distance] Loading {len(files)} audio files...")
    if len(files) == 0:                                        # fewer new files than ranks: nothing for this one
        dist.barrier()
        return

    kwargs.setdefault("audio_load_worker", workers)
    # a model loaded by an earlier call (baseline dir, then eval dir) is reused - unless another loader has taken the
    # engine's weight slot of this family in between (w2v2-base, then hubert-base, then w2v2-base again)
    kwargs.setdefault("load_model", ml.model is None or not getattr(ml, "owns_engine", lambda: True)())
    fad = FrechetAudioDistance(ml, **kwargs)
    workers = max(1, int(workers))

    chunks = _plan_chunks(files, ml, workers)
    with ThreadPoolExecutor(workers) as pool, ThreadPoolExecutor(1) as reader:
        writer = None                                          # embedding writes of batch k overlap the forward of batch k+1
        ahead = reader.submit(_read_native, chunks[0], ml, workers, 0)
        for k, part in enumerate(chunks):
            clips = ahead.result()
            if k + 1 < len(chunks):                            # chunk k+1 is read while chunk k is embedded
                ahead = reader.submit(_read_native, chunks[k + 1], ml, workers, (k + 1) & 1)
            clips = _convert_rest(part, clips, fad, pool)
            secs = [len(c) / ml.sr for c in clips]
            by_file = dict(zip(part, clips))
            # n outputs per file: the batch is cut n times shorter, so that the host copy of its outputs stays bounded
            for group in _batches(part, secs, _BATCH_AUDIO_SECONDS / len(names)):
                flats, rows = embed([by_file[f] for f in group])
                if writer is not None:
                    writer.result()
                writer = pool.submit(_save_outputs, ml, names, group, flats, rows, missing, workers)
        if writer is not None:
            writer.result()
    dist.barrier()
