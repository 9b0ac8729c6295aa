"""Embedding-model plugin surface (mirror of fadtk/model_loader.py:21-86, :89-108, :676-701).

``ModelLoader`` keeps the reference's contract verbatim - constructor arguments and attributes,
``load_model`` / ``_get_embedding`` / ``get_embedding`` / ``load_wav`` / ``enforce_min_len``,
picklable before ``load_model`` - so third-party plugins written against fadtk (README plugin
template, README.md:113-138) keep working.  ``VGGishModel`` is the H100-native implementation:
its forward is hand-written sm_90a CUDA behind the C ABI (include/fadtk_b200.h), not torchvggish.

One addition: ``embed_pcm_batch(list_of_int16_arrays)`` lets the batch driver push many clips
through the GPU in one launch sequence; the default implementation falls back to the per-clip
``get_embedding`` so plain plugins need not implement it.
"""
from __future__ import annotations

import logging
from abc import ABC, abstractmethod
from pathlib import Path

import numpy as np
import torch

from . import synth, weights

log = logging.getLogger(__name__)


class ModelLoader(ABC):
    """Load a model and get embeddings from it (fadtk/model_loader.py:21-86)."""

    def __init__(self, name: str, num_features: int, sr: int, min_len: int = -1):
        self.model = None
        self.sr = sr
        self.num_features = num_features
        self.name = name
        self.min_len = min_len
        self.device = torch.device('cuda') if torch.cuda.is_available() else torch.device('cpu')

    def get_embedding(self, audio: np.ndarray):
        embd = self._get_embedding(audio)
        if isinstance(embd, torch.Tensor):
            embd = embd.detach().cpu().numpy()
        # float32 embeddings are stored as float16, like the reference (model_loader.py:47-48)
        if embd.dtype == np.float32:
            embd = embd.astype(np.float16)
        return embd

    @abstractmethod
    def load_model(self):
        pass

    @abstractmethod
    def _get_embedding(self, audio: np.ndarray):
        """(n_frames, n_features) embedding of one clip."""

    def load_wav(self, wav_file: Path):
        pcm, sr = synth.read_wav(wav_file)              # PCM16 RIFF written by load_audio
        if pcm.ndim > 1:
            pcm = pcm[:, 0]
        wav_data = pcm / 32768.0                        # [-1.0, +1.0), float64 (model_loader.py:64-65)
        return self.enforce_min_len(wav_data)

    def enforce_min_len(self, audio: np.ndarray) -> np.ndarray:
        if self.min_len < 0:
            return audio
        need = self.min_len * self.sr
        if audio.shape[0] < need:
            log.warning(
                f"Audio is too short for {self.name}.\n"
                f"The model requires a minimum length of {self.min_len}s, audio is {audio.shape[0] / self.sr:.2f}s.\n"
                f"Padding with zeros.")
            audio = np.pad(audio, (0, int(np.ceil(need - audio.shape[0]))))
        return audio

    # ---- batched extension (not in the reference) -------------------------------------
    def embed_pcm_batch(self, clips):
        """list of int16 mono arrays at ``self.sr`` -> list of fp16 [n_i, d] arrays."""
        out = []
        for pcm in clips:
            wav = self.enforce_min_len(np.asarray(pcm).astype(np.int16) / 32768.0)
            out.append(self.get_embedding(wav))
        return out

    def embed_pcm_batch_flat(self, clips):
        """list of int16 mono arrays -> (fp16 [sum n_i, d] host array, rows per clip).  What the batch driver
        writes to the ``.npy`` caches; the native embedders produce it with ONE device -> host copy."""
        embs = self.embed_pcm_batch(clips)
        rows = [int(e.shape[0]) for e in embs]
        return (np.concatenate(embs) if len(embs) > 1 else np.ascontiguousarray(embs[0])), rows


class _DeviceBatch:
    """Shared by the native embedders: ``_embed_device(clips)`` returns one cuda fp16 tensor per clip.

    Weight ownership.  All loaders of a process share one native engine per GPU, and the engine holds ONE set of
    weights per model family (``_SLOT``): loading hubert-base replaces w2v2-base, HTSAT-base replaces HTSAT-tiny.
    The reference keeps every loader's model alive independently (two live FrechetAudioDistance objects, a
    dirs-outer / models-inner loop), so a loader records a token on the engine when it loads and checks it before
    every forward; if another loader took the slot in between, it reloads its own weights instead of silently
    embedding with the other model's."""

    _SLOT = None

    def _owner_token(self):
        return (type(self).__name__, getattr(self, "family", None), getattr(self, "size", None),
                getattr(self, "variant", None), getattr(self, "type", None),
                str(getattr(self, "checkpoint", None)), getattr(self, "seed", 0))

    def _claim(self):
        self._engine.owners[self._SLOT] = self._owner_token()

    def owns_engine(self) -> bool:
        eng = getattr(self, "_engine", None)
        return eng is not None and eng.owners.get(self._SLOT) == self._owner_token()

    def _ensure_loaded(self):
        if getattr(self, "_engine", None) is None:
            raise RuntimeError("load_model() has not been called")
        if not self.owns_engine():
            log.info(f"{self.name}: the engine's {self._SLOT} weights were replaced by another loader - reloading")
            self.load_model()

    def embed_pcm_batch(self, clips):
        return [t.cpu().numpy() for t in self._embed_device(clips)]

    def embed_pcm_batch_flat(self, clips):
        parts = self._embed_device(clips)
        rows = [int(p.shape[0]) for p in parts]
        flat = torch.cat(parts) if len(parts) > 1 else parts[0].contiguous()
        host = torch.empty(flat.shape, dtype=flat.dtype, pin_memory=True)
        host.copy_(flat)                                     # one D2H for the whole batch (synchronous: pinned destination)
        return host.numpy(), rows


_host_out = {}


def _pinned_like(t: torch.Tensor) -> torch.Tensor:
    """A pinned host tensor of t's shape from TWO alternating grow-only buffers per dtype: cudaHostAlloc of tens of MB
    per batch costs more than the copy it serves.  The returned array stays valid until the second next call with that
    dtype - the batch driver writes batch k to disk while batch k+1 is embedded (fad_batch.cache_embedding_files)."""
    n = t.numel()
    slot = _host_out.setdefault(t.dtype, {"turn": 0, "buf": [None, None]})
    slot["turn"] ^= 1
    buf = slot["buf"][slot["turn"]]
    if buf is None or buf.numel() < n:
        buf = torch.empty(max(n, 1), dtype=t.dtype, pin_memory=True)
        slot["buf"][slot["turn"]] = buf
    return buf[:n].view(t.shape)


def _data_address(a: np.ndarray) -> int:
    return a.__array_interface__["data"][0]                  # a.ctypes.data builds a ctypes object per call: 10x slower


def flat_pcm(clips) -> np.ndarray:
    """The int16 clips back to back as ONE array.  When they are consecutive views of one C-contiguous buffer - the
    batch driver's pinned staging buffer (fad_batch._read_native), the rows of a [clips, samples] array, slices of a
    long recording - the result is a view of that buffer: no host copy, and the H2D transfer that follows is a
    straight DMA when the buffer is pinned.  Anything else is concatenated."""
    if len(clips) == 1:
        return np.ascontiguousarray(clips[0])
    first = clips[0]
    owner = first
    while isinstance(owner.base, np.ndarray):
        owner = owner.base
    if owner.dtype == np.int16 and owner.flags.c_contiguous and first.dtype == np.int16:
        flat_owner = owner.reshape(-1)                         # a view: any C-contiguous shape is one run of samples
        ptr = _data_address(first)
        start = (ptr - _data_address(flat_owner)) // 2
        total = 0
        for c in clips:
            if c.dtype != np.int16 or c.ndim != 1 or not c.flags.c_contiguous or _data_address(c) != ptr + 2 * total:
                break
            total += c.shape[0]
        else:
            if 0 <= start and start + total <= flat_owner.shape[0]:
                return flat_owner[start:start + total]
    return np.concatenate(clips)


def _as_pcm16(audio: np.ndarray) -> np.ndarray:
    """The reference feeds ``int16 / 32768.0`` (load_wav); recover the integers exactly."""
    audio = np.asarray(audio)
    if audio.dtype == np.int16:
        return audio
    scaled = audio * 32768.0
    pcm = np.rint(scaled)
    if not np.array_equal(pcm, scaled) or pcm.min(initial=0) < -32768 or pcm.max(initial=0) > 32767:
        # arbitrary float waveforms: quantise like torchaudio.save(..., PCM_S16) would (fad.py:160)
        pcm = np.clip(np.rint(np.clip(audio, -1.0, 1.0) * 32768.0), -32768, 32767)
    return pcm.astype(np.int16)


class VGGishModel(_DeviceBatch, ModelLoader):
    """S. Hershey et al., "CNN Architectures for Large-Scale Audio Classification", ICASSP 2017.

    Same registry name, dimensionality, sample rate and minimum length as the reference
    (fadtk/model_loader.py:93-97).  PCA post-processing and the final ReLU are disabled as the
    reference does (:100-103); enabling either is not supported by the native path.
    """

    _SLOT = "vggish"

    def __init__(self, use_pca=False, use_activation=False, checkpoint=None, seed: int = 0):
        super().__init__("vggish", 128, 16000, min_len=1)
        if use_pca or use_activation:
            raise NotImplementedError("the GPU path implements the reference's default (no PCA, no final ReLU)")
        self.use_pca = use_pca
        self.use_activation = use_activation
        self.checkpoint = checkpoint
        self.seed = seed
        self._engine = None

    def __getstate__(self):                             # stay picklable after load_model()
        st = dict(self.__dict__)
        st["_engine"] = None
        st["model"] = None
        return st

    def load_model(self):
        from . import _native
        self._engine = _native.engine()
        state = weights.load_vggish_state(self.checkpoint, self.seed)
        self._engine.vggish_load(weights.pack_vggish(state))
        self.model = self._engine
        self.device = self._engine.torch_device
        self._claim()

    def _get_embedding(self, audio: np.ndarray):
        return self._embed_flat([_as_pcm16(audio)])[0]

    def _embed_device(self, clips):
        padded = []
        need = self.min_len * self.sr
        for c in clips:
            c = np.asarray(c, dtype=np.int16)
            if c.shape[0] < need:
                c = np.pad(c, (0, need - c.shape[0]))
            padded.append(c)
        return self._embed_flat(padded)

    def _embed_flat(self, clips):
        """list of int16 arrays -> list of fp16 cuda tensors [n_i, 128]."""
        emb, rows = self._embed_flat_device(clips)
        return list(torch.split(emb, [int(r) for r in rows]))

    # sub-batch of one pipelined forward: audio seconds (the copy of sub-batch k+1 overlaps the forward of sub-batch k)
    _PIPE_SECONDS = 2560.0

    def _embed_flat_device(self, clips):
        """list of int16 arrays -> (fp16 cuda tensor [sum n_i, 128], rows per clip).  Large batches are cut into
        sub-batches whose host -> device copies run on a second stream into two staging buffers, so the PCIe transfer
        of sub-batch k+1 hides behind the forward of sub-batch k (a 1000-clip batch is 320 MB of PCM: ~6 ms of PCIe
        against ~30 ms of forward)."""
        self._ensure_loaded()
        eng = self._engine
        dev = eng.torch_device
        lens = np.fromiter((len(c) for c in clips), dtype=np.int64, count=len(clips))
        offsets = np.zeros(len(clips) + 1, dtype=np.int64)
        np.cumsum(lens, out=offsets[1:])
        ex_start, rows = eng.vggish_plan(offsets)
        total_rows = int(rows.sum())
        emb = torch.empty((total_rows, 128), dtype=torch.float16, device=dev)
        limit = int(self._PIPE_SECONDS * self.sr)
        if offsets[-1] <= limit:                                 # small batch: one copy, one forward
            pcm = torch.from_numpy(flat_pcm(clips)).pin_memory().to(dev, non_blocking=True)
            eng.vggish_forward(pcm, torch.from_numpy(ex_start).to(dev), emb)
            return emb, rows
        cuts = [0]                                               # clip indices where sub-batches start
        for i in range(len(clips)):
            if offsets[i + 1] - offsets[cuts[-1]] > limit and i > cuts[-1]:
                cuts.append(i)
        cuts.append(len(clips))
        if getattr(self, "_pipe", None) is None or self._pipe["dev"] != dev:
            self._pipe = {"dev": dev, "copy": torch.cuda.Stream(device=dev), "stage": [None, None],
                          "ready": [torch.cuda.Event(), torch.cuda.Event()], "free": [torch.cuda.Event(), torch.cuda.Event()]}
        pipe = self._pipe
        main = torch.cuda.current_stream(dev)
        row_off = np.zeros(len(clips) + 1, dtype=np.int64)
        np.cumsum(rows, out=row_off[1:])
        ex_row = 0
        for j in range(len(cuts) - 1):
            a, b_ = cuts[j], cuts[j + 1]
            slot = j & 1
            n_samples = int(offsets[b_] - offsets[a])
            n_ex = int(row_off[b_] - row_off[a])
            src = torch.from_numpy(flat_pcm(clips[a:b_]))
            ex_j = torch.from_numpy(ex_start[ex_row:ex_row + n_ex] - offsets[a])
            if pipe["stage"][slot] is None or pipe["stage"][slot].numel() < n_samples:
                pipe["stage"][slot] = torch.empty(max(n_samples, limit + 64 * self.sr), dtype=torch.int16, device=dev)
            with torch.cuda.stream(pipe["copy"]):
                if j >= 2:
                    pipe["copy"].wait_event(pipe["free"][slot])
                stage = pipe["stage"][slot][:n_samples]
                stage.copy_(src, non_blocking=True)
                ex_dev = ex_j.to(dev, non_blocking=True)
                pipe["ready"][slot].record(pipe["copy"])
            main.wait_event(pipe["ready"][slot])
            stage.record_stream(main)
            ex_dev.record_stream(main)
            eng.vggish_forward(stage, ex_dev, emb[ex_row:ex_row + n_ex])
            pipe["free"][slot].record(main)
            ex_row += n_ex
        return emb, rows

    def embed_pcm_batch_flat(self, clips):
        """(fp16 [sum n_i, 128] host array, rows per clip): the pipelined device forward, then ONE device -> host copy."""
        need = self.min_len * self.sr
        if any(len(c) < need for c in clips):                    # short clips are zero-padded to min_len (model_loader.py:72-86)
            clips = [np.pad(np.asarray(c, dtype=np.int16), (0, need - len(c))) if len(c) < need else c for c in clips]
        emb, rows = self._embed_flat_device(clips)
        host = _pinned_like(emb)
        host.copy_(emb)                                          # synchronous: pinned destination
        return host.numpy(), [int(r) for r in rows]


class CLAPLaionModel(_DeviceBatch, ModelLoader):
    """CLAP from https://github.com/LAION-AI/CLAP, audio branch, H100-native.

    Same registry names, dimensionality and sample rate as the reference (model_loader.py:296-297):
    ``type='audio'`` = HTSAT-tiny (630k-audioset-best), ``type='music'`` = HTSAT-base
    (music_audioset_epoch_15_esc_90.14, model_loader.py:303,385) - same kernels, wider instantiations.
    One engine holds one CLAP variant at a time (as one reference process holds one model).
    The reference's per-window loop at batch one (model_loader.py:402-407) becomes one batched
    launch sequence over all 10-s windows of all clips.
    """

    _SLOT = "clap"

    def __init__(self, type: str = 'audio', checkpoint=None, seed: int = 0, max_chunks: int = 128):
        super().__init__(f"clap-laion-{type}", 512, 48000)
        self.type = type
        self.checkpoint = checkpoint
        self.seed = seed
        self.max_chunks = max_chunks                      # 10-s windows per launch sequence (~9 MB of workspace each)
        self._engine = None

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        st["model"] = None
        return st

    def load_model(self):
        if self.type not in ('audio', 'music'):
            raise ValueError(f"unknown CLAP-LAION type {self.type!r}")
        from . import _native, weights_clap
        self._engine = _native.engine()
        state = weights_clap.load_clap_state(self.checkpoint, self.seed, "tiny" if self.type == 'audio' else "base")
        self._engine.clap_load(weights_clap.pack_clap(state), max_chunks=self.max_chunks)
        self.model = self._engine
        self.device = self._engine.torch_device
        self._claim()

    def _get_embedding(self, audio: np.ndarray):
        return self._embed_flat([_as_pcm16(np.asarray(audio).reshape(-1))])[0]

    def _embed_device(self, clips):
        return self._embed_flat([np.asarray(c, dtype=np.int16) for c in clips])

    def _embed_flat(self, clips):
        self._ensure_loaded()
        eng = self._engine
        offsets = np.zeros(len(clips) + 1, dtype=np.int64)
        offsets[1:] = np.cumsum([len(c) for c in clips])
        plan = eng.clap_plan_frames(offsets)
        flat = torch.from_numpy(flat_pcm(clips))
        pcm = flat.pin_memory().to(eng.torch_device, non_blocking=True)
        emb = eng.clap_forward(pcm, eng.clap_plan_to_device(plan))
        return list(torch.split(emb, [int(r) for r in plan["rows_per_clip"]]))


class WhisperModel(_DeviceBatch, ModelLoader):
    """Whisper from https://huggingface.co/openai/whisper-<size>, H100-native (model_loader.py:636-672).

    Same registry names (``whisper-tiny|base|small|medium|large``), dimensionality and sample rate.  The
    reference's three transformers calls - feature extractor (clip padded / truncated to 30 s),
    ``WhisperModel`` forward with ``decoder_input_ids = [[sot, sot]]`` and ``last_hidden_state`` - are one
    batched launch sequence (fad_whisper_forward); every clip yields 2 rows of ``d_model`` features.
    """

    _SLOT = "whisper"

    DIMS = {'tiny': 384, 'base': 512, 'small': 768, 'medium': 1024, 'large': 1280}

    def __init__(self, size: str = 'small', checkpoint=None, seed: int = 0, max_clips: int = 16):
        super().__init__(f"whisper-{size}", self.DIMS[size], 16000)
        self.size = size
        self.checkpoint = checkpoint
        self.seed = seed
        self.max_clips = max_clips
        self._engine = None

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        st["model"] = None
        return st

    def load_model(self):
        from . import _native, weights_whisper
        self._engine = _native.engine()
        state, start = weights_whisper.load_whisper_state(self.checkpoint, self.seed, self.size)
        self._engine.whisper_load(weights_whisper.config_of(state), weights_whisper.pack_whisper(state, start), self.max_clips)
        self.model = self._engine
        self.device = self._engine.torch_device
        self._claim()

    def _get_embedding(self, audio: np.ndarray):
        return self._embed_flat([_as_pcm16(np.asarray(audio).reshape(-1))])[0]

    def _embed_device(self, clips):
        return self._embed_flat([np.asarray(c, dtype=np.int16) for c in clips])

    def _embed_flat(self, clips):
        self._ensure_loaded()
        eng = self._engine
        lens = np.array([len(c) for c in clips], dtype=np.int32)
        starts = np.zeros(len(clips), dtype=np.int64)
        starts[1:] = np.cumsum(lens[:-1])
        flat = torch.from_numpy(flat_pcm(clips))
        dev = eng.torch_device
        emb = eng.whisper_forward(flat.pin_memory().to(dev, non_blocking=True), torch.from_numpy(starts).to(dev),
                                  torch.from_numpy(lens).to(dev))
        return list(emb)                                   # [2, d_model] per clip


class EncodecEmbModel(_DeviceBatch, ModelLoader):
    """Encodec (https://github.com/facebookresearch/encodec) continuous encoder output, H100-native
    (model_loader.py:111-176).  ``variant='24k'`` (registry name ``encodec-emb``): the causal SEANet encoder
    of ``EncodecModel.encodec_model_24khz()`` on the whole file -> [T/320, 128].  ``variant='48k'``
    (``encodec-emb-48k``): the non-causal GroupNorm encoder of ``encodec_model_48khz()`` on 1-s segments with
    stride = segment (:139-152), the mono file duplicated to stereo as ``convert_audio`` does.
    """

    _SLOT = "encodec"

    def __init__(self, variant: str = '24k', checkpoint=None, seed: int = 0, max_chunk_samples: int = 16 * 240000):
        super().__init__('encodec-emb' if variant == '24k' else f"encodec-emb-{variant}", 128,
                         sr=24000 if variant == '24k' else 48000)
        self.variant = variant
        self.checkpoint = checkpoint
        self.seed = seed
        self.max_chunk_samples = max_chunk_samples
        self._engine = None

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        st["model"] = None
        return st

    def load_model(self):
        from . import _native, weights_encodec
        self._engine = _native.engine()
        state = weights_encodec.load_encodec_state(self.checkpoint, self.seed, self.variant)
        self._engine.encodec_load(weights_encodec.pack_encodec(state), self.max_chunk_samples, self.variant)
        self.model = self._engine
        self.device = self._engine.torch_device
        self._claim()

    def load_wav(self, wav_file):
        """The reference cuts files longer than 3 minutes (model_loader.py:171-173)."""
        wav = super().load_wav(wav_file)
        return wav[: 3 * 60 * self.sr]

    def _get_embedding(self, audio: np.ndarray):
        return self.embed_equal_length([_as_pcm16(np.asarray(audio).reshape(-1))])[0]

    def _embed_device(self, clips):
        """Clips of equal length share one launch sequence; others are embedded one length group at a time."""
        clips = [np.asarray(c, dtype=np.int16)[: 3 * 60 * self.sr] for c in clips]       # the reference's 3-minute cut (:171-173)
        out = [None] * len(clips)
        groups = {}
        for i, c in enumerate(clips):
            groups.setdefault(len(c), []).append(i)
        for _, idx in groups.items():
            for i, e in zip(idx, self.embed_equal_length([clips[i] for i in idx])):
                out[i] = e
        return out

    def embed_equal_length(self, clips):
        self._ensure_loaded()
        eng = self._engine
        pcm = torch.from_numpy(flat_pcm(clips).reshape(len(clips), -1)).pin_memory().to(eng.torch_device, non_blocking=True)
        if self.variant == '24k':
            return list(eng.encodec_forward(pcm))
        # 48 kHz: every clip is cut into 1-s segments that are encoded independently (model_loader.py:139-152)
        n, T = pcm.shape
        seg = 48000
        full = T // seg
        parts = []
        if full:
            parts.append(eng.encodec_forward(pcm[:, :full * seg].reshape(n * full, seg).contiguous()).reshape(n, full * 150, 128))
        if T - full * seg:
            parts.append(eng.encodec_forward(pcm[:, full * seg:].contiguous()))
        return list(torch.cat(parts, dim=1))


class Wav2VecFamilyModel(_DeviceBatch, ModelLoader):
    """wav2vec 2.0 / HuBERT / MERT hidden-state embedders, H100-native (model_loader.py:254-288, 525-596).

    One class for the three reference loaders whose checkpoints share the "group-norm conv feature encoder +
    post-LN transformer" architecture: ``w2v2-base[-k]`` (facebook/wav2vec2-base-960h), ``hubert-base[-k]``
    (facebook/hubert-base-ls960) and ``MERT-v1-95M[-k]`` (24 kHz).  The reference's processor + model call +
    ``hidden_states[layer]`` is one launch sequence that stops after ``layer`` transformer layers.
    Files longer than ``limit_minutes`` are truncated like the reference does.
    """

    _SLOT = "w2v"

    def __init__(self, family: str, name: str, layer: int, sr: int, checkpoint=None, seed: int = 0, limit_minutes: int = 6,
                 max_clips: int = 8, size: str = 'base'):
        from .weights_w2v import ARCH
        self.size = size
        self.arch = dict(ARCH[(family, size)])
        super().__init__(name, self.arch["d"], sr)
        self.family = family
        self.layer = layer
        self.limit = limit_minutes * 60 * sr
        self.checkpoint = checkpoint
        self.seed = seed
        self.max_clips = max_clips
        self._engine = None

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        st["model"] = None
        st["_packed"] = None
        return st

    def load_model(self):
        from . import _native, weights_w2v
        self._engine = _native.engine()
        env = {"w2v2": "FADTK_W2V2_CKPT", "hubert": "FADTK_HUBERT_CKPT", "mert": "FADTK_MERT_CKPT", "wavlm": "FADTK_WAVLM_CKPT"}[self.family]
        state = weights_w2v.load_w2v_state(self.checkpoint, self.seed, env=env, **self.arch)
        self._packed = (weights_w2v.config_of(state), weights_w2v.pack_w2v(state))
        self._max_len = self.sr * 30                           # workspace: max_clips pieces of up to 30 s
        self._engine.w2v_load(*self._packed, self.max_clips, max_len=self._max_len)
        self.model = self._engine
        self.device = self._engine.torch_device
        self._claim()

    def _get_embedding(self, audio: np.ndarray):
        pcm = _as_pcm16(np.asarray(audio).reshape(-1))
        if pcm.shape[0] > self.limit:
            log.warning(f"Audio is too long ({pcm.shape[0] / self.sr / 60:.2f} minutes > {self.limit / self.sr / 60:.2f} minutes). Truncating.")
            pcm = pcm[:self.limit]
        return self.embed_equal_length([pcm])[0]

    def _embed_device(self, clips):
        return [e[0] for e in self._embed_device_taps(clips, [self.layer])]

    def embed_equal_length(self, clips):
        return list(self.embed_equal_length_taps(clips, [self.layer])[0])

    def embed_pcm_batch_flat(self, clips):
        flat, rows = self.embed_pcm_batch_flat_taps(clips, [self.layer])
        return flat[0], rows

    # ---- several layers of one forward (fad_w2v_forward_taps): the per-layer sweep of fadtk_b200.layers
    def _embed_device_taps(self, clips, taps):
        """list of int16 arrays -> one cuda fp16 tensor [n_taps, n_i, d] per clip (hidden_states[taps[t]]).  Clips of
        equal length share one launch sequence; files over limit_minutes are truncated like the reference does."""
        clips = [np.asarray(c, dtype=np.int16)[:self.limit] for c in clips]
        out = [None] * len(clips)
        groups = {}
        for i, c in enumerate(clips):
            groups.setdefault(len(c), []).append(i)
        for _, idx in groups.items():
            emb = self.embed_equal_length_taps([clips[i] for i in idx], taps)
            for j, i in enumerate(idx):
                out[i] = emb[:, j]
        return out

    def embed_equal_length_taps(self, clips, taps):
        """equal-length int16 clips -> cuda fp16 [n_taps, n_clips, frames, d]"""
        self._ensure_loaded()
        eng = self._engine
        L = len(clips[0])
        if L > self._max_len:                                  # a long file (up to limit_minutes): one clip at a time
            self._max_len = L
            eng.w2v_load(*self._packed, 1, max_len=L)
            self.max_clips = 1
        pcm = torch.from_numpy(flat_pcm(clips).reshape(len(clips), -1)).pin_memory().to(eng.torch_device, non_blocking=True)
        return eng.w2v_forward_taps(pcm, taps)

    def embed_pcm_batch_flat_taps(self, clips, taps):
        """list of int16 arrays -> (fp16 host array [n_taps, sum n_i, d], rows per clip) with ONE device -> host copy:
        what the batch driver writes to the ``.npy`` caches of every tapped layer."""
        parts = self._embed_device_taps(clips, taps)
        rows = [int(p.shape[1]) for p in parts]
        flat = torch.cat(parts, dim=1) if len(parts) > 1 else parts[0].contiguous()
        host = torch.empty(flat.shape, dtype=flat.dtype, pin_memory=True)
        host.copy_(flat)                                     # synchronous: pinned destination
        return host.numpy(), rows


def _layer_name(prefix: str, size: str, layer: int) -> str:
    default = 12 if size in ('base', 'v1-95M') else 24
    return prefix + ("" if layer == default else f"-{layer}")


def W2V2Model(size: str, layer: int, **kw):
    return Wav2VecFamilyModel("w2v2", _layer_name(f"w2v2-{size}", size, layer), layer, 16000, size=size, **kw)


def HuBERTModel(size: str, layer: int, **kw):
    return Wav2VecFamilyModel("hubert", _layer_name(f"hubert-{size}", size, layer), layer, 16000, size=size, **kw)


def WavLMModel(size: str, layer: int, **kw):
    return Wav2VecFamilyModel("wavlm", _layer_name(f"wavlm-{size}", 'base' if size != 'large' else size, layer), layer, 16000, size=size, **kw)


def MERTModel(size: str = 'v1-95M', layer: int = 12, **kw):
    assert size == 'v1-95M', "only MERT-v1-95M is built"
    return Wav2VecFamilyModel("mert", _layer_name("MERT-v1-95M", size, layer), layer, 24000, size=size, **kw)


class UnbuiltModel(ModelLoader):
    """Registry entry whose forward pass has no H100-native implementation yet.

    The names stay valid ``choices`` for the CLI (fadtk/__main__.py:13,17); statistics / Frechet
    scoring from cached ``.npy`` embeddings or ``.npz`` statistics works for every name, only
    ``load_model`` (i.e. embedding raw audio) is unavailable.
    """

    def load_model(self):
        raise NotImplementedError(
            f"{self.name}: no sm_90a forward pass in fadtk_b200 yet (see DESIGN.md, scope table)")

    def _get_embedding(self, audio):
        raise NotImplementedError(self.name)


def _layered(prefix, dim, layers, default_layer):
    return [UnbuiltModel(prefix + ("" if v == default_layer else f"-{v}"), dim, 16000) for v in range(1, layers + 1)]


def get_all_models() -> list[ModelLoader]:
    """Same names, order and (num_features, sr) as fadtk/model_loader.py:676-701."""
    ms = [
        UnbuiltModel("clap-2023", 1024, 44100),
        CLAPLaionModel('audio'), CLAPLaionModel('music'),
        VGGishModel(),
        *[MERTModel('v1-95M', v) for v in range(1, 13)],
        EncodecEmbModel('24k'), EncodecEmbModel('48k'),
        *[W2V2Model('base', v) for v in range(1, 13)], *[W2V2Model('large', v) for v in range(1, 25)],
        *[HuBERTModel('base', v) for v in range(1, 13)], *[HuBERTModel('large', v) for v in range(1, 25)],
        *[WavLMModel('base', v) for v in range(1, 13)], *[WavLMModel('base-plus', v) for v in range(1, 13)],
        *[WavLMModel('large', v) for v in range(1, 25)],
        WhisperModel('tiny'), WhisperModel('small'), WhisperModel('base'), WhisperModel('medium'), WhisperModel('large'),
    ]
    return ms
