"""CPU restatement of the VGGish embedder the reference calls.

TEST INFRASTRUCTURE (see oracle/__init__.py).  PARITY UNPINNED for the network:
the reference obtains the model with ``torch.hub.load('harritaylor/torchvggish',
'vggish')`` (fadtk/model_loader.py:99) - an un-vendored, un-pinned hub dependency
whose source and weights are absent from the reference checkout and from this image.
What follows restates the *published* algorithm (Hershey et al., ICASSP 2017; the
AudioSet ``vggish_input`` / ``mel_features`` / ``vggish_params`` definitions that
torchvggish reuses), anchored on the reference's call site and its two
modifications:

* PCA/quantise post-processing disabled          (model_loader.py:100-101)
* the ReLU after the last Linear is removed       (model_loader.py:102-103)
* input is float64 mono in [-1, 1) at 16 kHz      (model_loader.py:64-65, :107-108)

Front-end arithmetic is float64 numpy (as upstream), the network is float32 torch
on CPU (as upstream when no GPU is present).  Weights use torchvggish's state-dict
key names, so a real ``vggish-10086976.pth`` can be dropped in unchanged.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

SAMPLE_RATE = 16000
WINDOW = 400            # 25 ms
HOP = 160               # 10 ms
FFT = 512               # next power of two >= WINDOW
N_BINS = FFT // 2 + 1   # 257
N_MEL = 64
MEL_LO_HZ = 125.0
MEL_HI_HZ = 7500.0
LOG_OFFSET = 0.01
EXAMPLE_FRAMES = 96     # 0.96 s, non-overlapping
CONV_KEYS = ("features.0", "features.3", "features.6", "features.8",
             "features.11", "features.13")
POOL_AFTER = (True, True, False, True, False, True)
FC_KEYS = ("embeddings.0", "embeddings.2", "embeddings.4")


def hz_to_mel(f):
    """HTK mel scale used by AudioSet's mel_features."""
    return 1127.0 * np.log(1.0 + np.asarray(f, dtype=np.float64) / 700.0)


def mel_matrix() -> np.ndarray:
    """[257, 64] triangular mel weights; the DC row is zeroed."""
    bins_mel = hz_to_mel(np.linspace(0.0, SAMPLE_RATE / 2.0, N_BINS))
    edges = np.linspace(hz_to_mel(MEL_LO_HZ), hz_to_mel(MEL_HI_HZ), N_MEL + 2)
    w = np.empty((N_BINS, N_MEL))
    for b in range(N_MEL):
        lo, mid, hi = edges[b:b + 3]
        rise = (bins_mel - lo) / (mid - lo)
        fall = (hi - bins_mel) / (hi - mid)
        w[:, b] = np.maximum(0.0, np.minimum(rise, fall))
    w[0, :] = 0.0
    return w


def periodic_hann() -> np.ndarray:
    return 0.5 - 0.5 * np.cos(2.0 * np.pi / WINDOW * np.arange(WINDOW))


def num_stft_frames(n_samples: int) -> int:
    return 1 + (n_samples - WINDOW) // HOP if n_samples >= WINDOW else 0


def num_examples(n_samples: int) -> int:
    t = num_stft_frames(n_samples)
    return 1 + (t - EXAMPLE_FRAMES) // EXAMPLE_FRAMES if t >= EXAMPLE_FRAMES else 0


def log_mel(wave: np.ndarray) -> np.ndarray:
    """float64 mono waveform -> [T, 64] log-mel (float64)."""
    wave = np.asarray(wave, dtype=np.float64)
    t = num_stft_frames(wave.shape[0])
    idx = np.arange(WINDOW)[None, :] + HOP * np.arange(t)[:, None]
    frames = wave[idx] * periodic_hann()
    mag = np.abs(np.fft.rfft(frames, FFT))
    return np.log(mag @ mel_matrix() + LOG_OFFSET)


def examples(wave: np.ndarray) -> np.ndarray:
    """waveform -> [n, 96, 64] float32 network input (tail frames dropped)."""
    lm = log_mel(wave)
    n = num_examples(np.asarray(wave).shape[0])
    return lm[: n * EXAMPLE_FRAMES].reshape(n, EXAMPLE_FRAMES, N_MEL).astype(np.float32)


def network(x: torch.Tensor, weights: dict) -> torch.Tensor:
    """[n, 96, 64] float32 -> [n, 128] float32 on CPU."""
    h = x[:, None, :, :]
    for key, pool in zip(CONV_KEYS, POOL_AFTER):
        h = F.relu(F.conv2d(h, weights[key + ".weight"], weights[key + ".bias"], padding=1))
        if pool:
            h = F.max_pool2d(h, 2, 2)
    # [n, 512, 6, 4] -> (time, mel, channel) order, as upstream's two transposes do
    h = h.permute(0, 2, 3, 1).reshape(h.shape[0], -1)
    for i, key in enumerate(FC_KEYS):
        h = F.linear(h, weights[key + ".weight"], weights[key + ".bias"])
        if i < 2:
            h = F.relu(h)
    return h


@torch.no_grad()
def embed(wave: np.ndarray, weights: dict, chunk: int = 256) -> np.ndarray:
    """What ``ModelLoader.get_embedding`` returns for VGGish: fp16 [n, 128].

    (model_loader.py:40-50: forward, ``.cpu()``, float32 -> float16.)
    """
    x = torch.from_numpy(examples(wave))
    outs = [network(x[i:i + chunk], weights) for i in range(0, x.shape[0], chunk)]
    if not outs:
        return np.zeros((0, 128), np.float16)
    return torch.cat(outs).numpy().astype(np.float16)


def load_wav_semantics(pcm16: np.ndarray, min_len_s: int = 1) -> np.ndarray:
    """``ModelLoader.load_wav`` + ``enforce_min_len`` (model_loader.py:63-86)."""
    wave = pcm16.astype(np.int16) / 32768.0
    need = min_len_s * SAMPLE_RATE
    if min_len_s >= 0 and wave.shape[0] < need:
        wave = np.pad(wave, (0, int(np.ceil(need - wave.shape[0]))))
    return wave
