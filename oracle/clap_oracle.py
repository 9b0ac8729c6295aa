"""CPU restatement of the CLAP-LAION audio embedder the reference calls.

TEST INFRASTRUCTURE (see oracle/__init__.py).  PARITY UNPINNED against the reference's own
dependency: ``laion_clap`` 1.1.7 + ``torchlibrosa`` 0.1.0 (uv.lock:417, :1735) are un-vendored and
not installable offline, and the checkpoint ``630k-audioset-best.pt`` (model_loader.py:301) is
absent.  What IS pinned: the network below is checked in tests/test_clap_oracle.py against an
independent implementation of the same published architecture - transformers'
``ClapAudioModelWithProjection`` (HTSAT-tiny, the port of laion_clap's htsat.py) - with shared
random weights, to fp32 round-off.  The front-end restates torchlibrosa's Spectrogram /
LogmelFilterBank with librosa's Slaney mel filters as summarised in SURVEY.md appendix B.

Reference call sites restated here (fadtk/model_loader.py):
  :389-411  _get_embedding: reshape(1,-1); int16 round trip; 10-s windows at 1-s hop, zero padded;
            ONE forward per window; concat -> [n_windows, 512]
  :413-418  float32_to_int16 = clip(x,-1,1)*32767 -> astype(int16) (truncation);
            int16_to_float32 = x/32767
  :382-387  CLAP_Module(enable_fusion=False, amodel='HTSAT-tiny'); get_audio_embedding_from_data(
            x, use_tensor=True) -> audio_projection(embedding) -> F.normalize(dim=-1)
State-dict keys follow transformers' ClapAudioModelWithProjection (minus the
``audio_model.audio_encoder.`` prefix), so HF-converted LAION checkpoints load directly.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

SR = 48000
N_FFT = 1024
HOP = 480
N_MEL = 64
FMIN, FMAX = 50.0, 14000.0
CHUNK = 10 * SR
FRAMES = CHUNK // HOP + 1          # 1001 (center=True)
SPEC = 256
WINDOW = 8
# HTSAT-tiny (clap-laion-audio) / HTSAT-base (clap-laion-music, model_loader.py:385): (embed dim, depths)
VARIANTS = {"tiny": (96, (2, 2, 6, 2)), "base": (128, (2, 2, 12, 2))}
EMBED, DEPTHS = VARIANTS["tiny"]
HEADS = (4, 8, 16, 32)


def config_of(sd: dict):
    """(embed dim, depths) read off a state dict."""
    embed = sd["patch_embed.proj.weight"].shape[0]
    depths = tuple(len({k.split(".")[3] for k in sd if k.startswith(f"layers.{i}.blocks.")}) for i in range(4))
    return embed, depths
OUT_DIM = 512


# ----------------------------------------------------------------------------- front-end
def _hz_to_mel_slaney(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, mels)


def _mel_to_hz_slaney(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filterbank() -> np.ndarray:
    """librosa.filters.mel(sr=48000, n_fft=1024, n_mels=64, fmin=50, fmax=14000): [64, 513],
    Slaney scale, area ('slaney') normalisation."""
    fft_f = np.linspace(0.0, SR / 2.0, N_FFT // 2 + 1)
    mel_f = _mel_to_hz_slaney(np.linspace(_hz_to_mel_slaney(FMIN), _hz_to_mel_slaney(FMAX), N_MEL + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fft_f[None, :]
    w = np.zeros((N_MEL, N_FFT // 2 + 1))
    for i in range(N_MEL):
        w[i] = np.maximum(0.0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    w *= (2.0 / (mel_f[2:N_MEL + 2] - mel_f[:N_MEL]))[:, None]
    return w


def quantize_like_reference(x: np.ndarray) -> np.ndarray:
    """model_loader.py:393,413-418: float -> int16 by truncation of x*32767 -> float32 / 32767."""
    x = np.clip(x, -1.0, 1.0)
    return ((x * 32767.0).astype(np.int16) / 32767.0).astype(np.float32)


def chunks_of(audio: np.ndarray):
    """model_loader.py:396-404: 10-s windows every second, each zero padded to 480 000 samples."""
    audio = audio.reshape(1, -1)
    out = []
    for i in range(0, audio.shape[1], SR):
        c = audio[:, i:i + CHUNK]
        if c.shape[1] < CHUNK:
            c = np.pad(c, ((0, 0), (0, CHUNK - c.shape[1])))
        out.append(c[0])
    return np.stack(out)


def log_mel(chunks: torch.Tensor) -> torch.Tensor:
    """[B, 480000] float32 -> [B, 1001, 64] float32: hann(1024, periodic), center/reflect,
    power spectrogram, Slaney mel, 10*log10(clamp(., 1e-10))."""
    win = torch.hann_window(N_FFT, periodic=True, dtype=torch.float32)
    spec = torch.stft(chunks, N_FFT, hop_length=HOP, win_length=N_FFT, window=win, center=True,
                      pad_mode="reflect", return_complex=True)
    power = spec.real ** 2 + spec.imag ** 2                           # [B, 513, 1001]
    mel = torch.from_numpy(mel_filterbank().astype(np.float32))      # [64, 513]
    m = torch.matmul(mel, power).transpose(1, 2)                      # [B, 1001, 64]
    return 10.0 * torch.log10(torch.clamp(m, min=1e-10))


# ------------------------------------------------------------------------------- network
def _rel_pos_index(ws: int = WINDOW, device=None) -> torch.Tensor:
    ar = torch.arange(ws, device=device)
    coords = torch.stack(torch.meshgrid(ar, ar, indexing="ij")).flatten(1)
    rel = (coords[:, :, None] - coords[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += ws - 1
    rel[:, :, 1] += ws - 1
    rel[:, :, 0] *= 2 * ws - 1
    return rel.sum(-1)                                                # [64, 64]


def _shift_mask(h: int, w: int, ws: int, shift: int, device=None, dtype=torch.float32) -> torch.Tensor:
    img = torch.zeros((1, h, w, 1), device=device, dtype=dtype)
    cnt = 0
    for hs in (slice(0, -ws), slice(-ws, -shift), slice(-shift, None)):
        for wsl in (slice(0, -ws), slice(-ws, -shift), slice(-shift, None)):
            img[:, hs, wsl, :] = cnt
            cnt += 1
    mw = _partition(img, ws).view(-1, ws * ws)
    m = mw.unsqueeze(1) - mw.unsqueeze(2)
    return m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0)    # [nW, 64, 64]


def _partition(x, ws):
    b, h, w, c = x.shape
    x = x.view(b, h // ws, ws, w // ws, ws, c)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(-1, ws, ws, c)


def _reverse(win, ws, h, w):
    c = win.shape[-1]
    x = win.view(-1, h // ws, w // ws, ws, ws, c)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(-1, h, w, c)


def _ln(x, sd, key):
    return F.layer_norm(x, (x.shape[-1],), sd[key + ".weight"], sd[key + ".bias"], 1e-5)


def _lin(x, sd, key, bias=True):
    return F.linear(x, sd[key + ".weight"], sd[key + ".bias"] if bias else None)


def swin_block(x, sd, pre, res, heads, shift):
    b, n, c = x.shape
    h = w = res
    ws = WINDOW
    if res <= ws:
        shift = 0
    y = _ln(x, sd, pre + "layernorm_before").view(b, h, w, c)
    if shift:
        y = torch.roll(y, (-shift, -shift), (1, 2))
    win = _partition(y, ws).view(-1, ws * ws, c)
    hd = c // heads
    q = _lin(win, sd, pre + "attention.self.query").view(-1, ws * ws, heads, hd).transpose(1, 2)
    k = _lin(win, sd, pre + "attention.self.key").view(-1, ws * ws, heads, hd).transpose(1, 2)
    v = _lin(win, sd, pre + "attention.self.value").view(-1, ws * ws, heads, hd).transpose(1, 2)
    att = q @ k.transpose(-1, -2) / math.sqrt(hd)
    bias = sd[pre + "attention.self.relative_position_bias_table"][_rel_pos_index(device=x.device).view(-1)]
    att = att + bias.view(ws * ws, ws * ws, heads).permute(2, 0, 1).unsqueeze(0)
    if shift:
        mask = _shift_mask(h, w, ws, shift, x.device, x.dtype)
        att = att.view(-1, mask.shape[0], heads, ws * ws, ws * ws) + mask.unsqueeze(1).unsqueeze(0)
        att = att.view(-1, heads, ws * ws, ws * ws)
    ctx = (att.softmax(-1) @ v).permute(0, 2, 1, 3).reshape(-1, ws * ws, c)
    ctx = _lin(ctx, sd, pre + "attention.output.dense").view(-1, ws, ws, c)
    y = _reverse(ctx, ws, h, w)
    if shift:
        y = torch.roll(y, (shift, shift), (1, 2))
    x = x + y.view(b, n, c)
    z = _lin(_ln(x, sd, pre + "layernorm_after"), sd, pre + "intermediate.dense")
    return x + _lin(F.gelu(z), sd, pre + "output.dense")


def patch_merge(x, sd, pre, res):
    b, n, c = x.shape
    x = x.view(b, res, res, c)
    x = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1)
    x = _ln(x.view(b, -1, 4 * c), sd, pre + "norm")
    return F.linear(x, sd[pre + "reduction.weight"])


def batch_norm(lm: torch.Tensor, sd: dict) -> torch.Tensor:
    """[B, 1001, 64] log-mel -> BatchNorm (eval) over mel bins"""
    x = (lm - sd["batch_norm.running_mean"]) / torch.sqrt(sd["batch_norm.running_var"] + 1e-5)
    return x * sd["batch_norm.weight"] + sd["batch_norm.bias"]


def fold_image(x: torch.Tensor) -> torch.Tensor:
    """[B, 1001, 64] BatchNorm-ed log-mel -> bicubic time resize to 1024 -> fold four 256-frame blocks along
    frequency -> [B, 1, 256, 256]."""
    x = x[:, None]                                                     # [B,1,T,F]
    x = F.interpolate(x, (SPEC * 4, N_MEL), mode="bicubic", align_corners=True)
    b = x.shape[0]
    x = x.reshape(b, 4, SPEC, N_MEL).permute(0, 1, 3, 2).contiguous()  # [B, 4, 64, 256]
    return x.reshape(b, 1, 4 * N_MEL, SPEC)


def mel_to_image(lm: torch.Tensor, sd: dict) -> torch.Tensor:
    """[B, 1001, 64] log-mel -> BatchNorm over mel bins -> bicubic time resize to 1024 ->
    fold four 256-frame blocks along frequency -> [B, 1, 256, 256]."""
    return fold_image(batch_norm(lm, sd))


def image_tokens(img: torch.Tensor, sd: dict) -> torch.Tensor:
    """[B, 1, 256, 256] -> 4x4/4 conv -> LayerNorm -> the residual stream entering block 0 [B, 4096, E]"""
    x = F.conv2d(img, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=4)
    return _ln(x.flatten(2).transpose(1, 2), sd, "patch_embed.norm")


def head(x: torch.Tensor, sd: dict) -> torch.Tensor:
    """the stream leaving the last block [B, 64, 8 E] -> final LayerNorm, token mean, projection, L2 norm [B, 512]"""
    x = _ln(x, sd, "norm").mean(1)                                     # token average -> [B, 8 E]
    x = _lin(F.relu(_lin(x, sd, "audio_projection.linear1")), sd, "audio_projection.linear2")
    return F.normalize(x, dim=-1)


@torch.no_grad()
def network(lm: torch.Tensor, sd: dict) -> torch.Tensor:
    """[B, 1001, 64] log-mel -> [B, 512] L2-normalised embedding, in the dtype and on the device of lm and sd."""
    x = image_tokens(mel_to_image(lm, sd), sd)                         # [B, 4096, 96]
    res = SPEC // 4
    _, depths = config_of(sd)
    for i, (depth, heads) in enumerate(zip(depths, HEADS)):
        for j in range(depth):
            x = swin_block(x, sd, f"layers.{i}.blocks.{j}.", res, heads, 0 if j % 2 == 0 else WINDOW // 2)
        if i < len(depths) - 1:
            x = patch_merge(x, sd, f"layers.{i}.downsample.", res)
            res //= 2
    return head(x, sd)


@torch.no_grad()
def embed(wave: np.ndarray, sd: dict, batch: int = 4) -> np.ndarray:
    """What ModelLoader.get_embedding returns for clap-laion-audio: fp16 [n_windows, 512]."""
    ch = torch.from_numpy(chunks_of(quantize_like_reference(np.asarray(wave, dtype=np.float64))))
    outs = [network(log_mel(ch[i:i + batch]), sd) for i in range(0, ch.shape[0], batch)]
    return torch.cat(outs).numpy().astype(np.float16)


def synthetic_state(seed: int = 0, variant: str = "tiny") -> dict:
    """Seeded random HTSAT (tiny | base) + projection parameters (float32), HF key names."""
    EMBED, DEPTHS = VARIANTS[variant]
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def lin(key, out_f, in_f, bias=True, std=None):
        sd[key + ".weight"] = torch.randn((out_f, in_f), generator=g) * (std or (1.0 / math.sqrt(in_f)))
        if bias:
            sd[key + ".bias"] = torch.randn((out_f,), generator=g) * 0.02

    def ln(key, n):
        sd[key + ".weight"] = 1.0 + 0.1 * torch.randn((n,), generator=g)
        sd[key + ".bias"] = 0.05 * torch.randn((n,), generator=g)

    sd["batch_norm.weight"] = 1.0 + 0.1 * torch.randn((N_MEL,), generator=g)
    sd["batch_norm.bias"] = 0.1 * torch.randn((N_MEL,), generator=g)
    sd["batch_norm.running_mean"] = -30.0 + 5.0 * torch.randn((N_MEL,), generator=g)
    sd["batch_norm.running_var"] = 200.0 + 50.0 * torch.rand((N_MEL,), generator=g)
    sd["patch_embed.proj.weight"] = torch.randn((EMBED, 1, 4, 4), generator=g) * 0.25
    sd["patch_embed.proj.bias"] = torch.randn((EMBED,), generator=g) * 0.02
    ln("patch_embed.norm", EMBED)
    c = EMBED
    for i, (depth, heads) in enumerate(zip(DEPTHS, HEADS)):
        for j in range(depth):
            p = f"layers.{i}.blocks.{j}."
            ln(p + "layernorm_before", c)
            for n in ("query", "key", "value"):
                lin(p + "attention.self." + n, c, c)
            sd[p + "attention.self.relative_position_bias_table"] = 0.2 * torch.randn(((2 * WINDOW - 1) ** 2, heads), generator=g)
            lin(p + "attention.output.dense", c, c)
            ln(p + "layernorm_after", c)
            lin(p + "intermediate.dense", 4 * c, c)
            lin(p + "output.dense", c, 4 * c)
        if i < len(DEPTHS) - 1:
            ln(f"layers.{i}.downsample.norm", 4 * c)
            lin(f"layers.{i}.downsample.reduction", 2 * c, 4 * c, bias=False)
            c *= 2
    ln("norm", c)
    lin("audio_projection.linear1", OUT_DIM, c)
    lin("audio_projection.linear2", OUT_DIM, OUT_DIM)
    return sd
