"""CPU restatement of the Encodec-24 kHz SEANet encoder as the reference uses it (test infrastructure only).

Reference call sites: fadtk/model_loader.py:123-130 (EncodecModel.encodec_model_24khz(), bandwidth irrelevant
for the encoder), :160-166 (``self.model.encoder(audio)`` -> [1, 128, T/320] -> transposed [T/320, 128]).
The ``encodec`` package (0.1.1, uv.lock) is not installed here; this restates its SEANetEncoder (causal
reflect-padded weight-normalised convs, ELU, residual blocks with conv shortcut, 2-layer LSTM with skip) and
tests/test_encodec_oracle.py pins it to transformers' independent port (EncodecModel.encoder) with shared
random weights.  Parity against the real facebook checkpoint is unpinned (no weights offline).
``conv_layer`` and ``lstm`` run one stage of the encoder (float64 by default) for the GPU stage tests
(tests/test_gpu_encodec_stages.py); ``encoder`` is built from them and takes a dtype too.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

# Deliberately NO import from fadtk_b200: the layer table and the weight-norm folding are restated here (torch's own
# ``torch._weight_norm``), so a bug in the product's weights_encodec.effective_weight / conv_table cannot hide behind
# an oracle that shares it.
LSTM_LAYERS = 2
_RATIOS = (2, 4, 5, 8)                                          # encoder order (encodec SEANetEncoder reverses [8, 5, 4, 2])


def conv_table():
    """(layer index in the Sequential, kind, Cin, Cout, kernel, stride) in execution order: conv(1 -> 32, k7);
    4 x [residual block, ELU, strided conv k = 2r]; LSTM; ELU; conv(512 -> 128, k7)"""
    t = [(0, "in", 1, 32, 7, 1)]
    ch, idx = 32, 1
    for r in _RATIOS:
        t += [(idx, "res", ch, ch, 3, 1), (idx + 2, "down", ch, 2 * ch, 2 * r, r)]
        ch, idx = 2 * ch, idx + 3
    t.append((idx + 2, "out", ch, 128, 7, 1))
    return t


def effective_weight(sd: dict, prefix: str) -> torch.Tensor:
    """torch.nn.utils.parametrizations.weight_norm (dim 0): w = g * v / ||v||, norm over every other dimension"""
    if prefix + ".conv.weight" in sd:                           # 48 kHz model: plain weights + GroupNorm
        return sd[prefix + ".conv.weight"]
    g = sd[prefix + ".conv.parametrizations.weight.original0"]
    v = sd[prefix + ".conv.parametrizations.weight.original1"]
    return torch._weight_norm(v, g, 0)


def _sconv(x, w, b, stride, causal=True):
    """x [B, C, T]; SConv1d: causal pads (k - stride) on the left; non-causal splits it (left gets the odd sample);
    the right side is extended so the last window is full; reflect."""
    k = w.shape[-1]
    pad_total = k - stride
    n_frames = (x.shape[-1] - k + pad_total) / stride + 1
    ideal = (math.ceil(n_frames) - 1) * stride + (k - pad_total)
    extra = ideal - x.shape[-1]
    if causal:
        x = _reflect_pad(x, pad_total, extra)
    else:
        right = pad_total // 2
        x = _reflect_pad(x, pad_total - right, right + extra)
    return F.conv1d(x, w.to(x.dtype), b.to(x.dtype), stride=stride)


def _reflect_pad(x, left, right):
    length = x.shape[-1]
    max_pad = max(left, right)
    extra = 0
    if length <= max_pad:                                      # encodec pad1d: tiny inputs get zeros first
        extra = max_pad - length + 1
        x = F.pad(x, (0, extra))
    y = F.pad(x, (left, right), mode="reflect")
    return y[..., : y.shape[-1] - extra] if extra else y


def conv_layers(sd: dict) -> list:
    """(state-dict prefix, stride) of every conv in the order the product loads them (weights_encodec.pack_encodec):
    the input conv, per stage the residual block's k = 3 conv, k = 1 conv and shortcut and the down conv, the last conv"""
    out = []
    for idx, kind, cin, cout, k, s in conv_table():
        if kind == "res":
            out += [(f"layers.{idx}.block.1", 1), (f"layers.{idx}.block.3", 1), (f"layers.{idx}.shortcut", 1)]
        else:
            out.append((f"layers.{idx}", s))
    return out


def is_causal(sd: dict) -> bool:
    return "layers.0.conv.weight" not in sd                    # 48 kHz: non-causal + GroupNorm(1, C) after every conv


@torch.no_grad()
def conv_layer(x: torch.Tensor, sd: dict, layer: int, elu_in: bool = False, groupnorm: bool = True,
               dtype=torch.float64) -> torch.Tensor:
    """conv `layer` of conv_layers(sd) on x [B, Cin, T] in `dtype`: ELU first if elu_in, then the padded conv and
    (48 kHz model, if groupnorm) its GroupNorm(1, Cout)"""
    prefix, stride = conv_layers(sd)[layer]
    x = x.to(dtype)
    if elu_in:
        x = F.elu(x)
    y = _sconv(x, effective_weight(sd, prefix).to(dtype), sd[prefix + ".conv.bias"], stride, is_causal(sd))
    if groupnorm and prefix + ".norm.weight" in sd:
        y = F.group_norm(y, 1, sd[prefix + ".norm.weight"].to(dtype), sd[prefix + ".norm.bias"].to(dtype), eps=1e-5)
    return y


@torch.no_grad()
def lstm(z: torch.Tensor, sd: dict, dtype=torch.float64) -> torch.Tensor:
    """The encoder's two LSTM layers with the skip: z [B, T, 512] -> LSTM(z) + z in `dtype`"""
    seq = z.to(dtype).transpose(0, 1)                          # [T, B, 512]
    hsz = seq.shape[-1]
    m = torch.nn.LSTM(hsz, hsz, LSTM_LAYERS)
    m.load_state_dict({k_.split("lstm.")[1]: v for k_, v in sd.items() if ".lstm." in k_})
    m = m.to(device=seq.device, dtype=dtype)
    return (m(seq)[0] + seq).transpose(0, 1)


@torch.no_grad()
def encoder(x: torch.Tensor, sd: dict, dtype=torch.float32) -> torch.Tensor:
    """[B, 1, T] (48 kHz: [B, 2, T]) -> [B, 128, ceil(T / 320)] in `dtype`"""
    layer = iter(range(len(conv_layers(sd))))

    def conv(t, elu_in=False):
        return conv_layer(t, sd, next(layer), elu_in, True, dtype)

    x = x.to(dtype)
    for idx, kind, cin, cout, k, s in conv_table():
        if kind == "in":
            x = conv(x)
        elif kind == "res":
            h = conv(x, True)
            h = conv(h, True)
            x = conv(x) + h
        elif kind == "down":
            x = conv(x, True)
        else:                                                  # LSTM with skip, ELU, last conv
            y = lstm(x.transpose(1, 2), sd, dtype)
            x = conv(y.transpose(1, 2), True)
    return x


@torch.no_grad()
def embed(wave: np.ndarray, sd: dict) -> np.ndarray:
    """What ModelLoader.get_embedding returns: fp16 [T/320, 128].  24 kHz: the whole file at once; 48 kHz
    (model_loader.py:139-152): mono duplicated to stereo (convert_audio), 1-s segments with stride = segment."""
    x = torch.from_numpy(np.asarray(wave, dtype=np.float32)).reshape(1, 1, -1)
    if "layers.0.conv.weight" not in sd:
        return encoder(x, sd)[0].transpose(0, 1).numpy().astype(np.float16)
    x = x.expand(1, 2, -1)
    seg = 48000
    outs = [encoder(x[:, :, o:o + seg], sd)[0].transpose(0, 1) for o in range(0, x.shape[-1], seg)]
    return torch.cat(outs).numpy().astype(np.float16)
