"""Whisper parameters: seeded synthetic set, checkpoint loading, device packing.

State-dict keys are those of ``transformers.WhisperModel`` (what the reference loads with
``WhisperModel.from_pretrained("openai/whisper-<size>")``, model_loader.py:660), so a real checkpoint's
``state_dict()`` packs directly.  No checkpoint exists offline: tests and benches use seeded synthetic
parameters with the real architecture (a small synthetic vocabulary - only the start-token row of
``decoder.embed_tokens`` is ever read).
"""
from __future__ import annotations

import math
import os
from pathlib import Path

import torch

from .weights import split_hi_lo_tiles

# size -> (d_model, heads, encoder layers, decoder layers); ffn = 4 d_model, head dim 64, 80 mel bins
SIZES = {"tiny": (384, 6, 4, 4), "base": (512, 8, 6, 6), "small": (768, 12, 12, 12),
         "medium": (1024, 16, 24, 24), "large": (1280, 20, 32, 32)}
N_MEL, SEQ, MAX_TARGET = 80, 1500, 448
SYNTH_VOCAB, SYNTH_START = 64, 1          # synthetic checkpoints: tiny vocabulary, start token 1


def synthetic_whisper_tensors(seed: int = 0, size: str = "small", layers: tuple | None = None):
    """Yields the (key, tensor) pairs of ``synthetic_whisper_state`` one at a time, in generation order."""
    d, heads, n_enc, n_dec = SIZES[size]
    if layers is not None:
        n_enc, n_dec = (int(n) for n in layers)
        if n_enc < 1 or n_dec < 1:
            raise ValueError("layers must be (encoder layers >= 1, decoder layers >= 1)")
    f = 4 * d
    g = torch.Generator().manual_seed(seed)

    def lin(key, out_f, in_f, bias=True):
        yield key + ".weight", torch.randn((out_f, in_f), generator=g) * (1.0 / math.sqrt(in_f))
        if bias:
            yield key + ".bias", torch.randn((out_f,), generator=g) * 0.02

    def ln(key, n):
        yield key + ".weight", 1.0 + 0.1 * torch.randn((n,), generator=g)
        yield key + ".bias", 0.05 * torch.randn((n,), generator=g)

    def attn(p):
        yield from lin(p + "k_proj", d, d, bias=False)
        yield from lin(p + "v_proj", d, d)
        yield from lin(p + "q_proj", d, d)
        yield from lin(p + "out_proj", d, d)

    yield "encoder.conv1.weight", torch.randn((d, N_MEL, 3), generator=g) * (1.0 / math.sqrt(3 * N_MEL))
    yield "encoder.conv1.bias", torch.randn((d,), generator=g) * 0.02
    yield "encoder.conv2.weight", torch.randn((d, d, 3), generator=g) * (1.0 / math.sqrt(3 * d))
    yield "encoder.conv2.bias", torch.randn((d,), generator=g) * 0.02
    yield "encoder.embed_positions.weight", 0.1 * torch.randn((SEQ, d), generator=g)
    for i in range(n_enc):
        p = f"encoder.layers.{i}."
        yield from attn(p + "self_attn.")
        yield from ln(p + "self_attn_layer_norm", d)
        yield from lin(p + "fc1", f, d)
        yield from lin(p + "fc2", d, f)
        yield from ln(p + "final_layer_norm", d)
    yield from ln("encoder.layer_norm", d)
    yield "decoder.embed_tokens.weight", 0.5 * torch.randn((SYNTH_VOCAB, d), generator=g)
    yield "decoder.embed_positions.weight", 0.1 * torch.randn((MAX_TARGET, d), generator=g)
    for i in range(n_dec):
        p = f"decoder.layers.{i}."
        yield from attn(p + "self_attn.")
        yield from ln(p + "self_attn_layer_norm", d)
        yield from attn(p + "encoder_attn.")
        yield from ln(p + "encoder_attn_layer_norm", d)
        yield from lin(p + "fc1", f, d)
        yield from lin(p + "fc2", d, f)
        yield from ln(p + "final_layer_norm", d)
    yield from ln("decoder.layer_norm", d)


def synthetic_whisper_state(seed: int = 0, size: str = "small", layers: tuple | None = None) -> dict:
    """Seeded parameters of whisper-``size``.  ``layers = (n_enc, n_dec)`` generates a shortened stack of that many
    encoder and decoder layers (same widths, its own draws after the first n_enc encoder layers); without it the
    state has the real depth."""
    return dict(synthetic_whisper_tensors(seed, size, layers))


def load_whisper_state(path=None, seed: int = 0, size: str = "small"):
    """-> (state dict, decoder_start_token_id).  ``path`` / $FADTK_WHISPER_CKPT: a torch-saved
    ``WhisperModel.state_dict()`` (optionally {"state_dict": ..., "decoder_start_token_id": n})."""
    from .weights import resolve_checkpoint
    path = resolve_checkpoint(path, "FADTK_WHISPER_CKPT", "whisper-" + size)
    if path is not None:
        from .weights import load_checkpoint_file
        raw = load_checkpoint_file(path)
        start = int(raw.pop("__meta__.decoder_start_token_id", 50258))
        raw = {k: v for k, v in raw.items() if not k.startswith("__meta__.")}
        sd = {k.removeprefix("model."): v.float().contiguous() for k, v in raw.items() if not k.startswith("proj_out")}
        return sd, start
    return synthetic_whisper_state(seed, size), SYNTH_START


def config_of(sd: dict) -> tuple:
    """(d_model, heads, encoder layers, decoder layers, ffn)"""
    d = sd["encoder.conv1.weight"].shape[0]
    n_enc = len({k.split(".")[2] for k in sd if k.startswith("encoder.layers.")})
    n_dec = len({k.split(".")[2] for k in sd if k.startswith("decoder.layers.")})
    return d, d // 64, n_enc, n_dec, sd["encoder.layers.0.fc1.weight"].shape[0]


def pack_whisper(sd: dict, decoder_start_token_id: int) -> list:
    """-> contiguous CPU tensors in the order fad_whisper_load expects (csrc/whisper_host.inc)."""
    d, heads, n_enc, n_dec, f = config_of(sd)
    fl = lambda t: t.float().contiguous()
    z = lambda n: torch.zeros((n,), dtype=torch.float32)
    out = []
    w1 = torch.zeros((d, 3, 128))                                      # k = tap*128 + mel bin (80 real)
    w1[:, :, :N_MEL] = sd["encoder.conv1.weight"].permute(0, 2, 1)
    out += [split_hi_lo_tiles(w1.reshape(d, 384)), fl(sd["encoder.conv1.bias"]),
            split_hi_lo_tiles(sd["encoder.conv2.weight"].permute(0, 2, 1).reshape(d, 3 * d).contiguous()),
            fl(sd["encoder.conv2.bias"]), fl(sd["encoder.embed_positions.weight"])]

    def qkv(p):
        w = torch.cat([sd[p + "q_proj.weight"], sd[p + "k_proj.weight"], sd[p + "v_proj.weight"]], 0)
        b = torch.cat([sd[p + "q_proj.bias"], z(d), sd[p + "v_proj.bias"]], 0)       # k_proj has no bias
        return split_hi_lo_tiles(w), fl(b)

    for i in range(n_enc):
        p = f"encoder.layers.{i}."
        qw, qb = qkv(p + "self_attn.")
        out += [fl(sd[p + "self_attn_layer_norm.weight"]), fl(sd[p + "self_attn_layer_norm.bias"]), qw, qb,
                split_hi_lo_tiles(sd[p + "self_attn.out_proj.weight"]), fl(sd[p + "self_attn.out_proj.bias"]),
                fl(sd[p + "final_layer_norm.weight"]), fl(sd[p + "final_layer_norm.bias"]),
                split_hi_lo_tiles(sd[p + "fc1.weight"]), fl(sd[p + "fc1.bias"]),
                split_hi_lo_tiles(sd[p + "fc2.weight"]), fl(sd[p + "fc2.bias"])]
    x0 = sd["decoder.embed_tokens.weight"][decoder_start_token_id][None, :] + sd["decoder.embed_positions.weight"][:2]
    out += [fl(sd["encoder.layer_norm.weight"]), fl(sd["encoder.layer_norm.bias"]), fl(x0)]
    for i in range(n_dec):
        p = f"decoder.layers.{i}."
        qw, qb = qkv(p + "self_attn.")
        c = p + "encoder_attn."
        ckv_w = torch.cat([sd[c + "k_proj.weight"], sd[c + "v_proj.weight"]], 0)
        ckv_b = torch.cat([z(d), sd[c + "v_proj.bias"]], 0)
        out += [fl(sd[p + "self_attn_layer_norm.weight"]), fl(sd[p + "self_attn_layer_norm.bias"]), qw, qb,
                split_hi_lo_tiles(sd[p + "self_attn.out_proj.weight"]), fl(sd[p + "self_attn.out_proj.bias"]),
                fl(sd[p + "encoder_attn_layer_norm.weight"]), fl(sd[p + "encoder_attn_layer_norm.bias"]),
                split_hi_lo_tiles(sd[c + "q_proj.weight"]), fl(sd[c + "q_proj.bias"]),
                split_hi_lo_tiles(ckv_w), fl(ckv_b),
                split_hi_lo_tiles(sd[c + "out_proj.weight"]), fl(sd[c + "out_proj.bias"]),
                fl(sd[p + "final_layer_norm.weight"]), fl(sd[p + "final_layer_norm.bias"]),
                split_hi_lo_tiles(sd[p + "fc1.weight"]), fl(sd[p + "fc1.bias"]),
                split_hi_lo_tiles(sd[p + "fc2.weight"]), fl(sd[p + "fc2.bias"])]
    out += [fl(sd["decoder.layer_norm.weight"]), fl(sd["decoder.layer_norm.bias"])]
    assert len(out) == 5 + 12 * n_enc + 3 + 20 * n_dec + 2
    return out
