"""Whisper one stage at a time, through the stage entries that call fad_whisper_forward's own launch code
(fad_whisper_logmel -> whisper_frontend + whisper_im2col1, fad_whisper_conv -> whisper_im2col1 / whisper_conv1 /
whisper_conv2, fad_whisper_enc_layer -> whisper_enc_layer, fad_whisper_encode -> the encoder loop with
whisper_enc_final, fad_whisper_dec_layer -> whisper_dec_layer), and the encoder and the whole forward at real clip
lengths, for every model size.  References are transformers' own WhisperModel (the reference's dependency, built by
oracle/whisper_oracle.build with the seeded synthetic weights), run in float64 on the GPU from exactly the values the
kernels read: encoder.conv1, encoder.conv2 with embed_positions, encoder.layers[l], decoder.layers[l] (causal mask over
the two start tokens, the kernel's fp16 encoder output as encoder_hidden_states), and the feature extractor's log-mel
restated in float64.  test_stage_composition_is_the_model (CPU) pins that composing these references is the model.
Stacks are shortened to 2 encoder + 2 decoder layers (weights_whisper.synthetic_whisper_state(layers=...)) except for
tiny, which runs its full 4 + 4.

Inputs and outputs sit in sentinel-NaN guarded buffers and the clips of a batch differ (music, noise, silence, a
full-scale square wave): an output left unwritten, a guard overwritten or a value of the neighbouring clip shows up.

Per-element bounds (float64, 1.001 margin; u = 2^-24):
  * front end, raw log10 mel of whisper_logmel_kernel.  With x_n the Hann-windowed frame and c_n = cos / sin of the
    DFT, the kernel's fp32 x_n (pcm 2^-15 exact, times the rounded Hann table) times the rounded table, summed by a
    400-step fma chain:  |d re| <= 403 u sum_n |x_n c_n| (same for im);  p = re^2 + im^2:
        |dp| <= (2 |re| + d re) d re + (2 |im| + d im) d im + 2 u p+,  p+ = (|re| + d re)^2 + (|im| + d im)^2;
    the <= 32-tap mel sum (rounded Slaney weights w, fma chain):  |d mel| <= (1 + u) sum w dp + 34 u sum w p+;
    log10f of max(mel, 1e-10f): log10((m + dm) / m) upwards, -log10(1 - dm / m) downwards (at most down to the clamp
    at -10), with m = max(mel, 1e-10) and dm = d mel + |1e-10f - 1e-10|, plus 2 ulp for log10f itself.
    The comparison is after the floor at clip_max - 8, as the model sees it: the floor is 1-Lipschitz, the clip max
    bound is the spread max(v +- b) - max(v), and an element surely under both floors is held to that spread alone.
  * conv stem, pre-activation: gpu_checks.gemm_bound (r_a = 0) + sum_j |w_j| e_a_j, with e_a the error of the operand
    the kernel reads: conv 0's features (max(x, c - 8) + 4) / 4 are fp32 (u |c - 8| for the floor, u |x + 4| for the
    add) rounded to fp16 (2^-11 |a| + 2^-25); conv 1 reads conv 0's fp16 output itself (e_a = 0).  K is 3 x 128 padded
    mel channels for conv 0 and 3 d for conv 1.
  * GELU: gpu_checks.gelu_out, conv 0 with its fp16 output; conv 1's fp32 add into the positional embedding:
    + 2^-24 |out|.
The layers (attention, LayerNorms, GEMMs with fp16 operands) and the taps are held to rms ceilings, about 3x the
largest level measured on the H100 (RMS_CEIL below).  Each layer is also held on its update out - x, which the stream
it adds to would otherwise hide.
"""
import hashlib
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fadtk_b200 import synth, weights_whisper as ww
from gpu_checks import (Guarded, check_bound, expect_rejected, gelu_out, gemm_bound, layer_metrics, on_fresh_engine,
                        report, report_stats, tap_metrics)
from oracle import whisper_oracle as wo

GUARD = 4096
MAX_CLIPS = 4
SIZES = list(ww.SIZES)
SOT = ww.SYNTH_START
N_SAMPLES, N_FRAMES, SEQ, N_FFT, HOP = 480000, 3000, 1500, 400, 160
U = 2.0 ** -24

# rms relative error ceilings (rms |kernel - fp64| / rms |fp64|), about 3x the largest level measured on an H100 80GB
# HBM3 (700 W) over the cases below, every size alike to within 10 %:
#   encoder layer 2.6e-4 (its update out - x 2.9e-4), decoder layer 2.8e-4 (update 2.9e-4), fad_whisper_encode 5.0e-4
#   (centred 4.4e-3, largest at 30 s), fad_whisper_forward 4.5e-4 (centred over its two rows 5.4e-3).
# The per-element bounds hold with room: max err / bound 0.029 for the front end, 0.24 for conv 0, 0.001 for conv 1
# (rms 2.2e-7, 3.1e-4 and 1.3e-6).
RMS_CEIL = {"enc_layer": 8e-4, "enc_update": 9e-4, "dec_layer": 8e-4, "dec_update": 9e-4,
            "encode": 1.5e-3, "encode_c": 1.3e-2, "forward": 1.4e-3, "forward_c": 1.6e-2}


def stack(size):
    """(encoder layers, decoder layers) of the stacks the stage tests run"""
    return None if size == "tiny" else (2, 2)


# ------------------------------------------------------------------------------------------------ models
_MODELS = {}


def model_state(size):
    """(state dict, float64 transformers WhisperModel on the GPU) of the seed-0 synthetic weights"""
    if size not in _MODELS:
        sd = ww.synthetic_whisper_state(0, size, layers=stack(size))
        model, _ = wo.build(sd, SOT)
        _MODELS[size] = (sd, model.double().to("cuda"))
    return _MODELS[size]


def load(engine, size, max_clips=MAX_CLIPS):
    token = ("whisper-stage-test", size, max_clips)
    if engine.owners.get("whisper") != token:
        sd = model_state(size)[0]
        engine.whisper_load(ww.config_of(sd), ww.pack_whisper(sd, SOT), max_clips)
        engine.owners["whisper"] = token


# ------------------------------------------------------------------------------------------------- inputs
def square(n):
    """full scale: +32767 / -32768 in runs of 37 samples"""
    return np.where((np.arange(n) // 37) % 2 == 0, 32767, -32768).astype(np.int16)


def make_clip(kind, n, seed=0):
    if kind == "silence":
        return np.zeros(n, np.int16)
    if kind == "square":
        return square(n)
    sec = max(n, 1600) / 16000
    base = synth.musiclike_clip(seed, sec, 16000) if kind == "music" else synth.noise_clip(seed, sec, 16000)
    return base[:n].copy()


def upload(clips):
    lens = np.array([len(c) for c in clips], dtype=np.int32)
    starts = np.zeros(len(clips), dtype=np.int64)
    starts[1:] = np.cumsum(lens[:-1])
    return (torch.from_numpy(np.concatenate(clips)).cuda(), torch.from_numpy(starts).cuda(), torch.from_numpy(lens).cuda())


STAGE_CLIPS = [("music", 160000), ("noise", 16000), ("silence", 48000), ("square", 480000)]


def stage_clips():
    """the four different clips of every stage batch"""
    return [make_clip(k, n, i) for i, (k, n) in enumerate(STAGE_CLIPS)]


# ------------------------------------------------------------------------------------------ front end, fp64
_MEL = {}


def mel_filters(device):
    """transformers' Slaney filter bank, float64 [201, 80]"""
    if device not in _MEL:
        import transformers as tr
        _MEL[device] = torch.from_numpy(tr.WhisperFeatureExtractor().mel_filters).to(device, torch.float64)
    return _MEL[device]


def frames64(clip, device):
    """the Hann-windowed frames [3000, 400] of the clip zero-padded / truncated to 30 s, centre, reflect"""
    x = torch.zeros(N_SAMPLES, dtype=torch.float64, device=device)
    n = min(len(clip), N_SAMPLES)
    x[:n] = torch.from_numpy(clip[:n].astype(np.float64) / 32768.0).to(device)
    xp = F.pad(x[None, None], (N_FFT // 2, N_FFT // 2), mode="reflect")[0, 0]
    n_ = torch.arange(N_FFT, dtype=torch.float64, device=device)
    hann = 0.5 - 0.5 * torch.cos(2 * math.pi * n_ / N_FFT)
    return xp.unfold(0, N_FFT, HOP)[:N_FRAMES] * hann


def ref_logmel(clip, device="cpu", bound=False):
    """float64 raw log10 mel [3000, 80] of one clip (and the per-element bound of the module docstring)"""
    fr = frames64(clip, device)
    X = torch.fft.rfft(fr, dim=1)
    p = X.real.square() + X.imag.square()
    W = mel_filters(device)
    mel = p @ W
    m = mel.clamp_min(1e-10)
    v = torch.log10(m)
    if not bound:
        return v
    k = torch.arange(N_FFT // 2 + 1, dtype=torch.float64, device=device)
    n_ = torch.arange(N_FFT, dtype=torch.float64, device=device)
    ang = 2 * math.pi * torch.remainder(n_[:, None] * k[None, :], N_FFT) / N_FFT
    A = fr.abs()
    dre = 403 * U * (A @ torch.cos(ang).abs())
    dim = 403 * U * (A @ torch.sin(ang).abs())
    re, im = X.real.abs(), X.imag.abs()
    pu = (re + dre).square() + (im + dim).square()
    dp = (2 * re + dre) * dre + (2 * im + dim) * dim + 2 * U * pu
    dm = (1 + U) * (dp @ W) + 34 * U * (pu @ W) + 2e-18
    t = dm / m
    up = torch.log10(1 + t)
    down = torch.where(t < 1, -torch.log10((1 - t).clamp_min(1e-300)), torch.full_like(t, math.inf))
    down = torch.minimum(down, v + 10 + 1e-6)
    b = (torch.maximum(up, down) + 2 * 2.0 ** -23 * v.abs()) * 1.001 + 1e-30
    return v, b


def floored(v, c):
    return torch.maximum(v, c - 8.0)


def features64(clips, device):
    """float64 input_features [B, 80, 3000] of the clips: the restated log-mel, floored at max - 8, (x + 4) / 4"""
    out = []
    for c in clips:
        v = ref_logmel(c, device)
        out.append(((floored(v, v.max()) + 4.0) / 4.0).T)
    return torch.stack(out)


def run_logmel(engine, clips):
    pcm, start, lens = upload(clips)
    n = len(clips)
    out = Guarded((n * N_FRAMES * 80 + n,), torch.float32, "cuda", GUARD)
    engine.whisper_logmel(pcm, start, lens, n, out.body)
    got = out.check()
    return got[:n * N_FRAMES * 80].view(n, N_FRAMES, 80), got[n * N_FRAMES * 80:]


FRONT_BATCHES = {
    # the left reflect reaches past the clip end; 5 clips > max_clips
    "short": [("music", 1), ("noise", 199), ("square", 200), ("music", 201), ("noise", 159)],
    # hop edges, 1 s (blocks wholly in the zero padding take the early out), the right reflect reads real samples
    "edges": [("square", 160), ("music", 161), ("noise", 16000), ("music", 479999), ("noise", 480000)],
    # the right reflect past 30 s, truncation, a silent clip next to a full-scale one
    "long": [("music", 480001), ("noise", 1000000), ("silence", 16000), ("square", 16000)],
}


@pytest.mark.gpu
@pytest.mark.parametrize("batch", list(FRONT_BATCHES))
def test_logmel_matches_fp64(engine, batch, capsys):
    """fad_whisper_logmel's raw log10 mel and per-clip max against the float64 restatement, within the fp32 bound of
    the module docstring, after the floor at max - 8."""
    load(engine, "tiny")
    clips = [make_clip(k, n, i) for i, (k, n) in enumerate(FRONT_BATCHES[batch])]
    raw, cmax = run_logmel(engine, clips)
    stats = {}
    for i, ((kind, n), clip) in enumerate(zip(FRONT_BATCHES[batch], clips)):
        v, b = ref_logmel(clip, "cuda", bound=True)
        c = v.max()
        c_lo, c_hi = (v - b).max(), (v + b).max()
        bc = torch.maximum(c_hi - c, c - c_lo) + 2 * U * (c - 8).abs()
        what = f"{kind} {n}"
        ck = cmax[i].double()
        assert (ck - c).abs().item() <= bc.item(), f"{what}: clip max {ck.item()!r}, want {c.item()!r} +- {bc.item():.3g}"
        fl = c - 8.0
        bound = torch.where(v - b > fl + bc, b, torch.where(v + b < fl - bc, bc.expand_as(b), torch.maximum(b, bc)))
        check_bound("logmel", what, floored(raw[i].double(), ck), floored(v, c), bound, stats, RMS_CEIL)
    report_stats(capsys, "whisper", stats, batch)


# ---------------------------------------------------------------------------------------------------- convs
def conv_mm(a, w, b, stride, pad):
    """Conv1d as one float64 GEMM: a [B, Cin, T], w [Cout, Cin, k] -> [B, Cout, T_out]"""
    k = w.shape[2]
    ap = F.pad(a, (pad, pad))
    T_out = (ap.shape[2] - k) // stride + 1
    cols = ap.unfold(2, k, stride)[:, :, :T_out]                         # [B, Cin, T_out, k]
    cols = cols.permute(0, 2, 3, 1).reshape(a.shape[0], T_out, k * a.shape[1])
    y = cols @ w.permute(0, 2, 1).reshape(w.shape[0], -1).T
    if b is not None:
        y = y + b
    return y.transpose(1, 2)


def conv_sums(a, w, stride, pad):
    """(S, sum |w|, sum |a|) of gpu_checks.gemm_bound for a GEMM conv; a [B, Cin, T] float64, w [Cout, Cin, k]"""
    S = conv_mm(a.abs(), w.abs(), None, stride, pad)
    ones = torch.ones((1, 1, w.shape[2]), dtype=a.dtype, device=a.device)
    sa = F.conv1d(F.pad(a.abs().sum(1, keepdim=True), (pad, pad)), ones, None, stride)
    return S, w.abs().flatten(1).sum(1)[None, :, None], sa


@torch.no_grad()
def conv0_reference(model, raw, cmax):
    """kernel raw log10 mel [B, 3000, 80] + clip max [B] -> (GELU(conv1(features)) [B, 3000, d], bound)"""
    x = raw.double().transpose(1, 2)
    c = cmax.double()[:, None, None]
    a = (floored(x, c) + 4.0) / 4.0
    ea = 2.0 ** -11 * a.abs() + 2.0 ** -25 + (2.0 ** -11 + 1) * U * ((c - 8).abs() + (a * 4).abs()) / 4
    conv = model.encoder.conv1
    y = conv_mm(a, conv.weight, conv.bias, 1, 1)
    e = gemm_bound(*conv_sums(a, conv.weight, 1, 1), 384, conv.bias, y) + conv_mm(ea, conv.weight.abs(), None, 1, 1)
    out, e = gelu_out(y, e, True)
    return out.transpose(1, 2), (e * 1.001).transpose(1, 2)


@torch.no_grad()
def conv1_reference(model, h1):
    """kernel conv 0 output fp16 [B, 3000, d] -> (embed_positions + GELU(conv2(h1)) [B, 1500, d], bound)"""
    a = h1.double().transpose(1, 2)
    conv = model.encoder.conv2
    y = conv_mm(a, conv.weight, conv.bias, 2, 1)
    e = gemm_bound(*conv_sums(a, conv.weight, 2, 1), 3 * a.shape[1], conv.bias, y)
    g, e = gelu_out(y, e, False)
    out = g.transpose(1, 2) + model.encoder.embed_positions.weight
    return out, (e.transpose(1, 2) + 2.0 ** -24 * out.abs()) * 1.001


def run_stem(engine, d, raw, cmax):
    """kernel raw log-mel -> (conv 0 output fp16 [B, 3000, d], conv 1 output fp32 [B, 1500, d]), guarded"""
    B = raw.shape[0]
    xin = Guarded(raw.shape, torch.float32, "cuda", GUARD, init=raw)
    cin = Guarded(cmax.shape, torch.float32, "cuda", GUARD, init=cmax)
    h1 = Guarded((B, N_FRAMES, d), torch.float16, "cuda", GUARD)
    engine.whisper_conv(0, xin.body, cin.body, B, h1.body)
    got0 = h1.check()
    assert xin.intact_input() and cin.intact_input(), "the input or its guard was modified"
    hin = Guarded(got0.shape, torch.float16, "cuda", GUARD, init=got0)
    x = Guarded((B, SEQ, d), torch.float32, "cuda", GUARD)
    engine.whisper_conv(1, hin.body, None, B, x.body)
    got1 = x.check()
    assert hin.intact_input(), "the input or its guard was modified"
    return got0, got1


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
def test_conv_stem_matches_fp64(engine, size, capsys):
    """conv 0 from the kernel's raw log-mel and clip max, conv 1 from conv 0's kernel output, four different clips in
    one batch: taps t = -1 and t = 3000 (conv 0) and t = -1 (conv 1) must read zeros, never the neighbouring clip."""
    load(engine, size)
    model = model_state(size)[1]
    d = model.config.d_model
    raw, cmax = run_logmel(engine, stage_clips())
    h1, x = run_stem(engine, d, raw, cmax)
    stats = {}
    ref0, b0 = conv0_reference(model, raw, cmax)
    ref1, b1 = conv1_reference(model, h1)
    for i, (kind, n) in enumerate(STAGE_CLIPS):
        check_bound("conv0", f"{size} {kind} {n}", h1[i], ref0[i], b0[i], stats, RMS_CEIL)
        check_bound("conv1", f"{size} {kind} {n}", x[i], ref1[i], b1[i], stats, RMS_CEIL)
    report_stats(capsys, "whisper", stats, size)


# ------------------------------------------------------------------------------------------------- layers
def enc_layer_ref(model, l, x):
    out = model.encoder.layers[l](x, None)
    return out[0] if isinstance(out, tuple) else out


def causal_mask(B, device):
    m = torch.zeros((B, 1, 2, 2), dtype=torch.float64, device=device)
    m[:, :, 0, 1] = torch.finfo(torch.float64).min
    return m


def dec_layer_ref(model, l, xd, enc):
    out = model.decoder.layers[l](xd, causal_mask(xd.shape[0], xd.device), enc, encoder_attention_mask=None,
                                  past_key_values=None, use_cache=False)
    return out[0] if isinstance(out, tuple) else out


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
def test_encoder_layers_match_fp64(engine, size, capsys):
    """Every encoder layer of the stack, each fed the previous stage's kernel output (layer 0: conv 1's)."""
    load(engine, size)
    model = model_state(size)[1]
    d = model.config.d_model
    raw, cmax = run_logmel(engine, stage_clips())
    x = run_stem(engine, d, raw, cmax)[1].clone()
    B = x.shape[0]
    lines = []
    for l in range(model.config.encoder_layers):
        xin = Guarded(x.shape, torch.float32, "cuda", GUARD, init=x)
        out = Guarded(x.shape, torch.float32, "cuda", GUARD)
        engine.whisper_enc_layer(l, xin.body, B, out.body)
        got = out.check()
        assert xin.intact_input(), "the input or its guard was modified"
        with torch.no_grad():
            ref = enc_layer_ref(model, l, x.double())
        rms, upd, mx = layer_metrics(got, x, ref)
        lines.append(f"layer {l}: rms {rms:.2e} update {upd:.2e} max {mx:.2e}")
        assert rms <= RMS_CEIL["enc_layer"] and upd <= RMS_CEIL["enc_update"] and mx <= 3 * RMS_CEIL["enc_layer"], \
            (size, l, rms, upd, mx)
        x = got.clone()
    with capsys.disabled():
        report("whisper", "enc_layer", size, "; ".join(lines))


def run_encode(engine, clips, d):
    pcm, start, lens = upload(clips)
    out = Guarded((len(clips), SEQ, d), torch.float16, "cuda", GUARD)
    engine.whisper_encode(pcm, start, lens, len(clips), out.body)
    return out.check()


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
def test_decoder_layers_match_fp64(engine, size, capsys):
    """Every decoder layer from the start rows embed_tokens[sot] + embed_positions[0, 1], each fed the previous
    layer's kernel output and the kernel's fp16 encoder output of four different clips."""
    load(engine, size)
    sd, model = model_state(size)
    d = model.config.d_model
    clips = stage_clips()
    B = len(clips)
    enc = run_encode(engine, clips, d)
    x0 = sd["decoder.embed_tokens.weight"][SOT][None, :] + sd["decoder.embed_positions.weight"][:2]
    xd = x0.float().cuda()[None].repeat(B, 1, 1).contiguous()
    ein = Guarded(enc.shape, torch.float16, "cuda", GUARD, init=enc)
    lines = []
    for l in range(model.config.decoder_layers):
        xin = Guarded(xd.shape, torch.float32, "cuda", GUARD, init=xd)
        out = Guarded(xd.shape, torch.float32, "cuda", GUARD)
        engine.whisper_dec_layer(l, xin.body, ein.body, B, out.body)
        got = out.check()
        assert xin.intact_input() and ein.intact_input(), "an input or its guard was modified"
        with torch.no_grad():
            ref = dec_layer_ref(model, l, xd.double(), enc.double())
        rms, upd, mx = layer_metrics(got, xd, ref)
        lines.append(f"layer {l}: rms {rms:.2e} update {upd:.2e} max {mx:.2e}")
        assert rms <= RMS_CEIL["dec_layer"] and upd <= RMS_CEIL["dec_update"] and mx <= 3 * RMS_CEIL["dec_layer"], \
            (size, l, rms, upd, mx)
        xd = got.clone()
    with capsys.disabled():
        report("whisper", "dec_layer", size, "; ".join(lines))


# ------------------------------------------------------------------------------------------------ taps
TAP_SECONDS = [1.0, 10.0, 30.0, 31.0]
TAP_CASES = [(s, sec) for s in SIZES for sec in TAP_SECONDS]


@pytest.mark.gpu
@pytest.mark.parametrize("size,sec", TAP_CASES, ids=[f"{s}-{int(sec)}s" for s, sec in TAP_CASES])
def test_encode_and_forward_match_fp64(engine, size, sec, capsys):
    """fad_whisper_encode against encoder(features).last_hidden_state and fad_whisper_forward against
    last_hidden_state for decoder_input_ids [[sot, sot]], a music and a noise clip per batch."""
    load(engine, size)
    model = model_state(size)[1]
    d = model.config.d_model
    n = int(sec * 16000)
    clips = [make_clip("music", n, 3), make_clip("noise", n, 4)]
    feats = features64(clips, "cuda")
    with torch.no_grad():
        enc_ref = model.encoder(feats).last_hidden_state
        ids = torch.full((len(clips), 2), SOT, dtype=torch.long, device="cuda")
        fwd_ref = model(encoder_outputs=(enc_ref,), decoder_input_ids=ids).last_hidden_state
    enc = run_encode(engine, clips, d)
    fwd = engine.whisper_forward(*upload(clips))
    torch.cuda.synchronize()
    assert fwd.shape == (len(clips), 2, d) and bool(torch.isfinite(fwd).all())
    er, ec, _ = tap_metrics(enc, enc_ref)
    fr, fc, _ = tap_metrics(fwd, fwd_ref)
    with capsys.disabled():
        report("whisper", "taps", f"{size} {sec:g} s", f"encode rms {er:.2e} centred {ec:.2e}; forward rms {fr:.2e} centred {fc:.2e}")
    assert er <= RMS_CEIL["encode"] and ec <= RMS_CEIL["encode_c"], (er, ec)
    assert fr <= RMS_CEIL["forward"] and fc <= RMS_CEIL["forward_c"], (fr, fc)


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["tiny", "medium"])
def test_outputs_independent_of_batch(engine, size):
    """A clip alone, inside a batch and across a max_clips chunk boundary (n = max_clips + 1) gives bitwise the same
    encoder output and embedding: the clip max is an exact atomic max and no GEMM row reads another."""
    load(engine, size)
    d = model_state(size)[1].config.d_model
    clips = [make_clip("music" if i % 2 else "noise", 16000 * (2 + i), 10 + i) for i in range(MAX_CLIPS + 1)]
    clips[1] = square(48000)
    enc = run_encode(engine, clips, d)
    fwd = engine.whisper_forward(*upload(clips))
    for i, c in enumerate(clips):
        one = run_encode(engine, [c], d)
        assert torch.equal(one[0].view(torch.int16), enc[i].view(torch.int16)), f"encoder: clip {i} depends on its batch"
        f1 = engine.whisper_forward(*upload([c]))
        assert torch.equal(f1[0].view(torch.int16), fwd[i].view(torch.int16)), f"forward: clip {i} depends on its batch"
    again = engine.whisper_forward(*upload(clips))
    assert torch.equal(again.view(torch.int16), fwd.view(torch.int16)), "two identical calls differ"


# ---------------------------------------------------------------------------------------------------- rejections
D_TINY = 384


def _conv_call(**over):
    def call(engine, outs):
        a = dict(c=1, B=2, x="ok", cmax="ok", out="ok")
        a.update(over)
        x = Guarded((2, N_FRAMES, D_TINY), torch.float32, "cuda", GUARD)
        cm = Guarded((2,), torch.float32, "cuda", GUARD)
        o = Guarded((2, N_FRAMES, D_TINY), torch.float32, "cuda", GUARD)
        outs.extend([o, cm])
        engine.whisper_conv(a["c"], x.ptr(a["x"]), cm.ptr(a["cmax"]), a["B"], o.ptr(a["out"]))
    return call


def _enc_layer_call(**over):
    def call(engine, outs):
        a = dict(l=0, B=2, x="ok", out="ok")
        a.update(over)
        x = Guarded((2, SEQ, D_TINY), torch.float32, "cuda", GUARD, init=torch.zeros((2, SEQ, D_TINY), device="cuda"))
        o = Guarded((2, SEQ, D_TINY), torch.float32, "cuda", GUARD)
        outs.append(o)
        engine.whisper_enc_layer(a["l"], x.ptr(a["x"]), a["B"], o.ptr(a["out"]))
    return call


def _dec_layer_call(**over):
    def call(engine, outs):
        a = dict(l=0, B=2, x="ok", enc="ok", out="ok")
        a.update(over)
        x = Guarded((2, 2, D_TINY), torch.float32, "cuda", GUARD, init=torch.zeros((2, 2, D_TINY), device="cuda"))
        e = Guarded((2, SEQ, D_TINY), torch.float16, "cuda", GUARD, init=torch.zeros((2, SEQ, D_TINY), device="cuda"))
        o = Guarded((2, 2, D_TINY), torch.float32, "cuda", GUARD)
        outs.append(o)
        engine.whisper_dec_layer(a["l"], x.ptr(a["x"]), e.ptr(a["enc"]), a["B"], o.ptr(a["out"]))
    return call


def _clips_call(entry, **over):
    def call(engine, outs):
        a = dict(n=2, pcm="ok", start="ok", out="ok")
        a.update(over)
        pcm, start, lens = upload([make_clip("noise", 1600), make_clip("noise", 800)])
        if entry == "encode":
            o = Guarded((2, SEQ, D_TINY), torch.float16, "cuda", GUARD)
            fn = engine.whisper_encode
        else:
            o = Guarded((2 * N_FRAMES * 80 + 2,), torch.float32, "cuda", GUARD)
            fn = engine.whisper_logmel
        outs.append(o)
        fn(pcm if a["pcm"] == "ok" else None, start if a["start"] == "ok" else None, lens, a["n"],
           o.ptr(a["out"]))
    return call


REJECT = [
    ("conv c 2", _conv_call(c=2), "fad_whisper_conv: c must be in [0, 2)"),
    ("conv c -1", _conv_call(c=-1), "fad_whisper_conv: c must be in [0, 2)"),
    ("conv B 0", _conv_call(B=0), "fad_whisper_conv: B must be in [1, max_clips]"),
    ("conv B beyond max_clips", _conv_call(B=MAX_CLIPS + 1), "fad_whisper_conv: B must be in [1, max_clips]"),
    ("conv null x", _conv_call(x="null"), "fad_whisper_conv: null x or out"),
    ("conv null out", _conv_call(c=0, out="null"), "fad_whisper_conv: null x or out"),
    ("conv misaligned x", _conv_call(x="odd"), "fad_whisper_conv: x and out must be 16-byte aligned"),
    ("conv misaligned out", _conv_call(c=0, out="odd"), "fad_whisper_conv: x and out must be 16-byte aligned"),
    ("conv 0 null clip_max", _conv_call(c=0, cmax="null"), "fad_whisper_conv: c = 0 needs a 4-byte aligned clip_max"),
    ("conv before any load", on_fresh_engine(_conv_call()), "fad_whisper_conv: fad_whisper_load has not been called"),
    ("enc layer l 4", _enc_layer_call(l=4), "fad_whisper_enc_layer: l must be in [0, enc_layers)"),
    ("enc layer l -1", _enc_layer_call(l=-1), "fad_whisper_enc_layer: l must be in [0, enc_layers)"),
    ("enc layer B beyond max_clips", _enc_layer_call(B=MAX_CLIPS + 1), "fad_whisper_enc_layer: B must be in [1, max_clips]"),
    ("enc layer null out", _enc_layer_call(out="null"), "fad_whisper_enc_layer: null x or out"),
    ("enc layer misaligned x", _enc_layer_call(x="odd"), "fad_whisper_enc_layer: x and out must be 16-byte aligned"),
    ("enc layer before any load", on_fresh_engine(_enc_layer_call()), "fad_whisper_enc_layer: fad_whisper_load has not been called"),
    ("dec layer l 4", _dec_layer_call(l=4), "fad_whisper_dec_layer: l must be in [0, dec_layers)"),
    ("dec layer B 0", _dec_layer_call(B=0), "fad_whisper_dec_layer: B must be in [1, max_clips]"),
    ("dec layer null x", _dec_layer_call(x="null"), "fad_whisper_dec_layer: null x or out"),
    ("dec layer misaligned out", _dec_layer_call(out="odd"), "fad_whisper_dec_layer: x and out must be 16-byte aligned"),
    ("dec layer null enc_out", _dec_layer_call(enc="null"), "fad_whisper_dec_layer: enc_out must be a 16-byte aligned pointer"),
    ("dec layer misaligned enc_out", _dec_layer_call(enc="odd"), "fad_whisper_dec_layer: enc_out must be a 16-byte aligned pointer"),
    ("dec layer before any load", on_fresh_engine(_dec_layer_call()), "fad_whisper_dec_layer: fad_whisper_load has not been called"),
    ("encode no clips", _clips_call("encode", n=0), "fad_whisper_encode: n_clips must be positive"),
    ("encode null pcm", _clips_call("encode", pcm="null"), "fad_whisper_encode: null pcm, clip_start, clip_len or out"),
    ("encode null out", _clips_call("encode", out="null"), "fad_whisper_encode: null pcm, clip_start, clip_len or out"),
    ("encode before any load", on_fresh_engine(_clips_call("encode")), "fad_whisper_encode: fad_whisper_load has not been called"),
    ("logmel no clips", _clips_call("logmel", n=0), "fad_whisper_logmel: n_clips must be positive"),
    ("logmel null clip_start", _clips_call("logmel", start="null"), "fad_whisper_logmel: null pcm, clip_start, clip_len or out"),
    ("logmel null out", _clips_call("logmel", out="null"), "fad_whisper_logmel: null pcm, clip_start, clip_len or out"),
    ("logmel before any load", on_fresh_engine(_clips_call("logmel")), "fad_whisper_logmel: fad_whisper_load has not been called"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("call,message", [c[1:] for c in REJECT], ids=[c[0] for c in REJECT])
def test_stage_entries_reject_invalid_arguments(engine, call, message):
    """Arguments the launch cannot honour fail with their message, launch nothing and write nothing."""
    load(engine, "tiny")
    expect_rejected(engine, call, message, [])


# ------------------------------------------------------------------------------------------ CPU: the references
@pytest.mark.parametrize("size", SIZES)
def test_stage_composition_is_the_model(size):
    """Composing the stage references (GELU(conv1) and GELU(conv2) as float64 GEMMs, embed_positions, the encoder
    layers, encoder.layer_norm, the start rows, the decoder layers with the causal mask, decoder.layer_norm) reproduces
    WhisperModel(features, decoder_input_ids = [[sot, sot]]) in float64, and the fp16 rows of whisper_oracle.embed."""
    sd = ww.synthetic_whisper_state(0, size, layers=stack(size))
    model, fe = wo.build(sd, SOT)
    md = model.double()
    clip = synth.musiclike_clip(5, 2.0, 16000)
    feats = torch.from_numpy(wo.features(clip / 32768.0, fe)).double()[None]
    ids = torch.tensor([[SOT, SOT]])
    with torch.no_grad():
        want_enc = md.encoder(feats).last_hidden_state
        want = md(feats, decoder_input_ids=ids).last_hidden_state
        enc = md.encoder
        x = F.gelu(conv_mm(feats, enc.conv1.weight, enc.conv1.bias, 1, 1))
        x = F.gelu(conv_mm(x, enc.conv2.weight, enc.conv2.bias, 2, 1)).transpose(1, 2) + enc.embed_positions.weight
        for l in range(len(enc.layers)):
            x = enc_layer_ref(md, l, x)
        e = enc.layer_norm(x)
        xd = (sd["decoder.embed_tokens.weight"][SOT].double()[None, :] + sd["decoder.embed_positions.weight"][:2].double())[None]
        for l in range(len(md.decoder.layers)):
            xd = dec_layer_ref(md, l, xd, e)
        got = md.decoder.layer_norm(xd)
    assert (e - want_enc).abs().max().item() <= 1e-10 * want_enc.abs().max().item()
    assert (got - want).abs().max().item() <= 1e-10 * want.abs().max().item()
    model.float()
    rows = wo.embed(clip / 32768.0, model, fe, SOT).astype(np.float64)
    ref = got[0].numpy()
    assert rows.shape == ref.shape
    assert np.sqrt(((rows - ref) ** 2).mean() / (ref ** 2).mean()) < 1e-3


FE_LENGTHS = [1, 200, 16000, 480001]


@pytest.mark.parametrize("n", FE_LENGTHS)
def test_fp64_logmel_is_the_feature_extractor(n):
    """The float64 front-end restatement against transformers' WhisperFeatureExtractor (an fp32 computation): the
    same features at its fp32 noise level."""
    import transformers as tr
    clip = make_clip("music", n, 7)
    want = wo.features(clip / 32768.0, tr.WhisperFeatureExtractor()).astype(np.float64)
    got = features64([clip], "cpu")[0].numpy()
    err = np.abs(got - want)
    assert err.max() <= 1e-4 and err.mean() <= 2e-6, (err.max(), err.mean())


# digests of synthetic_whisper_state(0, size): the tests and the benchmark depend on these exact tensors
STATE_SHA256 = {
    "tiny": "d47dcb43eda79e91b8f8886cc5e96a4291544dda644b36e7e25bdc1dbddbd2f0",
    "base": "893afb1d644199ed7fc92b706cfe75d61cb0647bd2c066e061e8f899175abcec",
    "small": "29e9253a8d2fddb4f5a90d36008bdc4f17605c88456b92144406c5b77ee60724",
    "medium": "e5c8ce42c97eddeb591d9cf34adc68af17c01b9d56d11106d6e3362681c45c28",
    "large": "3f244bec0fd56355aef98f2b14984456d02181889b7f56964f93bd43cd5dd1ab",
}


@pytest.mark.parametrize("size", SIZES)
def test_default_synthetic_states_unchanged(size):
    """Without `layers` the seeded state is bitwise the one every earlier release generated (hashed tensor by tensor,
    so the 1.5 B parameters of large never sit in memory at once); with it, only the first layers are generated and
    the encoder prefix matches the full state."""
    h = hashlib.sha256()
    prefix, in_prefix = {}, True                         # everything drawn before encoder layer 1
    for k, v in ww.synthetic_whisper_tensors(0, size):
        h.update(k.encode())
        h.update(v.contiguous().numpy().tobytes())
        in_prefix = in_prefix and not k.startswith("encoder.layers.1.")
        if in_prefix:
            prefix[k] = v
    assert h.hexdigest() == STATE_SHA256[size]
    short = ww.synthetic_whisper_state(0, size, layers=(1, 2))
    assert ww.config_of(short)[2:4] == (1, 2)
    assert len(prefix) == 5 + 15 and all(torch.equal(short[k], v) for k, v in prefix.items())
