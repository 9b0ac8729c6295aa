"""The Encodec encoders (encodec-emb, 24 kHz causal; encodec-emb-48k, non-causal with GroupNorm) one stage at a time,
through the stage entries that call the forward's own launch code (fad_encodec_conv -> enc_conv, fad_encodec_lstm ->
enc_lstm), and the whole forward at the clip lengths real files have, against the float64 restatement in
oracle/encodec_oracle.py (pinned to transformers' port by tests/test_encodec_oracle.py).  References run in float64
torch on the GPU from the exact fp32 inputs the kernels read.

Inputs live inside NaN-filled guard regions of at least (max padding + 2) time steps on each side, and neighbouring
clips of a batch differ: a tap read outside its clip shows up as NaN or as a wrong value in the output.  Outputs live
inside sentinel-filled buffers: every element must be written and no guard touched.

Conv bound (gpu_checks.gemm_bound, 1.001 margin), per output element y = b + sum_j w_j a_j over the K = k' Cin taps of
the GEMM row (k' = k, or k + (P - 1) stride when P time steps share a row): a_j = ELU(x) or x at the padded index, which
the kernel rounds to fp16 (r_a = 2^-11); S and sum_j |a_j| come from the same padded conv on |a| and |w|, and on |a| and
ones.  GroupNorm(1, C) after the conv (48 kHz): gpu_checks.ln_bound over each sample's N values, 1.001 margin.
An rms ceiling of about 3x the level measured on the H100 sits on top (RMS_CEIL below).  The LSTM (recurrent state
an fp16 hi/lo pair) and the whole forward are held to rms and max-abs ceilings of the same kind.
"""
import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import weights_encodec as we
from gpu_checks import (Guarded, check_bound, expect_rejected, gemm_bound, ln_bound, on_fresh_engine, report,
                        report_stats, rms_rel)
from oracle import encodec_oracle as eo

pytestmark = pytest.mark.gpu

GUARD = 256
MAX_CHUNK = 8 * 48000

# rms relative error (rms |kernel - fp64| / rms |fp64|), about 3x the largest level measured on an H100 80GB HBM3
# (700 W) over the cases below:
#   conv 3.9e-4 (the largest is a 1-sample input), conv + GroupNorm 2.6e-4, LSTM 8.1e-6 (max abs 6.3e-5 at TF 75),
#   whole forward 1.0e-3 (max |err| / max |ref| 1.1e-3, the fp16 embedding included)
# The largest max |err| / bound measured: conv 0.79, conv + GroupNorm 0.33.
RMS_CEIL = {"conv": 1.2e-3, "conv_gn": 8e-4, "lstm": 2.5e-5, "forward": 3e-3}
LSTM_MAX_ABS = 2e-4
FORWARD_MAX_ABS_REL = 3.5e-3                                     # max |err| / max |ref| of a whole embedding


def layer_table(variant):
    """(Cin, Cout, k, stride) per conv in the load order of fad_encodec_load"""
    t = [(2 if variant == "48k" else 1, 32, 7, 1)]
    ch = 32
    for r in we.RATIOS:
        t += [(ch, ch // 2, 3, 1), (ch // 2, ch, 1, 1), (ch, ch, 1, 1), (ch, 2 * ch, 2 * r, r)]
        ch *= 2
    t.append((512, 128, 7, 1))
    return t


_STATES = {}


def state(variant, dev):
    """seed-0 synthetic weights (what EncodecEmbModel loads under FADTK_SYNTHETIC) on the CPU and on the GPU"""
    if variant not in _STATES:
        sd = we.synthetic_encodec_state(0, variant)
        _STATES[variant] = (sd, {k: v.to(dev) for k, v in sd.items()})
    return _STATES[variant]


def load(engine, variant, max_chunk=MAX_CHUNK):
    """Load the variant's weights unless this module's load of them still holds the engine's Encodec slot."""
    token = ("encodec-stage-test", variant, max_chunk)
    if engine.owners.get("encodec") != token:
        engine.encodec_load(we.pack_encodec(state(variant, engine.torch_device)[0]), max_chunk, variant)
        engine.owners["encodec"] = token


@pytest.fixture(scope="module")
def dev(engine):
    return engine.torch_device


# ------------------------------------------------------------------------------------------------------ one conv
def conv_reference(x, sdg, layer, elu_in, groupnorm, K):
    """x fp32 [B, T_in, Cin] -> (y fp64 [B, T_out, Cout], per-element bound; see the module docstring)"""
    prefix, stride = eo.conv_layers(sdg)[layer]
    xt = x.double().transpose(1, 2)
    a = torch.nn.functional.elu(xt) if elu_in else xt
    y = eo.conv_layer(xt, sdg, layer, elu_in, False)
    w = eo.effective_weight(sdg, prefix).double()
    b = sdg[prefix + ".conv.bias"].double()
    causal = eo.is_causal(sdg)
    S = eo._sconv(a.abs(), w.abs(), torch.zeros_like(b), stride, causal)
    sum_a = eo._sconv(a.abs(), torch.ones_like(w), torch.zeros_like(b), stride, causal)
    sum_w = w.abs().flatten(1).sum(1)[None, :, None]
    e = gemm_bound(S, sum_w, sum_a, K, b, y, r_a=2.0 ** -11) * 1.001
    if groupnorm:
        g = sdg[prefix + ".norm.weight"].double()[None, :, None]
        beta = sdg[prefix + ".norm.bias"].double()[None, :, None]
        y, e = ln_bound(y, e, g, beta, (1, 2))
        e = e * 1.001
    return y.transpose(1, 2), e.transpose(1, 2)


def run_conv(engine, layer, x, variant, elu_in, groupnorm):
    """x fp32 [B, T_in, Cin] copied into a NaN-guarded buffer -> the checked output [B, T_out, Cout]"""
    B, T_in, cin = x.shape
    _, cout, k, s = layer_table(variant)[layer]
    xin = Guarded(x.shape, torch.float32, x.device, 16 * 512, init=x)   # covers the widest padding (12 steps) of 512 channels
    out = Guarded((B, -(-T_in // s), cout), torch.float32, x.device, GUARD)
    engine.encodec_conv(layer, xin.body, B, T_in, out.body, elu_in=elu_in, groupnorm=groupnorm)
    got = out.check()
    assert xin.intact_input(), "the input or its guard was modified"
    return got


def conv_input(dev, seed, B, T_in, cin):
    """B clips of different scales and offsets (unit-ish, half of them negative: ELU matters)"""
    g = torch.Generator(device=dev).manual_seed(seed)
    scale = torch.tensor([1.0, 0.3, 2.0, 0.7], device=dev)[torch.arange(B, device=dev) % 4]
    off = torch.tensor([0.0, 0.4, -0.3, 0.1], device=dev)[torch.arange(B, device=dev) % 4]
    return (torch.randn((B, T_in, cin), generator=g, device=dev) * scale[:, None, None] + off[:, None, None]).contiguous()


def check_conv(engine, dev, variant, layer, T_in, B, elu_in, groupnorm, seed, stats):
    cin, cout, k, s = layer_table(variant)[layer]
    P = we.time_pack(cout)
    T_out = -(-T_in // s)
    packed = P > 1 and T_out % P == 0
    K = (k + (P - 1) * s if packed else k) * cin
    x = conv_input(dev, seed, B, T_in, cin)
    got = run_conv(engine, layer, x, variant, elu_in, groupnorm)
    ref, bound = conv_reference(x, state(variant, dev)[1], layer, elu_in, groupnorm, K)
    what = f"{variant} layer {layer} T_in {T_in} B {B} elu {int(elu_in)} gn {int(groupnorm)}"
    check_bound("conv_gn" if groupnorm else "conv", what, got, ref, bound, stats, RMS_CEIL)
    return got, packed


def conv_lengths(variant, layer):
    """(long lengths: T_out a multiple of 8, then T_in = 1, 3, 5, 7 mod 8), (short lengths 1 .. k + 2, which reach past
    every padding of the layer: 1, 2, the padding and the padding + 1)"""
    _, _, k, s = layer_table(variant)[layer]
    return [64 * s, 200 * s] + [64 * s + r for r in (1, 3, 5, 7)], list(range(1, k + 3))


LAYERS = [(v, l) for v in ("24k", "48k") for l in range(18)]


@pytest.mark.parametrize("variant,layer", LAYERS, ids=[f"{v}-L{l}" for v, l in LAYERS])
def test_conv_matches_fp64(engine, dev, variant, layer, capsys):
    """Every conv at lengths that take the time-packed weights (T_out % P == 0) and the plain ones, at every short
    length up to past its padding, with and without the input ELU, and (48 kHz) with its GroupNorm."""
    load(engine, variant)
    longs, shorts = conv_lengths(variant, layer)
    cout = layer_table(variant)[layer][1]
    stats, paths = {}, set()
    for T_in in longs + shorts:
        for elu_in in (False, True):
            for gn in ((False, True) if variant == "48k" else (False,)):
                B = 2 if T_in * 2 <= MAX_CHUNK else 1
                _, packed = check_conv(engine, dev, variant, layer, T_in, B, elu_in, gn, 1000 * layer + T_in, stats)
                paths.add(packed)
    if we.time_pack(cout) > 1:
        assert paths == {True, False}, "the lengths do not cover both the packed and the plain weights"
    report_stats(capsys, "encodec", stats, f"{variant} layer {layer}")


@pytest.mark.parametrize("variant,layer", LAYERS, ids=[f"{v}-L{l}" for v, l in LAYERS])
def test_conv_short_single_clip(engine, dev, variant, layer):
    """One clip at every short length: a tap read outside the clip can only land in the input's NaN guard."""
    load(engine, variant)
    stats = {}
    for T_in in conv_lengths(variant, layer)[1]:
        for gn in ((False, True) if variant == "48k" else (False,)):
            check_conv(engine, dev, variant, layer, T_in, 1, True, gn, 7 * T_in + layer, stats)


def test_conv_clip_independent_of_batch(engine, dev):
    """A clip's conv output is bitwise the same alone and at the end of a batch (packed and plain, short and long)."""
    for variant in ("24k", "48k"):
        load(engine, variant)
        for layer in (0, 4, 5, 16, 17):
            s = layer_table(variant)[layer][3]
            for T_in in (3, 64 * s, 64 * s + 3):
                x = conv_input(dev, layer + T_in, 5, T_in, layer_table(variant)[layer][0])
                for gn in ((False, True) if variant == "48k" else (False,)):
                    full = run_conv(engine, layer, x, variant, True, gn)
                    one = run_conv(engine, layer, x[4:].contiguous(), variant, True, gn)
                    assert torch.equal(one, full[4:]), f"{variant} layer {layer} T_in {T_in}: a clip depends on its batch"


# ---------------------------------------------------------------------------------------------------------- LSTM
@pytest.mark.parametrize("TF", [1, 2, 75])
def test_lstm_matches_fp64(engine, dev, TF, capsys):
    """515 clips cross the 512-clip group boundary; the second group must not inherit the first group's state."""
    for variant in ("24k", "48k"):
        load(engine, variant)
        n = 515
        g = torch.Generator(device=dev).manual_seed(TF)
        z = (torch.randn((n, TF, 512), generator=g, device=dev) * (0.5 + torch.rand((n, 1, 1), generator=g, device=dev))).contiguous()
        zin = Guarded(z.shape, torch.float32, dev, GUARD, init=z)
        out = Guarded(z.shape, torch.float32, dev, GUARD)
        engine.encodec_lstm(zin.body, n, TF, out.body)
        got = out.check()
        ref = eo.lstm(z, state(variant, dev)[1])
        rms = rms_rel(got, ref)
        mx = (got.double() - ref).abs().max().item()
        rms_last = rms_rel(got[512:], ref[512:])
        with capsys.disabled():
            report("encodec", "lstm", f"{variant} TF {TF} clips {n}", f"rms rel err {rms:.3e} (second group {rms_last:.3e}), max abs {mx:.3e}")
        assert rms <= RMS_CEIL["lstm"] and rms_last <= RMS_CEIL["lstm"], (rms, rms_last)
        assert mx <= LSTM_MAX_ABS, mx
        again = Guarded(z.shape, torch.float32, dev, GUARD)
        engine.encodec_lstm(zin.body, n, TF, again.body)
        assert torch.equal(again.check(), got), "two identical calls differ"
        one = Guarded((1, TF, 512), torch.float32, dev, GUARD)
        engine.encodec_lstm(z[513:514].contiguous(), 1, TF, one.body)
        assert torch.equal(one.check(), got[513:514]), "a clip's LSTM output depends on its group"


# ---------------------------------------------------------------------------------------------------- whole forward
def pcm_clip(seed, n):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 24000.0
    x = 0.15 * rng.standard_normal(n) + 0.3 * np.sin(2 * np.pi * (110.0 + 30 * (seed % 7)) * t)
    return np.round(32767.0 * np.clip(x, -1.0, 1.0)).astype(np.int16)


def forward_reference(pcm, sdg, variant, dev):
    """fp64 [T / 320 frames, 128] of one int16 clip as the reference embeds it (48 kHz: stereo 1-s segments)"""
    x = torch.from_numpy(pcm.astype(np.float64) / 32768.0).to(dev).view(1, 1, -1)
    if variant == "24k":
        return eo.encoder(x, sdg, torch.float64)[0].T
    x = x.expand(1, 2, -1)
    return torch.cat([eo.encoder(x[:, :, o:o + 48000], sdg, torch.float64)[0].T for o in range(0, x.shape[-1], 48000)])


def check_forward(ml, variant, dev, lengths, capsys):
    sdg = state(variant, dev)[1]
    worst = 0.0
    for T in lengths:
        clips = [pcm_clip(T, T), pcm_clip(T + 1, T)]
        got = ml.embed_equal_length(clips)
        for g, c in zip(got, clips):
            ref = forward_reference(c, sdg, variant, dev)
            assert g.shape == ref.shape == (-(-T // 320), 128), (g.shape, ref.shape)
            assert bool(torch.isfinite(g).all()), f"{variant} T {T}: non-finite embedding"
            rms = rms_rel(g, ref)
            mx = ((g.double() - ref).abs().max() / ref.abs().max()).item()
            worst = max(worst, rms)
            with capsys.disabled():
                report("encodec", "forward", f"{variant} T {T}", f"rms rel err {rms:.3e}, max abs err / max |ref| {mx:.3e}")
            assert rms <= RMS_CEIL["forward"], (T, rms)
            assert mx <= FORWARD_MAX_ABS_REL, (T, mx)
    return worst


def test_forward_24k_matches_fp64(engine, dev, capsys):
    """encodec-emb on whole files at 1 .. 24001 samples: the conv inputs of clips up to 1920 samples (80 ms) get
    shorter than their padding somewhere in the stack; 319 .. 321 and 1919 .. 1921 straddle a frame."""
    ml = fk.EncodecEmbModel('24k', max_chunk_samples=MAX_CHUNK)
    ml.load_model()
    check_forward(ml, "24k", dev, [1, 7, 319, 320, 321, 1919, 1920, 1921, 24001], capsys)


def test_forward_48k_matches_fp64(engine, dev, capsys):
    """encodec-emb-48k on files of 48000 k + r samples: the remainder r is its own segment, short up to 960 samples."""
    ml = fk.EncodecEmbModel('48k', max_chunk_samples=MAX_CHUNK)
    ml.load_model()
    check_forward(ml, "48k", dev, [48000 + r for r in (1, 5, 960, 961, 47999)] + [2 * 48000 + 5], capsys)


@pytest.mark.parametrize("variant", ["24k", "48k"])
def test_embedding_independent_of_batch(engine, variant):
    """With 24 000-sample conv chunks, 515 clips of 0.25 s run in 129 conv chunks of 4 clips and two LSTM groups: every
    clip's embedding is bitwise what it is alone (the cache is filled one length group at a time)."""
    sr = 24000 if variant == "24k" else 48000
    ml = fk.EncodecEmbModel(variant, max_chunk_samples=24000)
    ml.load_model()
    n = sr // 4
    clips = [pcm_clip(i, n) for i in range(515)]
    batch = ml.embed_equal_length(clips)
    for i in (0, 5, 511, 513):
        one = ml.embed_equal_length([clips[i]])[0]
        assert torch.equal(one.view(torch.int16), batch[i].view(torch.int16)), f"clip {i} differs inside the batch"


# ------------------------------------------------------------------------------------------------------- rejections
def _conv_call(**over):
    def call(engine, outs):
        a = dict(layer=1, B=2, T_in=16, gn=0, x="ok", out="ok")
        a.update(over)
        dev = engine.torch_device
        x = Guarded((2, 16, 32), torch.float32, dev, GUARD, init=torch.zeros((2, 16, 32), device=dev))
        o = Guarded((2, 16, 32), torch.float32, dev, GUARD)
        outs.append(o)
        engine.encodec_conv(a["layer"], x.ptr(a["x"]), a["B"], a["T_in"], o.ptr(a["out"]), groupnorm=a["gn"])
    return call


def _lstm_call(**over):
    def call(engine, outs):
        a = dict(n=2, TF=3, z="ok", out="ok")
        a.update(over)
        dev = engine.torch_device
        z = Guarded((2, 3, 512), torch.float32, dev, GUARD, init=torch.zeros((2, 3, 512), device=dev))
        o = Guarded((2, 3, 512), torch.float32, dev, GUARD)
        outs.append(o)
        engine.encodec_lstm(z.ptr(a["z"]), a["n"], a["TF"], o.ptr(a["out"]))
    return call


REJECT = [
    # id, variant loaded, call, message
    ("conv layer 18", "24k", _conv_call(layer=18), "fad_encodec_conv: layer must be in [0, 18)"),
    ("conv layer -1", "48k", _conv_call(layer=-1), "fad_encodec_conv: layer must be in [0, 18)"),
    ("conv T_in 0", "24k", _conv_call(T_in=0), "fad_encodec_conv: T_in must be positive"),
    ("conv B 0", "24k", _conv_call(B=0), "fad_encodec_conv: B must be in [1, 4096]"),
    ("conv B 4097", "24k", _conv_call(B=4097, T_in=1), "fad_encodec_conv: B must be in [1, 4096]"),
    ("conv beyond the chunk", "24k", _conv_call(T_in=MAX_CHUNK), "fad_encodec_conv: B * T_in must be at most max_chunk_samples"),
    ("conv groupnorm at 24k", "24k", _conv_call(gn=1), "fad_encodec_conv: groupnorm needs the 48 kHz model"),
    ("conv null x", "48k", _conv_call(x="null"), "fad_encodec_conv: null x or out"),
    ("conv null out", "24k", _conv_call(out="null"), "fad_encodec_conv: null x or out"),
    ("conv misaligned x", "24k", _conv_call(x="odd"), "fad_encodec_conv: x and out must be 16-byte aligned"),
    ("conv misaligned out", "48k", _conv_call(out="odd", gn=1), "fad_encodec_conv: x and out must be 16-byte aligned"),
    ("conv before any load", None, on_fresh_engine(_conv_call()), "fad_encodec_conv: fad_encodec_load has not been called"),
    ("lstm no clips", "24k", _lstm_call(n=0), "fad_encodec_lstm: n_clips and TF must be positive"),
    ("lstm TF 0", "48k", _lstm_call(TF=0), "fad_encodec_lstm: n_clips and TF must be positive"),
    ("lstm TF beyond the chunk", "24k", _lstm_call(TF=MAX_CHUNK // 320 + 1),
     "fad_encodec_lstm: TF must be at most the frames of max_chunk_samples"),
    ("lstm null z", "24k", _lstm_call(z="null"), "fad_encodec_lstm: null z or out"),
    ("lstm misaligned out", "24k", _lstm_call(out="odd"), "fad_encodec_lstm: z and out must be 16-byte aligned"),
    ("lstm misaligned z", "48k", _lstm_call(z="odd"), "fad_encodec_lstm: z and out must be 16-byte aligned"),
    ("lstm before any load", None, on_fresh_engine(_lstm_call()), "fad_encodec_lstm: fad_encodec_load has not been called"),
]


@pytest.mark.parametrize("variant,call,message", [c[1:] for c in REJECT], ids=[c[0] for c in REJECT])
def test_stage_entries_reject_invalid_arguments(engine, variant, call, message):
    """Arguments the launch cannot honour fail with their message, launch nothing and write nothing."""
    if variant is not None:
        load(engine, variant)
    expect_rejected(engine, call, message, [])
