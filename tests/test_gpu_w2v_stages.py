"""The wav2vec family (w2v2, HuBERT, MERT, WavLM) one stage at a time, through the stage entries that call the forward's
own launch code (fad_w2v_normalize, fad_w2v_conv -> w2v_conv0 / w2v_conv, fad_w2v_posconv -> w2v_posconv, fad_w2v_layer
-> w2v_layer), and the whole forward tap by tap, at the clip lengths real files have.  References are transformers'
own modules (the reference's dependency) with the seeded synthetic weights, run in float64 on the GPU from exactly the
values the kernels read: feature_extractor.conv_layers[c], encoder.pos_conv_embed, encoder.layers[l] (WavLM layers get
layer 0's position bias), and the processor's normalisation restated in float64.  test_stage_composition_is_the_model
(CPU) pins that composing these references is the model.

Inputs and outputs sit in sentinel-NaN guarded buffers and the clips of a batch differ: an output left unwritten, a
guard overwritten or a value of the neighbouring clip shows up.  fad_w2v_conv fills the dead pitch rows of its input
with an fp16 NaN, so a valid output that reads one is non-finite.

Per-element bounds (float64, 1.001 margin), S = sum_j |w_j| |a_j| over the K = k Cin taps of an output:
  * normalize: out = (x - m) inv in fp32 with m, inv the fp32 roundings of the fp64 mean and 1 / sqrt(var + 1e-7):
        |d| <= 3 2^-23 |out| + 2^-24 inv |mean|  (the fp64 moments' own error included).  A wrong eps moves the +-1-LSB clip (var ~ 6e-10 << 1e-7) by far more.
  * GEMM conv (c >= 1, the positional conv), pre-activation: gpu_checks.gemm_bound, with r_a = 0 where the operand is
    the fp16 activation itself and 2^-11 where the kernel rounds it to fp16 (the positional conv's fp32 stream; the
    layer variant's conv 0, whose enc_im2col rounds the normalised waveform).
  * group variant conv 0 (CUDA cores, fp32 weights hi + lo, GroupNorm folded into (scale, shift) from fp64 moments):
        e = |scale| (10 2^-24 + 2^-20) S + 2^-23 (|y| + |shift|)
    (2^-20 S |scale| covers the hi + lo weight against the original, consistently in the conv and in its GroupNorm).
  * layer variant LayerNorm(512) over a row with conv errors e_i: gpu_checks.ln_bound.
  * GELU, fp32 or fp16 output: gpu_checks.gelu_out;  the positional conv's fp32 residual add: + 2^-24 |out|.
The layers (attention, two LayerNorms, two GEMMs with fp16 operands) and the whole forward are held to rms ceilings,
about 3x the level measured on the H100 (RMS_CEIL below), and the forward's taps also to a centred ceiling: under the
synthetic weights the hidden state is mostly a per-channel constant, and the per-frame fluctuation that FAD's covariance
measures is what the centred metric (per-(clip, channel) mean over frames removed from error and reference) sees.
"""
import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import synth, weights_w2v as ww
from gpu_checks import (Guarded, check_bound, expect_rejected, gelu_out, gemm_bound, layer_metrics, ln_bound,
                        on_fresh_engine, report, report_stats, tap_metrics)
from oracle import w2v_oracle as wo

GUARD = 4096
MAX_CLIPS = 2
KERNEL, STRIDE = ww.CONV_KERNEL, ww.CONV_STRIDE

# rms relative error ceilings (rms |kernel - fp64| / rms |fp64|), about 3x the largest level measured on an H100 80GB
# HBM3 (700 W) over the cases below:
#   conv group variant 2.3e-4 (max err / bound 0.994), layer variant 2.9e-4 (0.834), positional conv 9.9e-5 (0.056),
#   normalize 6.5e-7 (0.433), layer 2.7e-4 (its update out - x, layer_update: 3.2e-4), whole forward 8.4e-4 (centred
#   1.3e-3, mean error / fluctuation rms 2.1e-3, both largest at S = 2), long files 6.2e-4 (centred 9.7e-4)
RMS_CEIL = {"conv_group": 7e-4, "conv_layer": 9e-4, "posconv": 3e-4, "layer": 8e-4, "layer_update": 1e-3,
            "forward": 2.5e-3, "forward_c": 4e-3, "forward_m": 6e-3}

# name -> (weights arch, transformers family, sample rate); shortened stacks of 2 layers
MODELS = {"w2v2-base": (("w2v2", "base"), "w2v2", 16000), "hubert-large": (("hubert", "large"), "hubert", 16000),
          "wavlm-base": (("wavlm", "base"), "wavlm", 16000), "wavlm-large": (("wavlm", "large"), "wavlm", 16000),
          "MERT-v1-95M": (("mert", "v1-95M"), "hubert", 24000)}
LENGTHS = [400, 719, 720, 64000, 64010, 480000]


def frames(L):
    T = [L]
    for k, s in zip(KERNEL, STRIDE):
        T.append((T[-1] - k) // s + 1)
    return T


# ------------------------------------------------------------------------------------------------ references
def ref_normalize(pcm):
    """Wav2Vec2FeatureExtractor(do_normalize=True) in float64: pcm int16 [B, L] -> [B, L]"""
    x = pcm.double() / 32768.0
    m = x.mean(1, keepdim=True)
    return (x - m) / torch.sqrt(x.var(1, unbiased=False, keepdim=True) + 1e-7)


def position_bias(model, B, S):
    """layer 0's relative position bias, shaped as WavLMAttention passes it on to the later layers"""
    att = model.encoder.layers[0].attention
    return att.compute_bias(S, S).unsqueeze(0).repeat(B, 1, 1, 1).view(B * att.num_heads, S, S)


def run_layer(model, l, h, pb):
    layer = model.encoder.layers[l]
    return layer(h, position_bias=pb)[0] if pb is not None else layer(h)[0]


def is_stable(model):
    return bool(model.config.do_stable_layer_norm)


@torch.no_grad()
def ref_hidden_states(model, xn, wavlm):
    """float64 hidden_states[0 .. layers] of the model from the normalised waveform xn [B, L], composed of the modules
    the stage tests use."""
    h = xn[:, None]
    for conv in model.feature_extractor.conv_layers:
        h = conv(h)
    h = model.feature_projection(h.transpose(1, 2))
    h = h[0] if isinstance(h, tuple) else h
    enc = model.encoder
    h = h + enc.pos_conv_embed(h)
    if not is_stable(model):
        h = enc.layer_norm(h)
    hs = [h]
    pb = position_bias(model, h.shape[0], h.shape[1]) if wavlm else None
    for l in range(len(enc.layers)):
        h = run_layer(model, l, h, pb)
        hs.append(h)
    if is_stable(model):
        hs[-1] = enc.layer_norm(h)
    return hs


_MODELS = {}


def model_state(name, layers=2):
    """(state dict, float64 transformers model on the GPU) of the seed-0 synthetic weights, `layers` layers"""
    key = (name, layers)
    if key not in _MODELS:
        arch, family, sr = MODELS[name]
        a = dict(ww.ARCH[arch])
        a["layers"] = layers
        sd = ww.synthetic_w2v_state(0, **a)
        model, _ = wo.build(sd, family, sr)
        _MODELS[key] = (sd, model.double().to("cuda"))
    return _MODELS[key]


def load(engine, name, max_len, layers=2, max_clips=MAX_CLIPS):
    token = ("w2v-stage-test", name, layers, max_len, max_clips)
    if engine.owners.get("w2v") != token:
        sd = model_state(name, layers)[0]
        engine.w2v_load(ww.config_of(sd), ww.pack_w2v(sd), max_clips, max_len=max_len)
        engine.owners["w2v"] = token


# ------------------------------------------------------------------------------------------------- inputs
def sine30(n, sr):
    t = np.arange(n) / sr
    return np.round(16000 * np.sin(2 * np.pi * 30.0 * t)).astype(np.int16)


def clip_pair(case, L, sr):
    """two different clips of L samples"""
    sec = L / sr
    if case == 0:
        return [synth.musiclike_clip(L, sec, sr)[:L], sine30(L, sr)]
    return [synth.noise_clip(L + 1, sec, sr)[:L], np.zeros(L, np.int16)]


def pcm_tensor(clips):
    return torch.from_numpy(np.stack([np.resize(c, len(clips[0])) for c in clips])).cuda()


# ------------------------------------------------------------------------------------------------ normalize
def lsb_noise(n, seed):
    return np.random.default_rng(seed).integers(-1, 2, n).astype(np.int16)


def square(n):
    return np.where((np.arange(n) // 37) % 2 == 0, 32767, -32768).astype(np.int16)


def dc_clip(n, seed):
    return np.clip(synth.noise_clip(seed, n / 16000, 16000)[:n].astype(np.int32) // 8 + 12000, -32768, 32767).astype(np.int16)


@pytest.mark.gpu
@pytest.mark.parametrize("L", [400, 64000, 480000])
def test_normalize_matches_fp64(engine, L, capsys):
    """Music, noise, a DC offset, silence, +-1-LSB noise and a full-scale square wave in one batch: every clip is
    normalised with its own moments, within the fp32 bound of the module docstring."""
    clips = [synth.musiclike_clip(1, L / 16000, 16000)[:L], synth.noise_clip(2, L / 16000, 16000)[:L], dc_clip(L, 3),
             np.zeros(L, np.int16), lsb_noise(L, 4), square(L)]
    clips = [np.resize(c, L) for c in clips]
    pcm = torch.from_numpy(np.stack(clips)).cuda()
    out = Guarded((len(clips), L), torch.float32, "cuda", GUARD)
    engine.w2v_normalize(pcm, len(clips), L, out.body)
    got = out.check()
    ref = ref_normalize(pcm)
    x = pcm.double() / 32768.0
    mean = x.mean(1, keepdim=True)
    inv = 1.0 / torch.sqrt(x.var(1, unbiased=False, keepdim=True) + 1e-7)
    bound = (3 * 2.0 ** -23 * ref.abs() + 2.0 ** -24 * inv * mean.abs()) * 1.001 + 1e-30
    stats = {}
    for i, name in enumerate(("music", "noise", "dc", "silence", "lsb", "square")):
        check_bound("normalize", f"L {L} {name}", got[i], ref[i], bound[i], stats, RMS_CEIL)
    assert bool((got[3] == 0).all())
    report_stats(capsys, "w2v", stats, f"L {L}")


# ---------------------------------------------------------------------------------------------------- convs
def conv_sums(a, w, stride, groups=1, padding=0, drop_last=False):
    """(S, sum |w|, sum |a|, K) of gpu_checks.gemm_bound for a conv1d; a [B, Cin, T] float64, w [Cout, Cin/g, k]"""
    conv = lambda u, v: torch.nn.functional.conv1d(u, v, None, stride, padding, 1, groups)
    S = conv(a.abs(), w.abs())
    sa = conv(a.abs(), torch.ones_like(w))
    if drop_last:
        S, sa = S[..., :-1], sa[..., :-1]
    return S, w.abs().flatten(1).sum(1)[None, :, None], sa, w.shape[1] * w.shape[2]


@torch.no_grad()
def conv_reference(model, c, x):
    """x float64 [B, Cin, T_in] -> (module output [B, T_out, 512], per-element bound)"""
    mod = model.feature_extractor.conv_layers[c]
    w, b = mod.conv.weight, mod.conv.bias if mod.conv.bias is not None else torch.zeros(512, dtype=torch.float64, device=x.device)
    y = torch.nn.functional.conv1d(x, w, b, STRIDE[c])
    layer_variant = hasattr(mod, "layer_norm") and isinstance(mod.layer_norm, torch.nn.LayerNorm)
    if layer_variant:
        e = gemm_bound(*conv_sums(x, w, STRIDE[c]), b, y, r_a=2.0 ** -11 if c == 0 else 0.0)
        g, beta = mod.layer_norm.weight[None, :, None], mod.layer_norm.bias[None, :, None]
        y, e = ln_bound(y, e, g, beta, 1)
    elif c == 0:
        gn = mod.layer_norm                                                # GroupNorm(512, 512)
        S = torch.nn.functional.conv1d(x.abs(), w.abs(), None, STRIDE[c])
        yc = y - y.mean(2, keepdim=True)
        scale = gn.weight[None, :, None] / torch.sqrt(yc.square().mean(2, keepdim=True) + 1e-5)
        yn = yc * scale + gn.bias[None, :, None]
        shift = yn - (y - b[None, :, None]) * scale
        e = scale.abs() * (10 * 2.0 ** -24 + 2.0 ** -20) * S + 2.0 ** -23 * (yn.abs() + shift.abs())
        y = yn
    else:
        e = gemm_bound(*conv_sums(x, w, STRIDE[c]), b, y)
    want, bound = gelu_out(y, e, c < 6)
    bound = bound * 1.001
    ref = mod(x)
    assert (ref - want).abs().max().item() <= 1e-9 * max(1.0, want.abs().max().item()), "the bound's restatement is not the module"
    return ref.transpose(1, 2), bound.transpose(1, 2)


def run_conv(engine, c, x, B, L):
    """x (conv 0: fp32 [B, L]; else fp16 [B, T_c, 512]) guarded -> the checked compact output"""
    T = frames(L)
    xin = Guarded(x.shape, x.dtype, "cuda", GUARD, init=x)
    out = Guarded((B, T[c + 1], 512), torch.float32 if c == 6 else torch.float16, "cuda", GUARD)
    engine.w2v_conv(c, xin.body, B, L, out.body)
    got = out.check()
    assert xin.intact_input(), "the input or its guard was modified"
    return got


def check_conv_chain(engine, name, L, sr, capsys):
    """every conv c = 0..6 at length L, each fed the previous conv's kernel output (the values the forward feeds it)"""
    model = model_state(name)[1]
    kind = "conv_layer" if is_stable(model) else "conv_group"
    stats = {}
    for case in (0, 1):
        pcm = pcm_tensor(clip_pair(case, L, sr))
        x = ref_normalize(pcm).float()
        for c in range(7):
            got = run_conv(engine, c, x, 2, L)
            xin = x.double()[:, None] if c == 0 else x.double().transpose(1, 2)
            ref, bound = conv_reference(model, c, xin)
            check_bound(kind, f"{name} conv {c} L {L} case {case}", got, ref, bound, stats, RMS_CEIL)
            x = got
    report_stats(capsys, "w2v", stats, f"{name} L {L}")


CONV_CASES = [("w2v2-base", L, 16000) for L in LENGTHS] + [("w2v2-base", 720000, 24000)] + \
             [("hubert-large", L, 16000) for L in LENGTHS]


@pytest.mark.gpu
@pytest.mark.parametrize("name,L,sr", CONV_CASES, ids=[f"{n}-{L}" for n, L, _ in CONV_CASES])
def test_convs_match_fp64(engine, name, L, sr, capsys):
    """Both feature-encoder variants (group: w2v2-base, also MERT's at 24 kHz; layer: hubert-large), every conv, at the
    shortest clip (400 .. 719: one frame), 720, 64 000 (one dead pitch row per level) and 64 010 (63/32/17/9/5/3/2),
    and the 30-s batch maximum; music against a 30 Hz sine and noise against silence."""
    load(engine, name, max(L, 480000))
    check_conv_chain(engine, name, L, sr, capsys)


# ------------------------------------------------------------------------------------------- positional conv
def stream_input(B, S, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    scale = torch.tensor([1.0, 0.3], device="cuda")[torch.arange(B, device="cuda") % 2]
    off = torch.randn((B, 1, d), generator=g, device="cuda") * 0.5
    return (torch.randn((B, S, d), generator=g, device="cuda") * scale[:, None, None] + off).contiguous()


@torch.no_grad()
def posconv_reference(model, x):
    pc = model.encoder.pos_conv_embed
    xd = x.double()
    ref = xd + pc(xd)
    w = pc.conv.weight
    xt = xd.transpose(1, 2)
    y = torch.nn.functional.conv1d(xt, w, pc.conv.bias, 1, 64, 1, 16)[..., :-1]
    e = gemm_bound(*conv_sums(xt, w, 1, groups=16, padding=64, drop_last=True), pc.conv.bias, y, r_a=2.0 ** -11)
    _, e = gelu_out(y, e, False)
    bound = (e.transpose(1, 2) + 2.0 ** -24 * ref.abs()) * 1.001
    return ref, bound


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w2v2-base", "hubert-large"])
def test_posconv_matches_fp64(engine, name, capsys):
    """d = 768 (cg = 48) and 1024 (cg = 64) at S = 1, 2, 199, 1499: windows near a clip's edges must see zeros, not the
    neighbouring clip (whose stream differs)."""
    load(engine, name, 480000)
    model = model_state(name)[1]
    d = model.config.hidden_size
    stats = {}
    for S in (1, 2, 199, 1499):
        x = stream_input(2, S, d, S)
        xin = Guarded(x.shape, torch.float32, "cuda", GUARD, init=x)
        out = Guarded(x.shape, torch.float32, "cuda", GUARD)
        engine.w2v_posconv(xin.body, 2, S, out.body)
        got = out.check()
        assert xin.intact_input()
        ref, bound = posconv_reference(model, x)
        check_bound("posconv", f"{name} S {S}", got, ref, bound, stats, RMS_CEIL)
    report_stats(capsys, "w2v", stats, name)


# ------------------------------------------------------------------------------------------------- layers
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w2v2-base", "hubert-large", "wavlm-base", "wavlm-large"])
def test_layers_match_fp64(engine, name, capsys):
    """post-LN (w2v2-base), pre-LN (hubert-large), WavLM post-LN and pre-LN, both layers (layer 1 takes layer 0's
    position bias) at S = 1, 199, 1499."""
    load(engine, name, 480000)
    model = model_state(name)[1]
    d, wavlm = model.config.hidden_size, name.startswith("wavlm")
    worst = (0.0, "")
    for S in (1, 199, 1499):
        x = stream_input(2, S, d, 7 * S)
        if not is_stable(model):                          # post-LN: the stream entering a layer is a LayerNorm's output
            x = torch.nn.functional.layer_norm(x, (d,))
        for l in range(2):
            xin = Guarded(x.shape, torch.float32, "cuda", GUARD, init=x)
            out = Guarded(x.shape, torch.float32, "cuda", GUARD)
            engine.w2v_layer(l, xin.body, 2, S, out.body)
            got = out.check()
            assert xin.intact_input()
            with torch.no_grad():
                ref = run_layer(model, l, x.double(), position_bias(model, 2, S) if wavlm else None)
            rms, upd, mx = layer_metrics(got, x, ref)
            if upd > worst[0]:
                worst = (upd, f"S {S} layer {l}, rms rel err {rms:.3e}, max |err| / max |ref| {mx:.3e}")
            assert rms <= RMS_CEIL["layer"], (name, S, l, rms)
            assert upd <= RMS_CEIL["layer_update"], (name, S, l, upd)
            assert mx <= 3 * RMS_CEIL["layer"], (name, S, l, mx)
    with capsys.disabled():
        report("w2v", "layer", name, f"largest rms rel err of the update {worst[0]:.3e} ({worst[1]})")


# ------------------------------------------------------------------------------------------------ forward
FWD_CASES = [(n, L) for n in ("w2v2-base", "hubert-large", "wavlm-base", "wavlm-large") for L in LENGTHS] + \
            [("MERT-v1-95M", L) for L in (600, 1079, 1080, 96000, 96015, 720000)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,L", FWD_CASES, ids=[f"{n}-{L}" for n, L in FWD_CASES])
def test_forward_taps_match_fp64(engine, name, L, capsys):
    """Every tap hidden_states[k] of a 2-layer stack against the float64 model, two different clips per batch.  The
    centred metrics need S > 1 frames."""
    sr = MODELS[name][2]
    load(engine, name, max(L, 480000))
    model = model_state(name)[1]
    pcm = pcm_tensor(clip_pair(0, L, sr))
    with torch.no_grad():
        hs = ref_hidden_states(model, ref_normalize(pcm), name.startswith("wavlm"))
    S = frames(L)[7]
    lines = []
    for k, ref in enumerate(hs):
        got = engine.w2v_forward(pcm, k)
        assert got.shape == (2, S, model.config.hidden_size) and bool(torch.isfinite(got).all())
        rms, centred, mean_err = tap_metrics(got, ref)
        lines.append(f"tap {k}: rms {rms:.2e}" + (f" centred {centred:.2e} mean/fluct {mean_err:.2e}" if S > 1 else ""))
        assert rms <= RMS_CEIL["forward"], (k, rms)
        if S > 1:
            assert centred <= RMS_CEIL["forward_c"], (k, centred)
            assert mean_err <= RMS_CEIL["forward_m"], (k, mean_err)
    with capsys.disabled():
        report("w2v", "forward", f"{name} L {L}", "; ".join(lines))


@pytest.mark.gpu
def test_long_file_reload_matches_fp64(engine, capsys):
    """A 31-s file takes the >30-s path (the engine reloaded with max_clips = 1, max_len = L), a 10-s one the batch path;
    both at tap 1 against the float64 model."""
    ml = fk.Wav2VecFamilyModel("w2v2", "w2v2-base-1", 1, 16000, max_clips=2)
    ml.load_model()
    clips = [synth.musiclike_clip(31, 31.0, 16000), synth.noise_clip(10, 10.0, 16000)]
    got = ml.embed_pcm_batch(clips)
    assert ml.max_clips == 1
    sd = ww.synthetic_w2v_state(0, layers=1)
    model = wo.build(sd, "w2v2")[0].double().cuda()
    for g, c in zip(got, clips):
        pcm = torch.from_numpy(c[None]).cuda()
        with torch.no_grad():
            ref = ref_hidden_states(model, ref_normalize(pcm), False)[1]
        rms, centred, mean_err = tap_metrics(torch.as_tensor(np.asarray(g, dtype=np.float32)).cuda()[None], ref)
        with capsys.disabled():
            report("w2v", "long", f"{len(c)} samples", f"rms {rms:.2e} centred {centred:.2e} mean/fluct {mean_err:.2e}")
        assert rms <= RMS_CEIL["forward"] and centred <= RMS_CEIL["forward_c"] and mean_err <= RMS_CEIL["forward_m"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w2v2-base", "hubert-large", "wavlm-base"])
def test_forward_independent_of_batch(engine, name):
    """A clip alone, inside a batch and across a max_clips chunk boundary (n = max_clips + 1) is bitwise the same: the
    conv-0 GroupNorm moments are summed in a fixed order."""
    load(engine, name, 480000)
    clips = [synth.musiclike_clip(i, 4.0, 16000) for i in range(MAX_CLIPS + 1)]
    pcm = torch.from_numpy(np.stack(clips)).cuda()
    for tap in (0, 2):
        batch = engine.w2v_forward(pcm, tap)
        for i in range(MAX_CLIPS + 1):
            one = engine.w2v_forward(pcm[i:i + 1].contiguous(), tap)
            assert torch.equal(one[0].view(torch.int16), batch[i].view(torch.int16)), f"tap {tap}: clip {i} depends on its batch"
        again = engine.w2v_forward(pcm, tap)
        assert torch.equal(again.view(torch.int16), batch.view(torch.int16)), "two identical calls differ"


# ---------------------------------------------------------------------------------------------------- rejections
def _conv_call(**over):
    def call(engine, outs):
        a = dict(c=1, B=2, L=16000, x="ok", out="ok")
        a.update(over)
        x = Guarded((2, 16000), torch.float32, "cuda", GUARD)
        o = Guarded((2, 16000), torch.float32, "cuda", GUARD)
        outs.append(o)
        engine.w2v_conv(a["c"], x.ptr(a["x"]), a["B"], a["L"], o.ptr(a["out"]))
    return call


def _stream_call(entry, **over):
    def call(engine, outs):
        a = dict(l=0, B=2, S=10, x="ok", out="ok")
        a.update(over)
        x = Guarded((2, 10, 768), torch.float32, "cuda", GUARD, init=torch.zeros((2, 10, 768), device="cuda"))
        o = Guarded((2, 10, 768), torch.float32, "cuda", GUARD)
        outs.append(o)
        if entry == "layer":
            engine.w2v_layer(a["l"], x.ptr(a["x"]), a["B"], a["S"], o.ptr(a["out"]))
        else:
            engine.w2v_posconv(x.ptr(a["x"]), a["B"], a["S"], o.ptr(a["out"]))
    return call


def _normalize_call(**over):
    def call(engine, outs):
        a = dict(n=2, L=400, out="ok")
        a.update(over)
        pcm = torch.zeros((2, 400), dtype=torch.int16, device="cuda")
        o = Guarded((2, 400), torch.float32, "cuda", GUARD)
        outs.append(o)
        engine.w2v_normalize(pcm, a["n"], a["L"], o.ptr(a["out"]))
    return call


FRAMES_MAX = frames(32000)[7]
REJECT = [
    ("conv c 7", _conv_call(c=7), "fad_w2v_conv: c must be in [0, 7)"),
    ("conv c -1", _conv_call(c=-1), "fad_w2v_conv: c must be in [0, 7)"),
    ("conv L 399", _conv_call(L=399), "fad_w2v_conv: L must be at least 400 samples"),
    ("conv L beyond max_len", _conv_call(L=32001), "fad_w2v_conv: L must be at most max_len"),
    ("conv B beyond max_clips", _conv_call(B=MAX_CLIPS + 1), "fad_w2v_conv: B must be in [1, max_clips]"),
    ("conv B 0", _conv_call(B=0), "fad_w2v_conv: B must be in [1, max_clips]"),
    ("conv null x", _conv_call(x="null"), "fad_w2v_conv: null x or out"),
    ("conv misaligned x", _conv_call(x="odd"), "fad_w2v_conv: x and out must be 16-byte aligned"),
    ("conv misaligned out", _conv_call(c=0, out="odd"), "fad_w2v_conv: x and out must be 16-byte aligned"),
    ("conv before any load", on_fresh_engine(_conv_call()), "fad_w2v_conv: fad_w2v_load has not been called"),
    ("posconv S 0", _stream_call("posconv", S=0), "fad_w2v_posconv: S must be in [1, frames(max_len)]"),
    ("posconv S beyond max_len", _stream_call("posconv", S=FRAMES_MAX + 1), "fad_w2v_posconv: S must be in [1, frames(max_len)]"),
    ("posconv B beyond max_clips", _stream_call("posconv", B=MAX_CLIPS + 1), "fad_w2v_posconv: B must be in [1, max_clips]"),
    ("posconv misaligned out", _stream_call("posconv", out="odd"), "fad_w2v_posconv: x and out must be 16-byte aligned"),
    ("posconv before any load", on_fresh_engine(_stream_call("posconv")), "fad_w2v_posconv: fad_w2v_load has not been called"),
    ("layer l 2", _stream_call("layer", l=2), "fad_w2v_layer: l must be in [0, layers)"),
    ("layer l -1", _stream_call("layer", l=-1), "fad_w2v_layer: l must be in [0, layers)"),
    ("layer S beyond max_len", _stream_call("layer", S=FRAMES_MAX + 1), "fad_w2v_layer: S must be in [1, frames(max_len)]"),
    ("layer B beyond max_clips", _stream_call("layer", B=MAX_CLIPS + 1), "fad_w2v_layer: B must be in [1, max_clips]"),
    ("layer null x", _stream_call("layer", x="null"), "fad_w2v_layer: null x or out"),
    ("layer misaligned x", _stream_call("layer", x="odd"), "fad_w2v_layer: x and out must be 16-byte aligned"),
    ("layer before any load", on_fresh_engine(_stream_call("layer")), "fad_w2v_layer: fad_w2v_load has not been called"),
    ("normalize no clips", _normalize_call(n=0), "fad_w2v_normalize: n_clips and L must be positive"),
    ("normalize L 0", _normalize_call(L=0), "fad_w2v_normalize: n_clips and L must be positive"),
    ("normalize null out", _normalize_call(out="null"), "fad_w2v_normalize: null pcm or out"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("call,message", [c[1:] for c in REJECT], ids=[c[0] for c in REJECT])
def test_stage_entries_reject_invalid_arguments(engine, call, message):
    """Arguments the launch cannot honour fail with their message, launch nothing and write nothing."""
    load(engine, "w2v2-base", 32000)
    expect_rejected(engine, call, message, [])


# ------------------------------------------------------------------------------------------ CPU: the references
@pytest.mark.parametrize("name", list(MODELS))
def test_stage_composition_is_the_model(name):
    """Composing the stage references (the float64 normalisation, conv_layers[c], feature_projection, pos_conv_embed with
    its SamePad drop, the layers with layer 0's WavLM position bias, the stable-LN final LayerNorm) reproduces the
    transformers model the oracle drives, at every tap: float64 against float64, and the fp16 taps oracle/w2v_oracle.embed
    returns."""
    arch, family, sr = MODELS[name]
    a = dict(ww.ARCH[arch])
    a["layers"] = 2
    sd = ww.synthetic_w2v_state(0, **a)
    model, fe = wo.build(sd, family, sr)
    clip = synth.musiclike_clip(5, 0.5, sr)
    pcm = torch.from_numpy(clip[None])
    md = model.double()
    xn = ref_normalize(pcm)
    with torch.no_grad():
        want = md(xn, output_hidden_states=True).hidden_states
    x32 = fe(clip / 32768.0, sampling_rate=sr, return_tensors="np")["input_values"]
    assert np.abs(x32 - xn.numpy()).max() <= 1e-5 * np.abs(xn.numpy()).max()
    with torch.no_grad():
        got = ref_hidden_states(md, xn, family == "wavlm")
    assert len(got) == len(want) == 3
    for k, (g, w) in enumerate(zip(got, want)):
        assert (g - w).abs().max().item() <= 1e-10 * w.abs().max().item(), (name, k)
    model.float()
    for k in range(3):
        e = wo.embed(clip / 32768.0, model, fe, k, sr).astype(np.float64)
        ref = got[k][0].numpy()
        assert e.shape == ref.shape
        assert np.sqrt(((e - ref) ** 2).mean() / (ref ** 2).mean()) < 1e-3, (name, k)
