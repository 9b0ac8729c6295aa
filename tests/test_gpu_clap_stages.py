"""CLAP-LAION (HTSAT-tiny and HTSAT-base) one stage at a time, through the stage entries that call fad_clap_forward's
own launch code (fad_clap_logmel -> clap_logmel_kernel, fad_clap_patch_embed -> clap_patch_embed, fad_clap_block ->
clap_block, fad_clap_merge -> clap_merge, fad_clap_head -> clap_head), and the whole forward at real clip lengths.
References are oracle/clap_oracle.py (pinned to transformers' ClapAudioModelWithProjection by test_clap_oracle.py),
run in float64 on the GPU from exactly the values the kernels read, and a float64 restatement of the front end.
test_stage_composition_is_the_network (CPU) pins that composing these references is clap_oracle.network.

Inputs and outputs sit in sentinel-NaN guarded buffers and the windows of a batch differ (music, noise, silence, a
full-scale square wave with runs of +32767 and -32768): an output left unwritten, a guard overwritten or a value of the
neighbouring window shows up.

Per-element bounds (float64, u = 2^-24, gamma_n = n u / (1 - n u)):
  * front end, BatchNorm-ed log-mel of clap_logmel_kernel against the float64 STFT of the int16-round-tripped samples
    (centre, reflect, periodic Hann 1024, hop 480), the Slaney mel (50 Hz - 14 kHz), 10 log10(clamp(., 1e-10)) and
    the packed fp32 BatchNorm scale s / shift b.  The kernel's windowed samples a_n carry 2u |a_n| (rounded Hann table,
    product).  Its 512-point complex FFT of z_n = a_2n + i a_2n+1 runs 11 levels (two radix-4 stages = 4 add levels,
    the 16-point twiddles, the 32-point twiddles, 5 radix-2 shuffle levels), each a butterfly with fp32 twiddles of
    error mu <= 2u, so by Higham (Accuracy and Stability of Numerical Algorithms, 2nd ed., Thm 24.2) with
    eta = mu + gamma_4 (sqrt 2 + mu):
        ||dZ||_2 <= (2u + 11 eta / (1 - 11 eta)) ||Z||_2,   ||Z||_2 = sqrt(512) ||a||_2.
    The real-split post step X_k = (Z_k + conj Z_512-k) / 2 - i W^k (Z_k - conj Z_512-k) / 2 has |X_k| <=
    |Z_k| + |Z_512-k|, so it at most doubles the norm of dZ and adds 2 eta + 2u of its own:
        E = 1.01 (2 ||dZ||_2 + 2 (2 eta + 2u) ||Z||_2)  bounds |dX_k| for every bin k of the frame.
    Power p = re^2 + im^2:  |dp_k| <= 2 |X_k| E + E^2 + 2u (|X_k| + E)^2.  The mel band sums the fp32-rounded weights w
    by an fma chain of at most 32 taps:  |dm| <= (1 + u) sum w dp + (u + gamma_32) sum w (p + dp) + 1e-15 sum w p.
    A symmetric |err| <= bound cannot hold where the round-off exceeds the signal, so the kernel's value is held to the
    interval [10 log10(max(m - dm, 1e-10)), 10 log10(max(m + dm, 1e-10))] carried through x s + b, widened by the
    clamp's fp32 rounding (5.8e-8 dB), log10f (2 ulp) and the x 10 and BatchNorm roundings.  A silent frame has
    m = dm = 0: its interval is the clamp value alone.
  * patch embed, from the kernel's own frame pool and plan: the fp32 source coordinate s_t = fl(1000 t / 1023) is off
    by ds_t (computed exactly here); the cubic kernel (A = -0.75) has slope at most 1.35, so the four taps move by at
    most 4 * 1.35 ds_t M_t with M_t the largest |tap|; the fp32 coefficients (Horner, terms up to 36) carry 256 u each
    and the 4-tap fma chain gamma_4 * 1.5 M_t.  The 16-tap conv adds sum |w| e_pix + gamma_17 (|b| + sum |w| |pix|),
    then gpu_checks.ln_bound (with gamma_8 |y| for the LayerNorm's own sums).
  * patch merge: ln_bound over 4C from the exact fp32 stream (gamma_24 |y| for the sums), rounded to fp16
    (r_a = 2^-11), then gpu_checks.gemm_bound with K = 4C and b = 0, plus sum |w| e_ln (1 + 2^-11).
  * head: ln_bound per token (gamma_40 |y|), the fp32 64-token mean (gamma_16), two fp32 dot-product chains
    gamma_(K/32+6) sum |w| |x| + sum |w| e (ReLU is 1-Lipschitz), then the L2 normalisation: with n = ||h||,
    dn <= ||e||_2 + n (gamma_72 / 2 + 2u), |d out| <= (e + |out| dn) / (n - dn) + u |out|; the fp16 store adds
    2^-11 (|out| + e) + 2^-25.
Every bound carries a 1.001 margin.  The Swin blocks (attention, LayerNorms, GEMMs with fp16 operands), the head and
the whole forward are held to rms ceilings, about 3x the largest level measured on the H100 (RMS_CEIL below); each block also on
its update out - x, which the stream it adds to would otherwise hide.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fadtk_b200 import _native, synth, weights_clap as wc
from gpu_checks import (Guarded, check_bound, expect_rejected, gemm_bound, layer_metrics, ln_bound, on_fresh_engine,
                        report, report_stats)
from oracle import clap_oracle as co

GUARD = 4096
MAX_CHUNKS = 4
VARIANTS = list(wc.VARIANTS)
SR, HOP, N_FFT, FRAMES = 48000, 480, 1024, 1001
U = 2.0 ** -24


def gamma(n):
    return n * U / (1 - n * U)


# rms relative error ceilings (rms |kernel - fp64| / rms |fp64|), about 3x the largest level measured on an H100 80GB
# HBM3 (700 W) over the cases below, both variants alike to within 15 %:
#   Swin block 2.4e-4 (its update out - x 2.8e-4, max |err| / max |ref| 3.3e-4), head 2.2e-4 (the fp16 rounding of
#   unit rows: 2^-11 / sqrt(3) = 2.8e-4 rms), fad_clap_forward 2.3e-4 with 1 - cosine at most 4e-8 over 111 rows.
# The per-element bounds hold with room: max err / bound 0.87 for the front end (bins next to the clamp), 0.015 for the
# patch embed, 0.15 for the merges, 0.07 for the head (rms 4.6e-7 for the patch embed, 2.2e-4 for the merges).
# The head's bound is dominated by its fp16 store, so a wrong token mean (63 of 64 tokens: rms 1.4e-3) only shows in
# its rms.  "block_max" bounds a block's max |err| / max |ref| (measured 3.3e-4).
RMS_CEIL = {"block": 8e-4, "block_update": 9e-4, "block_max": 1e-3, "head": 7e-4, "forward": 7e-4}
COS_GAP = 1.2e-7                                      # 1 - cosine of every forward row against the float64 network


# ------------------------------------------------------------------------------------------------ models
_STATE = {}


def state(variant):
    """(state dict fp32 CPU, packed tensors, state dict float64 on the GPU) of the seed-0 synthetic weights"""
    if variant not in _STATE:
        sd = wc.synthetic_clap_state(0, variant)
        _STATE[variant] = (sd, wc.pack_clap(sd), {k: v.double().cuda() for k, v in sd.items()})
    return _STATE[variant]


def load(engine, variant, max_chunks=MAX_CHUNKS):
    token = ("clap-stage-test", variant, max_chunks)
    if engine.owners.get("clap") != token:
        engine.clap_load(state(variant)[1], max_chunks)
        engine.owners["clap"] = token


def block_geometry(variant):
    """[(stage, block in stage, res, C, heads, shift)] of every Swin block, stage-major"""
    embed, depths = wc.VARIANTS[variant]
    out, res, C = [], 64, embed
    for s, (depth, heads) in enumerate(zip(depths, co.HEADS)):
        for j in range(depth):
            out.append((s, j, res, C, heads, co.WINDOW // 2 if j % 2 == 1 and res > co.WINDOW else 0))
        res, C = res // 2, C * 2
    return out


# ------------------------------------------------------------------------------------------------- inputs
def square(n):
    """full scale: +32767 / -32768 in runs of 37 samples"""
    return np.where((np.arange(n) // 37) % 2 == 0, 32767, -32768).astype(np.int16)


def make_clip(kind, n, seed=0):
    if kind == "silence":
        return np.zeros(n, np.int16)
    if kind == "square":
        return square(n)
    sec = max(n, SR // 10) / SR
    base = synth.musiclike_clip(seed, sec, SR) if kind == "music" else synth.noise_clip(seed, sec, SR)
    return base[:n].copy()


def plan_of(clips):
    off = np.concatenate([[0], np.cumsum([len(c) for c in clips])]).astype(np.int64)
    return _native.Engine.clap_plan_frames(off)


def to_dev(plan):
    return {k: torch.from_numpy(v).cuda() for k, v in plan.items() if k != "rows_per_clip"}


def pcm_of(clips):
    return torch.from_numpy(np.concatenate(clips)).cuda()


def run_pool(engine, clips, plan):
    """kernel frame pool fp32 [n_pool, 64], guarded"""
    d = to_dev(plan)
    n = len(plan["pool_start"])
    out = Guarded((n, 64), torch.float32, "cuda", GUARD)
    engine.clap_pool(pcm_of(clips), d["pool_start"], d["pool_valid"], d["pool_frame"], n, out.body)
    return out.check("frame pool")


# ------------------------------------------------------------------------------------------ front end, fp64
_MEL = {}


def mel_weights(device):
    """the Slaney filter bank [64, 513], float64"""
    if device not in _MEL:
        _MEL[device] = torch.from_numpy(co.mel_filterbank()).to(device)
    return _MEL[device]


def window_frames(clip, device="cuda"):
    """the Hann-windowed frames [n_windows, 1001, 1024] (float64) of the reference's int16-round-tripped windows"""
    q = co.quantize_like_reference(clip.astype(np.float64) / 32768.0)
    ch = torch.from_numpy(co.chunks_of(q)).to(device, torch.float64)
    xp = F.pad(ch[:, None], (N_FFT // 2, N_FFT // 2), mode="reflect")[:, 0]
    n_ = torch.arange(N_FFT, dtype=torch.float64, device=device)
    hann = 0.5 - 0.5 * torch.cos(2 * math.pi * n_ / N_FFT)
    return xp.unfold(1, N_FFT, HOP)[:, :FRAMES] * hann


def ref_mel(clip, device="cuda", bound=False):
    """float64 mel power m [n_windows, 1001, 64] of one clip (and dm, the bound of the module docstring)"""
    fr = window_frames(clip, device)
    X = torch.fft.rfft(fr, dim=-1)
    A = X.abs()
    p = A.square()
    W = mel_weights(device)
    m = p @ W.T
    if not bound:
        return m
    mu = 2 * U
    eta = mu + gamma(4) * (math.sqrt(2) + mu)
    zn = math.sqrt(512) * fr.norm(dim=-1, keepdim=True)
    dz = (2 * U + 11 * eta / (1 - 11 * eta)) * zn
    E = 1.01 * (2 * dz + 2 * (2 * eta + 2 * U) * zn)
    dp = 2 * A * E + E.square() + 2 * U * (A + E).square()
    dm = (1 + U) * (dp @ W.T) + (U + gamma(32)) * ((p + dp) @ W.T) + 1e-15 * m
    return m, dm


CLAMP_DB = 10 * abs(math.log10(float(np.float32(1e-10))) + 10)


def logmel_interval(m, dm, s, b):
    """(midpoint, half width + rounding slack) of the kernel's BatchNorm-ed value, and where the interval reaches the
    clamp"""
    lo = 10 * torch.log10(torch.clamp(m - dm, min=1e-10))
    hi = 10 * torch.log10(torch.clamp(m + dm, min=1e-10))
    v = 10 * torch.log10(torch.clamp(m, min=1e-10))
    ya, yb = lo * s + b, hi * s + b
    mid, half = (ya + yb) / 2, (ya - yb).abs() / 2
    slack = s.abs() * (CLAMP_DB + 4 * 2.0 ** -23 * (v.abs() + 1e-3)) + 2 * U * ((v * s).abs() + b.abs()) + 2.0 ** -40
    return mid, (half + slack) * 1.001, (m - dm) <= 1e-10


FRONT_BATCHES = {
    # one sample (reflect of a lone sample, then zeros); the hop edge; the frames just short of one second
    "short": [("music", 1), ("noise", 479), ("square", 47999), ("silence", 48000)],
    # exactly 1 s and one sample more (a second window of one sample); exactly 10 s
    "edges": [("music", 48000), ("noise", 48001), ("square", 480000)],
    # 10 s + 1 sample; 25 s: windows share pool frames; a silent clip next to them
    "long": [("music", 480001), ("noise", 1200000), ("silence", 96000)],
}


@pytest.mark.gpu
@pytest.mark.parametrize("batch", list(FRONT_BATCHES))
def test_logmel_matches_fp64(engine, batch, capsys):
    """fad_clap_logmel's frame pool, gathered through fad_clap_plan_frames' frame_index window by window, against the
    float64 front end within the interval bound of the module docstring; silent frames sit exactly at the clamp."""
    load(engine, "tiny")
    pk = state("tiny")[1]
    s, b = pk[0].double().cuda(), pk[1].double().cuda()
    clips = [make_clip(k, n, i) for i, (k, n) in enumerate(FRONT_BATCHES[batch])]
    plan = plan_of(clips)
    pool = run_pool(engine, clips, plan)
    fi = torch.from_numpy(plan["frame_index"]).cuda().long()
    got_all = pool[fi]                                                   # [n_windows, 1001, 64]
    stats, lines, row = {}, [], 0
    clamp_value = None
    for (kind, n), clip, rows in zip(FRONT_BATCHES[batch], clips, plan["rows_per_clip"]):
        m, dm = ref_mel(clip, bound=True)
        assert m.shape[0] == rows
        got = got_all[row:row + rows]
        row += rows
        mid, bound, at_clamp = logmel_interval(m, dm, s, b)
        check_bound("logmel", f"{kind} {n}", got, mid, bound, stats, {})
        lines.append(f"{kind} {n}: {at_clamp.double().mean().item():.2%} of bins reach the clamp")
        silent = (m == 0)
        if bool(silent.any()):
            # every silent frame of a bin holds the same bits, 10 log10f(1e-10f) s + b, in every clip
            hi = torch.where(silent, got, -math.inf).reshape(-1, 64).amax(0)
            lo = torch.where(silent, got, math.inf).reshape(-1, 64).amin(0)
            seen = silent.reshape(-1, 64).any(0)
            assert torch.equal(hi[seen], lo[seen]), f"{kind} {n}: silent frames differ"
            if clamp_value is None:
                clamp_value = torch.full_like(hi, math.nan)
            both = seen & ~torch.isnan(clamp_value)
            assert torch.equal(hi[both], clamp_value[both]), f"{kind} {n}: clamp value differs between clips"
            clamp_value = torch.where(seen, hi, clamp_value)
    assert row == got_all.shape[0]
    report_stats(capsys, "clap", stats, batch)
    with capsys.disabled():
        report("clap", "logmel", batch, "; ".join(lines))


# ----------------------------------------------------------------------------------------------- patch embed
STAGE_CLIPS = [("music", 48000), ("noise", 24000), ("silence", 48000), ("square", 48000)]   # one window each


def stage_clips():
    return [make_clip(k, n, i) for i, (k, n) in enumerate(STAGE_CLIPS)]


def cubic_w(x):
    """torch's cubic convolution weights (A = -0.75) of the four taps at fraction x, float64"""
    A = -0.75

    def near(t):
        return ((A + 2) * t - (A + 3)) * t * t + 1

    def far(t):
        return ((A * t - 5 * A) * t + 8 * A) * t - 4 * A
    return [far(x + 1), near(x), near(1 - x), far(2 - x)]


def fold(x):
    """[B, 1024, 64] resized log-mel -> [B, 1, 256, 256] image (clap_oracle.fold_image without the resize)"""
    b = x.shape[0]
    return x.reshape(b, 4, 256, 64).permute(0, 1, 3, 2).reshape(b, 1, 256, 256)


@torch.no_grad()
def patch_embed_reference(lm, sd64, ln_sum=8):
    """BatchNorm-ed log-mel [B, 1001, 64] (float64) -> (stream entering block 0 [B, 4096, E], bound)"""
    img = co.fold_image(lm)
    t = torch.arange(1024, dtype=torch.float64)
    s_exact = t * 1000.0 / 1023.0
    s32 = torch.from_numpy((np.arange(1024, dtype=np.float32) * np.float32(1000.0)) / np.float32(1023.0)).double()
    ds = (s32 - s_exact).abs().to(lm.device)
    i0 = torch.floor(s_exact).long()
    taps = torch.stack([(i0 - 1 + k).clamp(0, FRAMES - 1) for k in range(4)]).to(lm.device)   # [4, 1024]
    M = lm.abs()[:, taps, :].amax(1)                                                           # [B, 1024, 64]
    e_pix = M * (4 * 1.35 * ds[None, :, None] + 4 * 256 * U + gamma(4) * 1.5)
    e_img = fold(e_pix)
    w, bias = sd64["patch_embed.proj.weight"], sd64["patch_embed.proj.bias"]
    y = F.conv2d(img, w, bias, stride=4)
    e = F.conv2d(e_img, w.abs(), None, stride=4) + gamma(17) * (bias.abs()[None, :, None, None]
                                                               + F.conv2d(img.abs(), w.abs(), None, stride=4))
    y = y.flatten(2).transpose(1, 2)
    e = e.flatten(2).transpose(1, 2) + gamma(ln_sum) * y.abs()
    out, bnd = ln_bound(y, e, sd64["patch_embed.norm.weight"], sd64["patch_embed.norm.bias"], -1)
    return out, bnd * 1.001


def run_patch_embed(engine, pool, plan):
    fi = plan["frame_index"]
    B = fi.shape[0]
    E = wc.VARIANTS[engine.owners["clap"][1]][0]
    pin = Guarded(pool.shape, torch.float32, "cuda", GUARD, init=pool)
    fin = Guarded(fi.shape, torch.float32, "cuda", GUARD)                 # an int32 buffer behind a float32 sentinel
    fin.body.view(torch.int32).copy_(torch.from_numpy(fi))
    fin.init = fin.body.clone()
    out = Guarded((B, 4096, E), torch.float32, "cuda", GUARD)
    engine.clap_patch_embed(pin.body, pool.shape[0], fin.body, B, out.body)
    got = out.check("patch embed")
    assert pin.intact_input() and fin.guards_intact() and torch.equal(fin.body.view(torch.int32), fin.init.view(torch.int32)), \
        "an input or its guard was modified"
    return got


# ------------------------------------------------------------------------------------------- stage chain
_CHAIN = {}


def chain(engine, variant):
    """Every stage on the GPU, each fed the previous stage's kernel output: {"lm": BatchNorm-ed log-mel [B, 1001, 64]
    gathered from the kernel's pool, "x0": patch embed, "blocks": [(blk, x in, out)], "merges": [(s, x in, out)],
    "final": the stream leaving the last block}"""
    load(engine, variant)
    if variant in _CHAIN:
        return _CHAIN[variant]
    clips = stage_clips()
    plan = plan_of(clips)
    pool = run_pool(engine, clips, plan)
    x = run_patch_embed(engine, pool, plan)
    B = x.shape[0]
    res = {"lm": pool[torch.from_numpy(plan["frame_index"]).cuda().long()].double(), "x0": x, "blocks": [], "merges": []}
    geo = block_geometry(variant)
    _, depths = wc.VARIANTS[variant]
    for blk, (s, j, r, C, heads, shift) in enumerate(geo):
        xin = Guarded(x.shape, torch.float32, "cuda", GUARD, init=x)
        out = Guarded(x.shape, torch.float32, "cuda", GUARD)
        engine.clap_block(blk, xin.body, B, out.body)
        got = out.check(f"block {blk}")
        assert xin.intact_input(), "the input or its guard was modified"
        res["blocks"].append((blk, x, got.clone()))
        x = got.clone()
        if j == depths[s] - 1 and s < 3:
            xin = Guarded(x.shape, torch.float32, "cuda", GUARD, init=x)
            out = Guarded((B, x.shape[1] // 4, 2 * x.shape[2]), torch.float32, "cuda", GUARD)
            engine.clap_merge(s, xin.body, B, out.body)
            got = out.check(f"merge {s}")
            assert xin.intact_input(), "the input or its guard was modified"
            res["merges"].append((s, x, got.clone()))
            x = got.clone()
    res["final"] = x
    _CHAIN[variant] = res
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_patch_embed_matches_fp64(engine, variant, capsys):
    """fad_clap_patch_embed from the kernel's own frame pool and plan (every window touches the time clamp at t = 0
    and t = 1023), four different windows in one batch, per element."""
    ch = chain(engine, variant)
    sd64 = state(variant)[2]
    ref, bound = patch_embed_reference(ch["lm"], sd64)
    stats = {}
    for i, (kind, n) in enumerate(STAGE_CLIPS):
        check_bound("patch_embed", f"{variant} {kind} {n}", ch["x0"][i], ref[i], bound[i], stats, {})
    report_stats(capsys, "clap", stats, variant)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_blocks_match_fp64(engine, variant, capsys):
    """Every Swin block (res 64, 32, 16, 8; shifted blocks at res >= 16), each fed the stream the GPU produced for the
    block before it, against float64 clap_oracle.swin_block on that same input."""
    ch = chain(engine, variant)
    sd64 = state(variant)[2]
    geo = block_geometry(variant)
    lines, worst = [], [0.0, 0.0, 0.0]
    for blk, x, got in ch["blocks"]:
        s, j, res, C, heads, shift = geo[blk]
        with torch.no_grad():
            ref = co.swin_block(x.double(), sd64, f"layers.{s}.blocks.{j}.", res, heads, shift)
        rms, upd, mx = layer_metrics(got, x, ref)
        worst = [max(a, b) for a, b in zip(worst, (rms, upd, mx))]
        lines.append(f"{blk} (res {res}{' shifted' if shift else ''}): rms {rms:.2e} update {upd:.2e} max {mx:.2e}")
        assert rms <= RMS_CEIL["block"] and upd <= RMS_CEIL["block_update"] and mx <= RMS_CEIL["block_max"], \
            (variant, blk, rms, upd, mx)
    with capsys.disabled():
        report("clap", "block", variant, "; ".join(lines))
        report("clap", "block", variant, f"largest rms {worst[0]:.3e} update {worst[1]:.3e} max/max {worst[2]:.3e}")


@torch.no_grad()
def merge_reference(x, sd64, s, res):
    """stream [B, res^2, C] (float64 of the kernel's fp32) -> (merged [B, res^2 / 4, 2 C], bound)"""
    pre = f"layers.{s}.downsample."
    b, n, c = x.shape
    xv = x.view(b, res, res, c)
    xc = torch.cat([xv[:, 0::2, 0::2], xv[:, 1::2, 0::2], xv[:, 0::2, 1::2], xv[:, 1::2, 1::2]], -1).view(b, -1, 4 * c)
    yn, e_ln = ln_bound(xc, gamma(24) * xc.abs(), sd64[pre + "norm.weight"], sd64[pre + "norm.bias"], -1)
    W = sd64[pre + "reduction.weight"]
    y = yn @ W.T
    S = yn.abs() @ W.abs().T
    sum_w = W.abs().sum(1)[None, :, None]
    sum_a = yn.abs().sum(-1, keepdim=True).transpose(1, 2)
    zero = torch.zeros(W.shape[0], dtype=torch.float64, device=x.device)
    e = gemm_bound(S.transpose(1, 2), sum_w, sum_a, 4 * c, zero, y.transpose(1, 2), r_a=2.0 ** -11).transpose(1, 2)
    e = e + (e_ln * (1 + 2.0 ** -11)) @ W.abs().T
    return y, e * 1.001


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_merges_match_fp64(engine, variant, capsys):
    """All three patch merges, each from the stream the GPU produced for it, per element."""
    ch = chain(engine, variant)
    sd64 = state(variant)[2]
    stats = {}
    assert [s for s, _, _ in ch["merges"]] == [0, 1, 2]
    for s, x, got in ch["merges"]:
        with torch.no_grad():
            want = co.patch_merge(x.double(), sd64, f"layers.{s}.downsample.", 64 >> s)
        ref, bound = merge_reference(x.double(), sd64, s, 64 >> s)
        assert (ref - want).abs().max().item() <= 1e-10 * want.abs().max().item()
        check_bound("merge", f"{variant} merge {s}", got, ref, bound, stats, {})
    report_stats(capsys, "clap", stats, variant)


@torch.no_grad()
def head_reference(x, sd64):
    """stream leaving the last block [B, 64, 8 E] -> (embedding [B, 512], bound)"""
    D = x.shape[-1]
    yn, e = ln_bound(x, gamma(40) * x.abs(), sd64["norm.weight"], sd64["norm.bias"], -1)
    pooled = yn.mean(1)
    ep = e.mean(1) + gamma(16) * yn.abs().mean(1)
    W1, b1 = sd64["audio_projection.linear1.weight"], sd64["audio_projection.linear1.bias"]
    W2, b2 = sd64["audio_projection.linear2.weight"], sd64["audio_projection.linear2.bias"]
    z1 = pooled @ W1.T + b1
    e1 = gamma(D // 32 + 6) * (pooled.abs() @ W1.abs().T + b1.abs()) + ep @ W1.abs().T
    h1 = F.relu(z1)
    h2 = h1 @ W2.T + b2
    e2 = gamma(512 // 32 + 6) * (h1 @ W2.abs().T + b2.abs()) + e1 @ W2.abs().T
    n = h2.norm(dim=-1, keepdim=True)
    dn = e2.norm(dim=-1, keepdim=True) + n * (gamma(72) / 2 + 2 * U)
    out = h2 / n
    eo = (e2 + out.abs() * dn) / (n - dn) + U * out.abs()
    eo = eo + 2.0 ** -11 * (out.abs() + eo) + 2.0 ** -25
    return out, eo * 1.001


def run_head(engine, x):
    B = x.shape[0]
    xin = Guarded(x.shape, torch.float32, "cuda", GUARD, init=x)
    out = Guarded((B, 512), torch.float16, "cuda", GUARD)
    engine.clap_head(xin.body, B, out.body)
    got = out.check("head")
    assert xin.intact_input(), "the input or its guard was modified"
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_head_matches_fp64(engine, variant, capsys):
    """fad_clap_head from the stream the GPU produced for it, per element and in rms, against clap_oracle.head."""
    ch = chain(engine, variant)
    sd64 = state(variant)[2]
    got = run_head(engine, ch["final"])
    ref, bound = head_reference(ch["final"].double(), sd64)
    with torch.no_grad():
        want = co.head(ch["final"].double(), sd64)
    assert (ref - want).abs().max().item() <= 1e-12
    stats = {}
    for i, (kind, n) in enumerate(STAGE_CLIPS):
        check_bound("head", f"{variant} {kind} {n}", got[i], ref[i], bound[i], stats, RMS_CEIL)
    report_stats(capsys, "clap", stats, variant)


# --------------------------------------------------------------------------------------- whole forward
FORWARD_SECONDS = [1.0, 2.5, 10.0, 10.0 + 1 / SR, 25.0, 61.0]


@torch.no_grad()
def reference_rows(clip, sd64, batch=8):
    """float64 embedding rows [n_windows, 512] of one clip: the float64 front end, then clap_oracle.network"""
    m = ref_mel(clip)
    lm = 10 * torch.log10(torch.clamp(m, min=1e-10))
    return torch.cat([co.network(lm[i:i + batch], sd64) for i in range(0, lm.shape[0], batch)])


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_forward_matches_fp64(engine, variant, capsys):
    """fad_clap_forward over clips of 1, 2.5, 10, 10 s + 1 sample, 25 and 61 s in one call (61 windows span many
    max_chunks chunks): the rows of each clip are fad_clap_plan's count, each close in cosine to the float64 network
    and all of them within an rms ceiling."""
    load(engine, variant)
    sd64 = state(variant)[2]
    clips = [make_clip("music" if i % 2 == 0 else "noise", int(round(sec * SR)), 40 + i)
             for i, sec in enumerate(FORWARD_SECONDS)]
    plan = plan_of(clips)
    _, _, rows = _native.Engine.clap_plan(np.concatenate([[0], np.cumsum([len(c) for c in clips])]).astype(np.int64))
    assert np.array_equal(plan["rows_per_clip"], rows)
    assert list(rows) == [1, 3, 10, 11, 25, 61]
    got = engine.clap_forward(pcm_of(clips), engine.clap_plan_to_device(plan))
    torch.cuda.synchronize()
    assert got.shape == (int(rows.sum()), 512) and bool(torch.isfinite(got).all())
    ref = torch.cat([reference_rows(c, sd64) for c in clips])
    g = got.double()
    cos = (g * ref).sum(1) / (g.norm(dim=1) * ref.norm(dim=1))
    rms = ((g - ref).square().mean().sqrt() / ref.square().mean().sqrt()).item()
    with capsys.disabled():
        report("clap", "forward", variant, f"{got.shape[0]} rows: min cosine {cos.min().item():.8f}, rms {rms:.3e}, "
                                           f"max |err| {(g - ref).abs().max().item():.3e}")
    assert 1 - cos.min().item() <= COS_GAP, cos.min().item()
    assert rms <= RMS_CEIL["forward"], rms


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_outputs_independent_of_batch(engine, variant):
    """A clip's rows are bitwise the same alone, inside a batch and split across a max_chunks chunk boundary; two
    identical calls give the same result."""
    load(engine, variant)
    clips = [make_clip("music", 72000, 50), make_clip("noise", 130000, 51), square(96000), make_clip("silence", 48000)]
    plan = plan_of(clips)
    rows = plan["rows_per_clip"]
    assert list(rows) == [2, 3, 2, 1]
    start = np.concatenate([[0], np.cumsum(rows)])
    assert start[1] < MAX_CHUNKS < start[2], "clip 1 must have windows in the first and the second chunk"
    got = engine.clap_forward(pcm_of(clips), engine.clap_plan_to_device(plan))
    for i, c in enumerate(clips):
        one = engine.clap_forward(pcm_of([c]), engine.clap_plan_to_device(plan_of([c])))
        assert torch.equal(one.view(torch.int16), got[start[i]:start[i + 1]].view(torch.int16)), \
            f"clip {i} depends on its batch"
    again = engine.clap_forward(pcm_of(clips), engine.clap_plan_to_device(plan))
    assert torch.equal(again.view(torch.int16), got.view(torch.int16)), "two identical calls differ"


@pytest.mark.gpu
def test_streams_need_no_vector_alignment(engine):
    """The stage entries only copy the caller's streams, so x and out may sit at any element offset: block 0 from a
    buffer 4 bytes past 16-byte alignment into another gives bitwise the aligned result."""
    ch = chain(engine, "tiny")
    _, x, want = ch["blocks"][0]
    B, n = x.shape[0], x.numel()
    xin = Guarded((n + 1,), torch.float32, "cuda", GUARD)
    xin.body[1:].copy_(x.flatten())
    out = Guarded((n + 1,), torch.float32, "cuda", GUARD)
    engine.clap_block(0, xin.body[1:], B, out.body[1:])
    torch.cuda.synchronize()
    assert out.guards_intact() and out.body[:1].view(torch.int32).item() == out.bits
    assert torch.equal(out.body[1:].view(x.shape), want)


# ---------------------------------------------------------------------------------------------------- rejections
E_TINY = 96


class _Addr:
    """a raw device address one byte past a tensor's start: misaligned for every element type"""

    def __init__(self, t):
        self.addr = t.data_ptr() + 1

    def data_ptr(self):
        return self.addr


def _arg(g, kind):
    return _Addr(g.body) if kind == "byte" else g.ptr(kind)


def _patch_call(**over):
    def call(engine, outs):
        a = dict(B=2, n_pool=4, pool="ok", fi="ok", out="ok")
        a.update(over)
        pool = Guarded((4, 64), torch.float32, "cuda", GUARD, init=torch.zeros((4, 64), device="cuda"))
        fi = Guarded((2, FRAMES), torch.float32, "cuda", GUARD, init=torch.zeros((2, FRAMES), device="cuda"))
        o = Guarded((2, 4096, E_TINY), torch.float32, "cuda", GUARD)
        outs.append(o)
        engine.clap_patch_embed(_arg(pool, a["pool"]), a["n_pool"], _arg(fi, a["fi"]), a["B"], o.ptr(a["out"]))
    return call


def _stream_call(entry, **over):
    def call(engine, outs):
        a = dict(i=1, B=2, x="ok", out="ok")
        a.update(over)
        shape = (2, 64, 8 * E_TINY) if entry == "head" else (2, 4096, E_TINY)
        x = Guarded(shape, torch.float32, "cuda", GUARD, init=torch.zeros(shape, device="cuda"))
        if entry == "head":
            o = Guarded((2, 512), torch.float16, "cuda", GUARD)
            outs.append(o)
            engine.clap_head(x.ptr(a["x"]), a["B"], _arg(o, a["out"]))
            return
        o = Guarded(shape, torch.float32, "cuda", GUARD)
        outs.append(o)
        fn = engine.clap_block if entry == "block" else engine.clap_merge
        fn(a["i"], x.ptr(a["x"]), a["B"], o.ptr(a["out"]))
    return call


def _pool_call(entry, **over):
    def call(engine, outs):
        a = dict(n_pool=None, n_chunks=None, pcm="ok", start="ok", valid="ok", frame="ok", fi="ok", out="ok")
        a.update(over)
        clip = make_clip("noise", 48000)
        plan = plan_of([clip])
        d = to_dev(plan)
        n_pool = len(plan["pool_start"]) if a["n_pool"] is None else a["n_pool"]
        n_chunks = plan["frame_index"].shape[0] if a["n_chunks"] is None else a["n_chunks"]
        pick = lambda t, k: t if a[k] == "ok" else (_Addr(t) if a[k] == "byte" else None)
        pcm = pick(pcm_of([clip]), "pcm")
        ps, pv, pf = pick(d["pool_start"], "start"), pick(d["pool_valid"], "valid"), pick(d["pool_frame"], "frame")
        if entry == "logmel":
            o = Guarded((len(plan["pool_start"]), 64), torch.float32, "cuda", GUARD)
            outs.append(o)
            engine.clap_pool(pcm, ps, pv, pf, n_pool, _arg(o, a["out"]))
        else:
            o = Guarded((1, 512), torch.float16, "cuda", GUARD)
            outs.append(o)
            engine.clap_forward_raw(pcm, ps, pv, pf, n_pool, pick(d["frame_index"], "fi"), n_chunks, _arg(o, a["out"]))
    return call


PE, BL, MG, HD = "fad_clap_patch_embed", "fad_clap_block", "fad_clap_merge", "fad_clap_head"
LM, FW = "fad_clap_logmel", "fad_clap_forward"
POOL_NULL = "null pcm, pool_start, pool_valid or pool_frame"
POOL_ALIGN = "pcm, pool_start, pool_valid and pool_frame must be aligned to their element size"
REJECT = [
    ("patch B 0", _patch_call(B=0), f"{PE}: B must be in [1, max_chunks]"),
    ("patch B beyond max_chunks", _patch_call(B=MAX_CHUNKS + 1), f"{PE}: B must be in [1, max_chunks]"),
    ("patch n_pool 0", _patch_call(n_pool=0), f"{PE}: n_pool must be positive"),
    ("patch null pool", _patch_call(pool="null"), f"{PE}: null pool, frame_index or x_out"),
    ("patch null frame_index", _patch_call(fi="null"), f"{PE}: null pool, frame_index or x_out"),
    ("patch null out", _patch_call(out="null"), f"{PE}: null pool, frame_index or x_out"),
    ("patch misaligned pool", _patch_call(pool="byte"), f"{PE}: pool and frame_index must be 4-byte aligned"),
    ("patch misaligned frame_index", _patch_call(fi="byte"), f"{PE}: pool and frame_index must be 4-byte aligned"),
    ("patch before any load", on_fresh_engine(_patch_call()), f"{PE}: fad_clap_load has not been called"),
    ("block blk 12", _stream_call("block", i=12), f"{BL}: blk must be in [0, n_blocks)"),
    ("block blk -1", _stream_call("block", i=-1), f"{BL}: blk must be in [0, n_blocks)"),
    ("block B 0", _stream_call("block", i=0, B=0), f"{BL}: B must be in [1, max_chunks]"),
    ("block B beyond max_chunks", _stream_call("block", i=0, B=MAX_CHUNKS + 1), f"{BL}: B must be in [1, max_chunks]"),
    ("block null x", _stream_call("block", i=0, x="null"), f"{BL}: null x or out"),
    ("block null out", _stream_call("block", i=0, out="null"), f"{BL}: null x or out"),
    ("block before any load", on_fresh_engine(_stream_call("block", i=0)), f"{BL}: fad_clap_load has not been called"),
    ("merge s 3", _stream_call("merge", i=3), f"{MG}: s must be in [0, 3)"),
    ("merge s -1", _stream_call("merge", i=-1), f"{MG}: s must be in [0, 3)"),
    ("merge B 0", _stream_call("merge", i=0, B=0), f"{MG}: B must be in [1, max_chunks]"),
    ("merge B beyond max_chunks", _stream_call("merge", i=0, B=MAX_CHUNKS + 1), f"{MG}: B must be in [1, max_chunks]"),
    ("merge null x", _stream_call("merge", i=0, x="null"), f"{MG}: null x or out"),
    ("merge null out", _stream_call("merge", i=0, out="null"), f"{MG}: null x or out"),
    ("merge before any load", on_fresh_engine(_stream_call("merge", i=0)), f"{MG}: fad_clap_load has not been called"),
    ("head B 0", _stream_call("head", B=0), f"{HD}: B must be in [1, max_chunks]"),
    ("head B beyond max_chunks", _stream_call("head", B=MAX_CHUNKS + 1), f"{HD}: B must be in [1, max_chunks]"),
    ("head null x", _stream_call("head", x="null"), f"{HD}: null x or out"),
    ("head null out", _stream_call("head", out="null"), f"{HD}: null x or out"),
    ("head misaligned out", _stream_call("head", out="byte"), f"{HD}: out must be 2-byte aligned"),
    ("head before any load", on_fresh_engine(_stream_call("head")), f"{HD}: fad_clap_load has not been called"),
    ("logmel n_pool -1", _pool_call("logmel", n_pool=-1), f"{LM}: n_pool must be >= 0"),
    ("logmel null pcm", _pool_call("logmel", pcm="null"), f"{LM}: {POOL_NULL}"),
    ("logmel null pool_start", _pool_call("logmel", start="null"), f"{LM}: {POOL_NULL}"),
    ("logmel null pool_valid", _pool_call("logmel", valid="null"), f"{LM}: {POOL_NULL}"),
    ("logmel null pool_frame", _pool_call("logmel", frame="null"), f"{LM}: {POOL_NULL}"),
    ("logmel misaligned pcm", _pool_call("logmel", pcm="byte"), f"{LM}: {POOL_ALIGN}"),
    ("logmel misaligned pool_start", _pool_call("logmel", start="byte"), f"{LM}: {POOL_ALIGN}"),
    ("logmel misaligned pool_valid", _pool_call("logmel", valid="byte"), f"{LM}: {POOL_ALIGN}"),
    ("logmel misaligned pool_frame", _pool_call("logmel", frame="byte"), f"{LM}: {POOL_ALIGN}"),
    ("logmel null out", _pool_call("logmel", out="null"), f"{LM}: null out"),
    ("logmel misaligned out", _pool_call("logmel", out="byte"), f"{LM}: out must be 4-byte aligned"),
    ("logmel before any load", on_fresh_engine(_pool_call("logmel")), f"{LM}: fad_clap_load has not been called"),
    ("forward n_pool -1", _pool_call("forward", n_pool=-1), f"{FW}: n_pool must be >= 0"),
    ("forward n_chunks -1", _pool_call("forward", n_chunks=-1), f"{FW}: n_chunks must be >= 0"),
    ("forward null pcm", _pool_call("forward", pcm="null"), f"{FW}: {POOL_NULL}"),
    ("forward null pool_start", _pool_call("forward", start="null"), f"{FW}: {POOL_NULL}"),
    ("forward null pool_valid", _pool_call("forward", valid="null"), f"{FW}: {POOL_NULL}"),
    ("forward null pool_frame", _pool_call("forward", frame="null"), f"{FW}: {POOL_NULL}"),
    ("forward misaligned pool_start", _pool_call("forward", start="byte"), f"{FW}: {POOL_ALIGN}"),
    ("forward null frame_index", _pool_call("forward", fi="null"), f"{FW}: null frame_index or emb_out"),
    ("forward null out", _pool_call("forward", out="null"), f"{FW}: null frame_index or emb_out"),
    ("forward windows without a pool", _pool_call("forward", n_pool=0), f"{FW}: windows need a non-empty frame pool"),
    ("forward misaligned frame_index", _pool_call("forward", fi="byte"),
     f"{FW}: frame_index and emb_out must be aligned to their element size"),
    ("forward misaligned out", _pool_call("forward", out="byte"),
     f"{FW}: frame_index and emb_out must be aligned to their element size"),
    ("forward before any load", on_fresh_engine(_pool_call("forward")), f"{FW}: fad_clap_load has not been called"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("call,message", [c[1:] for c in REJECT], ids=[c[0] for c in REJECT])
def test_stage_entries_reject_invalid_arguments(engine, call, message):
    """Arguments the launch cannot honour fail with their message, launch nothing and write nothing."""
    load(engine, "tiny")
    expect_rejected(engine, call, message, [])


@pytest.mark.gpu
def test_empty_plan_is_valid(engine):
    """An empty plan (no clips, or only empty clips) hands over null pointers with zero counts: the forward and the
    front end accept it and launch nothing."""
    load(engine, "tiny")
    launches = engine.launches
    engine.clap_forward_raw(None, None, None, None, 0, None, 0, None)
    engine.clap_pool(None, None, None, None, 0, None)
    out = engine.clap_forward(torch.zeros(0, dtype=torch.int16, device="cuda"), engine.clap_plan_to_device(plan_of([])))
    torch.cuda.synchronize()
    assert out.shape == (0, 512) and engine.launches == launches


# ------------------------------------------------------------------------------------------ CPU: the references
@pytest.mark.parametrize("variant", VARIANTS)
def test_stage_composition_is_the_network(variant):
    """Composing the stage references as the GPU tests wire them (BatchNorm, patch_embed_reference, the blocks of
    block_geometry, the three merges, the head) reproduces clap_oracle.network in float64 to 1e-10."""
    sd64 = {k: v.double() for k, v in wc.synthetic_clap_state(1, variant).items()}
    g = torch.Generator().manual_seed(2)
    lm = (-30.0 + 12.0 * torch.randn((2, FRAMES, 64), generator=g)).double()
    _, depths = wc.VARIANTS[variant]
    with torch.no_grad():
        want = co.network(lm, sd64)
        x, _ = patch_embed_reference(co.batch_norm(lm, sd64), sd64)
        for s, j, res, C, heads, shift in block_geometry(variant):
            assert x.shape[1:] == (res * res, C)
            x = co.swin_block(x, sd64, f"layers.{s}.blocks.{j}.", res, heads, shift)
            if j == depths[s] - 1 and s < 3:
                x, _ = merge_reference(x, sd64, s, res)
        got, _ = head_reference(x, sd64)
    assert (got - want).abs().max().item() <= 1e-10


def test_oracle_masks_follow_device_and_dtype():
    """The shift mask and relative-position index are transformers' own (ClapAudioLayer.get_attn_mask,
    ClapAudioSelfAttention.create_relative_position_index) in fp32 on the CPU, bit for bit, and their float64 versions
    are the same values; the fp32 CPU network is bitwise the composition of its fp32 stages."""
    tr = pytest.importorskip("transformers")
    from transformers.models.clap import modeling_clap as mc
    cfg = tr.ClapAudioConfig()
    for res in (64, 32, 16):
        layer = mc.ClapAudioLayer(cfg, 96, (res, res), 4, shift_size=4)
        layer.window_size = 8
        want = layer.get_attn_mask(res, res, torch.float32, "cpu")
        got = co._shift_mask(res, res, 8, 4)
        assert got.dtype == torch.float32 and torch.equal(got, want)
        assert torch.equal(co._shift_mask(res, res, 8, 4, "cpu", torch.float64), want.double())
    att = mc.ClapAudioSelfAttention(cfg, 96, 4, 8)
    assert torch.equal(co._rel_pos_index(), att.create_relative_position_index())
    sd = wc.synthetic_clap_state(1, "tiny")
    g = torch.Generator().manual_seed(3)
    lm = -30.0 + 12.0 * torch.randn((1, FRAMES, 64), generator=g)
    with torch.no_grad():
        want = co.network(lm, sd)
        x = co.image_tokens(co.fold_image(co.batch_norm(lm, sd)), sd)
        _, depths = wc.VARIANTS["tiny"]
        for s, j, res, C, heads, shift in block_geometry("tiny"):
            x = co.swin_block(x, sd, f"layers.{s}.blocks.{j}.", res, heads, shift)
            if j == depths[s] - 1 and s < 3:
                x = co.patch_merge(x, sd, f"layers.{s}.downsample.", res)
        got = co.head(x, sd)
    assert got.dtype == torch.float32 and torch.equal(got, want)


@pytest.mark.parametrize("n", [1, 48001, 480000])
def test_fp64_front_end_is_the_oracle_front_end(n):
    """The float64 front end against clap_oracle.log_mel (fp32 torch.stft): the same log-mel at its fp32 noise level
    in bins within 60 dB of the window's peak."""
    clip = make_clip("music", n, 7)
    ch = torch.from_numpy(co.chunks_of(co.quantize_like_reference(clip / 32768.0)))
    want = co.log_mel(ch).double()
    got = 10 * torch.log10(torch.clamp(ref_mel(clip, "cpu"), min=1e-10))
    assert got.shape == want.shape
    loud = want > want.amax((1, 2), keepdim=True) - 60.0
    err = (got - want).abs()
    assert err[loud].max().item() <= 1e-3, err[loud].max().item()
