"""The attention and LayerNorm kernels of the transformer embedders, one launch at a time, through the stage entries that
call the forwards' own launch code: the CLAP Swin window attention (fad_window_attention), WavLM's gated relative
position bias (fad_wavlm_gate, fad_attention_bias), the Whisper decoder's self- and cross-attention
(fad_decoder_self_attention, fad_cross_attention) and every LayerNorm (fad_layernorm -> clap_ln).

References are fp64 (torch on the GPU), computed from the exact fp16 / fp32 inputs the kernel reads.  Every output
lives inside a buffer whose guard regions (256 elements on each side) and unwritten elements hold a NaN sentinel: each
test checks that every element was written and that no guard was touched.  Identical calls must be bitwise equal, and a
unit (a window image, a clip, a row) must come out bitwise the same at another batch position and in a call of another
size.

Attention bound, per output element o = sum_k p_k v_k (p the softmax of the scores s_k), with A = sum_k p_k |v_k|:
  * P is rounded to fp16 before P V:                  2^-11 A, plus 2^-25 per fp16-subnormal p_k (p_k < 2^-13), that is
                                                      2^-25 sum_{p_k < 2^-13} |v_k|
  * score error delta_k (natural-log units): the fp32 dot product (fp16 products exact, at most hd fp32 adds),
    the scale, the bias and mask adds and the exp argument, each at most 2^-22 of its magnitude, and ex2 / __expf
    (2^-21 relative):  delta_k = 2^-22 (hd sum_j |q_j k_j| scale + |bias_k| + |s_k| + |s_k - max s|) + 2^-21.
    A relative error delta_k of p_k moves o by at most sum_k p_k delta_k (|v_k| + |o|)
  * fp32 accumulation of P V: `acc` A, acc = 2^-22 per mma.sync k-step (+ 2), or 2^-24 per sequential fp32 add
  * the fp16 rounding of the output:                  2^-11 |o| + 2^-25
An rms ceiling of about 3x the level measured on the H100 sits on top (RMS_CEIL below).
"""
import math

import numpy as np
import pytest
import torch

from fadtk_b200 import _native
from fadtk_b200 import weights_clap
from gpu_checks import Guarded, check_bound, expect_rejected
from oracle import clap_oracle as co

pytestmark = pytest.mark.gpu

GUARD = 256
U = 2.0 ** -24

# rms relative error (rms |kernel - fp64| / rms |fp64|), about 3x the largest level measured per kernel on an H100 80GB
# HBM3 (700 W) over the cases below:
#   window attention 2.7e-4, WavLM biased attention 2.2e-4, decoder self-attention 1.4e-4, cross-attention 2.2e-4,
#   WavLM gate 9.5e-8, LayerNorm fp32 output 1.7e-5 (the |mean| = 1e3 std rows), fp16 output 2.1e-4
# The largest max |err| / bound measured: window 0.81, biased 0.55, decoder 0.47, cross 0.30, gate 0.18, LayerNorm fp32
# 0.24, LayerNorm fp16 0.997 (its half-ulp rounding term is attained; the kernel is deterministic, so this is stable).
RMS_CEIL = {"window": 8e-4, "bias": 6.5e-4, "dec_self": 4.5e-4, "cross": 6.5e-4, "gate": 3e-7, "ln32": 5e-5, "ln16": 6.5e-4}


@pytest.fixture(scope="module")
def dev(engine):
    return engine.torch_device


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _same(a, b):
    return torch.equal(a.view(torch.int16) if a.dtype == torch.float16 else a, b.view(torch.int16) if b.dtype == torch.float16 else b)


def _check(got, ref, bound, kind, what, capsys):
    rms, ratio = check_bound(kind, what, got, ref, bound, {}, RMS_CEIL)
    with capsys.disabled():
        print(f"\n[{kind}] {what}: rms rel err {rms:.3e}, max err / bound {ratio:.3f}")


def attention_reference(q, k, v, bias, scale, acc):
    """q [..., Lq, hd], k / v [..., Lk, hd] (fp64 of the kernel's fp16 inputs), bias broadcastable to [..., Lq, Lk]
    -> (o fp64, per-element bound of the fp16 kernel output; see the module docstring)."""
    hd = q.shape[-1]
    s = (q @ k.transpose(-1, -2)) * scale + bias
    mag = (q.abs() @ k.abs().transpose(-1, -2)) * scale
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    p = e / e.sum(-1, keepdim=True)
    o = p @ v
    a = p @ v.abs()
    delta = 2.0 ** -22 * (hd * mag + bias.abs() + s.abs() + (s - m).abs()) + 2.0 ** -21
    pd = p * delta
    sub = (p < 2.0 ** -13).double() @ v.abs()
    bound = (2.0 ** -11 * o.abs() + (2.0 ** -11 + acc) * a + pd @ v.abs() + pd.sum(-1, keepdim=True) * o.abs()
             + 2.0 ** -25 * sub) * 1.001 + 2.0 ** -25
    return o, bound


# ----------------------------------------------------------------------------------------------- window attention
# (head dim, C, res, heads): HTSAT-tiny and HTSAT-base, stages 0..3
WINDOW = [(24, 96, 64, 4), (24, 192, 32, 8), (24, 384, 16, 16), (24, 768, 8, 32),
          (32, 128, 64, 4), (32, 256, 32, 8), (32, 512, 16, 16), (32, 1024, 8, 32)]


def window_problem(dev, seed, n_img, C, res, heads):
    """qkv fp16 [n_windows * 64, 3 C] with per-head score scales 0.3 .. 10 (scores up to about +-30 in every fourth
    head) and value scales 1/4 .. 4, and relbias [heads][64][64] = table[_rel_pos_index] of a random per-head table
    as large as that head's scores."""
    g = _gen(dev, seed)
    hd = C // heads
    rows = n_img * res * res
    sig2 = torch.tensor([0.3, 1.0, 3.0, 10.0], device=dev)[torch.arange(heads, device=dev) % 4]
    vsc = 2.0 ** (torch.arange(heads, device=dev) % 5 - 2).float()
    qk = torch.randn((rows, 2, heads, hd), generator=g, device=dev) * sig2.sqrt()[None, None, :, None]
    v = torch.randn((rows, 1, heads, hd), generator=g, device=dev) * vsc[None, None, :, None]
    qkv = torch.cat([qk, v], 1).reshape(rows, 3 * C).half().contiguous()
    table = torch.randn((225, heads), generator=g, device=dev) * sig2
    relbias = table[co._rel_pos_index().to(dev)].permute(2, 0, 1).contiguous()        # [heads, 64 (query), 64 (key)]
    return qkv, relbias


def window_reference(qkv, relbias, C, heads, res, shift):
    hd = C // heads
    n_win = qkv.shape[0] // 64
    t = qkv.double().view(n_win, 64, 3, heads, hd).permute(2, 0, 3, 1, 4)             # [3, win, head, 64, hd]
    bias = relbias.double()[None]
    if shift:
        mask = co._shift_mask(res, res, 8, shift).to(qkv.device).double()            # [windows per image, 64, 64]
        bias = bias + mask.repeat(n_win // mask.shape[0], 1, 1)[:, None]
    o, bound = attention_reference(t[0], t[1], t[2], bias, 1.0 / math.sqrt(hd), 6 * 2.0 ** -22)
    return o.permute(0, 2, 1, 3).reshape(n_win * 64, C), bound.permute(0, 2, 1, 3).reshape(n_win * 64, C)


def run_window(engine, qkv, C, heads, relbias, res, shift):
    out = Guarded((qkv.shape[0], C), torch.float16, qkv.device, GUARD)
    engine.window_attention(qkv, qkv.shape[0] // 64, C, heads, relbias, res, shift, out.body)
    return out.check()


@pytest.mark.parametrize("hd,C,res,heads", WINDOW)
def test_window_attention_matches_fp64(engine, dev, hd, C, res, heads, capsys):
    n_img = 3
    per_img = res * res
    qkv, relbias = window_problem(dev, C + res, n_img, C, res, heads)
    for shift in ((0, 4) if res > 8 else (0,)):
        out = run_window(engine, qkv, C, heads, relbias, res, shift)
        ref, bound = window_reference(qkv, relbias, C, heads, res, shift)
        _check(out, ref, bound, "window", f"hd {hd} C {C} res {res} shift {shift}", capsys)
        assert _same(out, run_window(engine, qkv, C, heads, relbias, res, shift)), "two identical calls differ"
        one = run_window(engine, qkv[2 * per_img:].contiguous(), C, heads, relbias, res, shift)
        assert _same(one, out[2 * per_img:]), "an image's output depends on its batch position"


def test_window_attention_grid_stride(engine, dev, capsys):
    """More (window, head) units than the launch cap (num_sms * 32 blocks x 4 warps): warps loop over units."""
    hd, C, res, heads = 24, 192, 32, 8
    cap = torch.cuda.get_device_properties(dev).multi_processor_count * 32 * 4
    n_img = cap // (16 * heads) + 5
    assert n_img * 16 * heads > cap
    qkv, relbias = window_problem(dev, 99, n_img, C, res, heads)
    out = run_window(engine, qkv, C, heads, relbias, res, 4)
    ref, bound = window_reference(qkv, relbias, C, heads, res, 4)
    _check(out, ref, bound, "window", f"{n_img} images, {n_img * 16 * heads} units > cap {cap}", capsys)
    k = n_img - 2
    one = run_window(engine, qkv[k * res * res:(k + 1) * res * res].contiguous(), C, heads, relbias, res, 4)
    assert _same(one, out[k * res * res:(k + 1) * res * res]), "an image's output depends on its batch position"


# ------------------------------------------------------------------------------------------------------- WavLM
def gate_reference(x, w, b, c, heads):
    """WavLMAttention.forward steps 1-3 in fp64 -> (gate [rows, heads], bound)."""
    xh = x.double().view(x.shape[0], heads, 64)
    w64, b64 = w.double(), b.double()
    p = xh @ w64.t() + b64                                                        # [rows, heads, 8]
    dp = 64 * U * (xh.abs() @ w64.abs().t() + b64.abs())
    s = p.view(x.shape[0], heads, 2, 4).sum(-1)
    ds = dp.view(x.shape[0], heads, 2, 4).sum(-1) + 3 * U * p.abs().view(x.shape[0], heads, 2, 4).sum(-1)
    sg = torch.sigmoid(s)
    dsg = 0.25 * ds + 3 * U
    ga, gb = sg[..., 0], sg[..., 1]
    c64 = c.double()[None]
    gate = ga * (gb * c64 - 1.0) + 2.0
    bound = dsg[..., 0] * (gb * c64 - 1.0).abs() + ga * c64.abs() * dsg[..., 1] + 4 * U * (ga * gb * c64.abs() + ga + 2.0)
    return gate, bound * 1.001


@pytest.mark.parametrize("rows,heads", [(149 * 3, 12), (1499 * 2, 16), (40000, 16)])
def test_wavlm_gate_matches_fp64(engine, dev, rows, heads, capsys):
    """rows = 40 000 x 16 heads is more than the grid (num_sms * 16 blocks of 256) covers: the grid-stride loop runs."""
    d = heads * 64
    g = _gen(dev, rows + heads)
    x = torch.randn((rows, d), generator=g, device=dev) * 2.0
    w = torch.randn((8, 64), generator=g, device=dev) * 0.3
    b = torch.randn((8,), generator=g, device=dev)
    c = 1.0 + torch.randn((heads,), generator=g, device=dev)
    out = Guarded((rows, heads), torch.float32, dev, GUARD)
    engine.wavlm_gate(x, w, b, c, rows, heads, d, out.body)
    got = out.check()
    ref, bound = gate_reference(x, w, b, c, heads)
    _check(got, ref, bound, "gate", f"rows {rows} heads {heads}", capsys)
    again = Guarded((rows, heads), torch.float32, dev, GUARD)
    engine.wavlm_gate(x, w, b, c, rows, heads, d, again.body)
    assert torch.equal(again.check(), got)
    part = Guarded((101, heads), torch.float32, dev, GUARD)
    engine.wavlm_gate(x[rows - 101:].contiguous(), w, b, c, 101, heads, d, part.body)
    assert torch.equal(part.check(), got[rows - 101:])


def bias_problem(dev, seed, n_clips, S, d):
    heads = d // 64
    g = _gen(dev, seed)
    sig2 = torch.tensor([0.3, 1.0, 3.0, 10.0], device=dev)[torch.arange(heads, device=dev) % 4]
    vsc = 2.0 ** (torch.arange(heads, device=dev) % 5 - 2).float()
    qk = torch.randn((n_clips * S, 2, heads, 64), generator=g, device=dev) * sig2.sqrt()[None, None, :, None]
    v = torch.randn((n_clips * S, 1, heads, 64), generator=g, device=dev) * vsc[None, None, :, None]
    qkv = torch.cat([qk, v], 1).reshape(n_clips * S, 3 * d).half().contiguous()
    relb = (torch.randn((heads, 2 * S - 1), generator=g, device=dev) * sig2[:, None] * 0.5).contiguous()
    gate = (torch.rand((n_clips * S, heads), generator=g, device=dev) * 3.0 + 0.5).contiguous()    # the gate's range (1, 3) and beyond
    return qkv, relb, gate


def bias_reference(qkv, relb, gate, n_clips, S, d):
    heads = d // 64
    t = qkv.double().view(n_clips, S, 3, heads, 64).permute(2, 0, 3, 1, 4)              # [3, clip, head, S, 64]
    dist = torch.arange(S, device=qkv.device)[None, :] - torch.arange(S, device=qkv.device)[:, None] + S - 1
    rb = relb.double()[:, dist]                                                          # [head, S (query), S (key)]
    gq = gate.double().view(n_clips, S, heads).permute(0, 2, 1)[..., None]              # [clip, head, S, 1]
    acc = (2 * math.ceil(S / 16) + 2) * 2.0 ** -22                                      # k-steps + online-softmax rescales
    o, bound = attention_reference(t[0], t[1], t[2], gq * rb[None], 0.125, acc)
    return o.permute(0, 2, 1, 3).reshape(n_clips * S, d), bound.permute(0, 2, 1, 3).reshape(n_clips * S, d)


def run_bias(engine, qkv, n_clips, S, d, relb, gate):
    out = Guarded((n_clips * S, d), torch.float16, qkv.device, GUARD)
    engine.attention_bias(qkv, n_clips, S, d, relb, gate, out.body)
    return out.check()


@pytest.mark.parametrize("d", [768, 1024])
@pytest.mark.parametrize("S", [49, 64, 65, 149, 499, 1499])
def test_wavlm_biased_attention_matches_fp64(engine, dev, S, d, capsys):
    """Ragged query and key tiles (S = 49, 65, 149, 499, 1499) and the 30-s length whose distances reach 1498."""
    n_clips = 3 if S < 1000 else 2
    qkv, relb, gate = bias_problem(dev, S * 7 + d, n_clips, S, d)
    out = run_bias(engine, qkv, n_clips, S, d, relb, gate)
    ref, bound = bias_reference(qkv, relb, gate, n_clips, S, d)
    _check(out, ref, bound, "bias", f"S {S} d {d}", capsys)
    assert _same(out, run_bias(engine, qkv, n_clips, S, d, relb, gate)), "two identical calls differ"
    last = slice((n_clips - 1) * S, n_clips * S)
    one = run_bias(engine, qkv[last].contiguous(), 1, S, d, relb, gate[last].contiguous())
    assert _same(one, out[last]), "a clip's output depends on its batch position"


# ------------------------------------------------------------------------------------------------ Whisper decoder
DEC_D = [384, 512, 768, 1024, 1280]


def _dec_qkv(dev, seed, rows, d):
    heads = d // 64
    g = _gen(dev, seed)
    sig2 = torch.tensor([0.3, 1.0, 3.0, 10.0], device=dev)[torch.arange(heads, device=dev) % 4]
    vsc = 2.0 ** (torch.arange(heads, device=dev) % 5 - 2).float()
    x = torch.randn((rows, 3, heads, 64), generator=g, device=dev)
    x[:, :2] *= sig2.sqrt()[None, None, :, None]
    x[:, 2] *= vsc[None, :, None]
    return x


@pytest.mark.parametrize("n_clips", [1, 5])
@pytest.mark.parametrize("d", DEC_D)
def test_decoder_self_attention_matches_fp64(engine, dev, d, n_clips, capsys):
    """Token 0 attends to itself only (its output is v0, bitwise); token 1 to both.  d = 384 with an odd clip count
    leaves (clip, head) units that do not fill the last 4-warp block."""
    heads = d // 64
    qkv = _dec_qkv(dev, d + n_clips, 2 * n_clips, d).reshape(2 * n_clips, 3 * d).half().contiguous()
    out = Guarded((2 * n_clips, d), torch.float16, dev, GUARD)
    engine.decoder_self_attention(qkv, n_clips, d, out.body)
    got = out.check()
    assert _same(got[0::2], qkv[0::2, 2 * d:].contiguous()), "token 0 is not v0"
    t = qkv.double().view(n_clips, 2, 3, heads, 64).permute(2, 0, 3, 1, 4)
    causal = torch.tensor([[0.0, -1e30], [0.0, 0.0]], device=dev, dtype=torch.float64)
    ref, bound = attention_reference(t[0], t[1], t[2], causal, 0.125, 8 * U)
    ref, bound = (z.permute(0, 2, 1, 3).reshape(2 * n_clips, d) for z in (ref, bound))
    _check(got, ref, bound + 2.0 ** -25, "dec_self", f"d {d} clips {n_clips}", capsys)
    again = Guarded((2 * n_clips, d), torch.float16, dev, GUARD)
    engine.decoder_self_attention(qkv, n_clips, d, again.body)
    assert _same(again.check(), got)
    one = Guarded((2, d), torch.float16, dev, GUARD)
    engine.decoder_self_attention(qkv[-2:].contiguous(), 1, d, one.body)
    assert _same(one.check(), got[-2:]), "a clip's output depends on its batch position"


CROSS = [(d, 1500) for d in DEC_D] + [(d, S) for d in (384, 1280) for S in (1, 127, 129)]


@pytest.mark.parametrize("d,S", CROSS)
def test_cross_attention_matches_fp64(engine, dev, d, S, capsys):
    heads, n_clips = d // 64, 3
    x = _dec_qkv(dev, d * 3 + S, n_clips * S, d)
    kv = x[:, 1:].reshape(n_clips * S, 2 * d).half().contiguous()
    qg = _gen(dev, S + 1)
    sig2 = torch.tensor([0.3, 1.0, 3.0, 10.0], device=dev)[torch.arange(heads, device=dev) % 4]
    q = (torch.randn((n_clips * 2, heads, 64), generator=qg, device=dev) * sig2.sqrt()[None, :, None]).reshape(n_clips * 2, d)
    q = q.half().contiguous()
    out = Guarded((n_clips * 2, d), torch.float16, dev, GUARD)
    engine.cross_attention(q, kv, n_clips, S, d, out.body)
    got = out.check()
    qq = q.double().view(n_clips, 2, heads, 64).permute(0, 2, 1, 3)
    kk = kv.double().view(n_clips, S, 2, heads, 64).permute(2, 0, 3, 1, 4)
    zero = torch.zeros((), dtype=torch.float64, device=dev)
    ref, bound = attention_reference(qq, kk[0], kk[1], zero, 0.125, (S + 4) * U)
    ref, bound = (z.permute(0, 2, 1, 3).reshape(n_clips * 2, d) for z in (ref, bound))
    _check(got, ref, bound, "cross", f"d {d} S {S}", capsys)
    again = Guarded((n_clips * 2, d), torch.float16, dev, GUARD)
    engine.cross_attention(q, kv, n_clips, S, d, again.body)
    assert _same(again.check(), got)
    one = Guarded((2, d), torch.float16, dev, GUARD)
    engine.cross_attention(q[2:4].contiguous(), kv[S:2 * S].contiguous(), 1, S, d, one.body)
    assert _same(one.check(), got[2:4]), "a clip's output depends on its batch position"


# -------------------------------------------------------------------------------------------------------- LayerNorm
# width -> (CHUNKS, lanes per row) of the dispatch in clap_host.inc
LN_WIDTHS = {96: (3, 8), 192: (3, 16), 384: (3, 32), 768: (6, 32), 1536: (12, 32), 128: (4, 8), 256: (4, 16),
             512: (4, 32), 1024: (8, 32), 2048: (16, 32), 1280: (10, 32)}
EPS = float(np.float32(1e-5))


def ln_rows(dev, seed, rows, width):
    """fp32 rows of four kinds: |mean| = 1e3 std, constant (dyadic, so the kernel's mean is exact), one outlier of
    1e3 in unit-variance noise, and plain rows at scales 1e-3 .. 1e2."""
    g = _gen(dev, seed)
    x = torch.randn((rows, width), generator=g, device=dev)
    kind = torch.arange(rows, device=dev) % 8
    x[kind == 0] = x[kind == 0] * 0.5 + 500.0
    x[kind == 1] = (torch.randint(-40, 40, ((kind == 1).sum().item(), 1), generator=g, device=dev).float() / 4.0)
    out_col = torch.randint(0, width, ((kind == 2).sum().item(),), generator=g, device=dev)
    x[torch.nonzero(kind == 2).flatten(), out_col] = 1e3
    scale = 10.0 ** torch.randint(-3, 3, (rows, 1), generator=g, device=dev).float()
    plain = kind >= 3
    x[plain] = x[plain] * scale[plain]
    gamma = 1.0 + 0.3 * torch.randn((width,), generator=g, device=dev)
    beta = 0.5 * torch.randn((width,), generator=g, device=dev)
    return x.contiguous(), gamma, beta


def ln_reference(xr, gamma, beta, gelu, width):
    """xr [rows, width]: the rows the kernel normalises, fp32.  -> (y fp64, bound of the fp32 result, bound of fp16).
    Lane sums: CHUNKS groups of 4 then log2(L) shuffle levels, so the mean and the variance carry at most
    depth = CHUNKS + 2 + log2(L) roundings of 2^-24 of their sums of magnitudes; rsqrtf 2^-22; the affine 3 roundings;
    GELU (erff 2 ulp) amplifies by at most 1.13.  fp16 output: + 2^-11 |y| + 2^-25."""
    chunks, lanes = LN_WIDTHS[width]
    depth = chunks + 2 + math.log2(lanes)
    x = xr.double()
    mu = x.mean(-1, keepdim=True)
    xc = x - mu
    rstd = 1.0 / torch.sqrt(xc.square().mean(-1, keepdim=True) + EPS)
    g, b = gamma.double(), beta.double()
    y = xc * rstd * g + b
    dmu = (depth + 1) * U * x.abs().mean(-1, keepdim=True)                  # the sum, then the division by the width
    # variance: its sum (depth + 3 roundings with the subtraction and the square) and the mean's error squared;
    # rstd takes half of that relative error, + rsqrtf (2^-22) and the eps add; then (x - mean) * rstd * gamma
    rr = 0.5 * ((depth + 3) * U + dmu.square() * rstd.square()) + 2.0 ** -22 + U + 3 * U
    dy = dmu * rstd * g.abs() + xc.abs() * rstd * g.abs() * rr + 2 * U * (b.abs() + y.abs()) + 1e-38
    if gelu:
        yg = 0.5 * y * (1.0 + torch.special.erf(y / math.sqrt(2.0)))
        dy = 1.13 * dy + 0.5 * y.abs() * 2.0 ** -22 + 2 * U * yg.abs()
        y = yg
    return y, dy * 1.001, (dy + 2.0 ** -11 * y.abs()) * 1.001 + 2.0 ** -25


def run_ln(engine, x, gamma, beta, rows, C, ld_out, res=0, shift=0, mode=0, gelu=False, want32=True, alias=False):
    width = 4 * C if mode else C
    o16 = Guarded((rows, ld_out), torch.float16, x.device, GUARD)
    o32 = Guarded((rows, width), torch.float32, x.device, GUARD) if want32 and not alias else None
    engine.layernorm(x, gamma, beta, rows, C, ld_out, o16.body, x if alias else (o32.body if o32 else None),
                     res=res, shift=shift, mode=mode, gelu=gelu)
    out16 = o16.check()
    assert not bool(out16[:, width:].view(torch.int16).any()), "columns past the width are not +0"
    return out16, (o32.check() if o32 else None)


def check_ln(engine, x, xr, gamma, beta, rows, C, ld_out, what, capsys, **kw):
    """LayerNorm of the kernel rows xr (fp32 result within its bound, fp16 = fp32.half() bitwise, fp16 alone the same)."""
    width = xr.shape[1]
    out16, out32 = run_ln(engine, x, gamma, beta, rows, C, ld_out, **kw)
    y, b32, b16 = ln_reference(xr, gamma, beta, kw.get("gelu", False), width)
    _check(out32, y, b32, "ln32", what, capsys)
    _check(out16[:, :width], y, b16, "ln16", what, capsys)
    assert _same(out16[:, :width], out32.half()), "fp16 output != fp32 output rounded"
    alone, _ = run_ln(engine, x, gamma, beta, rows, C, ld_out, want32=False, **kw)
    assert _same(alone, out16), "fp16 output differs without the fp32 copy"
    assert _same(run_ln(engine, x, gamma, beta, rows, C, ld_out, **kw)[1], out32), "two identical calls differ"
    return out16, out32


@pytest.mark.parametrize("width", list(LN_WIDTHS))
def test_layernorm_rows_as_is(engine, dev, width, capsys):
    """Every width of the dispatch; 1003 rows leave a partial warp; ld_out > width (padding exactly +0)."""
    rows, ld_out = 1003, width + 12
    x, gamma, beta = ln_rows(dev, width, rows, width)
    out16, out32 = check_ln(engine, x, x, gamma, beta, rows, width, ld_out, f"width {width}", capsys)
    const = torch.arange(rows, device=dev) % 8 == 1
    assert torch.equal(out32[const], beta.expand(int(const.sum()), width)), "a constant row does not give beta exactly"
    part16, part32 = run_ln(engine, x[500:537].contiguous(), gamma, beta, 37, width, ld_out)
    assert _same(part16, out16[500:537]) and torch.equal(part32, out32[500:537]), "a row depends on its position"


def test_layernorm_gelu(engine, dev, capsys):
    """Exact-erf GELU after the affine (wav2vec2 / HuBERT layer-norm feature encoder, width 512)."""
    rows, width = 1003, 512
    x, gamma, beta = ln_rows(dev, 7, rows, width)
    check_ln(engine, x, x, gamma, beta, rows, width, width, "width 512 GELU", capsys, gelu=True)


@pytest.mark.parametrize("width", [512, 768, 1024])
def test_layernorm_fp32_copy_in_place(engine, dev, width):
    """Post-LN encoders write the normalised row back over the stream (out_f32 = x): the same values as a separate copy."""
    rows = 1003
    x, gamma, beta = ln_rows(dev, width + 1, rows, width)
    want16, want32 = run_ln(engine, x, gamma, beta, rows, width, width)
    got16, _ = run_ln(engine, x, gamma, beta, rows, width, width, alias=True)
    assert torch.equal(x, want32), "in-place fp32 copy differs from the separate one"
    assert _same(got16, want16)


def _window_perm(n_img, res, shift):
    tokens = torch.arange(n_img * res * res).view(n_img, res, res, 1)
    return co._partition(torch.roll(tokens, (-shift, -shift), (1, 2)), 8).reshape(-1)


@pytest.mark.parametrize("shift", [0, 4])
@pytest.mark.parametrize("res,C", [(64, 96), (64, 128), (32, 192), (32, 256), (16, 384), (16, 512)])
def test_layernorm_window_ordered(engine, dev, res, C, shift, capsys):
    """Row o normalises the token of window-ordered row o (the oracle's partition of the cyclically shifted grid)."""
    n_img = 2
    rows = n_img * res * res
    x, gamma, beta = ln_rows(dev, res + C + shift, rows, C)
    perm = _window_perm(n_img, res, shift).to(dev)
    out16, out32 = check_ln(engine, x, x[perm], gamma, beta, rows, C, C + 4, f"res {res} C {C} shift {shift}", capsys,
                            res=res, shift=shift)
    one16, one32 = run_ln(engine, x[res * res:].contiguous(), gamma, beta, res * res, C, C + 4, res=res, shift=shift)
    assert _same(one16, out16[res * res:]) and torch.equal(one32, out32[res * res:]), "an image depends on its position"


@pytest.mark.parametrize("res,C", [(64, 96), (32, 192), (16, 384), (64, 128), (32, 256), (16, 512)])
def test_layernorm_patch_merge_gather(engine, dev, res, C, capsys):
    """Output row (b, i, j) on the res/2 grid normalises [x(2i,2j), x(2i+1,2j), x(2i,2j+1), x(2i+1,2j+1)] (width 4 C),
    the concatenation of the Swin patch merging; each of the four parts has its own scale so a swap cannot cancel."""
    n_img = 3
    x, _, _ = ln_rows(dev, res * 3 + C, n_img * res * res, C)
    par = torch.arange(res, device=dev) % 2
    part_scale = torch.tensor([1.0, 2.0, 0.5, 4.0], device=dev)[par[:, None] + 2 * par[None, :]]    # [y, x]
    x = (x.view(n_img, res, res, C) * part_scale[None, :, :, None]).contiguous()
    _, gamma, beta = ln_rows(dev, C, 1, 4 * C)
    xi = x.view(n_img, res, res, C)
    merged = torch.cat([xi[:, 0::2, 0::2], xi[:, 1::2, 0::2], xi[:, 0::2, 1::2], xi[:, 1::2, 1::2]], -1)
    rows = n_img * (res // 2) ** 2
    check_ln(engine, x.view(-1, C), merged.reshape(rows, 4 * C), gamma, beta, rows, C, 4 * C + 8,
             f"merge res {res} C {C}", capsys, res=res, mode=1)


# ------------------------------------------------------------------------------------------------------- rejections
def _window_call(**over):
    def call(engine, outs):
        dev = engine.torch_device
        a = dict(n_windows=4, C=96, heads=4, res=16, shift=0, offset=0)
        a.update(over)
        qkv = torch.zeros((8 * 64, 3 * 128), dtype=torch.float16, device=dev)
        relbias = torch.zeros((32, 64, 64), device=dev)
        o = Guarded((8 * 64, 128), torch.float16, dev, GUARD)
        outs.append(o)
        engine.window_attention(qkv, a["n_windows"], a["C"], a["heads"], relbias, a["res"], a["shift"],
                                o.buf[GUARD + a["offset"]:])
    return call


def _bias_call(**over):
    def call(engine, outs):
        dev = engine.torch_device
        a = dict(n_clips=2, S=65, d=768)
        a.update(over)
        qkv = torch.zeros((2 * 65, 3 * 768), dtype=torch.float16, device=dev)
        o = Guarded((2 * 65, 768), torch.float16, dev, GUARD)
        outs.append(o)
        engine.attention_bias(qkv, a["n_clips"], a["S"], a["d"], torch.zeros((12, 129), device=dev),
                              torch.zeros((130, 12), device=dev), o.body)
    return call


def _gate_call(**over):
    def call(engine, outs):
        dev = engine.torch_device
        a = dict(rows=10, heads=12, d=768)
        a.update(over)
        o = Guarded((10, 12), torch.float32, dev, GUARD)
        outs.append(o)
        engine.wavlm_gate(torch.zeros((10, 768), device=dev), torch.zeros((8, 64), device=dev), torch.zeros(8, device=dev),
                          torch.ones(12, device=dev), a["rows"], a["heads"], a["d"], o.body)
    return call


def _bias_table_s0(engine, outs):
    _native.Engine.wavlm_bias_table(np.zeros((320, 12), np.float32), 0)


def _dec_call(d):
    def call(engine, outs):
        dev = engine.torch_device
        o = Guarded((4, 1024), torch.float16, dev, GUARD)
        outs.append(o)
        engine.decoder_self_attention(torch.zeros((4, 3 * 1024), dtype=torch.float16, device=dev), 2, d, o.body)
    return call


def _cross_call(**over):
    def call(engine, outs):
        dev = engine.torch_device
        a = dict(n_clips=2, S=100, d=384)
        a.update(over)
        o = Guarded((4, 384), torch.float16, dev, GUARD)
        outs.append(o)
        kv = torch.zeros((2 * 8000, 2 * 384), dtype=torch.float16, device=dev)
        engine.cross_attention(torch.zeros((4, 384), dtype=torch.float16, device=dev), kv, a["n_clips"], a["S"], a["d"],
                               o.body)
    return call


def _ln_call(**over):
    def call(engine, outs):
        dev = engine.torch_device
        a = dict(rows=512, C=128, ld_out=128, res=16, shift=0, mode=0, out32="own", offset=0, gamma=True)
        a.update(over)
        x = torch.zeros((2048, 512), device=dev)
        gamma = torch.ones(2048, device=dev)
        o16 = Guarded((2048, 512), torch.float16, dev, GUARD)
        o32 = Guarded((2048, 512), torch.float32, dev, GUARD)
        outs += [o16, o32]
        out32 = {"own": o32.body, "x": x, "none": None}[a["out32"]]
        engine.layernorm(x, gamma if a["gamma"] else None, gamma, a["rows"], a["C"], a["ld_out"], o16.buf[GUARD + a["offset"]:],
                         out32, res=a["res"], shift=a["shift"], mode=a["mode"])
    return call


REJECT = [
    # id, call, message
    ("window head dim 16", _window_call(C=64), "fad_window_attention: head dim C / heads must be 24 or 32"),
    ("window res not a power of two", _window_call(res=12, n_windows=1), "fad_window_attention: res must be a power of two >= 8"),
    ("window shift at res 8", _window_call(res=8, shift=4, n_windows=1), "fad_window_attention: shift must be 0, or in (0, 8) when res > 8"),
    ("window shift 8", _window_call(shift=8), "fad_window_attention: shift must be 0, or in (0, 8) when res > 8"),
    ("window partial image", _window_call(n_windows=6), "fad_window_attention: n_windows must be a positive multiple of (res / 8)^2"),
    ("window misaligned out", _window_call(offset=4), "fad_window_attention: qkv, relbias and out must be 16-byte aligned"),
    ("bias d not heads x 64", _bias_call(d=800), "fad_attention_bias: d must be a positive multiple of 64"),
    ("bias S 0", _bias_call(S=0), "fad_attention_bias: S must be positive"),
    ("bias no clips", _bias_call(n_clips=0), "fad_attention_bias: n_clips must be in [1, 65535]"),
    ("gate d not heads x 64", _gate_call(d=700), "fad_wavlm_gate: d must be heads * 64"),
    ("gate no rows", _gate_call(rows=0), "fad_wavlm_gate: rows must be positive"),
    ("bias table S 0", _bias_table_s0, "fad_wavlm_bias_table: heads and S must be positive"),
    ("decoder d 96", _dec_call(96), "fad_decoder_self_attention: d must be a positive multiple of 64"),
    ("cross S beyond shared memory", _cross_call(S=7000),
     "fad_cross_attention: S must be positive and its 2 S fp32 scores must fit in shared memory"),
    ("cross S 0", _cross_call(S=0), "fad_cross_attention: S must be positive and its 2 S fp32 scores must fit in shared memory"),
    ("cross d 96", _cross_call(d=96), "fad_cross_attention: d must be a positive multiple of 64"),
    ("cross no clips", _cross_call(n_clips=0), "fad_cross_attention: n_clips must be in [1, 65535]"),
    ("ln ld_out below width", _ln_call(ld_out=124), "clap_ln: ld_out must be a multiple of 4 and at least the width"),
    ("ln ld_out not a multiple of 4", _ln_call(ld_out=130), "clap_ln: ld_out must be a multiple of 4 and at least the width"),
    ("ln unknown mode", _ln_call(mode=2), "clap_ln: mode must be 0 (rows as they are or window-ordered) or 1 (patch-merge gather)"),
    ("ln merge without res", _ln_call(mode=1, res=0, ld_out=512), "clap_ln: the patch-merge gather needs res"),
    ("ln window rows aliased", _ln_call(out32="x"), "clap_ln: out_f32 may alias x only as the same rows in token order (mode 0, res 0)"),
    ("ln merge rows aliased", _ln_call(out32="x", mode=1, rows=64, ld_out=512),
     "clap_ln: out_f32 may alias x only as the same rows in token order (mode 0, res 0)"),
    ("ln res not a power of two", _ln_call(res=12, rows=144), "clap_ln: res must be 0 or a power of two >= 8"),
    ("ln shift without res", _ln_call(res=0, shift=4), "clap_ln: shift needs res"),
    ("ln shift not below res", _ln_call(shift=16), "clap_ln: shift must be in [0, res), and 0 in mode 1"),
    ("ln partial image", _ln_call(rows=500), "clap_ln: window-ordered rows must be whole images"),
    ("ln no rows", _ln_call(rows=0, res=0), "clap_ln: rows and C must be positive"),
    ("ln misaligned out", _ln_call(offset=2), "clap_ln: x, gamma, beta and out_f32 must be 16-byte aligned, out 8-byte aligned"),
    ("ln null gamma", _ln_call(gamma=False), "clap_ln: null x, gamma, beta or out"),
    ("ln unsupported width", _ln_call(C=640, ld_out=640, res=0), "unsupported LayerNorm width"),
]


@pytest.mark.parametrize("call,message", [c[1:] for c in REJECT], ids=[c[0] for c in REJECT])
def test_stage_entries_reject_invalid_arguments(engine, call, message):
    """Arguments the launch cannot honour fail with their message, launch nothing and write nothing."""
    expect_rejected(engine, call, message, [])
