"""The wgmma GEMM behind every convolution and Linear layer (csrc/conv_gemm.cuh) called the way the models call it:
through fad_linear (clap_gemm: ragged K and N, overlapping A rows, GELU / ELU, fused residual, fp16 and fp32 outputs)
and fad_umma_layer (3x3 convolutions).

References are fp64, computed from the exact fp16 A and the fp32 weights the packing started from.  Weight padding
(columns past k_cols, rows past n_cols) and bias padding hold non-zero values, so reading past k_cols or storing
past n_cols changes a result.  Every output lives inside a buffer whose unused part and guard regions (leading 256
elements, two extra rows and 256 trailing elements) hold a NaN sentinel: every test checks that the sentinel is
intact and that every output element was written.
"""
import math

import numpy as np
import pytest
import torch
from scipy.special import erf

from fadtk_b200 import weights as wts
from gpu_checks import Guarded, expect_rejected, rms_rel
from oracle import clap_oracle as co

pytestmark = pytest.mark.gpu

GUARD = 256
ACT_NONE, ACT_RELU, ACT_GELU, ACT_ELU = 0, 1, 2, 3


def _pad(v, m):
    return (v + m - 1) // m * m


@pytest.fixture(scope="module")
def dev(engine):
    return engine.torch_device


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def make_problem(dev, seed, rows, k_cols, n_cols, split_w, w_scale=0.5, a=None):
    """A fp16 [rows, k_cols] (unless given), fp32 weights [n_cols, k_cols] and bias [n_cols], and their packed
    device forms with non-zero padding.  split_w = 0 draws fp16-representable weights, so both modes start from
    the weights the reference uses."""
    g = _gen(dev, seed)
    if a is None:
        a = torch.randn((rows, k_cols), generator=g, device=dev).to(torch.float16)
    Np, Kp = _pad(n_cols, 128), _pad(k_cols, 64)
    full = 0.25 + torch.randn((Np, Kp), generator=g, device=dev) * w_scale      # padding: non-zero, finite
    w32 = torch.randn((n_cols, k_cols), generator=g, device=dev) * w_scale
    if not split_w:
        w32 = w32.half().float()
    full[:n_cols, :k_cols] = w32
    packed = wts.split_hi_lo_tiles(full) if split_w else full.half()
    bias_full = 3.0 + torch.randn((Np,), generator=g, device=dev)                  # padding: non-zero
    bias = torch.randn((n_cols,), generator=g, device=dev) * 0.5
    bias_full[:n_cols] = bias
    return a, w32, bias, packed.contiguous(), bias_full.contiguous()


def act64(x, act):
    if act == ACT_RELU:
        return x.clamp_min(0.0)
    if act == ACT_GELU:
        return 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))
    if act == ACT_ELU:
        return torch.where(x > 0, x, torch.expm1(x))
    return x


def reference(a, w32, bias, act):
    """(fp64 result, fp64 bound on |kernel - result| at the fp32-accumulation level)."""
    a64, w64 = a.double(), w32.double()
    pre = a64 @ w64.t() + bias.double()
    # fp32 accumulation over K (wgmma truncation, chunk sums, hi/lo weights: 2^-22 relative per weight) is far below
    # 2^-20 of sum |a w|; + the rounding of the bias add and of the activation (GELU/ELU: ~2.3e-7 of |x|)
    mag = a64.abs() @ w64.abs().t()
    pre_bound = 2.0 ** -20 * mag + 2.0 ** -22 * pre.abs() + 1e-30
    bound = pre_bound * (1.2 if act in (ACT_GELU, ACT_ELU) else 1.0) + (3e-7 * pre.abs() if act in (ACT_GELU, ACT_ELU) else 0.0)
    return act64(pre, act), bound


def check_f32(out32, ref, bound, what):
    err = (out32.double() - ref).abs()
    ratio = (err / bound).max().item()
    assert ratio <= 1.0, f"{what}: max |err| / bound = {ratio:.3g} (max err {err.max().item():.3g})"
    rms = (err.square().mean().sqrt() / ref.square().mean().sqrt().clamp_min(1e-30)).item()
    assert rms <= 2e-6, f"{what}: rms relative error {rms:.3g} is above the fp32-accumulation level"


def run_linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, split_w, lda=0, want=("16", "32"),
               resid=None, resid_C=0, resid_res=0, resid_shift=0):
    dev = a.device
    o16 = Guarded((rows, n_cols), torch.float16, dev, GUARD, GUARD + 2 * n_cols) if "16" in want else None
    o32 = Guarded((rows, n_cols), torch.float32, dev, GUARD, GUARD + 2 * n_cols) if "32" in want else None
    engine.linear(a, rows, k_cols, packed, bias_full, n_cols, act, lda=lda, split_w=split_w,
                  out16=o16.body if o16 else None, out32=o32.body if o32 else None,
                  resid=resid, resid_C=resid_C, resid_res=resid_res, resid_shift=resid_shift)
    for o in (o16, o32):
        if o is not None:
            o.check()
    return (o16.body if o16 else None), (o32.body if o32 else None)


def check_all_outputs(engine, a, rows, k_cols, w32, bias, packed, bias_full, n_cols, act, split_w, lda=0, ref=None):
    """fp32 alone, fp16 alone, both together: the fp32 result is at the reference's accumulation level, and all
    three calls store the same f (bitwise: fp16 == fp32.half())."""
    _, out32 = run_linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, split_w, lda, want=("32",))
    out16, _ = run_linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, split_w, lda, want=("16",))
    both16, both32 = run_linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, split_w, lda, want=("16", "32"))
    assert torch.equal(both32, out32), "fp32 output differs when fp16 is stored too"
    assert torch.equal(both16.view(torch.int16), out32.half().view(torch.int16)), "fp16 output (with fp32) != fp32.half()"
    assert torch.equal(out16.view(torch.int16), out32.half().view(torch.int16)), "fp16 output (alone) != fp32.half()"
    if ref is None:
        ref = reference(a, w32, bias, act)
    check_f32(out32, *ref, f"rows={rows} K={k_cols} N={n_cols} act={act} split_w={split_w}")
    return out32


# ----------------------------------------------------------------------------------------------- a. shapes and edges
SHAPES = [
    # rows,   K,     N,  act, split_w
    (1, 64, 48, ACT_NONE, 1),
    (127, 80, 96, ACT_RELU, 0),
    (128, 96, 128, ACT_GELU, 1),
    (129, 384, 200, ACT_ELU, 1),
    (1000, 576, 288, ACT_GELU, 0),          # 9 k-steps: uneven 5 + 4 chunks
    (129, 1536, 384, ACT_NONE, 1),
    (1000, 3584, 2048, ACT_RELU, 1),
    (127, 12288, 1536, ACT_NONE, 1),
    (129, 12288, 48, ACT_ELU, 0),
    (40000, 384, 384, ACT_GELU, 1),         # 939 tiles on 132 SMs: every CTA runs 7 or 8 tiles
    (40000, 96, 48, ACT_ELU, 0),            # 313 tiles, not a multiple of the SM count
    # CLAP HTSAT tiny (C = 96 .. 768) and base (C = 128 .. 1024): qkv, proj, fc1 (GELU), fc2, patch-merge reduction
    (4096, 96, 288, ACT_NONE, 1),
    (4096, 128, 128, ACT_NONE, 1),
    (2048, 192, 768, ACT_GELU, 1),
    (1024, 1024, 256, ACT_NONE, 1),
    (1024, 1536, 384, ACT_NONE, 1),
    (512, 2048, 1024, ACT_NONE, 1),
    (256, 768, 2304, ACT_NONE, 1),
    (256, 4096, 1024, ACT_NONE, 1),
    # Whisper tiny / small: conv1 (K = 3 x 128 padded mel taps) and conv2 (K = 3 d), GELU
    (3000, 384, 384, ACT_GELU, 1),
    (1500, 2304, 768, ACT_GELU, 1),
    # wav2vec feature conv0 (K = 64), Encodec ELU convs and LSTM input / recurrent GEMMs, last conv
    (2000, 64, 512, ACT_NONE, 1),
    (1000, 64, 128, ACT_ELU, 1),
    (1000, 96, 16, ACT_ELU, 1),
    (300, 512, 2048, ACT_NONE, 1),
    (64, 1024, 2048, ACT_NONE, 1),
    (500, 3584, 128, ACT_NONE, 1),
]


@pytest.mark.parametrize("rows,k_cols,n_cols,act,split_w", SHAPES)
def test_linear_matches_fp64_reference(engine, dev, rows, k_cols, n_cols, act, split_w):
    seed = rows * 7 + k_cols * 13 + n_cols * 17 + act
    a, w32, bias, packed, bias_full = make_problem(dev, seed, rows, k_cols, n_cols, split_w)
    check_all_outputs(engine, a, rows, k_cols, w32, bias, packed, bias_full, n_cols, act, split_w)


# ---------------------------------------------------------------------------------------------- b. overlapping rows
OVERLAP = [
    # T rows of C channels, window taps, stride, N, act, outputs: the wav2vec feature convs and positional conv
    (4001, 512, 3, 2, 512, ACT_GELU),       # K = 1536, lda = 1024
    (4000, 512, 2, 2, 512, ACT_GELU),       # K = 1024, lda = 1024 (adjacent windows)
    (40001, 512, 3, 2, 512, ACT_NONE),      # 20000 rows: persistent CTAs over overlapping rows
    (600, 48, 128, 1, 48, ACT_GELU),        # positional conv group: K = 128 x 48, lda = 48, N = 48
]


@pytest.mark.parametrize("T,C,taps,stride,n_cols,act", OVERLAP)
def test_linear_overlapping_rows(engine, dev, T, C, taps, stride, n_cols, act):
    g = _gen(dev, T + C + taps)
    x = torch.randn((T, C), generator=g, device=dev).to(torch.float16)
    k_cols, lda = taps * C, stride * C
    a_ref = x.reshape(-1).unfold(0, k_cols, lda)                        # [rows, K] windows, lda apart
    rows = a_ref.shape[0]
    _, w32, bias, packed, bias_full = make_problem(dev, T * 3 + n_cols, rows, k_cols, n_cols, 1, a=a_ref,
                                                   w_scale=1.0 / math.sqrt(k_cols))
    check_all_outputs(engine, x, rows, k_cols, w32, bias, packed, bias_full, n_cols, act, 1, lda=lda,
                      ref=reference(a_ref, w32, bias, act))


# ------------------------------------------------------------------------------------------------ c. fused residual
def _resid_case(engine, dev, seed, rows, k_cols, n_cols, act, resid_C, res, shift, perm):
    a, w32, bias, packed, bias_full = make_problem(dev, seed, rows, k_cols, n_cols, 1)
    _, out32 = run_linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, 1, want=("32",))
    check_f32(out32, *reference(a, w32, bias, act), "residual GEMM")
    before = torch.randn((rows, resid_C), generator=_gen(dev, seed + 1), device=dev)
    expect = before.clone()
    expect[perm] = before[perm] + out32[:, :resid_C]                     # row r adds into token perm[r]
    # the residual alone (how the transformer blocks call it), then together with both outputs
    for want in ((), ("16", "32")):
        r = Guarded((rows, resid_C), torch.float32, dev, GUARD, GUARD + 2 * resid_C, init=before)
        o16, o32 = run_linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, 1, want=want,
                              resid=r.body, resid_C=resid_C, resid_res=res, resid_shift=shift)
        assert r.guards_intact(), "residual guard region overwritten"
        bad = (r.body != expect).any(1).nonzero().flatten()
        assert bad.numel() == 0, f"residual rows {bad[:8].tolist()} (of {bad.numel()}) differ from x + C scattered"
        if want:
            assert torch.equal(o32, out32)
            assert torch.equal(o16.view(torch.int16), out32.half().view(torch.int16))


PLAIN_RESID = [
    # rows, K, N, act, resid_C
    (3000, 1152, 384, ACT_GELU, 384),       # Whisper tiny conv2 + residual
    (1000, 2304, 768, ACT_NONE, 768),       # Whisper small fc2 / wav2vec fc2 shape
    (2000, 64, 128, ACT_NONE, 128),         # Encodec residual 1x1 conv, time-packed (resid_C = n_cols)
    (2000, 16, 32, ACT_NONE, 32),           # the same layer unpacked
    (300, 96, 200, ACT_GELU, 192),          # resid_C < n_cols, ragged last group
    (40000, 96, 96, ACT_NONE, 96),          # persistent CTAs: residual rows prefetched for the next tile
]


@pytest.mark.parametrize("rows,k_cols,n_cols,act,resid_C", PLAIN_RESID)
def test_linear_fused_residual(engine, dev, rows, k_cols, n_cols, act, resid_C):
    perm = torch.arange(rows, device=dev)
    _resid_case(engine, dev, rows + k_cols + n_cols, rows, k_cols, n_cols, act, resid_C, 0, 0, perm)


WINDOW_RESID = [
    # res, C, batch, K (proj: C, fc2: 4 C)
    (64, 96, 2, 96),
    (32, 192, 2, 768),
    (16, 384, 3, 384),
    (8, 768, 2, 3072),
]


@pytest.mark.parametrize("shift", [0, 4])
@pytest.mark.parametrize("res,C,batch,k_cols", WINDOW_RESID)
def test_linear_window_ordered_residual(engine, dev, res, C, batch, k_cols, shift):
    """Swin blocks add the window-ordered GEMM rows back into token order: the row -> token map comes from the
    oracle's own window partition of the cyclically shifted token grid."""
    tokens = torch.arange(batch * res * res).view(batch, res, res, 1)
    perm = co._partition(torch.roll(tokens, (-shift, -shift), (1, 2)), 8).reshape(-1)
    assert torch.equal(perm.sort().values, torch.arange(batch * res * res))
    _resid_case(engine, dev, res * 1000 + C + shift, batch * res * res, k_cols, C, ACT_NONE, C, res, shift, perm.to(dev))


# ------------------------------------------------------------------------------------- d. activations, isolated
def _bias_grid():
    f32 = np.float32
    grid = [np.linspace(-20.0, 20.0, 16001, dtype=np.float64).astype(f32)]
    edges = [0.0, -0.0, 1e-30, -1e-30, 1e-38, -1e-38, 1e-45, -1e-45, 1e-7, -1e-7, 1e-3, -1e-3]
    for x0 in (-1.0 / 16.0, 4.3 * math.sqrt(2.0), -4.3 * math.sqrt(2.0), 3.5 * math.sqrt(2.0), -3.5 * math.sqrt(2.0)):
        c = f32(x0)
        edges += [c, np.nextafter(c, f32(-np.inf)), np.nextafter(c, f32(np.inf))]
        edges += list(np.linspace(float(c) - 1e-3, float(c) + 1e-3, 41))
    grid.append(np.array(edges, dtype=f32))
    g = np.concatenate(grid)
    return np.concatenate([g, np.zeros(_pad(g.size, 8) - g.size, dtype=f32)])


def _act_exact(x64, act):
    if act == ACT_RELU:
        return np.maximum(x64, 0.0)
    if act == ACT_GELU:
        return 0.5 * x64 * (1.0 + erf(x64 / math.sqrt(2.0)))
    return np.where(x64 > 0, x64, np.expm1(x64))


def _act_bound(x64, ref, act):
    """The error budgets stated next to gelu_erf / elu_ex2: GELU: erf to 1.4e-7 (plus the rounding of 1 +- (1 - e),
    2^-23 of the bracket) times |x| / 2, plus a few ulps of the result; ELU: 2^-22 absolute on the ex2 branch,
    ~1e-7 relative on the Taylor branch (x > -1/16)."""
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    if act == ACT_RELU:
        return np.zeros_like(x64)
    if act == ACT_GELU:
        return 0.5 * np.abs(x64) * (1.4e-7 + 2.0 ** -23) + 4 * ulp
    taylor = (x64 > -0.0625) & (x64 <= 0)
    return np.where(x64 > 0, 0.0, np.where(taylor, 2e-7 * np.abs(ref), 2.0 ** -22)) + 2 * ulp


@pytest.mark.parametrize("act", [ACT_RELU, ACT_GELU, ACT_ELU], ids=["relu", "gelu", "elu"])
def test_activation_on_exact_zero_accumulator(engine, dev, act):
    """Zero weights: the accumulator is exactly 0, so column j of the output is act(bias[j]) with no GEMM noise."""
    grid = _bias_grid()
    n_cols, k_cols, rows = grid.size, 64, 130
    Np = _pad(n_cols, 128)
    bias_full = torch.full((Np,), 5.0, device=dev)
    bias_full[:n_cols] = torch.from_numpy(grid).to(dev)
    packed = torch.zeros((2 * Np, k_cols), dtype=torch.float16, device=dev)
    a = torch.randn((rows, k_cols), generator=_gen(dev, 5), device=dev).to(torch.float16)
    _, out32 = run_linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, 1, want=("32",))
    assert (out32 == out32[0]).all(), "rows of a zero-weight GEMM differ"
    got = out32[0].double().cpu().numpy()
    x64 = grid.astype(np.float64)
    ref = _act_exact(x64, act)
    err = np.abs(got - ref)
    bound = _act_bound(x64, ref, act)
    worst = int(np.argmax(err - bound))
    assert (err <= bound).all(), f"act {act}: x = {x64[worst]!r}: got {got[worst]!r}, want {ref[worst]!r} (bound {bound[worst]:.3g})"


@pytest.mark.parametrize("act", [ACT_RELU, ACT_GELU, ACT_ELU], ids=["relu", "gelu", "elu"])
def test_activation_applied_to_the_same_accumulator(engine, dev, act):
    """Random A and W: the kernel is deterministic, so out(act) is act applied to out(none) within the same bounds."""
    rows, k_cols, n_cols = 1000, 384, 384
    a, _, _, packed, bias_full = make_problem(dev, 77, rows, k_cols, n_cols, 1, w_scale=1.0 / math.sqrt(k_cols))
    bias_full[:n_cols] *= 8.0                                                 # spread x over [-10, 10]
    _, pre = run_linear(engine, a, rows, k_cols, packed, bias_full, n_cols, ACT_NONE, 1, want=("32",))
    _, post = run_linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, 1, want=("32",))
    x64 = pre.double().cpu().numpy()
    ref = _act_exact(x64, act)
    err = np.abs(post.double().cpu().numpy() - ref)
    assert (err <= _act_bound(x64, ref, act)).all(), f"act {act}: max err {err.max():.3g}"


# -------------------------------------------------------------------------------------- e. weight-split precision
def _split_errors(engine, dev, kind, k):
    """rms relative error of the fp32 output per weight mode against fp64 from the fp32 weights."""
    g = _gen(dev, 1000 + k)
    if kind == "conv":
        nb, hh, ww, cin, cout, taps = 8, 12, 8, 512, 256, 9
    else:
        nb, hh, ww, cin, cout, taps = 256, 1, 1, k, 256, 1
    x = torch.randn((nb, hh, ww, cin), generator=g, device=dev).to(torch.float16)
    w32 = torch.randn((cout, taps * cin), generator=g, device=dev) * (2.0 / (taps * cin)) ** 0.5
    b = torch.randn((cout,), generator=g, device=dev) * 0.1
    if taps == 9:
        wt = w32.double().reshape(cout, 3, 3, cin).permute(0, 3, 1, 2)
        ref = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), wt, b.double(), padding=1).permute(0, 2, 3, 1)
    else:
        ref = (x.double().reshape(nb, cin) @ w32.double().t() + b.double()).reshape(nb, 1, 1, cout)
    packs = {0: w32.half().contiguous(), 1: wts.split_hi_lo_tiles(w32)}
    errs = {}
    for mode in (0, 1):
        _, out32 = engine.umma_layer(x, packs[mode], b, taps, False, False, want_f32=True, split_w=mode)
        errs[f"layer{mode}"] = rms_rel(out32, ref)
    if taps == 1:
        a = x.reshape(nb, cin)
        for mode in (0, 1):
            _, out32 = run_linear(engine, a, nb, cin, packs[mode], b, cout, ACT_NONE, mode, want=("32",))
            errs[f"linear{mode}"] = rms_rel(out32, ref.reshape(nb, cout))
    return errs


# about 3x the largest rms relative error measured per mode (see test_hi_lo_weights_remove_fp16_rounding)
SPLIT_CEIL = {0: 6e-4, 1: 4.5e-6}


@pytest.mark.parametrize("kind,k", [("fc", 4096), ("fc", 12288), ("conv", 9 * 512)])
def test_hi_lo_weights_remove_fp16_rounding(engine, dev, kind, k, capsys):
    """Each weight mode against fp64 from the fp32 weights.  The hi/lo pair must remove the fp16 weight rounding
    (mode 1 <= mode 0 / 100), each below an absolute ceiling.

    Measured on an H100 80GB HBM3 (rms relative error of the fp32 output; fad_linear and fad_umma_layer agree):
        K = 4096:          mode 0 2.07e-4   mode 1 1.02e-6
        K = 12288:         mode 0 2.05e-4   mode 1 1.50e-6
        9 x 512 conv:      mode 0 2.07e-4   mode 1 1.06e-6
    Mode 1 is ~1e-6, not the ~1e-7 22 bits would give: at |w| ~ sqrt(2 / K) the lo parts are fp16 subnormals
    (spacing 2^-24), so the pair keeps about 20 bits of each weight.  That physical limit puts 'mode 1 <= mode 0 / 100'
    close to its bound (1.37x margin at K = 12288): the seeds are fixed and the kernel is deterministic, so it is
    stable, but smaller weights (a larger K or another weight scale) move mode 1 towards the bound."""
    errs = _split_errors(engine, dev, kind, k)
    with capsys.disabled():
        print(f"\n[split precision] {kind} K={k}: " + "  ".join(f"{n}={v:.3e}" for n, v in errs.items()))
    for path in ("layer", "linear"):
        if f"{path}0" not in errs:
            continue
        e0, e1 = errs[f"{path}0"], errs[f"{path}1"]
        assert e0 <= SPLIT_CEIL[0], errs
        assert e1 <= e0 / 100 and e1 <= SPLIT_CEIL[1], errs


# ------------------------------------------------------------------------------------------ f. accumulation bias
@pytest.mark.parametrize("weights", ["fp32", "fp16-exact"])
@pytest.mark.parametrize("kind,k", [("fc", 4096), ("fc", 12288), ("conv", 9 * 512)])
def test_accumulation_is_unbiased(engine, dev, kind, k, weights, capsys):
    """The tensor core truncates when it accumulates: uncorrected, a 512-long chunk of positive-leaning products
    comes out scaled by 1 - 512 x 1.06e-9 = 1 - 5.4e-7.  The per-chunk unshrink must leave |slope - 1| <= 1.5e-7,
    slope = <out, ref> / <ref, ref> over all outputs (split weights with non-zero lo parts, post-ReLU-like activations).

    Measured on an H100 80GB HBM3, slope - 1:      K = 4096    K = 12288   9 x 512 conv
        unshrink counting 2 x 512 per chunk         -1.8e-8     +7.4e-8     +2.8e-8
        counting only the 512 hi products           -5.6e-7     -4.7e-7     -5.1e-7
    (the lo-part wgmmas share the accumulator and truncate it like the hi ones).
    Weights exact in fp16 packed as hi/lo pairs have all-zero lo parts, whose wgmmas add exact zeros and do not
    truncate, so the count is decided per weight tensor.  Measured, fp16-exact weights:
        per-tensor count (lo parts found zero)       -9.6e-9     +8.7e-9     +3.6e-9
        2 x 512 counted regardless of the weights   +5.3e-7     +5.5e-7     +5.4e-7"""
    g = _gen(dev, 2000 + k)
    if kind == "conv":
        nb, hh, ww, cin, cout, taps = 16, 12, 8, 512, 512, 9
    else:
        nb, hh, ww, cin, cout, taps = 512, 1, 1, k, 512, 1
    x = torch.relu(torch.randn((nb, hh, ww, cin), generator=g, device=dev) + 0.3).to(torch.float16)
    w32 = torch.randn((cout, taps * cin), generator=g, device=dev) * (2.0 / (taps * cin)) ** 0.5
    if weights == "fp16-exact":
        w32 = w32.half().float()
    b = torch.zeros(cout, device=dev)
    packed = wts.split_hi_lo_tiles(w32)
    if taps == 9:
        wt = w32.double().reshape(cout, 3, 3, cin).permute(0, 3, 1, 2)
        ref = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), wt, padding=1).permute(0, 2, 3, 1).reshape(-1)
        _, out32 = engine.umma_layer(x, packed, b, taps, False, False, want_f32=True, split_w=1)
    else:
        ref = (x.double().reshape(nb, cin) @ w32.double().t()).reshape(-1)
        _, out32 = run_linear(engine, x.reshape(nb, cin), nb, cin, packed, b, cout, ACT_NONE, 1, want=("32",))
    o = out32.double().reshape(-1)
    slope = ((o * ref).sum() / (ref * ref).sum()).item()
    with capsys.disabled():
        print(f"\n[accumulation bias] {kind} K={taps * cin} {weights} weights: slope - 1 = {slope - 1:+.3e}")
    assert abs(slope - 1.0) <= 1.5e-7, f"slope - 1 = {slope - 1:+.3e}"


# -------------------------------------------------------------------------------- g. persistence and determinism
@pytest.mark.parametrize("act,split_w", [(ACT_GELU, 1), (ACT_NONE, 0)])
def test_rows_do_not_depend_on_tile_position(engine, dev, act, split_w):
    """A row's outputs are bitwise the same whether it is computed in a 129-row call or at another tile position
    of a 40 000-row call (every CTA runs several tiles there), and two identical calls are bitwise equal."""
    rows, k_cols, n_cols, off = 40000, 384, 384, 25037
    a, _, _, packed, bias_full = make_problem(dev, 31 + act, rows, k_cols, n_cols, split_w)
    big16, big32 = run_linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, split_w)
    again16, again32 = run_linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, split_w)
    assert torch.equal(big32, again32) and torch.equal(big16.view(torch.int16), again16.view(torch.int16))
    small16, small32 = run_linear(engine, a[off:off + 129], 129, k_cols, packed, bias_full, n_cols, act, split_w)
    assert torch.equal(small32, big32[off:off + 129]), "fp32 rows depend on their tile position"
    assert torch.equal(small16.view(torch.int16), big16[off:off + 129].view(torch.int16))


# ------------------------------------------------------------------------------------------------- h. rejections
REJECT = [
    # id, arguments, the clap_gemm message
    ("n_cols not a multiple of 8", dict(n_cols=44), "n_cols must be a positive multiple of 8"),
    ("fp32-only n_cols not a multiple of 8", dict(n_cols=36, want=("32",)), "n_cols must be a positive multiple of 8"),
    ("k_cols not a multiple of 8", dict(k_cols=60), "k_cols must be a positive multiple of 8"),
    ("lda not a multiple of 8", dict(lda=100), "lda must be a multiple of 8"),
    ("resid_C not a multiple of 32", dict(resid_C=48), "resid_C must be a positive multiple of 32 and at most n_cols"),
    ("resid_C above n_cols", dict(n_cols=96, resid_C=128), "resid_C must be a positive multiple of 32 and at most n_cols"),
    ("window resolution not a power of two", dict(resid_C=96, resid_res=12), "resid_res must be a power of two >= 8"),
    ("window shift not below the resolution", dict(resid_C=96, resid_res=8, resid_shift=8), "resid_shift must be in [0, resid_res)"),
    ("rows not whole window images", dict(resid_C=96, resid_res=16), "window-ordered rows must be whole images"),
    ("misaligned fp32 output", dict(misalign="out32"), "A, W, bias, outputs and residual must be 16-byte aligned"),
    ("misaligned fp16 output", dict(misalign="out16"), "A, W, bias, outputs and residual must be 16-byte aligned"),
    ("unknown activation", dict(act=4), "act must be 0 (none), 1 (ReLU), 2 (GELU) or 3 (ELU)"),
    ("E4M3 low-part mode", dict(split_w=2), "split_w must be 0 or 1"),
    ("null bias", dict(no_bias=True), "null A, W or bias"),
    ("no output", dict(want=()), "no output"),
]


@pytest.mark.parametrize("case,message", [c[1:] for c in REJECT], ids=[c[0] for c in REJECT])
def test_linear_rejects_invalid_arguments(engine, dev, case, message):
    """Arguments the epilogue or TMA cannot honour fail with clap_gemm's message, launch nothing and write nothing."""
    rows, k_cols, n_cols = 192, case.get("k_cols", 128), case.get("n_cols", 128)
    a = torch.randn((rows, 256), generator=_gen(dev, 3), device=dev).to(torch.float16)
    packed = torch.randn((2 * 128, 128), generator=_gen(dev, 4), device=dev).to(torch.float16)
    bias = None if case.get("no_bias") else torch.randn((128,), generator=_gen(dev, 5), device=dev)
    want = case.get("want", ("16", "32"))
    o16 = Guarded((rows, 128), torch.float16, dev, GUARD, GUARD + 256)
    o32 = Guarded((rows, 128), torch.float32, dev, GUARD, GUARD + 256)
    r = Guarded((rows, 128), torch.float32, dev, GUARD, GUARD + 256)
    resid_C = case.get("resid_C", 0)
    out16 = o16.body if "16" in want else None
    out32 = o32.body if "32" in want else None
    if case.get("misalign") == "out32":
        out32 = o32.ptr("odd")
    if case.get("misalign") == "out16":
        out16 = o16.buf[GUARD + 4:]

    def call(engine, outs):
        engine.linear(a, rows, k_cols, packed, bias, n_cols, case.get("act", ACT_NONE), lda=case.get("lda", 0),
                      split_w=case.get("split_w", 1), out16=out16, out32=out32, resid=r.body if resid_C else None,
                      resid_C=resid_C, resid_res=case.get("resid_res", 0), resid_shift=case.get("resid_shift", 0))
    expect_rejected(engine, call, "clap_gemm: " + message, [o16, o32, r])


def _umma_layer_split_w_2(engine, outs):
    dev = engine.torch_device
    x = torch.zeros((1, 1, 1, 64), dtype=torch.float16, device=dev)
    w = torch.zeros((2 * 128, 64), dtype=torch.float16, device=dev)
    engine.umma_layer(x, w, torch.zeros(128, device=dev), 1, False, False, want_f32=True, split_w=2)


def _stats_tensor_core_1(engine, outs):
    e = torch.zeros((16, 64), dtype=torch.float16, device=engine.torch_device)
    engine.stats_accumulate(e, e[0], engine.stats_new(64), tensor_core=1)


MODE_REJECT = [
    # id, call, message: the other stage entries whose mode number comes from the caller
    ("fad_umma_layer split_w 2", _umma_layer_split_w_2, "fad_umma_layer: split_w must be 0 (fp16 weights) or 1 (fp16 hi/lo pair)"),
    ("fad_stats_accumulate tensor_core 1", _stats_tensor_core_1,
     "fad_stats_accumulate: tensor_core must be 0 (DMMA) or 2 (CUDA-core fp64)"),
]


@pytest.mark.parametrize("call,message", [c[1:] for c in MODE_REJECT], ids=[c[0] for c in MODE_REJECT])
def test_stage_entries_reject_unknown_modes(engine, call, message):
    """A mode the library does not have fails with its message and launches nothing."""
    expect_rejected(engine, call, message, [])
