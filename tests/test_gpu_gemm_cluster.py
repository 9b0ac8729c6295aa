"""The CTA pairing of the wgmma GEMM (csrc/conv_gemm.cuh): clusters of two CTAs compute neighbouring M tiles of one
N tile and share each weight box by TMA multicast.  With an odd number of M tiles the last pair's second CTA is a
spare that must store nothing.

Every case is checked against the fp64 reference the way tests/test_gpu_gemm.py checks it, and again with the input
shifted by an odd number of M tiles (128 rows, or whole images that make an odd number of tiles), which moves every
tile to the other rank of its pair and flips the parity of the tile count: the shared rows must come out bitwise
the same.  Outputs sit between NaN sentinels, with a trailing guard longer than a spare tile can reach.
"""
import pytest
import torch

from fadtk_b200 import _native
from fadtk_b200 import weights as wts
from gpu_checks import SENTINEL, Guarded
from test_gpu_gemm import ACT_ELU, ACT_GELU, ACT_NONE, ACT_RELU, _gen, check_f32, make_problem, reference

pytestmark = pytest.mark.gpu
GUARD = 256


# ------------------------------------------------------------------------------------------ plain geometry (Linear)
def linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, split_w, resid=None, resid_C=0):
    """fad_linear into fenced fp16 and fp32 outputs (and the fenced residual); 256 rows of trailing guard cover the
    rows of a spare tile, which start at the next multiple of 128 at or after `rows`."""
    dev = a.device
    o16 = Guarded((rows, n_cols), torch.float16, dev, GUARD, 256 * n_cols)
    o32 = Guarded((rows, n_cols), torch.float32, dev, GUARD, 256 * n_cols)
    r = Guarded((rows, resid_C), torch.float32, dev, GUARD, 256 * resid_C, init=resid) if resid is not None else None
    engine.linear(a, rows, k_cols, packed, bias_full, n_cols, act, split_w=split_w, out16=o16.body, out32=o32.body,
                  resid=r.body if r else None, resid_C=resid_C)
    for o, what in ((o16, "fp16 output"), (o32, "fp32 output"), (r, "residual")):
        if o is not None:
            o.check(what)
    assert torch.equal(o16.body.view(torch.int16), o32.body.half().view(torch.int16)), "fp16 output != fp32.half()"
    return o32.body, (r.body if r else None)


PLAIN = [
    # rows, K, N, act, split_w: M tiles (and after the 128-row shift) x N tiles
    (100, 192, 256, ACT_GELU, 1),       # a single tile (1 -> 2) x 2: its pair's rank 1 is a spare
    (549, 384, 384, ACT_NONE, 1),       # 5 -> 6 tiles x 3
    (200, 256, 4096, ACT_RELU, 1),      # 2 -> 3 x 32 N tiles: 32 -> 64 units, fewer than the CTA pairs
    (50, 256, 4096, ACT_NONE, 0),       # 1 -> 2 x 32, fp16 weights
    (300, 128, 128, ACT_ELU, 1),        # 3 -> 4 x 1: 2 units
    (40000, 96, 96, ACT_ELU, 0),        # 313 -> 314 x 1, ragged N: persistent pairs, fp16 weights
    (20000, 576, 384, ACT_GELU, 0),     # 157 -> 158 x 3, 9 k-steps, fp16 weights
]


@pytest.mark.parametrize("rows,k_cols,n_cols,act,split_w", PLAIN)
def test_linear_rows_same_on_either_rank(engine, rows, k_cols, n_cols, act, split_w):
    dev = engine.torch_device
    a, w32, bias, packed, bias_full = make_problem(dev, rows + 3 * k_cols + n_cols, rows, k_cols, n_cols, split_w)
    out32, _ = linear(engine, a, rows, k_cols, packed, bias_full, n_cols, act, split_w)
    check_f32(out32, *reference(a, w32, bias, act), f"rows={rows} K={k_cols} N={n_cols}")
    pad = torch.randn((128, k_cols), generator=_gen(dev, 9), device=dev).to(torch.float16)
    shifted, _ = linear(engine, torch.cat([pad, a]), rows + 128, k_cols, packed, bias_full, n_cols, act, split_w)
    assert torch.equal(shifted[128:].view(torch.int32), out32.view(torch.int32)), \
        "rows differ when their tile moves to the other CTA of the pair"


@pytest.mark.parametrize("rows", [1000, 100])
def test_fused_residual_same_on_either_rank(engine, rows):
    """8 -> 9 and 1 -> 2 M tiles: the residual rows get x + C exactly, and a spare CTA adds nothing anywhere."""
    dev = engine.torch_device
    k_cols, n_cols, resid_C = 256, 384, 384
    a, w32, bias, packed, bias_full = make_problem(dev, 7 + rows, rows, k_cols, n_cols, 1)
    before = torch.randn((rows + 128, resid_C), generator=_gen(dev, 8), device=dev)
    pad = torch.randn((128, k_cols), generator=_gen(dev, 9), device=dev).to(torch.float16)
    out32, r = linear(engine, a, rows, k_cols, packed, bias_full, n_cols, ACT_NONE, 1, resid=before[128:], resid_C=resid_C)
    check_f32(out32, *reference(a, w32, bias, ACT_NONE), "residual GEMM")
    assert torch.equal(r, before[128:] + out32), "residual rows differ from x + C"
    shifted, r2 = linear(engine, torch.cat([pad, a]), rows + 128, k_cols, packed, bias_full, n_cols, ACT_NONE, 1,
                         resid=before, resid_C=resid_C)
    assert torch.equal(shifted[128:], out32) and torch.equal(r2[128:], r)


# ------------------------------------------------------------------------------------------- convolution geometry
def umma_layer(engine, x, packed, bias, cout, relu, pool, split_w):
    """fad_umma_layer (3x3 convolution) into fenced outputs: fp16 and fp32 un-pooled, fp16 pooled.  The trailing
    guard is 8 images long: a spare tile's pixels belong to the images after the last (partial) image group."""
    nb, hh, ww, cin = x.shape
    oh, ow = (hh // 2, ww // 2) if pool else (hh, ww)
    shape, tail = (nb, oh, ow, cout), 8 * oh * ow * cout
    o16 = Guarded(shape, torch.float16, x.device, GUARD, tail)
    o32 = None if pool else Guarded(shape, torch.float32, x.device, GUARD, tail)
    _native._check(_native.lib().fad_umma_layer(
        engine._h, x.data_ptr(), nb, hh, ww, cin, packed.data_ptr(), bias.data_ptr(), cout, 9, relu, int(pool),
        split_w, o16.body.data_ptr(), _native._ptr(o32.body if o32 else None), _native._stream()))
    o16.check("fp16 output")
    if o32 is None:
        return o16.body
    o32.check("fp32 output")
    assert torch.equal(o16.body.view(torch.int16), o32.body.half().view(torch.int16)), "fp16 output != fp32.half()"
    return o32.body


CONV = [
    # NB, H, W, Cin, Cout, pool, split_w, images per shift: M tiles (before -> after the shift) x N tiles
    (5, 24, 16, 64, 256, False, 1, 1),      # 16 x 8 boxes, 3 tiles per image: 15 -> 18 x 2
    (3, 24, 16, 128, 128, True, 1, 1),      # pooled: 9 -> 12 x 1
    (10, 12, 8, 64, 512, True, 0, 4),       # 8 x 4 x 4-image boxes, 3 tiles per group: 9 -> 12 x 4, partial last group
    (7, 12, 8, 128, 256, False, 0, 4),      # 6 -> 9 x 2, fp16 weights
]


@pytest.mark.parametrize("nb,hh,ww,cin,cout,pool,split_w,shift", CONV)
def test_conv_rows_same_on_either_rank(engine, nb, hh, ww, cin, cout, pool, split_w, shift):
    dev = engine.torch_device
    g = _gen(dev, nb * 100 + cin + cout)
    x = torch.randn((nb + shift, hh, ww, cin), generator=g, device=dev).to(torch.float16)
    w32 = torch.randn((cout, 9 * cin), generator=g, device=dev) * (2.0 / (9 * cin)) ** 0.5
    if not split_w:
        w32 = w32.half().float()
    bias = torch.randn((cout,), generator=g, device=dev) * 0.1
    packed = (wts.split_hi_lo_tiles(w32) if split_w else w32.half()).contiguous()
    mine = x[shift:].contiguous()
    out = umma_layer(engine, mine, packed, bias, cout, ACT_RELU, pool, split_w)

    wt = w32.double().reshape(cout, 3, 3, cin).permute(0, 3, 1, 2)
    xd = mine.double().permute(0, 3, 1, 2)
    pre = torch.nn.functional.conv2d(xd, wt, bias.double(), padding=1)
    mag = torch.nn.functional.conv2d(xd.abs(), wt.abs(), padding=1)
    bound = 2.0 ** -20 * mag + 2.0 ** -22 * pre.abs() + 1e-30
    ref = pre.clamp_min(0.0)
    if pool:
        # the kernel pools fp16-rounded values: the max of the window's errors plus one fp16 rounding
        ref, bound = torch.nn.functional.max_pool2d(ref, 2), torch.nn.functional.max_pool2d(bound, 2)
        ref, bound = ref.permute(0, 2, 3, 1), bound.permute(0, 2, 3, 1)
        err = (out.double() - ref).abs()
        assert (err <= bound + 2.0 ** -11 * (ref.abs() + bound) + 2.0 ** -24).all(), f"max err {err.max().item():.3g}"
    else:
        check_f32(out, ref.permute(0, 2, 3, 1), bound.permute(0, 2, 3, 1), f"conv NB={nb} {hh}x{ww} {cin}->{cout}")

    shifted = umma_layer(engine, x, packed, bias, cout, ACT_RELU, pool, split_w)
    bits = SENTINEL[out.dtype][0]
    assert torch.equal(shifted[shift:].view(bits), out.view(bits)), \
        "images differ when their tiles move to the other CTA of the pair"
