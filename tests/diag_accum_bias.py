"""Diagnostic (not a test): does tensor-core fp32 accumulation shrink results systematically?

For each layer shape, run the tensor-core layer on post-ReLU-like operands and regress its fp32
output on the exact fp64 result computed from the SAME fp16 operands:
    slope - 1  = <out, ref> / <ref, ref> - 1     (systematic scale error)
    rms        = |out - slope*ref| / |ref|       (unbiased noise)
Usage (GPU box):  python tests/diag_accum_bias.py
"""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from fadtk_b200 import _native  # noqa: E402

SHAPES = [  # NB, H, W, Cin, Cout, taps
    (64, 1, 1, 12288, 4096, 1), (64, 1, 1, 4096, 4096, 1), (8, 12, 8, 512, 512, 9),
    (8, 24, 16, 256, 256, 9), (8, 48, 32, 64, 128, 9), (64, 1, 1, 4096, 128, 1),
]


def main():
    eng = _native.engine(0, max_examples=64)
    dev = eng.torch_device
    g = torch.Generator(device="cpu").manual_seed(0)
    for nb, hh, ww, cin, cout, taps in SHAPES:
        x = torch.relu(torch.randn((nb, hh, ww, cin), generator=g) + 0.3).to(torch.float16).to(dev)
        w = (torch.randn((cout, taps * cin), generator=g) * (2.0 / (taps * cin)) ** 0.5).to(torch.float16).to(dev)
        b = torch.zeros(cout, device=dev)
        _, out32 = eng.umma_layer(x, w, b, taps, False, False, want_f32=True)
        from fadtk_b200 import weights as wts
        _, out32s = eng.umma_layer(x, wts.split_hi_lo_tiles(w.float().cpu()).to(dev), b, taps, False, False, want_f32=True, split_w=True)
        if taps == 9:
            wt = w.double().reshape(cout, 3, 3, cin).permute(0, 3, 1, 2).contiguous()
            ref = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), wt, padding=1).permute(0, 2, 3, 1)
            ref32 = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), padding=1).permute(0, 2, 3, 1)
        else:
            ref = (x.double().reshape(nb, cin) @ w.double().t()).reshape(nb, 1, 1, cout)
            ref32 = (x.float().reshape(nb, cin) @ w.float().t()).reshape(nb, 1, 1, cout)
        o = out32.double()
        slope = (o * ref).sum() / (ref * ref).sum()
        rms = ((o - slope * ref).norm() / ref.norm()).item()
        s32 = (ref32.double() * ref).sum() / (ref * ref).sum()
        # magnitude-wise: mean of (|out| - |ref|) / mean |ref|
        shrink = ((o.abs() - ref.abs()).mean() / ref.abs().mean()).item()
        os_ = out32s.double(); slope_s = (os_ * ref).sum() / (ref * ref).sum()
        print(f"K={taps * cin:6d} N={cout:5d}: split-W slope-1 = {slope_s.item() - 1:+.3e} rms {((os_ - slope_s * ref).norm() / ref.norm()).item():.2e} | fp16-W slope-1 = {slope.item() - 1:+.3e}  |.|-shrink = {shrink:+.3e}  "
              f"noise rms = {rms:.2e}   (torch fp32 CUDA slope-1 = {s32.item() - 1:+.3e})")


if __name__ == "__main__":
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    main()
