"""Fixed cost per output tile of the wgmma GEMM (csrc/conv_gemm.cuh), separated from the cost per k-step.

Times fad_umma_layer on one 3x3-convolution geometry with fixed M and N (conv3_1's: 24 x 16 pixels, 256 output
channels, one 10 000-example chunk: 30 000 M tiles x 2 N tiles) while K is swept over Cin in {64, 128, 256, 512}
(9, 18, 36, 72 k-steps), with fp16 hi/lo weights (split, what the product runs) and plain fp16 weights.  Per mode it
fits

    us per tile = intercept + slope x k-steps

by least squares, where us per tile = median ms / tiles per CTA.  The slope is the main loop (ideally the pure wgmma
issue time: 1024 clk per k-step with split weights, 512 with fp16), the intercept what each tile costs on top of it
(epilogue, pipeline refill).  Both are also given in SM clocks at the median of the clock samples nvidia-smi took while
the timed launches ran; on a power-capped card single samples scatter widely, so the fit itself is done in time.

The first line is the card, power limit and max SM clock, read in the same process.
    python benchmarks/gemm_tile_overhead.py [--examples 10000] [--reps 20]"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

os.environ.setdefault("FADTK_SYNTHETIC", "1")
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from fadtk_b200 import _native, weights  # noqa: E402

HH, WW, COUT = 24, 16, 256
CINS = [64, 128, 256, 512]


def smi(query):
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--examples", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    print(json.dumps({"gpu": smi("name,power.limit,clocks.max.sm"), "examples": args.examples}), flush=True)
    eng = _native.engine(0)
    dev = eng.torch_device
    nb = args.examples
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    m_tiles = nb * (HH // 8) * (WW // 16)             # 16 x 8 x 1 pixel boxes
    units = (m_tiles + 1) // 2 * (COUT // 128)
    pairs = min(units, sms // 2)                       # one CTA per SM, clusters of two
    tiles_per_cta = units / pairs
    fits, clocks = {}, []
    for label, split in (("split", 1), ("fp16", 0)):
        pts = []
        for cin in CINS:
            torch.manual_seed(1)
            k = 9 * cin
            x = (torch.randn(nb, HH, WW, cin, device=dev) * 0.5).to(torch.float16)
            w32 = torch.randn(COUT, k) * (2.0 / k) ** 0.5
            bias = torch.randn(COUT, device=dev) * 0.1
            w = (weights.split_hi_lo_tiles(w32, 128) if split else w32.to(torch.float16)).to(dev).contiguous()
            for _ in range(3):
                eng.umma_layer(x, w, bias, 9, 1, 0, split_w=split)
            torch.cuda.synchronize()
            n = args.reps
            evs = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
            evs[0].record()
            for i in range(n):                          # one event per launch: a single slow launch must not hide in a mean
                eng.umma_layer(x, w, bias, 9, 1, 0, split_w=split)
                evs[i + 1].record()
            mhz = [float(smi("clocks.sm")) for _ in range(3)]     # sampled while the launches above run
            torch.cuda.synchronize()
            per = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(n))
            ms = per[n // 2]
            ks = k // 64
            us = ms * 1e3 / tiles_per_cta
            pts.append((ks, us))
            clocks += mhz
            print(json.dumps({"mode": label, "cin": cin, "ksteps": ks, "ms": round(ms, 4), "min_ms": round(per[0], 4),
                              "max_ms": round(per[-1], 4), "sm_mhz_samples": mhz, "tiles_per_cta": round(tiles_per_cta, 1),
                              "us_per_tile": round(us, 3)}), flush=True)
            del x, w
        ks_arr = np.array([p[0] for p in pts], dtype=np.float64)
        us_arr = np.array([p[1] for p in pts])
        slope, intercept = np.polyfit(ks_arr, us_arr, 1)
        fits[label] = {"intercept_us": round(float(intercept), 3), "slope_us_per_kstep": round(float(slope), 4),
                       "max_residual_us": round(float(np.abs(us_arr - (intercept + slope * ks_arr)).max()), 3)}
    mhz = float(np.median(clocks))
    for f in fits.values():
        f["intercept_clk"] = round(f["intercept_us"] * mhz)
        f["slope_clk_per_kstep"] = round(f["slope_us_per_kstep"] * mhz)
    print(json.dumps({"fit": fits, "median_sm_mhz": mhz, "power_limit_w": smi("power.limit")}), flush=True)


if __name__ == "__main__":
    main()
