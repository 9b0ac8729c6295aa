"""Timing / profiling driver for the fp64 tensor-pipe (DMMA) kernels: exact Gram statistics, the
Newton-Schulz Frechet chain, the batched per-song chain.  One JSON line; run it under ncu for the
captures in profiles/ (SURVEY.md section 8 rows a8, a9, a12; VERDICT rows N1, N2).

    python benchmarks/fp64_kernels.py [--reps 5] [--what stats,frechet,batched]

Roofline denominators: HBM from MEASURED_PEAKS.json; the fp64 tensor-pipe rate is measured live
(`fad_bench_dmma_peak`: register-only DMMA issue loop) because MEASURED_PEAKS.json has no fp64 entry.
Algorithmic work: statistics 2 N d^2 FLOP (full Gram; the kernel computes the upper tile triangle,
(d/64)(d/64+1)/2 * 64*64 * 2N - reported as `issued`) and N d 2 bytes; Newton-Schulz 6 d^3 per iteration.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

import os as _os
_os.environ.setdefault("FADTK_SYNTHETIC", "1")      # benchmarks run the real architectures on seeded random weights (no checkpoints offline)
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from fadtk_b200 import _native  # noqa: E402


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, out


def spectrum_cov(rng, d, n, decay):
    """covariance of n samples with a power-law spectrum (cond ~ d^decay), like the real fma_pop statistics"""
    basis, _ = np.linalg.qr(rng.standard_normal((d, d)))
    scale = np.arange(1, d + 1, dtype=np.float64) ** (-decay / 2.0)
    x = rng.standard_normal((n, d)) * scale @ basis.T + rng.standard_normal(d) * 0.1
    return x.mean(0), np.cov(x, rowvar=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--what", default="peak,stats,frechet,batched")
    ap.add_argument("--songs", type=int, default=5000)
    ap.add_argument("--dims", default="128,512,768,1024", help="Frechet dimensions")
    ap.add_argument("--stats-shapes", default="100000x128,937500x128,500000x512,50000x768")
    args = ap.parse_args()
    what = set(args.what.split(","))
    torch.cuda.set_device(0)
    eng = _native.Engine(0, max_examples=64)
    dev = eng.torch_device
    peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text()) if (ROOT / "MEASURED_PEAKS.json").exists() else {}
    hbm = peaks.get("hbm_gbs", 6650.0)
    out = {"hbm_peak_gbs": hbm, "hbm_peak_source": "MEASURED_PEAKS.json" if peaks else "fallback (H100 SXM data sheet, not measured)"}
    dmma = eng.dmma_peak_tflops() if "peak" in what else None
    if dmma:
        dmma = max(dmma, eng.dmma_peak_tflops())
    out["dmma_peak_tflops"] = dmma
    out["dmma_peak_source"] = "measured live: fad_bench_dmma_peak (register-only m8n8k4 f64 issue loop, 4 CTAs x 8 warps per SM)"
    rng = np.random.default_rng(0)

    if "stats" in what:
        rows = []
        for n, d in (tuple(int(v) for v in sh.split("x")) for sh in args.stats_shapes.split(",")):
            emb = torch.randn((n, d), device=dev, dtype=torch.float32).mul_(1.5).add_(0.3).to(torch.float16)
            shift = emb[:1024].float().mean(0).to(torch.float16)
            for mode, name in ((0, "dmma"), (2, "simt")):
                acc = eng.stats_new(d)
                ms, _ = timed(lambda: eng.stats_accumulate(emb, shift, acc.zero_(), tensor_core=mode), args.reps)
                flop = 2.0 * n * d * d
                nt = d // 64
                rows.append({"n": n, "d": d, "kernel": name, "ms": ms, "algorithmic_tflops": flop / ms / 1e9,
                             "issued_tflops": flop * (nt + 1) / (2 * nt) / ms / 1e9 if mode == 0 else None,
                             "algorithmic_gbs": n * d * 2 / ms / 1e6, "frac_hbm": n * d * 2 / ms / 1e6 / hbm,
                             "frac_dmma": (flop * (nt + 1) / (2 * nt) / ms / 1e9 / dmma) if (dmma and mode == 0) else None})
            del emb
        out["stats"] = rows

    if "frechet" in what:
        rows = []
        for d, n in ((int(v), 4000 + 4 * int(v)) for v in args.dims.split(",")):
            m1, c1 = spectrum_cov(rng, d, n, 2.0)
            m2, c2 = spectrum_cov(rng, d, n, 2.2)
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
            a = (t(m1), t(c1), t(m2), t(c2))
            launches0 = eng.launches
            ms, res = timed(lambda: eng.frechet(*a), args.reps)
            launches = (eng.launches - launches0) // (args.reps + 1)
            base = _native.Baseline(eng, a[0], a[1])
            ms_pre, res2 = timed(lambda: base.frechet(a[2], a[3]), args.reps)
            rows.append({"d": d, "ms_full": ms, "ms_presqrt": ms_pre, "launches_full": launches,
                         "fad": float(res[0].item()), "resid": float(res[2].item()),
                         "fad_presqrt_rel_diff": abs(float(res2[0].item()) - float(res[0].item())) / abs(float(res[0].item()))})
        out["frechet"] = rows

    if "batched" in what:
        d, rows_per, songs = 128, 750, args.songs
        mix = (rng.standard_normal((d, d)) / np.sqrt(d)).astype(np.float32)
        base_rows = (rng.standard_normal((20000, d)).astype(np.float32) @ mix).astype(np.float64)
        base = _native.Baseline(eng, base_rows.mean(0), np.cov(base_rows, rowvar=False))
        emb = (torch.randn((songs * rows_per, d), device=dev) @ torch.from_numpy(mix).to(dev)).mul_(1.1).to(torch.float16)
        offs = torch.arange(0, songs + 1, device=dev, dtype=torch.int64) * rows_per
        ms, res = timed(lambda: base.frechet_batched(emb, offs), max(1, args.reps // 2))
        out["batched"] = {"songs": songs, "rows": rows_per, "d": d, "ms": ms, "songs_per_s": songs / ms * 1e3,
                          "finite": bool(torch.isfinite(res[:, 0]).all().item()), "fad_mean": float(res[:, 0].mean().item())}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
