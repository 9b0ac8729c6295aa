"""Per-sample realism at user sizes: one fad_realism call (the baseline's k-NN radii over the m x m square, the median
and pruning, then the realism pass over the m x n rectangle) next to fad_prdc_counts on the same rows, which evaluates
the same m n pairs with the ball-count epilogue.  Whole calls are timed with CUDA events (median of REALISM_PAIRS_REPS
calls, default 5, after a warm-up); a separate torch.profiler run of the same calls splits fad_realism into its
kernels (median device time per kernel over the calls).

Shapes: m = n = 100 000 at d = 128 (VGGish), 512 (CLAP) and 768 (Whisper-small), and m = 100 000, n = 10 000 at
d = 128 (a small eval set against a large baseline); rows with a common offset, rounded to fp16, as prdc_pairs.py.
k = REALISM_K (default 3).  Rates are ALGORITHMIC: tensor FLOP = 3 x 2 d per pair (hi.hi, hi.lo, lo.hi), m^2 pairs
for the radii, m n for the realism and counts passes.  The first line is the card, power limit and max SM clock, read
in the same process; the last field of every record says whether two calls gave bitwise-equal outputs.  JSON lines
on stdout.
"""
import json
import os
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402
from fadtk_b200 import _native  # noqa: E402
from prdc_pairs import PEAK_FP16, smi, timed  # noqa: E402

SHAPES = [("vggish", 100_000, 100_000, 128), ("clap", 100_000, 100_000, 512),
          ("whisper-small", 100_000, 100_000, 768), ("vggish-small-eval", 100_000, 10_000, 128)]
KERNELS = {"radii": "prdc_tile_kernel<0>", "realism": "prdc_tile_kernel<4>"}


def kernel_ms(fn, reps: int) -> dict:
    """median device milliseconds per call of each library kernel fn launches, from torch.profiler"""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "fad::" in e.name:
            per.setdefault(e.name, []).append(e.device_time_total / 1e3)
    out = {}
    for name, ts in per.items():
        short = name.split("(")[0].replace("void ", "").replace("fad::", "")
        out[short] = round(float(np.median(ts)) * len(ts) / reps, 3)
    return out


def main():
    assert torch.cuda.is_available(), "realism_pairs.py measures on the GPU"
    name, plimit, max_mhz = [s.strip() for s in smi("name,power.limit,clocks.max.sm").split(",")]
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"gpu": name, "power_limit_w": plimit, "max_sm_mhz": max_mhz, "sms": props.multi_processor_count}),
          flush=True)
    eng = _native.engine(0)
    dev = eng.torch_device
    reps = int(os.environ.get("REALISM_PAIRS_REPS", "5"))
    k = int(os.environ.get("REALISM_K", "3"))
    for label, m, n, d in SHAPES:
        g = torch.Generator(device=dev).manual_seed(7)
        mu = 40.0 * torch.randn(d, device=dev, generator=g)
        z = (mu + 1.8 * torch.randn(m + n, d, device=dev, generator=g)).to(torch.float16).contiguous()
        z[m:] += 0.25
        a = eng.realism(z, m, k)                                        # warm-up of every pass
        radii = torch.cat([a[0], torch.ones(n, dtype=torch.float32, device=dev)])
        eng.prdc_counts(z, m, radii)
        b = eng.realism(z, m, k)
        torch.cuda.synchronize()
        bitwise = all(torch.equal(p, q) for p, q in zip(a[:4], b[:4])) and a[4] == b[4]
        ms_call = timed(lambda: eng.realism(z, m, k), reps)
        ms_counts = timed(lambda: eng.prdc_counts(z, m, radii), reps)
        per_kernel = kernel_ms(lambda: eng.realism(z, m, k), reps)
        rec = {"shape": label, "m": m, "n": n, "d": d, "k": k, "reps": reps, "realism_call_ms": round(ms_call, 3),
               "kernels_ms": per_kernel}
        stages = [("counts", ms_counts, float(m) * n)]
        for stage, kern in KERNELS.items():
            ms = next((v for kname, v in per_kernel.items() if kern in kname), None)
            if ms is not None:
                stages.append((stage, ms, float(m) * m if stage == "radii" else float(m) * n))
        for stage, ms, pairs in stages:
            flop = pairs * 3 * 2 * d
            rec[stage] = {"ms": round(ms, 3), "tensor_tflops": flop / (ms * 1e-3) / 1e12,
                          "datasheet_tensor_ms": round(flop / PEAK_FP16 * 1e3, 3)}
        real = a[1].cpu().numpy()
        rec["values"] = {"threshold_sq": a[4], "realism_median": float(np.median(real.astype(np.float64))),
                         "share_realism_ge_1": float(np.mean(real >= 1.0))}
        rec["bitwise_equal_two_runs"] = bitwise
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
