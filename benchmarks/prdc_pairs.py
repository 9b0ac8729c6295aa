"""Precision / recall / density / coverage passes at user sizes: the k-NN radii (fad_knn_radii_sq, the full m x m and
n x n squares) and the ball counts (fad_prdc_counts, the m x n rectangle), timed apart with CUDA events (median of
PRDC_PAIRS_REPS calls, default 5) after a warm-up.

Shapes: m = n = 100 000 at d = 128 (VGGish) and d = 512 (CLAP), m = n = 50 000 at d = 768 (Whisper-small); rows with
a common offset, rounded to fp16, as benchmarks/kad_pairs.py.  k = PRDC_K (default 5).  Rates are ALGORITHMIC: the
pairs each pass evaluates (m^2 + n^2 for the radii, m n for the counts), tensor FLOP = 3 x 2 d per pair (hi.hi, hi.lo,
lo.hi).  The first line is the card, power limit and max SM clock, read in the same process; the last field of every
record says whether two runs gave bitwise-equal outputs.  JSON lines on stdout.
"""
import json
import os
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from fadtk_b200 import _native  # noqa: E402

SHAPES = [("vggish", 100_000, 100_000, 128), ("clap", 100_000, 100_000, 512), ("whisper-small", 50_000, 50_000, 768)]
PEAK_FP16 = 989e12            # H100 SXM data sheet, dense fp16, 700 W


def smi(query: str) -> str:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def timed(fn, reps: int) -> float:
    """median milliseconds of one call, CUDA events around each call"""
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    evs[0].record()
    for i in range(reps):
        fn()
        evs[i + 1].record()
    torch.cuda.synchronize()
    return float(np.median([evs[i].elapsed_time(evs[i + 1]) for i in range(reps)]))


def main():
    assert torch.cuda.is_available(), "prdc_pairs.py measures on the GPU"
    name, plimit, max_mhz = [s.strip() for s in smi("name,power.limit,clocks.max.sm").split(",")]
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"gpu": name, "power_limit_w": plimit, "max_sm_mhz": max_mhz, "sms": props.multi_processor_count}),
          flush=True)
    eng = _native.engine(0)
    dev = eng.torch_device
    reps = int(os.environ.get("PRDC_PAIRS_REPS", "5"))
    k = int(os.environ.get("PRDC_K", "5"))
    for label, m, n, d in SHAPES:
        g = torch.Generator(device=dev).manual_seed(7)
        mu = 40.0 * torch.randn(d, device=dev, generator=g)
        z = (mu + 1.8 * torch.randn(m + n, d, device=dev, generator=g)).to(torch.float16).contiguous()
        z[m:] += 0.25
        radii = eng.knn_radii_sq(z, m, k)                               # warm-up of both passes
        inside, flags = eng.prdc_counts(z, m, radii)
        torch.cuda.synchronize()
        radii2 = eng.knn_radii_sq(z, m, k)
        inside2, flags2 = eng.prdc_counts(z, m, radii2)
        torch.cuda.synchronize()
        bitwise = bool(torch.equal(radii, radii2) and torch.equal(inside, inside2) and torch.equal(flags, flags2))
        ms_radii = timed(lambda: eng.knn_radii_sq(z, m, k), reps)
        ms_counts = timed(lambda: eng.prdc_counts(z, m, radii), reps)
        rec = {"shape": label, "m": m, "n": n, "d": d, "k": k, "reps": reps}
        for stage, ms, pairs in (("radii", ms_radii, float(m) * m + float(n) * n), ("counts", ms_counts, float(m) * n)):
            flop = pairs * 3 * 2 * d
            rec[stage] = {"ms": round(ms, 3), "pairs_per_s": pairs / (ms * 1e-3),
                          "tensor_tflops": flop / (ms * 1e-3) / 1e12,
                          "datasheet_tensor_ms": round(flop / PEAK_FP16 * 1e3, 3)}
        ins, fl = inside.cpu().numpy(), flags.cpu().numpy()
        rec["values"] = {"precision": float(np.count_nonzero(ins)) / n, "recall": float(np.count_nonzero(fl & 2)) / m,
                         "density": float(ins.sum(dtype=np.int64)) / (k * n),
                         "coverage": float(np.count_nonzero(fl & 1)) / m}
        rec["bitwise_equal_two_runs"] = bitwise
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
