"""Kernel Audio Distance stages at user sizes: the bandwidth selection (fad_kad_median_sq, three radix passes over the
baseline pair triangle) and the kernel sums (fad_kad_sums, one pass over the pair triangle of [X; Y]), timed apart with
CUDA events over repeated launches after a warm-up.

Shapes: m = n = 100 000 at d = 128 (VGGish), 100 000 at d = 512 (CLAP), 50 000 at d = 768 (Whisper-small); rows with a
common offset, rounded to fp16.  Rates are ALGORITHMIC: pairs = (m + n)(m + n - 1) / 2 for the sums and m (m - 1) / 2
per radix pass; tensor FLOP = 2 d per pair for each of the three fp16 products (hi.hi, hi.lo, lo.hi) the kernel issues;
one ex2 per pair.  The bound is the larger of tensor time (FLOP over the data-sheet dense fp16 rate, 989 TFLOP/s) and
MUFU time (16 ex2 per clock per SM at the max SM clock); the card's power limit can keep the kernel below either.
The first line is the card, power limit and max SM clock, read in the same process; the last field of every record
says whether two runs gave bitwise-equal results.  JSON lines on stdout.
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
EX2_PER_CLK_SM = 16


def smi(query: str) -> str:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def timed(fn, reps: int) -> float:
    """median milliseconds of one call, CUDA events around each launch"""
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    evs[0].record()
    for i in range(reps):
        fn()
        evs[i + 1].record()
    torch.cuda.synchronize()
    return float(np.median([evs[i].elapsed_time(evs[i + 1]) for i in range(reps)]))


def main():
    assert torch.cuda.is_available(), "kad_pairs.py measures on the GPU"
    name, plimit, max_mhz = [s.strip() for s in smi("name,power.limit,clocks.max.sm").split(",")]
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"gpu": name, "power_limit_w": plimit, "max_sm_mhz": max_mhz, "sms": props.multi_processor_count}),
          flush=True)
    eng = _native.engine(0)
    dev = eng.torch_device
    reps = int(os.environ.get("KAD_PAIRS_REPS", "5"))
    ex2_rate = EX2_PER_CLK_SM * props.multi_processor_count * float(max_mhz) * 1e6
    for label, m, n, d in SHAPES:
        g = torch.Generator(device=dev).manual_seed(7)
        mu = 40.0 * torch.randn(d, device=dev, generator=g)
        z = (mu + 1.8 * torch.randn(m + n, d, device=dev, generator=g)).to(torch.float16).contiguous()
        z[m:] += 0.25
        x = z[:m]
        sq = eng.kad_median_sq(x)                                       # warm-up of both stages
        sigma = (0.5 * (sq[0].sqrt() + sq[1].sqrt())).reshape(1).contiguous()
        sums = eng.kad_sums(z, m, sigma)
        torch.cuda.synchronize()
        sq2, sums2 = eng.kad_median_sq(x), eng.kad_sums(z, m, sigma)
        torch.cuda.synchronize()
        bitwise = bool(torch.equal(sq, sq2) and torch.equal(sums, sums2))
        ms_med = timed(lambda: eng.kad_median_sq(x), reps)
        ms_sum = timed(lambda: eng.kad_sums(z, m, sigma), reps)
        rec = {"shape": label, "m": m, "n": n, "d": d, "reps": reps}
        for stage, ms, pairs in (("median", ms_med, 3 * m * (m - 1) / 2), ("sums", ms_sum, (m + n) * (m + n - 1) / 2)):
            flop = pairs * 3 * 2 * d
            t_tensor = flop / PEAK_FP16
            t_mufu = pairs / ex2_rate if stage == "sums" else 0.0
            rec[stage] = {"ms": round(ms, 3), "pairs_per_s": pairs / (ms * 1e-3), "tensor_tflops": flop / (ms * 1e-3) / 1e12,
                          "ex2_per_s": (pairs / (ms * 1e-3)) if stage == "sums" else 0.0,
                          "datasheet_tensor_ms": round(t_tensor * 1e3, 3), "mufu_ms_at_max_clock": round(t_mufu * 1e3, 3),
                          "bound": "tensor" if t_tensor >= t_mufu else "mufu",
                          "share_of_bound": max(t_tensor, t_mufu) / (ms * 1e-3)}
        rec["sums"]["values"] = [float(v) for v in sums.cpu()]
        rec["bandwidth"] = float(sigma.cpu())
        rec["bitwise_equal_two_runs"] = bitwise
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
