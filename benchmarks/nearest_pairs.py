"""The k nearest distinct baseline groups at user sizes: one fad_nearest call next to fad_realism's tile pass on the same
rows, which evaluates the same m n pairs with a max / argmin epilogue.  Whole fad_nearest calls are timed with CUDA
events (median of NEAREST_PAIRS_REPS calls, default 5, after a warm-up); a torch.profiler run of fad_realism gives its
tile pass (prdc_tile_kernel<4>) alone, and one of fad_nearest splits it into the tile pass and the run merge.

Shapes: m = n = 100 000 at d = 128 (VGGish), 512 (CLAP) and 768 (Whisper-small) with k = 1, 5, 16; m = 100 000,
n = 10 000 at d = 128 (a small eval set against a large baseline); and at d = 128, k = 5 the baseline cut into
VGGish-like 10-row groups against one-row groups.  Rows with a common offset, rounded to fp16, as prdc_pairs.py.
The first line is the card, power limit and max SM clock, read in the same process; the last field of every record
says whether two calls gave bitwise-equal outputs.  JSON lines on stdout.
"""
import json
import os
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import torch  # noqa: E402
from fadtk_b200 import _native  # noqa: E402
from prdc_pairs import smi, timed  # noqa: E402
from realism_pairs import kernel_ms  # noqa: E402

CASES = ([("vggish", 100_000, 100_000, 128, k, 1) for k in (1, 5, 16)] +
         [("clap", 100_000, 100_000, 512, k, 1) for k in (1, 5, 16)] +
         [("whisper-small", 100_000, 100_000, 768, k, 1) for k in (1, 5, 16)] +
         [("vggish-small-eval", 100_000, 10_000, 128, 5, 1), ("vggish-10-row-groups", 100_000, 100_000, 128, 5, 10)])


def runs(m: int, n: int) -> int:
    """the X column runs per Y tile, cut as fad_nearest cuts them"""
    tx, ty = -(-m // 128), -(-n // 128)
    return -(-tx // max(4, -(-(tx * ty) // 8192)))


def main():
    assert torch.cuda.is_available(), "nearest_pairs.py measures on the GPU"
    name, plimit, max_mhz = [s.strip() for s in smi("name,power.limit,clocks.max.sm").split(",")]
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"gpu": name, "power_limit_w": plimit, "max_sm_mhz": max_mhz, "sms": props.multi_processor_count}),
          flush=True)
    eng = _native.engine(0)
    dev = eng.torch_device
    reps = int(os.environ.get("NEAREST_PAIRS_REPS", "5"))
    only = os.environ.get("NEAREST_PAIRS_ONLY")
    realism_ms = {}
    for label, m, n, d, k, group in CASES:
        if only and only not in label:
            continue
        g = torch.Generator(device=dev).manual_seed(7)
        mu = 40.0 * torch.randn(d, device=dev, generator=g)
        z = (mu + 1.8 * torch.randn(m + n, d, device=dev, generator=g)).to(torch.float16).contiguous()
        z[m:] += 0.25
        off = None
        if group > 1:
            off = torch.cat([torch.arange(0, m, group, device=dev), torch.tensor([m], device=dev)]).to(torch.int64)
        a = eng.nearest(z, m, k, off)
        b = eng.nearest(z, m, k, off)
        torch.cuda.synchronize()
        bitwise = all(torch.equal(p, q) for p, q in zip(a, b))
        ms_call = timed(lambda: eng.nearest(z, m, k, off), reps)
        per_kernel = kernel_ms(lambda: eng.nearest(z, m, k, off), reps)
        key = (m, n, d)
        if key not in realism_ms:                        # the realism tile pass over the same rows
            eng.realism(z, m, 3)
            realism_ms[key] = next(v for kname, v in kernel_ms(lambda: eng.realism(z, m, 3), reps).items()
                                   if "prdc_tile_kernel<4>" in kname)
        tile = next((v for kname, v in per_kernel.items() if "prdc_tile_kernel<5>" in kname), None)
        rec = {"shape": label, "m": m, "n": n, "d": d, "k": k, "group_rows": group, "reps": reps,
               "nearest_call_ms": round(ms_call, 3), "nearest_tile_ms": tile, "realism_tile_ms": realism_ms[key],
               "tile_over_realism": round(tile / realism_ms[key], 3) if tile else None, "kernels_ms": per_kernel,
               "part_mb": round(2 * 4 * n * k * runs(m, n) / 1e6, 1),
               "rank1_distance_median": float(a[1][:, 0].sqrt().median()), "bitwise_equal_two_runs": bitwise}
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
