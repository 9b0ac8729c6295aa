"""KAD permutation tests at user sizes: the label generation (fad_perm_labels) and the permutation sums
(fad_kad_perm_sums: all labellings' tile passes) at m = n = 100 000 rows, d = 128 and 512, B = 999, next to the same
run's fad_kad_sums; and calc_kad_comparison at 10 000 + 10 000 rows against a 100 000-row baseline.  CUDA events
around repeated calls after a warm-up.  Rates are ALGORITHMIC: 6 d (the three fp16 distance products) + 2 x (padded
labellings) tensor FLOP per pair.  The first line is the card, power limit and max SM clock, read in the same process.
JSON lines on stdout; KAD_TEST_SHAPES=small runs a tenth of the rows."""
import json
import os
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import fadtk_b200 as fk  # noqa: E402
from fadtk_b200 import _native  # noqa: E402

PEAK_FP16 = 989e12            # H100 SXM data sheet, dense fp16, 700 W


def smi(query: str) -> str:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def timed(fn, reps: int) -> float:
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    evs[0].record()
    for i in range(reps):
        fn()
        evs[i + 1].record()
    torch.cuda.synchronize()
    return float(np.median([evs[i].elapsed_time(evs[i + 1]) for i in range(reps)]))


def rows(n, d, seed, dev, shift=0.0):
    g = torch.Generator(device=dev).manual_seed(7)
    mu = 40.0 * torch.randn(d, device=dev, generator=g)
    g.manual_seed(seed)
    return (mu + shift + 1.8 * torch.randn(n, d, device=dev, generator=g)).to(torch.float16).contiguous()


def main():
    assert torch.cuda.is_available(), "kad_test_pairs.py measures on the GPU"
    name, plimit, max_mhz = [s.strip() for s in smi("name,power.limit,clocks.max.sm").split(",")]
    print(json.dumps({"gpu": name, "power_limit_w": plimit, "max_sm_mhz": max_mhz}), flush=True)
    eng = _native.engine(0)
    dev = eng.torch_device
    reps = int(os.environ.get("KAD_TEST_REPS", "3"))
    scale = 10 if os.environ.get("KAD_TEST_SHAPES") == "small" else 1
    B = 999
    padded = -(-(B + 1) // 64) * 64
    for d in (128, 512):
        m = n = 100_000 // scale
        z = torch.cat([rows(m, d, 1, dev), rows(n, d, 2, dev, 0.25)])
        sq = eng.kad_median_sq(z[:m])
        sigma = (0.5 * (sq[0].sqrt() + sq[1].sqrt())).reshape(1).contiguous()
        eng.kad_perm_sums(z, m, sigma, B, 0)
        eng.perm_labels(m + n, m, B, 0)
        eng.kad_sums(z, m, sigma)
        torch.cuda.synchronize()
        ms_lab = timed(lambda: eng.perm_labels(m + n, m, B, 0), reps)
        ms_perm = timed(lambda: eng.kad_perm_sums(z, m, sigma, B, 0), reps)
        ms_kad = timed(lambda: eng.kad_sums(z, m, sigma), reps)
        N = m + n
        pairs = N * (N - 1) / 2
        flop = pairs * (6 * d + 2 * padded)
        print(json.dumps({"d": d, "m": m, "n": n, "B": B, "labels_ms": round(ms_lab, 3),
                          "perm_sums_ms": round(ms_perm, 3), "tile_pass_ms_excl_labels": round(ms_perm - ms_lab, 3),
                          "tflops": flop / ((ms_perm - ms_lab) * 1e-3) / 1e12,
                          "share_of_datasheet_fp16": flop / PEAK_FP16 / ((ms_perm - ms_lab) * 1e-3),
                          "kad_sums_ms": round(ms_kad, 3), "kad_sums_x_B_plus_1_ms": round(ms_kad * (B + 1), 1)}),
              flush=True)
        if d == 128:
            # where the time goes: the pass at 1, 8 and 16 blocks of 64 labellings (label time taken out).  The marginal
            # time of a block against its data-sheet tensor time says how busy the label product keeps the tensor
            # pipe; the one-block pass is mostly the distance product and the epilogue.
            per = {}
            for b_run in (63, 511, 1023):
                eng.kad_perm_sums(z, m, sigma, b_run, 0)
                t_lab = timed(lambda: eng.perm_labels(m + n, m, b_run, 0), reps)
                per[(b_run + 1) // 64] = timed(lambda: eng.kad_perm_sums(z, m, sigma, b_run, 0), reps) - t_lab
            block_ms = (per[16] - per[1]) / 15
            block_tensor_ms = pairs * 2 * 64 / PEAK_FP16 * 1e3
            dist_tensor_ms = pairs * 6 * d / PEAK_FP16 * 1e3
            print(json.dumps({"d": d, "blocks_1_8_16_ms": [round(per[k], 3) for k in (1, 8, 16)],
                              "ms_per_label_block": round(block_ms, 3),
                              "label_block_datasheet_tensor_ms": round(block_tensor_ms, 3),
                              "label_product_share_of_datasheet": block_tensor_ms / block_ms,
                              "one_block_pass_ms": round(per[1], 3),
                              "distance_datasheet_tensor_ms": round(dist_tensor_ms, 3)}), flush=True)
    # the comparison test: 10 000 + 10 000 rows against 100 000 baseline rows
    d = 128
    x = rows(100_000 // scale, d, 3, dev).cpu()
    a, b = rows(10_000 // scale, d, 4, dev, 0.1).cpu(), rows(10_000 // scale, d, 5, dev).cpu()
    fk.calc_kad_comparison(x, a, b, permutations=B)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fk.calc_kad_comparison(x, a, b, permutations=B)
    torch.cuda.synchronize()
    print(json.dumps({"comparison": {"m": x.shape[0], "n_a": a.shape[0], "n_b": b.shape[0], "B": B, "d": d,
                                     "s": round(time.perf_counter() - t0, 3), "p_value": r.p_value,
                                     "difference": r.difference}}), flush=True)


if __name__ == "__main__":
    main()
