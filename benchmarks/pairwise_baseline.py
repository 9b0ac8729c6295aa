"""A prepared baseline against the unprepared calls, at user sizes: the one-off preparation (prepare_pairwise_baseline:
bandwidth, S_xx and radius lists of k_max = 16) and, per eval set, KAD, PRDC at k = 5 and realism at k = 3 with the
baseline rows (every call redoes the baseline's m x m work) and with the preparation (the eval work only).  Every
call is the public Python function on device tensors, timed with CUDA events around it (median of
PAIRWISE_BASELINE_REPS calls, default 3; 1 at m = 1 000 000) after a warm-up; each record says whether the prepared
PRDC and realism results equal the unprepared ones (bitwise) and the relative difference of the two KAD values.

Shapes: m x n = 100 000 x 10 000 and 100 000 x 100 000 at d = 128 (VGGish), 1 000 000 x 10 000 at d = 128 (a large
baseline, a small eval set) and 100 000 x 10 000 at d = 512 (CLAP); rows with a common offset, rounded to fp16, as
prdc_pairs.py.  The first line is the card, power limit and max SM clock, read in the same process.  JSON lines on
stdout.
"""
import json
import os
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import fadtk_b200 as fk  # noqa: E402
from prdc_pairs import smi, timed  # noqa: E402

SHAPES = [(100_000, 10_000, 128), (100_000, 100_000, 128), (1_000_000, 10_000, 128), (100_000, 10_000, 512)]


def main():
    assert torch.cuda.is_available(), "pairwise_baseline.py measures on the GPU"
    name, plimit, max_mhz = [s.strip() for s in smi("name,power.limit,clocks.max.sm").split(",")]
    print(json.dumps({"gpu": name, "power_limit_w": plimit, "max_sm_mhz": max_mhz}), flush=True)
    dev = torch.device("cuda", 0)
    for m, n, d in SHAPES:
        reps = 1 if m >= 1_000_000 else int(os.environ.get("PAIRWISE_BASELINE_REPS", "3"))
        g = torch.Generator(device=dev).manual_seed(7)
        mu = 40.0 * torch.randn(d, device=dev, generator=g)
        x = (mu + 1.8 * torch.randn(m, d, device=dev, generator=g)).to(torch.float16).contiguous()
        y = (mu + 0.25 + 1.8 * torch.randn(n, d, device=dev, generator=g)).to(torch.float16).contiguous()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pb = fk.prepare_pairwise_baseline(x)
        torch.cuda.synchronize()
        rec = {"m": m, "n": n, "d": d, "reps": reps, "prepare_ms": round((time.perf_counter() - t0) * 1e3, 1)}
        calls = {"kad": lambda b: fk.calc_kernel_audio_distance(b, y),
                 "prdc_k5": lambda b: fk.calc_prdc(b, y, 5),
                 "realism_k3": lambda b: fk.calc_realism(b, y, 3)}
        for metric, fn in calls.items():
            got_p, got_u = fn(pb), fn(x)                  # warm-up, and the results compared below
            ms_u = timed(lambda: fn(x), reps)
            ms_p = timed(lambda: fn(pb), reps)
            if metric == "kad":
                same = abs(got_p.score - got_u.score) / abs(got_u.score)
            elif metric == "prdc_k5":
                same = got_p == got_u
            else:
                same = all(np.array_equal(getattr(got_p, a), getattr(got_u, a))
                           for a in ("realism", "nearest", "nearest_distance"))
            rec[metric] = {"unprepared_ms": round(ms_u, 2), "prepared_ms": round(ms_p, 2),
                           "kad_rel_diff" if metric == "kad" else "bitwise_equal": same}
        print(json.dumps(rec), flush=True)
        del pb, x, y
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
