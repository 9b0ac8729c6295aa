"""Sharded Kernel Audio Distance (fad_kad_*_sharded): what each rank's share of the pair tiles costs, per stage.

Under torchrun (R ranks, one GPU each; the library's NCCL communicator):
    torchrun --nproc-per-node R benchmarks/kad_sharded.py
each stage (bandwidth = fad_kad_median_sq_sharded, sums = fad_kad_sums_sharded) is timed with CUDA events, warm-up
first, median of 5 calls, and the maximum over the ranks is reported; the exchange is also timed on its own (one
all-reduce of the same bytes).  Every rank asserts that its outputs are bitwise equal to the unsharded entries'.

In one process (`python benchmarks/kad_sharded.py`), the same cut into R = 1, 2, 4, 8 shards runs as local shards on
one GPU, one shard after another, and torch.profiler gives each shard's tile-kernel time: the maximum over the shards
is what each of R ranks would spend in the tile passes (the exchange and the replicated prologue not included).

Shapes: m = n = 100 000 rows at d = 128 and d = 512 (KAD_SHARDED_BIG=1 adds 500 000 + 500 000 at d = 512); rows with a
common offset, rounded to fp16.  The wave model: a pass over U units on R ranks takes ceil(U / (132 R)) waves of
persistent CTAs (132 SMs).  The first line is the card, power limit and SM count.  JSON lines on stdout.
"""
import json
import math
import os
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from fadtk_b200 import _native, dist  # noqa: E402

SHAPES = [("vggish", 100_000, 100_000, 128), ("clap", 100_000, 100_000, 512)]
BIG = [("clap-500k", 500_000, 500_000, 512)]
REPS = 5


def smi(query: str, index: int) -> str:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", str(index)],
                         capture_output=True, text=True)
    return out.stdout.strip()


def timed(fn, reps: int = REPS) -> float:
    """median milliseconds of one call, CUDA events around each call (after one warm-up call)"""
    fn()
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    evs[0].record()
    for i in range(reps):
        fn()
        evs[i + 1].record()
    torch.cuda.synchronize()
    return float(np.median([evs[i].elapsed_time(evs[i + 1]) for i in range(reps)]))


def data(dev, m, n, d):
    g = torch.Generator(device=dev).manual_seed(7)
    mu = 40.0 * torch.randn(d, device=dev, generator=g)
    z = (mu + 1.8 * torch.randn(m + n, d, device=dev, generator=g)).to(torch.float16).contiguous()
    z[m:] += 0.25
    return z


def units(rows):
    return (-(-rows // 128) + 1) // 2


def waves(u, r, sms):
    return math.ceil(u / (sms * r))


def tile_ms(fn, mode: int):
    """per launch of kad_tile_kernel<mode> in one call of fn, in launch order: milliseconds (torch.profiler)"""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.device_time / 1e3 for e in prof.events()
            if e.device_type == torch.autograd.DeviceType.CUDA and f"kad_tile_kernel<{mode}>" in e.name]


def local(eng, shapes, sms):
    for label, m, n, d in shapes:
        z = data(eng.torch_device, m, n, d)
        x = z[:m]
        sq = eng.kad_median_sq(x)
        sigma = (0.5 * (sq[0].sqrt() + sq[1].sqrt())).reshape(1).contiguous()
        sums = eng.kad_sums(z, m, sigma)
        rec = {"mode": "local", "shape": label, "m": m, "n": n, "d": d, "sums_units": units(m + n),
               "bandwidth_units": units(m), "whole_call_ms": {"bandwidth": round(timed(lambda: eng.kad_median_sq(x)), 3),
                                                              "sums": round(timed(lambda: eng.kad_sums(z, m, sigma)), 3)}}
        for r in (1, 2, 4, 8):
            assert torch.equal(eng.kad_median_sq_sharded(x, local_shards=r), sq), r
            assert torch.equal(eng.kad_sums_sharded(z, m, sigma, local_shards=r), sums), r
            t_sum = tile_ms(lambda: eng.kad_sums_sharded(z, m, sigma, local_shards=r), 0)
            t_med = tile_ms(lambda: eng.kad_median_sq_sharded(x, local_shards=r), 1)
            n_med = len(t_med) // 3                                  # launches per radix pass (empty shards launch none)
            rec[f"R{r}"] = {"sums_tile_max_ms": round(max(t_sum), 3), "sums_tile_ms": [round(t, 3) for t in t_sum],
                            "bandwidth_tile_max_ms": round(sum(max(t_med[p * n_med:(p + 1) * n_med]) for p in range(3)), 3),
                            "waves_sums": waves(units(m + n), r, sms), "waves_bandwidth": waves(units(m), r, sms)}
        rec["bitwise_equal_to_unsharded"] = True
        print(json.dumps(rec), flush=True)


def collective(eng, shapes, sms):
    r = dist.world_size()
    for label, m, n, d in shapes:
        z = data(eng.torch_device, m, n, d)
        x = z[:m]
        sq = eng.kad_median_sq(x)
        sigma = (0.5 * (sq[0].sqrt() + sq[1].sqrt())).reshape(1).contiguous()
        sums = eng.kad_sums(z, m, sigma)
        assert torch.equal(eng.kad_median_sq_sharded(x), sq) and torch.equal(eng.kad_sums_sharded(z, m, sigma), sums)
        ms = {"bandwidth": timed(lambda: eng.kad_median_sq_sharded(x)),
              "sums": timed(lambda: eng.kad_sums_sharded(z, m, sigma))}
        # the exchanges alone: three all-reduces of the [2][2048] histogram, one of the units x 3 partials
        hist = torch.zeros(2 * 2048, dtype=torch.float64, device=eng.torch_device)
        part = torch.zeros(3 * units(m + n), dtype=torch.float64, device=eng.torch_device)
        ex = {"bandwidth": timed(lambda: [eng.allreduce_sum_(hist) for _ in range(3)]),
              "sums": timed(lambda: eng.allreduce_sum_(part))}
        rec = {"mode": "torchrun", "ranks": r, "shape": label, "m": m, "n": n, "d": d,
               "ms_max_over_ranks": {k: round(dist.max_over_ranks(v), 3) for k, v in ms.items()},
               "exchange_ms_max_over_ranks": {k: round(dist.max_over_ranks(v), 3) for k, v in ex.items()},
               "waves_sums": waves(units(m + n), r, sms), "waves_bandwidth": waves(units(m), r, sms),
               "bitwise_equal_to_unsharded": True}
        if dist.rank() == 0:
            print(json.dumps(rec), flush=True)


def main():
    assert torch.cuda.is_available(), "kad_sharded.py measures on the GPU"
    dist.init_from_env()
    dev = torch.cuda.current_device()
    eng = _native.engine(dev)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    name, plimit = [s.strip() for s in smi("name,power.limit", dev).split(",")]
    if dist.rank() == 0:
        print(json.dumps({"gpu": name, "power_limit_w": plimit, "sms": sms, "ranks": dist.world_size()}), flush=True)
    shapes = SHAPES + (BIG if os.environ.get("KAD_SHARDED_BIG") == "1" else [])
    if dist.is_distributed():
        assert dist.enable_native_allreduce(eng), "needs the library's NCCL communicator (nccl backend)"
        collective(eng, shapes, sms)
    else:
        local(eng, shapes, sms)
    dist.shutdown()


if __name__ == "__main__":
    main()
