"""Sharded precision, recall, density and coverage (fad_knn_radii_sq_sharded, fad_prdc_counts_sharded): what each
rank's share of the radii and ball-count tiles costs, per pass.

Under torchrun (R ranks, one GPU each; the library's NCCL communicator):
    torchrun --nproc-per-node R benchmarks/prdc_sharded.py
each pass (radii, counts) is timed with CUDA events, warm-up first, median of 5 calls, and the maximum over the ranks is
reported; the exchange is also timed on its own (one all-reduce of the same bytes).  Every rank asserts that its
outputs are bitwise equal to the unsharded entries'.

In one process (`python benchmarks/prdc_sharded.py`), the same cut into R = 1, 2, 4, 8 shards runs as local shards on
one GPU, one shard after another, and torch.profiler gives each shard's tile-kernel time: the maximum over the shards
is what each of R ranks would spend in the tile passes (the exchange and the replicated prologue not included).

Shapes: m = n = 100 000 rows at d = 128 and d = 512, k = 5; rows with a common offset, rounded to fp16 (kad_sharded.py's
data).  Radii units are whole tile rows (Tx units of Tx tiles, then Ty of Ty tiles), counts units runs of about
G = max(4, ceil(Tx Ty / 8192)) column tiles.  The wave model: a pass over U units on R ranks takes ceil(U / (132 R))
waves of persistent CTAs (132 SMs).  The first line is the card, power limit and SM count.  JSON lines on stdout.
"""
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from fadtk_b200 import _native, dist  # noqa: E402
from kad_sharded import data, smi, timed, waves  # noqa: E402

SHAPES = [("vggish", 100_000, 100_000, 128), ("clap", 100_000, 100_000, 512)]
K = 5


def units(m, n):
    """(radii units, tiles per radii unit at m = n, counts units, tiles per counts unit at most)"""
    tx, ty = -(-m // 128), -(-n // 128)
    g = max(4, -(-(tx * ty) // 8192))
    cuts = -(-ty // g)
    return tx + ty, tx, tx * cuts, -(-ty // cuts)


def tile_ms(fn, pass_: int):
    """per launch of prdc_tile_kernel<pass_> in one call of fn, in launch order: milliseconds (torch.profiler)"""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.device_time / 1e3 for e in prof.events()
            if e.device_type == torch.autograd.DeviceType.CUDA and f"prdc_tile_kernel<{pass_}>" in e.name]


def local(eng, sms):
    for label, m, n, d in SHAPES:
        z = data(eng.torch_device, m, n, d)
        radii = eng.knn_radii_sq(z, m, K)
        inside, flags = eng.prdc_counts(z, m, radii)
        ur, tr, uc, tc = units(m, n)
        rec = {"mode": "local", "shape": label, "m": m, "n": n, "d": d, "k": K,
               "radii_units": ur, "radii_tiles_per_unit": tr, "counts_units": uc, "counts_tiles_per_unit_max": tc,
               "whole_call_ms": {"radii": round(timed(lambda: eng.knn_radii_sq(z, m, K)), 3),
                                 "counts": round(timed(lambda: eng.prdc_counts(z, m, radii)), 3)}}
        for r in (1, 2, 4, 8):
            assert torch.equal(eng.knn_radii_sq_sharded(z, m, K, local_shards=r), radii), r
            got_in, got_fl = eng.prdc_counts_sharded(z, m, radii, local_shards=r)
            assert torch.equal(got_in, inside) and torch.equal(got_fl, flags), r
            t_r = tile_ms(lambda: eng.knn_radii_sq_sharded(z, m, K, local_shards=r), 0)
            t_c = tile_ms(lambda: eng.prdc_counts_sharded(z, m, radii, local_shards=r), 1)
            rec[f"R{r}"] = {"radii_tile_max_ms": round(max(t_r), 3), "radii_tile_ms": [round(t, 3) for t in t_r],
                            "counts_tile_max_ms": round(max(t_c), 3), "counts_tile_ms": [round(t, 3) for t in t_c],
                            "waves_radii": waves(ur, r, sms), "waves_counts": waves(uc, r, sms)}
        rec["bitwise_equal_to_unsharded"] = True
        print(json.dumps(rec), flush=True)


def collective(eng, sms):
    r = dist.world_size()
    for label, m, n, d in SHAPES:
        z = data(eng.torch_device, m, n, d)
        radii = eng.knn_radii_sq(z, m, K)
        inside, flags = eng.prdc_counts(z, m, radii)
        assert torch.equal(eng.knn_radii_sq_sharded(z, m, K), radii)
        got_in, got_fl = eng.prdc_counts_sharded(z, m, radii)
        assert torch.equal(got_in, inside) and torch.equal(got_fl, flags)
        ms = {"radii": timed(lambda: eng.knn_radii_sq_sharded(z, m, K)),
              "counts": timed(lambda: eng.prdc_counts_sharded(z, m, radii))}
        # the exchanges alone: one all-reduce of the same bytes, (m + n) x 4 (radii) and (n + 2 m) x 4 (counts)
        ex_r = torch.zeros(-(-(m + n) // 2), dtype=torch.float64, device=eng.torch_device)
        ex_c = torch.zeros(-(-(n + 2 * m) // 2), dtype=torch.float64, device=eng.torch_device)
        ex = {"radii": timed(lambda: eng.allreduce_sum_(ex_r)), "counts": timed(lambda: eng.allreduce_sum_(ex_c))}
        ur, _, uc, _ = units(m, n)
        rec = {"mode": "torchrun", "ranks": r, "shape": label, "m": m, "n": n, "d": d, "k": K,
               "ms_max_over_ranks": {k: round(dist.max_over_ranks(v), 3) for k, v in ms.items()},
               "exchange_ms_max_over_ranks": {k: round(dist.max_over_ranks(v), 3) for k, v in ex.items()},
               "waves_radii": waves(ur, r, sms), "waves_counts": waves(uc, r, sms),
               "bitwise_equal_to_unsharded": True}
        if dist.rank() == 0:
            print(json.dumps(rec), flush=True)


def main():
    assert torch.cuda.is_available(), "prdc_sharded.py measures on the GPU"
    dist.init_from_env()
    dev = torch.cuda.current_device()
    eng = _native.engine(dev)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    name, plimit = [s.strip() for s in smi("name,power.limit", dev).split(",")]
    if dist.rank() == 0:
        print(json.dumps({"gpu": name, "power_limit_w": plimit, "sms": sms, "ranks": dist.world_size()}), flush=True)
    if dist.is_distributed():
        assert dist.enable_native_allreduce(eng), "needs the library's NCCL communicator (nccl backend)"
        collective(eng, sms)
    else:
        local(eng, sms)
    dist.shutdown()


if __name__ == "__main__":
    main()
