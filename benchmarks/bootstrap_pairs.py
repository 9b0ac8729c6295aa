"""The bootstrap intervals at user sizes, B = 999: the stages of fad_frechet_boot timed one by one through the stage
entries - multiplicities (fad_boot_counts), unit records (fad_unit_records), weighted record sums
(fad_boot_record_sums), Frechet chains of the B + 1 resamples (fad_frechet_records) - and the whole KAD pass
(fad_kad_boot_sums: multiplicities, row weights, the weighted label product over the eval rows' pair tiles, unit
terms) at VGGish-like (5 000 files x 10 rows, d = 128), CLAP-like (5 000 x 10, d = 512) and MERT-like (1 000 x 750,
d = 768) shapes, with the whole FAD call at the first shape.  CUDA events around each call after a small warm-up.  FLOP
model from shapes: records N d^2, sums 2 (B + 1) F R(d), chains (B + 1) x iterations x 3 x 2 d^3; shares are of the DMMA
rate fad_bench_dmma_peak measures in the same run.  The first line is the card, power limit and max SM clock.  JSON
lines on stdout; BOOTSTRAP_SHAPES=small runs a tenth of the files and B = 99."""
import json
import os
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402
from fadtk_b200 import _native  # noqa: E402
from fadtk_b200.utils import DeviceStatistics  # noqa: E402


def smi(query: str) -> str:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return r, e0.elapsed_time(e1)


def main():
    small = os.environ.get("BOOTSTRAP_SHAPES") == "small"
    dev = torch.device("cuda")
    eng = _native.engine()
    print(json.dumps({"gpu": smi("name"), "power_limit_w": smi("power.limit"), "max_sm_clock_mhz": smi("clocks.max.sm")}))
    peak = eng.dmma_peak_tflops() * 1e12
    print(json.dumps({"dmma_peak_tflops_measured": peak / 1e12}))
    B = 99 if small else 999
    iters = 60
    shapes = [("vggish-like", 128, 5000, 10), ("clap-like", 512, 5000, 10), ("mert-like", 768, 1000, 750)]
    for name, d, files, rows in shapes:
        F = files // 10 if small else files
        N = F * rows
        g = torch.Generator(device=dev).manual_seed(d)
        mix = torch.randn(d, d, generator=g, device=dev, dtype=torch.float32) / d ** 0.5
        emb = (torch.randn(N, d, generator=g, device=dev) @ mix + 0.3).to(torch.float16).contiguous()
        offs = torch.arange(F + 1, device=dev, dtype=torch.int64) * rows
        xb = (torch.randn(4 * d, d, generator=g, device=dev) @ mix).to(torch.float16).contiguous()
        st = DeviceStatistics(d, eng)
        st.add(xb)
        mu, cov = st.finalize()
        base = _native.Baseline(eng, mu, cov)
        sq = eng.kad_median_sq(xb).cpu()
        sig = torch.tensor([0.5 * (float(sq[0]) ** 0.5 + float(sq[1]) ** 0.5)], dtype=torch.float64, device=dev)
        gu = torch.ones(F, dtype=torch.float64, device=dev)
        # warm-up on a few units
        w_offs = offs[:9].contiguous()
        base.frechet_boot(emb, w_offs, 3, 0)
        eng.kad_boot_sums(emb[:int(w_offs[-1])], w_offs, sig, gu[:8].contiguous(), 3, 0)
        shift = emb.float().mean(0).to(torch.float16)
        cnt, t_counts = timed(lambda: eng.boot_counts(F, B, 0))
        rec, t_rec = timed(lambda: eng.unit_records(emb, offs, shift))
        sums, t_sums = timed(lambda: eng.boot_record_sums(rec, cnt, d))
        del rec
        _, t_chain = timed(lambda: base.frechet_records(sums, shift))
        del sums
        _, t_kad = timed(lambda: eng.kad_boot_sums(emb, offs, sig, gu, B, 0))
        R = 1 + d + d * (d + 1) // 2
        fl = {"records": N * d * d * 2.0, "sums": 2.0 * (B + 1) * F * R, "chains": (B + 1) * iters * 3 * 2.0 * d ** 3}
        res = {"shape": name, "d": d, "files": F, "rows_per_file": rows, "B": B, "counts_ms": round(t_counts, 3)}
        for k, t in (("records", t_rec), ("sums", t_sums), ("chains", t_chain)):
            res[f"{k}_ms"] = round(t, 2)
            res[f"{k}_tflop"] = fl[k] / 1e12
            res[f"{k}_share_of_dmma"] = round(fl[k] / (t * 1e-3) / peak, 3)
        res["kad_pass_ms"] = round(t_kad, 2)
        if name == "vggish-like":
            _, t_all = timed(lambda: base.frechet_boot(emb, offs, B, 0))
            res["fad_whole_call_ms"] = round(t_all, 2)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
