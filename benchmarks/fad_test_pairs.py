"""The FAD comparison at user sizes, B = 999: the three stages of fad_frechet_perm timed one by one through the stage
entries - unit records (fad_unit_records), labelled sums (fad_perm_record_sums), Frechet chains of all 2 (B + 1)
labelled statistics (fad_frechet_records) - at VGGish-like (2 x 5 000 files x 10 rows, d = 128), CLAP-like (2 x 5 000 x
10, d = 512) and MERT-like (2 x 1 000 x 750, d = 768) shapes, with the whole call at the first shape, and one call of
the per-set path (DeviceStatistics.add_gather + Baseline.frechet) for scale.  CUDA events around each call after a
small warm-up.  FLOP model from shapes: records N d^2, sums 2 x 2 (B + 1) F R(d), chains 2 (B + 1) x iterations x 3 x
2 d^3; shares are of the DMMA rate fad_bench_dmma_peak measures in the same run.  The first line is the card, power
limit and max SM clock.  JSON lines on stdout; FAD_TEST_SHAPES=small runs a tenth of the files and B = 99."""
import json
import os
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
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
    small = os.environ.get("FAD_TEST_SHAPES") == "small"
    dev = torch.device("cuda")
    eng = _native.engine()
    print(json.dumps({"gpu": smi("name"), "power_limit_w": smi("power.limit"), "max_sm_clock_mhz": smi("clocks.max.sm")}))
    peak = eng.dmma_peak_tflops() * 1e12
    print(json.dumps({"dmma_peak_tflops_measured": peak / 1e12}))
    B = 99 if small else 999
    iters = 60
    shapes = [("vggish-like", 128, 5000, 10), ("clap-like", 512, 5000, 10), ("mert-like", 768, 1000, 750)]
    for name, d, files, rows in shapes:
        files = files // 10 if small else files
        F, N = 2 * files, 2 * files * rows
        g = torch.Generator(device=dev).manual_seed(d)
        mix = torch.randn(d, d, generator=g, device=dev, dtype=torch.float32) / d ** 0.5
        emb = (torch.randn(N, d, generator=g, device=dev) @ mix + 0.3).to(torch.float16).contiguous()
        offs = torch.arange(F + 1, device=dev, dtype=torch.int64) * rows
        xb = (torch.randn(4 * d, d, generator=g, device=dev) @ mix).to(torch.float16)
        st = DeviceStatistics(d, eng)
        st.add(xb.contiguous())
        mu, cov = st.finalize()
        base = _native.Baseline(eng, mu, cov)
        # warm-up on a few units
        w_offs = offs[:9].contiguous()
        base.frechet_perm(emb, w_offs, 4, 3, 0)
        shift = emb.float().mean(0).to(torch.float16)
        rec, t_rec = timed(lambda: eng.unit_records(emb, offs, shift))
        bits = eng.perm_labels(F, files, B, 0)
        sums, t_sums = timed(lambda: eng.perm_record_sums(rec, bits, d))
        del rec
        _, t_chain = timed(lambda: base.frechet_records(sums, shift))
        del sums
        R = 1 + d + d * (d + 1) // 2
        fl = {"records": N * d * d * 2.0, "sums": 2.0 * 2 * (B + 1) * F * R,
              "chains": 2.0 * (B + 1) * iters * 3 * 2 * d ** 3}
        res = {"shape": name, "d": d, "files": F, "rows_per_file": rows, "B": B}
        for k, t in (("records", t_rec), ("sums", t_sums), ("chains", t_chain)):
            res[f"{k}_ms"] = round(t, 2)
            res[f"{k}_tflop"] = fl[k] / 1e12
            res[f"{k}_share_of_dmma"] = round(fl[k] / (t * 1e-3) / peak, 3)
        if name == "vggish-like":
            _, t_all = timed(lambda: base.frechet_perm(emb, offs, files, B, 0))
            res["whole_call_ms"] = round(t_all, 2)
        idx = torch.arange(files * rows, device=dev, dtype=torch.int64)

        def per_set():
            s = DeviceStatistics(d, eng)
            s.add_gather(emb, idx)
            m, c = s.finalize()
            return base.frechet(m.contiguous(), c)
        per_set()
        _, t_set = timed(per_set)
        res["per_set_call_ms"] = round(t_set, 2)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
