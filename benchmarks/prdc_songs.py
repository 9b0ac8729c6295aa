"""Per-song precision, recall, density and coverage at user sizes: fad_knn_song_radii_sq (the baseline radii once and
every song's radii within the song) and fad_prdc_song_counts (one X x Y counts rectangle with per-song covered /
recalled counts), each timed with CUDA events over repeated calls after a warm-up; in the same run, calc_prdc on the
whole eval set (fad_knn_radii_sq + fad_prdc_counts), and the per-file loop a user would otherwise write -
calc_prdc(X, Y_k) once per song, which redoes the baseline radii every time - timed on a few songs and scaled to all of
them (labelled as scaled).

Shapes, k = 5, rows with a common offset rounded to fp16: a 100 000-row baseline against 10 000 songs x 10 rows at
d = 128 (VGGish), 1 250 songs x 750 rows at d = 128 (Encodec, 10-s clips at 75 frames/s) and 1 000 songs x 10 rows at
d = 512 (CLAP); and one 100 000-row song against m = 2 000, whose counts run on Tx = 16 CTAs (one span).  The first
line is the card, power limit and max SM clock, read in the same process; each record says whether two calls gave
bitwise-equal outputs.  JSON lines on stdout.
"""
import json
import os
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from fadtk_b200 import _native  # noqa: E402
from fadtk_b200.fad import calc_prdc  # noqa: E402

SHAPES = [("vggish", 100_000, 10_000, 10, 128), ("encodec", 100_000, 1_250, 750, 128), ("clap", 100_000, 1_000, 10, 512),
          ("one_long_song", 2_000, 1, 100_000, 128)]
K = 5
LOOP_SONGS = 3


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
    assert torch.cuda.is_available(), "prdc_songs.py measures on the GPU"
    name, plimit, max_mhz = [s.strip() for s in smi("name,power.limit,clocks.max.sm").split(",")]
    print(json.dumps({"gpu": name, "power_limit_w": plimit, "max_sm_mhz": max_mhz,
                      "sms": torch.cuda.get_device_properties(0).multi_processor_count}), flush=True)
    eng = _native.engine(0)
    dev = eng.torch_device
    reps = int(os.environ.get("PRDC_SONGS_REPS", "5"))
    for label, m, songs, rows, d in SHAPES:
        g = torch.Generator(device=dev).manual_seed(11)
        mu = 40.0 * torch.randn(d, device=dev, generator=g)
        n = songs * rows
        z = (mu + 1.8 * torch.randn(m + n, d, device=dev, generator=g)).to(torch.float16).contiguous()
        z[m:] += 0.25
        offsets = torch.arange(0, n + 1, rows, dtype=torch.int64, device=dev)
        ra = eng.knn_song_radii_sq(z, m, offsets, K)                      # warm-up
        ca = eng.prdc_song_counts(z, m, offsets, ra)
        rb = eng.knn_song_radii_sq(z, m, offsets, K)
        cb = eng.prdc_song_counts(z, m, offsets, rb)
        torch.cuda.synchronize()
        same = bool(torch.equal(ra, rb) and torch.equal(ca[0], cb[0]) and torch.equal(ca[1], cb[1]))
        ms_radii = timed(lambda: eng.knn_song_radii_sq(z, m, offsets, K), reps)
        ms_counts = timed(lambda: eng.prdc_song_counts(z, m, offsets, ra), reps)

        wr = eng.knn_radii_sq(z, m, K)                                     # the whole eval set, same rows
        eng.prdc_counts(z, m, wr)
        ms_whole_radii = timed(lambda: eng.knn_radii_sq(z, m, K), reps)
        ms_whole_counts = timed(lambda: eng.prdc_counts(z, m, wr), reps)

        rec = {"shape": label, "m": m, "songs": songs, "rows_per_song": rows, "d": d, "k": K, "reps": reps,
               "song_radii_ms": round(ms_radii, 3), "song_counts_ms": round(ms_counts, 3),
               "per_song_total_ms": round(ms_radii + ms_counts, 3),
               "whole_set_radii_ms": round(ms_whole_radii, 3), "whole_set_counts_ms": round(ms_whole_counts, 3),
               "bitwise_equal_two_runs": same}
        if songs > 1:
            calc_prdc(z[:m], z[m:m + rows], k=K)                           # warm-up of the per-file path
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for s in range(LOOP_SONGS):
                calc_prdc(z[:m], z[m + s * rows:m + (s + 1) * rows], k=K)
            torch.cuda.synchronize()
            loop_ms = (time.perf_counter() - t0) * 1e3 / LOOP_SONGS
            rec.update({"loop_ms_per_song": round(loop_ms, 3), "loop_songs_timed": LOOP_SONGS,
                        "loop_all_songs_s_scaled": round(loop_ms * songs / 1e3, 1)})
        print(json.dumps(rec), flush=True)
        del z, ra, rb, ca, cb, wr
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
