"""Per-song Kernel Audio Distance at user sizes: fad_kad_song_sums (every song's S_yy,k and S_xy,k plus the baseline's
S_xx in one call) timed with CUDA events over repeated calls after a warm-up, and, for comparison, the per-file loop a
user would otherwise write - calc_kernel_audio_distance(X, Y_k) once per song, which redoes the bandwidth selection and
the baseline's pair triangle every time - timed on a few songs and scaled to all of them.

Shapes: a 100 000-row baseline against 10 000 songs x 10 rows at d = 128 (VGGish), 1 250 songs x 750 rows at d = 128
(Encodec, 10-s clips at 75 frames/s) and 1 000 songs x 10 rows at d = 512 (CLAP); rows with a common offset, rounded
to fp16.  Pairs are ALGORITHMIC: m (m - 1) / 2 + m n_total + sum n_k (n_k - 1) / 2.  The first line is the card, power
limit and max SM clock, read in the same process; each record says whether two calls gave bitwise-equal sums.  JSON
lines on stdout.
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
from fadtk_b200.fad import calc_kernel_audio_distance  # noqa: E402

SHAPES = [("vggish", 100_000, 10_000, 10, 128), ("encodec", 100_000, 1_250, 750, 128), ("clap", 100_000, 1_000, 10, 512)]
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
    assert torch.cuda.is_available(), "kad_songs.py measures on the GPU"
    name, plimit, max_mhz = [s.strip() for s in smi("name,power.limit,clocks.max.sm").split(",")]
    print(json.dumps({"gpu": name, "power_limit_w": plimit, "max_sm_mhz": max_mhz,
                      "sms": torch.cuda.get_device_properties(0).multi_processor_count}), flush=True)
    eng = _native.engine(0)
    dev = eng.torch_device
    reps = int(os.environ.get("KAD_SONGS_REPS", "5"))
    for label, m, songs, rows, d in SHAPES:
        g = torch.Generator(device=dev).manual_seed(11)
        mu = 40.0 * torch.randn(d, device=dev, generator=g)
        n = songs * rows
        z = (mu + 1.8 * torch.randn(m + n, d, device=dev, generator=g)).to(torch.float16).contiguous()
        z[m:] += 0.25
        offsets = torch.arange(0, n + 1, rows, dtype=torch.int64, device=dev)
        sq = eng.kad_median_sq(z[:m])
        sigma = (0.5 * (sq[0].sqrt() + sq[1].sqrt())).reshape(1).contiguous()
        a = eng.kad_song_sums(z, m, offsets, sigma)                    # warm-up
        b = eng.kad_song_sums(z, m, offsets, sigma)
        torch.cuda.synchronize()
        ms = timed(lambda: eng.kad_song_sums(z, m, offsets, sigma), reps)
        ms_sigma = timed(lambda: eng.kad_median_sq(z[:m]), reps)
        pairs = m * (m - 1) / 2 + m * n + songs * rows * (rows - 1) / 2

        calc_kernel_audio_distance(z[:m], z[m:m + rows])                # warm-up of the per-file path
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in range(LOOP_SONGS):
            calc_kernel_audio_distance(z[:m], z[m + k * rows:m + (k + 1) * rows])
        torch.cuda.synchronize()
        loop_ms = (time.perf_counter() - t0) * 1e3 / LOOP_SONGS
        rec = {"shape": label, "m": m, "songs": songs, "rows_per_song": rows, "d": d, "reps": reps,
               "song_sums_ms": round(ms, 3), "pairs_per_s": pairs / (ms * 1e-3),
               "bandwidth_ms": round(ms_sigma, 3), "per_song_total_ms": round(ms + ms_sigma, 3),
               "loop_ms_per_song": round(loop_ms, 3), "loop_songs_timed": LOOP_SONGS,
               "loop_all_songs_s_scaled": round(loop_ms * songs / 1e3, 1),
               "s_xx": float(a[0]), "bitwise_equal_two_runs": bool(torch.equal(a, b))}
        print(json.dumps(rec), flush=True)
        del z, a, b
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
