"""Per-layer time of the wgmma GEMM on the eight VGGish tensor-core layers at the benchmark's shapes (one 10 000-example
chunk per launch, stage entry fad_umma_layer), with fp16 hi/lo weights (split_w = 1, what the product runs) and with
plain fp16 weights (split_w = 0).

Split weights issue twice the tensor work of plain ones but move only 1.5x the bytes per k-step, so the split / plain
time ratio on the big layers says what bounds them: ~1.5 = feeding the tensor cores from L2, ~2 = issuing wgmmas.

Per layer and mode: median / min / max ms over one CUDA event per launch; TFLOP/s algorithmic (2 M N K once) and issued
(x2 for split weights); and the bytes moved from L2 into shared memory per launch, as implied by the tile count,
k-steps and stage size, over the median time.  The L2 bytes are given for one CTA per 128 x 128 tile loading its whole
stage ("unpaired") and for CTA pairs that share each weight box by TMA multicast ("paired": per pair and k-step, two A
boxes and one weight box).  The first line is the card, power limit and max SM clock, read in the same process.
    python benchmarks/vggish_layers.py [--examples 10000] [--reps 10]"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

os.environ.setdefault("FADTK_SYNTHETIC", "1")
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402
from fadtk_b200 import _native, weights  # noqa: E402

# the kVgg table of csrc/fadtk_b200.cu: name, H, W, Cin, Cout, taps, relu, pool
LAYERS = [
    ("conv2", 48, 32, 64, 128, 9, 1, 1), ("conv3_1", 24, 16, 128, 256, 9, 1, 0), ("conv3_2", 24, 16, 256, 256, 9, 1, 1),
    ("conv4_1", 12, 8, 256, 512, 9, 1, 0), ("conv4_2", 12, 8, 512, 512, 9, 1, 1),
    ("fc1", 1, 1, 12288, 4096, 1, 1, 0), ("fc2", 1, 1, 4096, 4096, 1, 1, 0), ("fc3", 1, 1, 4096, 128, 1, 0, 0),
]
A_BYTES = 128 * 64 * 2                               # one 128-row x 64-K fp16 A box per k-step


def m_tiles(nb, hh, ww):
    """128-row output tiles of one launch (make_geom's pixel boxes)"""
    if hh == 1 and ww == 1:
        return -(-nb // 128)
    bw = min(ww, 16)
    bh = 1
    while bh * 2 <= 128 // bw and hh % (bh * 2) == 0:
        bh *= 2
    bn = 128 // (bw * bh)
    return -(-nb // bn) * (hh // bh) * (ww // bw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--examples", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": gpu[torch.cuda.current_device()] if gpu else None, "examples": args.examples}))
    eng = _native.engine(0)
    dev = eng.torch_device
    nb = args.examples
    for name, hh, ww, cin, cout, taps, relu, pool in LAYERS:
        torch.manual_seed(1)
        k = taps * cin
        x = (torch.randn(nb, hh, ww, cin, device=dev) * 0.5).to(torch.float16)
        w32 = torch.randn(cout, k) * (2.0 / k) ** 0.5
        bias = torch.randn(cout, device=dev) * 0.1
        mt, nt, ks = m_tiles(nb, hh, ww), cout // 128, k // 64
        flop = 2.0 * nb * hh * ww * cout * k
        rec = {"layer": name, "m_tiles": mt, "n_tiles": nt, "ksteps": ks}
        for label, split in (("split", 1), ("fp16", 0)):
            w = (weights.split_hi_lo_tiles(w32, 128) if split else w32.to(torch.float16)).to(dev).contiguous()
            for _ in range(3):
                eng.umma_layer(x, w, bias, taps, relu, pool, split_w=split)
            torch.cuda.synchronize()
            n = args.reps
            evs = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
            evs[0].record()
            for i in range(n):                          # one event per launch: a single slow launch must not hide in a mean
                eng.umma_layer(x, w, bias, taps, relu, pool, split_w=split)
                evs[i + 1].record()
            torch.cuda.synchronize()
            per = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(n))
            ms = per[n // 2]
            w_box = (2 if split else 1) * 128 * 64 * 2
            unpaired = float(mt * nt * ks * (A_BYTES + w_box))
            paired = float(-(-mt // 2) * nt * ks * (2 * A_BYTES + w_box))
            rec[label] = {"ms": round(ms, 4), "min_ms": round(per[0], 4), "max_ms": round(per[-1], 4),
                          "tflops": round(flop / ms / 1e9, 1), "issued_tflops": round((2 if split else 1) * flop / ms / 1e9, 1),
                          "l2_gb_unpaired": round(unpaired / 1e9, 2), "l2_tb_s_unpaired": round(unpaired / ms / 1e9, 2),
                          "l2_gb_paired": round(paired / 1e9, 2), "l2_tb_s_paired": round(paired / ms / 1e9, 2)}
            del w
        rec["split_over_fp16"] = round(rec["split"]["ms"] / rec["fp16"]["ms"], 3)
        print(json.dumps(rec), flush=True)
        del x


if __name__ == "__main__":
    main()
