"""Per-shape rate of the wgmma GEMM kernel on the Linear layers of the transformer forwards (stage entry
fad_umma_layer, H = W = 1): split weights, and plain fp16 weights for scale.
TFLOP/s are ALGORITHMIC (2 M N K once).  One JSON list on stdout."""
import json
import os
import sys
from pathlib import Path

os.environ.setdefault("FADTK_SYNTHETIC", "1")
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402
from fadtk_b200 import _native, weights  # noqa: E402

SHAPES = [  # name, rows, K, N, act (0 none, 2 GELU)
    ("whisper-small qkv (64 clips)", 96000, 768, 2304, 0), ("whisper-small out", 96000, 768, 768, 0),
    ("whisper-small fc1+GELU", 96000, 768, 3072, 2), ("whisper-small fc2", 96000, 3072, 768, 0),
    ("clap stage2 qkv (500 windows)", 512000, 192, 576, 0), ("clap stage2 fc1+GELU", 512000, 192, 768, 2),
    ("clap stage2 fc2", 512000, 768, 192, 0),
    ("clap stage3 qkv", 128000, 384, 1152, 0), ("clap stage3 fc1+GELU", 128000, 384, 1536, 2), ("clap stage3 fc2", 128000, 1536, 384, 0),
]
eng = _native.engine(0)
dev = eng.torch_device
out = []
for name, rows, K, N, act in SHAPES:
    torch.manual_seed(1)
    npad = (N + 127) // 128 * 128                       # the product pads the weight rows to whole 128-column tiles
    x = (torch.randn(rows, K, device=dev) * 0.5).to(torch.float16).reshape(rows, 1, 1, K)
    w32 = torch.zeros(npad, K)
    w32[:N] = torch.randn(N, K) / K ** 0.5
    bias = torch.zeros(npad, dtype=torch.float32, device=dev)
    rec = {"layer": name, "rows": rows, "K": K, "N": N, "act": act}
    for label, split in (("split", True), ("fp16", False)):
        w = (weights.split_hi_lo_tiles(w32, 128) if split else w32.to(torch.float16)).to(dev).contiguous()
        for _ in range(3):
            eng.umma_layer(x, w, bias, 1, act, 0, split_w=split)
        torch.cuda.synchronize()
        n = int(os.environ.get("LINEAR_SHAPES_REPS", "10"))
        evs = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
        evs[0].record()
        for i in range(n):                                  # one event per launch: a single slow launch must not hide in a mean
            eng.umma_layer(x, w, bias, 1, act, 0, split_w=split)
            evs[i + 1].record()
        torch.cuda.synchronize()
        per = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(n))
        ms = per[n // 2]
        rec[label] = {"ms": round(ms, 4), "min_ms": round(per[0], 4), "max_ms": round(per[-1], 4), "tflops": round(2.0 * rows * K * N / ms / 1e9, 1)}
    out.append(rec)
    del x, w
print(json.dumps(out))
