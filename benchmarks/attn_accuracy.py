"""Error statistics of the two encoder-attention kernels against an fp64 reference on the same fp16 inputs:
rms and mean (signed) error of the output, relative to the rms of the exact output.  $1 = score scale (peakedness)."""
import json
import os
import sys
from pathlib import Path

os.environ.setdefault("FADTK_SYNTHETIC", "1")
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402
from fadtk_b200 import _native  # noqa: E402

eng = _native.Engine(0, max_examples=16)
dev = eng.torch_device
out = []
for S, d, n, scale in ((199, 768, 8, 1.0), (199, 768, 8, 2.5), (1500, 768, 2, 1.0), (1500, 768, 2, 2.5), (499, 768, 4, 4.0)):
    g = torch.Generator(device="cpu").manual_seed(S + int(scale * 10))
    qkv = torch.randn((n * S, 3 * d), generator=g)
    qkv[:, :2 * d] *= scale
    qkv[:, 2 * d:] += 0.3                                  # values with a non-zero mean: a scale bias shows up as a mean error
    qkv = qkv.to(torch.float16).to(dev)
    x = qkv.double().view(n, S, 3, d // 64, 64)
    q, k, v = (x[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    p = torch.softmax(q @ k.transpose(-1, -2) / 8.0, dim=-1)
    want = (p @ v).permute(0, 2, 1, 3).reshape(n * S, d)
    rms = want.pow(2).mean().sqrt().item()
    row = {"S": S, "score_scale": scale, "max_p_mean": p.max(-1).values.mean().item()}
    for name, legacy in (("wgmma", False), ("mma_sync", True)):
        got = eng.attention(qkv, n, legacy=legacy).double()
        err = got - want
        row[name] = {"rms_rel": err.pow(2).mean().sqrt().item() / rms, "mean_rel": err.mean().item() / rms,
                     "scale_bias": ((got * want).sum() / (want * want).sum()).item() - 1.0}
    out.append(row)
print(json.dumps(out))
