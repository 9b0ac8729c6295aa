"""Does the wgmma GEMM (fp16 activations, fp16 hi/lo weights, fp32 register accumulation cut every 512 of K) carry a SYSTEMATIC
per-output-channel error?  fp32 outputs of fad_umma_layer vs an fp64 product of the same fp16 activations and fp32 weights:
rms error, error of the per-channel mean over all rows, and what that would be if the errors were independent."""
import json
import os
import sys
from pathlib import Path

os.environ.setdefault("FADTK_SYNTHETIC", "1")
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402
from fadtk_b200 import _native, weights as wts  # noqa: E402

eng = _native.Engine(0, max_examples=16)
dev = eng.torch_device
out = []
for rows, K, N, act, mean_in in ((25600, 768, 768, 0, 0.0), (25600, 768, 3072, 2, 0.0), (25600, 3072, 768, 0, 0.3), (25600, 768, 768, 0, 0.5)):
    g = torch.Generator(device="cpu").manual_seed(K + N)
    x = (torch.randn((rows, K), generator=g) + mean_in).to(torch.float16)
    w32 = torch.randn((N, K), generator=g) * (1.0 / K) ** 0.5
    b = torch.randn((N,), generator=g) * 0.1
    xd = x.to(dev).view(rows, 1, 1, K).contiguous()
    row = {"rows": rows, "K": K, "N": N, "activation": {0: "none", 2: "gelu"}[act], "input_mean": mean_in}
    for name, split in (("split_hi_lo", 1), ("fp16_weights", 0)):
        wd = (wts.split_hi_lo_tiles(w32) if split else w32.to(torch.float16)).to(dev)
        _, got = eng.umma_layer(xd, wd, b.to(dev), 1, act, False, want_f32=True, split_w=split)
        ref = x.to(dev).double() @ (w32.to(dev).double().t() if split else w32.to(torch.float16).to(dev).double().t()) + b.to(dev).double()
        if act == 2:
            ref = torch.nn.functional.gelu(ref)
        err = got.view(rows, N).double() - ref
        rms = ref.pow(2).mean().sqrt().item()
        row[name] = {"rms_rel": err.pow(2).mean().sqrt().item() / rms,
                     "channel_mean_err_rms_rel": err.mean(0).pow(2).mean().sqrt().item() / rms,
                     "expected_if_independent": err.pow(2).mean().sqrt().item() / rms / rows ** 0.5,
                     "global_mean_err_rel": err.mean().item() / rms,
                     "scale_bias": ((got.view(rows, N).double() * ref).sum() / (ref * ref).sum()).item() - 1.0}
    out.append(row)
print(json.dumps(out))
