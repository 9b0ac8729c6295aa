"""VGGish parameters: seeded synthetic set, checkpoint loading, device packing.

There is no network in the build or GPU containers, so unless a real
``vggish-10086976.pth`` (torchvggish release file, model_loader.py:99) is supplied
the engine runs on *seeded synthetic* parameters with the real architecture.  The
state-dict uses torchvggish's key names, so the same dict feeds the CUDA path
(packed by ``pack_vggish``) and the CPU oracle byte-for-byte.
"""
from __future__ import annotations

import math
from pathlib import Path

import numpy as np
import torch

# (state-dict key, Cin, Cout, maxpool after?)
VGGISH_CONVS = (
    ("features.0", 1, 64, True),
    ("features.3", 64, 128, True),
    ("features.6", 128, 256, False),
    ("features.8", 256, 256, True),
    ("features.11", 256, 512, False),
    ("features.13", 512, 512, True),
)
# (state-dict key, in, out, relu after?) - the ReLU after the last Linear is removed
# by the reference (model_loader.py:102-103)
VGGISH_FCS = (
    ("embeddings.0", 512 * 6 * 4, 4096, True),
    ("embeddings.2", 4096, 4096, True),
    ("embeddings.4", 4096, 128, False),
)


def synthetic_vggish_state(seed: int = 0) -> dict:
    """He-normal convolutions / linears with small random biases, float32, on CPU."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for key, cin, cout, _ in VGGISH_CONVS:
        std = math.sqrt(2.0 / (9 * cin))
        sd[key + ".weight"] = torch.randn((cout, cin, 3, 3), generator=g) * std
        sd[key + ".bias"] = torch.randn((cout,), generator=g) * 0.05
    for key, fin, fout, relu in VGGISH_FCS:
        std = math.sqrt((2.0 if relu else 1.0) / fin)
        sd[key + ".weight"] = torch.randn((fout, fin), generator=g) * std
        sd[key + ".bias"] = torch.randn((fout,), generator=g) * 0.05
    return sd


class MissingCheckpoint(RuntimeError):
    """No pretrained checkpoint could be resolved and synthetic weights were not explicitly allowed."""


_warned = set()


def resolve_checkpoint(path, env: str, what: str):
    """-> Path of the real checkpoint to load, or None when seeded SYNTHETIC weights may be used.

    The reference always loads pretrained weights (torch.hub / HF / direct URLs, model_loader.py:99, 301, 657);
    scores from random weights are meaningless and would be cached under the same ``embeddings/<model>`` and
    ``stats/<model>`` paths.  So: an explicit path (argument or ``$<env>``) that does not exist is an error, and
    with no path at all the loader refuses to run unless ``FADTK_SYNTHETIC=1`` (tests, bench.py, smoke) opts in."""
    import logging
    import os
    path = path or os.environ.get(env)
    if path:
        if Path(path).exists():
            return Path(path)
        raise MissingCheckpoint(f"{what}: checkpoint {path!r} (argument or ${env}) does not exist")
    if os.environ.get("FADTK_SYNTHETIC", "") == "1":
        if what not in _warned:
            _warned.add(what)
            logging.getLogger("fadtk_b200").warning(
                "%s: FADTK_SYNTHETIC=1 - running on SEEDED RANDOM weights (real architecture); "
                "scores are not comparable with pretrained-model FAD", what)
        return None
    raise MissingCheckpoint(
        f"{what}: no pretrained checkpoint - pass checkpoint=... or set ${env} (there is no network to download it); "
        "set FADTK_SYNTHETIC=1 to run on seeded random weights (tests / benchmarks only)")


def load_checkpoint_file(path) -> dict:
    """A checkpoint as a flat {name: tensor} dict: ``.safetensors`` (what Hugging Face publishes today) or a torch
    pickle (``pytorch_model.bin`` / ``.pt`` / ``.pth``, optionally wrapped in {"state_dict": ...}).  Published
    weight-normalised convolutions come in two spellings - ``weight_g`` / ``weight_v`` (torch.nn.utils.weight_norm,
    every older checkpoint) and ``parametrizations.weight.original0`` / ``original1`` (torch >= 2.1) - the older one is
    renamed to the newer, which is what the packers read."""
    path = Path(path)
    if path.suffix == ".safetensors":
        from safetensors.torch import load_file
        raw = load_file(str(path), device="cpu")
    else:
        raw = torch.load(path, map_location="cpu")
        if isinstance(raw, dict) and "state_dict" in raw and isinstance(raw["state_dict"], dict):
            extra = {k: v for k, v in raw.items() if k != "state_dict" and not isinstance(v, dict)}
            raw = dict(raw["state_dict"], **{f"__meta__.{k}": v for k, v in extra.items()})
    out = {}
    for k, v in raw.items():
        if k.endswith(".weight_g"):
            k = k[:-len("weight_g")] + "parametrizations.weight.original0"
        elif k.endswith(".weight_v"):
            k = k[:-len("weight_v")] + "parametrizations.weight.original1"
        out[k] = v
    return out


def load_vggish_state(path=None, seed: int = 0) -> dict:
    """Real checkpoint ``path`` (or $FADTK_VGGISH_CKPT); seeded synthetic only under FADTK_SYNTHETIC=1."""
    path = resolve_checkpoint(path, "FADTK_VGGISH_CKPT", "vggish")
    if path is not None:
        sd = load_checkpoint_file(path)
        return {k: v.float().contiguous() for k, v in sd.items()
                if k.startswith(("features.", "embeddings."))}
    return synthetic_vggish_state(seed)


LAYER_NAMES = ("conv2", "conv3_1", "conv3_2", "conv4_1", "conv4_2", "fc1", "fc2", "fc3")
ALL_LAYERS_SPLIT = 0xFF


def split_hi_lo_tiles(w32: torch.Tensor, tile: int = 128) -> torch.Tensor:
    """fp32 [Cout, K] -> fp16 [2*Cout, K]: per 128-row tile, the hi rows (fp16(w)) followed by the
    lo rows (fp16(w - hi)); hi + lo carries 22 bits of the weight."""
    cout, k = w32.shape
    hi = w32.to(torch.float16)
    lo = (w32 - hi.float()).to(torch.float16)
    out = torch.stack([hi.view(cout // tile, tile, k), lo.view(cout // tile, tile, k)], dim=1)
    return out.reshape(2 * cout, k).contiguous()


def pack_vggish(sd: dict, split_mask: int = ALL_LAYERS_SPLIT) -> dict:
    """Re-lay the state-dict for the sm_90a kernels (all on CPU, contiguous).

    ``split_mask`` bit i (LAYER_NAMES order) stores that layer's weights as an fp16 hi/lo pair
    (split_hi_lo_tiles); default: every tensor-core layer.


    conv1   : float32 [64, 9]                     (CUDA-core stencil, fp32 input)
    conv2-6 : float16 [Cout, 9*Cin], k = (kh*3+kw)*Cin + cin   (UMMA B operand, K-major)
    fc1-3   : float16 [out, in]                   (already K-major; fc1's input order is
                                                   the NHWC flatten the upstream uses)
    biases  : float32
    """
    out = {}
    key, _, cout, _ = VGGISH_CONVS[0]
    out["conv1.w"] = sd[key + ".weight"].reshape(cout, 9).float().contiguous()
    out["conv1.b"] = sd[key + ".bias"].float().contiguous()
    def lay(w32, layer_idx):
        if (split_mask >> layer_idx) & 1:
            return split_hi_lo_tiles(w32.float().contiguous())
        return w32.to(torch.float16).contiguous()

    for i, (key, cin, cout, _) in enumerate(VGGISH_CONVS[1:], start=2):
        w = sd[key + ".weight"].permute(0, 2, 3, 1).reshape(cout, 9 * cin)
        out[f"conv{i}.w"] = lay(w, i - 2)
        out[f"conv{i}.b"] = sd[key + ".bias"].float().contiguous()
    for i, (key, fin, fout, _) in enumerate(VGGISH_FCS, start=1):
        out[f"fc{i}.w"] = lay(sd[key + ".weight"], 4 + i)
        out[f"fc{i}.b"] = sd[key + ".bias"].float().contiguous()
    out["split_mask"] = int(split_mask)
    return out


def state_fingerprint(sd: dict) -> str:
    import hashlib
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(np.ascontiguousarray(sd[k].numpy()).tobytes()[:4096])
    return h.hexdigest()[:16]
