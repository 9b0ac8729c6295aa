"""How much of the w2v2-base FAD parity error is the attention kernel and how much is chance: FAD(gpu) vs FAD(cpu oracle) for
several independent 8 + 8 clip sets (4 s clips).  One JSON line."""
import json
import os
import sys
from pathlib import Path

os.environ.setdefault("FADTK_SYNTHETIC", "1")
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
import fadtk_b200 as fk  # noqa: E402
from fadtk_b200 import synth, weights_w2v as ww  # noqa: E402
from oracle import fad_oracle as fo, w2v_oracle as wo  # noqa: E402

ml = fk.W2V2Model('base', 12, max_clips=8)
ml.load_model()
sd = ww.synthetic_w2v_state(0)
model, fe = wo.build(sd, "w2v2")
out = []
for seed in range(int(sys.argv[1]) if len(sys.argv) > 1 else 4):
    sets = {"base": [synth.noise_clip(100 * seed + i, 4.0, 16000) for i in range(8)],
            "eval": [synth.musiclike_clip(100 * seed + i, 4.0, 16000) for i in range(8)]}
    gpu = {k: np.concatenate(ml.embed_pcm_batch(v)) for k, v in sets.items()}
    cpu = {k: np.concatenate([wo.embed(c / 32768.0, model, fe, 12) for c in v]) for k, v in sets.items()}
    fg = fk.calc_frechet_distance(*fk.calc_embd_statistics(gpu["base"]), *fk.calc_embd_statistics(gpu["eval"]))
    fc = fo.frechet_distance(*fo.embd_statistics(cpu["base"]), *fo.embd_statistics(cpu["eval"]))
    out.append({"seed": seed, "fad_gpu": float(fg), "fad_cpu": float(fc), "rel": float((fg - fc) / fc)})
print(json.dumps({"sets": out}))
