"""The per-layer sweep's forward against one forward per layer: full-depth synthetic w2v2-base (12 layers, post-LN) and
hubert-large (24 layers, pre-LN) weights on 8 clips of 10 s.  Timed with CUDA events after a warm-up, alternating
the two, median of the repeats:
  * taps: ONE fad_w2v_forward_taps call writing layers 1..layers (the registry's range), and
  * per-layer: the sum of the fad_w2v_forward calls that stop at layer 1, 2, .., layers (what one directory pass per
    registry name runs on the GPU).
Both must produce bitwise equal outputs.  Time only.  The first line is the card and its power limit, read in the same
run; then one JSON line per model."""
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402
from fadtk_b200 import _native, synth, weights_w2v as ww  # noqa: E402

CLIPS, SECONDS, SR, REPEATS = 8, 10.0, 16000, 5


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
    eng = _native.engine()
    print(json.dumps({"gpu": smi("name"), "power_limit_w": smi("power.limit"), "max_sm_clock_mhz": smi("clocks.max.sm")}),
          flush=True)
    n = int(SECONDS * SR)
    pcm = torch.stack([torch.from_numpy(synth.musiclike_clip(i, SECONDS, SR)[:n]) for i in range(CLIPS)]).cuda()
    for name, arch in (("w2v2-base", ("w2v2", "base")), ("hubert-large", ("hubert", "large"))):
        sd = ww.synthetic_w2v_state(0, **ww.ARCH[arch])
        eng.w2v_load(ww.config_of(sd), ww.pack_w2v(sd), CLIPS, max_len=n)
        del sd
        layers = int(ww.ARCH[arch]["layers"])
        taps = list(range(1, layers + 1))
        per_layer = lambda: [eng.w2v_forward(pcm, k) for k in taps]          # noqa: E731
        tapped = lambda: eng.w2v_forward_taps(pcm, taps)                     # noqa: E731
        per_layer(), tapped()                                                # warm-up: workspaces, modules, bias tables
        torch.cuda.synchronize()
        t_taps, t_layers = [], []
        for _ in range(REPEATS):
            one, t = timed(per_layer)
            t_layers.append(t)
            del one
            out, t = timed(tapped)
            t_taps.append(t)
        # the check: a NaN-filled output (no stale values of an earlier call can pass) against fresh per-layer outputs
        out.fill_(float("nan"))
        eng.w2v_forward_taps(pcm, taps, out=out)
        one = per_layer()
        equal = all(torch.equal(out[t].view(torch.int16), one[t].view(torch.int16)) for t in range(layers))
        med = lambda v: sorted(v)[len(v) // 2]                               # noqa: E731
        print(json.dumps({"model": name, "layers": layers, "clips": CLIPS, "seconds": SECONDS, "frames": int(out.shape[2]),
                          "taps_ms": round(med(t_taps), 2), "per_layer_sum_ms": round(med(t_layers), 2),
                          "ratio": round(med(t_layers) / med(t_taps), 2), "taps_ms_all": [round(t, 2) for t in t_taps],
                          "per_layer_sum_ms_all": [round(t, 2) for t in t_layers], "bitwise_equal": equal}), flush=True)
        del out, one
        if not equal:
            raise SystemExit(f"{name}: the tapped forward differs from the per-layer forward")


if __name__ == "__main__":
    main()
