"""Several layers of one wav2vec-family forward (fad_w2v_forward_taps) and the per-layer sweep built on it
(fadtk_b200.layers).

  * Every slice of a tapped call is bitwise what fad_w2v_forward writes for that layer alone, for the five
    architectures of test_gpu_w2v_stages.MODELS on a 3-layer stack, at the shortest clip, either side of a frame
    boundary, 10 s and 30 s, with n_clips = max_clips + 1 so that every call crosses a chunk boundary.  The accuracy of
    fad_w2v_forward against float64 is test_gpu_w2v_stages.test_forward_taps_match_fp64's.
  * Rejected calls launch nothing and write nothing.
  * End to end at full depth (MERT-v1-95M: 12 layers, hubert-large: 24, pre-LN) on directories of mixed-length WAVs:
    the sweep's caches are byte-identical to one `embeds -m <name>` pass per layer, its FADs equal
    `python -m fadtk_b200 <name>`'s exactly, and a rerun after some caches were deleted writes exactly those.
"""
import os
import shutil

import numpy as np
import pytest
import torch

from fadtk_b200 import _native, cli, layers, synth, weights_w2v as ww
from gpu_checks import Guarded, expect_rejected, on_fresh_engine
from test_gpu_w2v_stages import MODELS

GUARD = 4096
MAX_CLIPS = 2
N_LAYERS = 3
TAP_SETS = [[0, 1, 2, 3], [1, 3], [2], [3]]


def load(engine, name, max_len, max_clips=MAX_CLIPS):
    token = ("w2v-layers-test", name, N_LAYERS, max_len, max_clips)
    if engine.owners.get("w2v") != token:
        arch = dict(ww.ARCH[MODELS[name][0]])
        arch["layers"] = N_LAYERS
        sd = ww.synthetic_w2v_state(0, **arch)
        engine.w2v_load(ww.config_of(sd), ww.pack_w2v(sd), max_clips, max_len=max_len)
        engine.owners["w2v"] = token


def clips_of(L, sr):
    """max_clips + 1 different clips of L samples"""
    sec = L / sr
    return [synth.musiclike_clip(1, sec, sr)[:L], synth.noise_clip(L + 1, sec, sr)[:L],
            np.round(12000 * np.sin(2 * np.pi * 55.0 * np.arange(L) / sr)).astype(np.int16)]


CASES = [(n, L) for n in MODELS for L in ((400, 719, 720, 160000, 480000) if MODELS[n][2] == 16000
                                          else (400, 1079, 1080, 240000, 720000))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,L", CASES, ids=[f"{n}-{L}" for n, L in CASES])
def test_taps_are_bitwise_the_one_tap_forward(engine, name, L):
    sr = MODELS[name][2]
    load(engine, name, max(L, 720000))
    pcm = torch.from_numpy(np.stack([np.resize(c, L) for c in clips_of(L, sr)])).cuda()
    n = pcm.shape[0]
    assert n == MAX_CLIPS + 1
    one = [engine.w2v_forward(pcm, k) for k in range(N_LAYERS + 1)]
    S, d = one[0].shape[1:]
    for taps in TAP_SETS:
        out = Guarded((len(taps), n, S, d), torch.float16, "cuda", GUARD)
        got = engine.w2v_forward_taps(pcm, taps, out=out.body)
        assert got.data_ptr() == out.body.data_ptr()
        out.check()
        for t, k in enumerate(taps):
            assert torch.equal(out.body[t].view(torch.int16), one[k].view(torch.int16)), f"taps {taps}: slice {t} (layer {k})"
    again = engine.w2v_forward_taps(pcm, TAP_SETS[0])
    assert torch.equal(again.view(torch.int16), torch.stack(one).view(torch.int16))


# ---------------------------------------------------------------------------------------------------- rejections
MAX_LEN = 32000


def _taps_call(taps=(1, 3), L=16000, out="ok", n=3):
    def call(engine, outs):
        pcm = torch.zeros((n, max(L, 1)), dtype=torch.int16, device="cuda")
        o = Guarded((4, 3, 49, 768), torch.float16, "cuda", GUARD)
        outs.append(o)
        engine.w2v_forward_taps(pcm, list(taps), out=o.ptr(out))
    return call


def _raw_call(handle="ok", pcm="ok", taps="ok", out="ok", n=3):
    """straight through the C ABI: the arguments the Python wrapper never passes"""
    def call(engine, outs):
        import ctypes as C
        x = torch.zeros((3, 16000), dtype=torch.int16, device="cuda")
        o = Guarded((2, 3, 49, 768), torch.float16, "cuda", GUARD)
        outs.append(o)
        arr = (C.c_int * 2)(1, 3)
        _native._check(_native.lib().fad_w2v_forward_taps(
            engine._h if handle == "ok" else None, x.data_ptr() if pcm == "ok" else None, n, 16000,
            arr if taps == "ok" else None, 2, o.body.data_ptr() if out == "ok" else None, _native._stream()))
    return call


M = "fad_w2v_forward_taps: "
REJECT = [
    ("null handle", _raw_call(handle=None), M + "fad_w2v_load has not been called"),
    ("before any load", on_fresh_engine(_taps_call()), M + "fad_w2v_load has not been called"),
    ("null pcm", _raw_call(pcm=None), M + "null pcm, taps or out"),
    ("null taps", _raw_call(taps=None), M + "null pcm, taps or out"),
    ("null out", _raw_call(out=None), M + "null pcm, taps or out"),
    ("no clips", _raw_call(n=0), M + "n_clips must be positive"),
    ("no taps", _taps_call(taps=()), M + "n_taps must be in [1, layers + 1]"),
    ("too many taps", _taps_call(taps=(0, 1, 2, 3, 4)), M + "n_taps must be in [1, layers + 1]"),
    ("taps decreasing", _taps_call(taps=(3, 1)), M + "taps must be strictly increasing in [0, layers]"),
    ("taps repeated", _taps_call(taps=(1, 1)), M + "taps must be strictly increasing in [0, layers]"),
    ("tap beyond layers", _taps_call(taps=(1, 4)), M + "taps must be strictly increasing in [0, layers]"),
    ("tap negative", _taps_call(taps=(-1, 2)), M + "taps must be strictly increasing in [0, layers]"),
    ("misaligned out", _taps_call(out="odd"), M + "out must be 16-byte aligned"),
    ("L beyond max_len", _taps_call(L=MAX_LEN + 1), M + "L must be at most max_len"),
    ("L 399", _taps_call(L=399), M + "L must be at least 400 samples"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("call,message", [c[1:] for c in REJECT], ids=[c[0] for c in REJECT])
def test_forward_taps_rejects_invalid_arguments(engine, call, message):
    load(engine, "w2v2-base", MAX_LEN)
    expect_rejected(engine, call, message, [])


# ------------------------------------------------------------------------------------------- end to end, full depth
def _write_dirs(root, sr):
    """baseline and eval directories of mixed-length WAVs at the model rate; the eval set has one 31-s file (the
    loader's one-clip reload)"""
    for kind, secs in (("base", (4.0, 5.5, 5.5, 7.25, 3.0)), ("eval", (2.5, 6.0, 6.0, 4.75, 31.0))):
        (root / kind).mkdir(parents=True)
        for i, s in enumerate(secs):
            clip = synth.musiclike_clip(10 * i + len(kind), s, sr, baseline=(kind == "base"))
            synth.write_wav(root / kind / f"f{i}.wav", clip, sr)


def _npy(root):
    return {str(p.relative_to(root)): p for p in sorted(root.rglob("embeddings/*/*.npy"))}


def _scores(csv):
    return {r.split(",")[0]: r.split(",")[3] for r in csv.read_text().splitlines()[1:]}


@pytest.fixture
def cached_weights(monkeypatch):
    """The seeded synthetic weights generated and packed once per architecture: the one-layer reference below loads
    the same checkpoint once per registry name."""
    load_state, pack = ww.load_w2v_state, ww.pack_w2v
    states, packs = {}, {}

    def load_cached(path=None, seed=0, env="FADTK_W2V_CKPT", **cfg):
        key = (path, seed, env, tuple(sorted(cfg.items())))
        if key not in states:
            states[key] = load_state(path, seed, env, **cfg)
        return states[key]

    def pack_cached(sd):
        if id(sd) not in packs:
            packs[id(sd)] = (sd, pack(sd))
        return packs[id(sd)][1]
    monkeypatch.setattr(ww, "load_w2v_state", load_cached)
    monkeypatch.setattr(ww, "pack_w2v", pack_cached)


@pytest.mark.gpu
@pytest.mark.parametrize("model,sr", [("MERT-v1-95M", 24000), ("hubert-large", 16000)])
def test_sweep_equals_one_run_per_layer(model, sr, tmp_path, cached_weights, capsys):
    assert os.environ.get("FADTK_SYNTHETIC") == "1"
    n = layers.n_layers(model)
    names = layers.layer_names(model, range(1, n + 1))
    _write_dirs(tmp_path / "sweep", sr)
    shutil.copytree(tmp_path / "sweep", tmp_path / "single")
    base, ev = tmp_path / "sweep" / "base", tmp_path / "sweep" / "eval"
    assert layers.main([model, str(base), str(ev), str(tmp_path / "sweep.csv"), "-w", "4"]) == 0
    sb, se = tmp_path / "single" / "base", tmp_path / "single" / "eval"
    assert cli.embeds_main(["-m", *names, "-d", str(sb), str(se), "-w", "4"]) == 0
    for name in names:
        assert cli.score_main([name, str(sb), str(se), str(tmp_path / "single.csv"), "-w", "4"]) == 0
    a, b = _npy(tmp_path / "sweep"), _npy(tmp_path / "single")
    assert sorted(a) == sorted(b) and len(a) == 10 * n
    for rel in a:
        assert a[rel].read_bytes() == b[rel].read_bytes(), rel
    fad_sweep, fad_single = _scores(tmp_path / "sweep.csv"), _scores(tmp_path / "single.csv")
    assert list(fad_sweep) == names and fad_sweep == fad_single
    with capsys.disabled():
        print(f"\n[w2v layers] {model}: " + ", ".join(f"{k}: {fad_sweep[k]}" for k in names[:3]) + ", ...", flush=True)

    # a rerun after some caches of some layers are deleted writes exactly those
    gone = [f"base/embeddings/{names[0]}/f1.npy", f"eval/embeddings/{names[n // 2]}/f4.npy",
            f"eval/embeddings/{names[n // 2]}/f0.npy", f"base/embeddings/{names[-1]}/f3.npy"]
    for rel in gone:
        (tmp_path / "sweep" / rel).unlink()
    mtimes = {rel: p.stat().st_mtime_ns for rel, p in _npy(tmp_path / "sweep").items()}
    assert layers.main([model, str(base), str(ev), str(tmp_path / "rerun.csv"), "-w", "4"]) == 0
    after = _npy(tmp_path / "sweep")
    assert sorted(after) == sorted(b)
    for rel, p in after.items():
        assert p.read_bytes() == b[rel].read_bytes(), rel
        if rel not in gone:
            assert p.stat().st_mtime_ns == mtimes[rel], f"{rel} was rewritten"
    assert _scores(tmp_path / "rerun.csv") == fad_single
