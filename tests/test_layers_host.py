"""The per-layer sweep of the wav2vec family (fadtk_b200.layers, fad_batch.cache_tapped_embedding_files) without a GPU:
--layers parsing, the layer names against the registry, the directory flow with a stub tapped loader (one cache per
layer, only missing caches written, the batch bound), the statistics-file check before any embedding, and the CSV rows."""
import os
from pathlib import Path

import numpy as np
import pytest

import fadtk_b200 as fk
from fadtk_b200 import cli, fad_batch, layers, synth
from fadtk_b200.model_loader import ModelLoader, Wav2VecFamilyModel


# --------------------------------------------------------------------------------------------------- --layers
@pytest.mark.parametrize("spec,n,want", [
    ("all", 12, list(range(1, 13))), (None, 24, list(range(1, 25))), ("1-12", 12, list(range(1, 13))),
    ("3", 12, [3]), ("7,2,2,5", 12, [2, 5, 7]), ("1-3,10-12,2", 12, [1, 2, 3, 10, 11, 12]), (" 4 - 6 , 24", 24, [4, 5, 6, 24]),
    ([5, 1, 5], 12, [1, 5]), (range(1, 4), 12, [1, 2, 3])])
def test_parse_layers(spec, n, want):
    assert layers.parse_layers(spec, n) == want


@pytest.mark.parametrize("spec,n,message", [
    ("0", 12, "outside 1..12"), ("13", 12, "13 outside 1..12"), ("1-25", 24, "25 outside 1..24"), ("0-2", 12, "0 outside"),
    ("5-3", 12, "is empty"), ("x", 12, "expected 'all'"), ("", 12, "expected 'all'"), ("1-", 12, "expected 'all'"),
    ("1,,2", 12, "expected 'all'"), ([], 12, "no layer given"), ([0, 3], 12, "0 outside")])
def test_parse_layers_rejects(spec, n, message):
    with pytest.raises(ValueError, match=message):
        layers.parse_layers(spec, n)


def test_command_line_rejects_layers_and_models_with_a_message(capsys):
    with pytest.raises(SystemExit) as e:
        layers.main(["MERT-v1-95M", "base", "eval", "--layers", "0-12"])
    assert e.value.code == 2 and "0 outside 1..12" in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        layers.main(["vggish", "base", "eval"])
    assert e.value.code == 2 and "invalid choice: 'vggish'" in capsys.readouterr().err


@pytest.mark.parametrize("model", ["vggish", "MERT-v1-95M-3", "whisper-small", "clap-laion-audio", "nope"])
def test_api_refuses_a_non_w2v_model(model, tmp_path):
    with pytest.raises(ValueError, match="is not a wav2vec-family checkpoint"):
        fk.score_layers(model, tmp_path, tmp_path)
    with pytest.raises(ValueError, match="is not a wav2vec-family checkpoint"):
        fk.cache_layer_embeddings(tmp_path, model)


# ------------------------------------------------------------------------------------------------------- names
@pytest.mark.parametrize("model", list(layers.CHECKPOINTS))
def test_layer_names_are_the_registry_names(model):
    """For every checkpoint and every layer the sweep's names are the registry's, and each name's loader is that
    checkpoint at that layer."""
    ck = layers.checkpoint_loader(model)
    assert isinstance(ck, Wav2VecFamilyModel) and ck.layer == ck.arch["layers"] == layers.n_layers(model)
    registry = [m for m in fk.get_all_models() if isinstance(m, Wav2VecFamilyModel)
                and (m.family, m.size) == (ck.family, ck.size)]
    n = layers.n_layers(model)
    assert len(registry) == n
    assert layers.layer_names(model, range(1, n + 1)) == [m.name for m in sorted(registry, key=lambda m: m.layer)]
    assert layers.layer_names(model, [n]) == [model]


# ------------------------------------------------------------------------------------------------ directory flow
def _features(c, t):
    """[seconds, 4] fp16 rows of a clip at tap t: simple statistics that differ per tap"""
    return np.stack([[c[:16000 * (k + 1)].astype(np.float64).mean() + t, c.min(), c.max(), len(c) + 10 * t]
                     for k in range(max(1, len(c) // 16000))]).astype(np.float16)


class TapStub(ModelLoader):
    """A tapped loader in the shape of Wav2VecFamilyModel.embed_pcm_batch_flat_taps; records every call."""

    def __init__(self, layer=None):
        super().__init__("stub" if layer is None else f"stub-{layer}", 4, 16000)
        self.layer = layer
        self.calls = []

    def load_model(self):
        pass

    def _get_embedding(self, audio):
        raise NotImplementedError

    def embed_pcm_batch(self, clips):                        # the one-layer path: what embeds -m stub-<layer> writes
        return [_features(c, self.layer) for c in clips]

    def embed_pcm_batch_flat_taps(self, clips, taps):
        self.calls.append(([len(c) for c in clips], list(taps)))
        per = [[_features(c, t) for c in clips] for t in taps]
        return np.stack([np.concatenate(p) for p in per]), [len(e) for e in per[0]]


TAPS = [1, 3, 5]
NAMES = [f"stub-{t}" for t in TAPS]


def _directory(root: Path):
    rng = np.random.default_rng(11)
    clips = {f"c{i}.wav": rng.integers(-3000, 3000, size=16000 * (1 + i % 3) + 37 * i, dtype=np.int16) for i in range(7)}
    root.mkdir(parents=True, exist_ok=True)
    for name, pcm in clips.items():
        synth.write_wav(root / name, pcm, 16000)
    return clips


def _caches(root: Path):
    return {p.relative_to(root): p for p in sorted((root / "embeddings").rglob("*.npy"))}


def test_tapped_flow_writes_one_cache_per_layer_as_the_one_layer_flow_does(tmp_path):
    clips = _directory(tmp_path / "sweep")
    _directory(tmp_path / "single")
    ml = TapStub()
    fad_batch.cache_tapped_embedding_files(tmp_path / "sweep", ml, TAPS, NAMES, workers=3, load_model=False)
    assert sorted(sum((c[0] for c in ml.calls), [])) == sorted(len(c) for c in clips.values())     # each file once
    assert all(c[1] == TAPS for c in ml.calls)
    for t in TAPS:                                                  # the one-layer flow, one directory pass per name
        fad_batch.cache_embedding_files(tmp_path / "single", TapStub(t), workers=3, load_model=False)
    sweep, single = _caches(tmp_path / "sweep"), _caches(tmp_path / "single")
    assert sorted(sweep) == sorted(single) and len(sweep) == len(clips) * len(TAPS)
    for rel, p in sweep.items():
        assert p.read_bytes() == single[rel].read_bytes(), rel
    for t, name in zip(TAPS, NAMES):
        for f, pcm in clips.items():
            np.testing.assert_array_equal(np.load(tmp_path / "sweep" / "embeddings" / name / (Path(f).stem + ".npy")),
                                          _features(pcm, t))


def test_tapped_flow_writes_only_the_missing_caches(tmp_path):
    clips = _directory(tmp_path)
    ml = TapStub()
    fad_batch.cache_tapped_embedding_files(tmp_path, ml, TAPS, NAMES, workers=2, load_model=False)
    ml.calls.clear()
    fad_batch.cache_tapped_embedding_files(tmp_path, ml, TAPS, NAMES, workers=2, load_model=False)
    assert ml.calls == []                                           # everything cached: nothing embedded
    before = {rel: (p.read_bytes(), p.stat().st_mtime_ns) for rel, p in _caches(tmp_path).items()}
    old = 1_000_000_000 * 10 ** 9                                   # an mtime no write of this run can produce
    for p in _caches(tmp_path).values():
        os.utime(p, ns=(old, old))
    gone = [Path("embeddings") / "stub-3" / "c2.npy", Path("embeddings") / "stub-1" / "c2.npy",
            Path("embeddings") / "stub-5" / "c4.npy"]
    for rel in gone:
        (tmp_path / rel).unlink()
    fad_batch.cache_tapped_embedding_files(tmp_path, ml, TAPS, NAMES, workers=2, load_model=False)
    assert sorted(sum((c[0] for c in ml.calls), [])) == sorted(len(clips[f]) for f in ("c2.wav", "c4.wav"))
    after = _caches(tmp_path)
    assert sorted(after) == sorted(before)
    for rel, p in after.items():
        assert p.read_bytes() == before[rel][0], rel
        assert (p.stat().st_mtime_ns != old) == (rel in gone), rel


def test_tapped_flow_divides_the_batch_seconds_by_the_tap_count(tmp_path, monkeypatch):
    clips = _directory(tmp_path)
    monkeypatch.setattr(fad_batch, "_BATCH_AUDIO_SECONDS", 9.0)
    ml = TapStub()
    fad_batch.cache_tapped_embedding_files(tmp_path, ml, TAPS, NAMES, workers=2, load_model=False)
    secs = [sum(c[0]) / 16000 for c in ml.calls]
    assert all(s <= 3.0 or len(c[0]) == 1 for s, c in zip(secs, ml.calls)), secs   # 9 s / 3 taps, or a single file
    assert sum(len(c[0]) for c in ml.calls) == len(clips) and len(ml.calls) >= 4
    single = TapStub()
    fad_batch.cache_tapped_embedding_files(tmp_path, single, [2], ["stub-2"], workers=2, load_model=False)
    assert max(sum(c[0]) / 16000 for c in single.calls) > 3.0                # one tap: the whole 9-s budget


def test_tapped_flow_needs_one_name_per_tap(tmp_path):
    with pytest.raises(ValueError, match="one registry name per tap"):
        fad_batch.cache_tapped_embedding_files(tmp_path, TapStub(), [1, 2], ["a"])


# --------------------------------------------------------------------------------------------- statistics files
def test_npz_baseline_lacking_a_layer_fails_before_any_embedding(tmp_path, monkeypatch):
    calls = []
    monkeypatch.setattr(fad_batch, "cache_tapped_embedding_files", lambda *a, **k: calls.append(a))
    _directory(tmp_path / "eval")
    d = 768
    keys = {}
    for name in layers.layer_names("MERT-v1-95M", [1, 2, 4]):            # layer 3 missing
        keys[f"{name}.mu"], keys[f"{name}.cov"] = np.zeros(d), np.eye(d)
    keys["MERT-v1-95M-3.mu"] = np.zeros(d)                                 # mu without cov is not enough
    np.savez(tmp_path / "base.npz", **keys)
    with pytest.raises(ValueError, match="doesn't contain data for MERT-v1-95M-3$"):
        fk.score_layers("MERT-v1-95M", str(tmp_path / "base.npz"), str(tmp_path / "eval"), layers="1-4")
    with pytest.raises(ValueError, match="MERT-v1-95M-3, MERT-v1-95M$"):
        fk.score_layers("MERT-v1-95M", tmp_path / "base.npz", tmp_path / "eval", layers=[1, 3, 12])
    assert calls == [] and not (tmp_path / "eval" / "embeddings").exists()


def test_named_baseline_is_checked_too(tmp_path, monkeypatch):
    calls = []
    monkeypatch.setattr(fad_batch, "cache_tapped_embedding_files", lambda *a, **k: calls.append(a))
    monkeypatch.setenv("FADTK_STATS_DIR", str(tmp_path))
    np.savez(tmp_path / "mini_pop.npz", **{"hubert-base-2.mu": np.zeros(768), "hubert-base-2.cov": np.eye(768)})
    _directory(tmp_path / "eval")
    with pytest.raises(ValueError, match="doesn't contain data for hubert-base-1$"):
        fk.score_layers("hubert-base", "mini_pop", str(tmp_path / "eval"), layers="1,2")
    assert calls == []


# ---------------------------------------------------------------------------------------------------- output
def test_command_line_table_and_csv_rows(tmp_path, monkeypatch, capsys):
    got = {}

    def fake(model, baseline, eval, layers_, workers):
        got.update(model=model, baseline=baseline, eval=eval, layers=layers_, workers=workers)
        return [(n, 0.5 + k) for k, n in enumerate(layers.layer_names(model, layers.parse_layers(layers_, 24)))]
    monkeypatch.setattr(layers, "score_layers", fake)
    csv = tmp_path / "out" / "fad.csv"
    assert layers.main(["hubert-large", "fma_pop", "ev dir", str(csv), "--layers", "24,2-3", "-w", "3"]) == 0
    assert got == dict(model="hubert-large", baseline="fma_pop", eval="ev dir", layers="24,2-3", workers=3)
    out = capsys.readouterr().out.splitlines()
    assert out[0].split() == ["layer", "model", "FAD"]
    assert [ln.split() for ln in out[1:]] == [["2", "hubert-large-2", "0.5"], ["3", "hubert-large-3", "1.5"],
                                              ["24", "hubert-large", "2.5"]]
    lines = csv.read_text().splitlines(keepends=True)
    assert lines[0] == cli.CSV_HEADER
    rows = [ln.rstrip("\n").split(",") for ln in lines[1:]]
    assert [r[:5] for r in rows] == [["hubert-large-2", "fma_pop", "ev dir", "0.5", "None"],
                                     ["hubert-large-3", "fma_pop", "ev dir", "1.5", "None"],
                                     ["hubert-large", "fma_pop", "ev dir", "2.5", "None"]]
    assert all(float(r[5]) > 0 for r in rows)
    # a second run appends under the same header, as a shell loop over `python -m fadtk_b200 <name>` would
    layers.main(["hubert-large", "fma_pop", "ev dir", str(csv), "--layers", "2"])
    assert csv.read_text().count(cli.CSV_HEADER) == 1 and len(csv.read_text().splitlines()) == 5
