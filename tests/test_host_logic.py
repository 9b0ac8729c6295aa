"""CPU tests: plugin surface, cache paths, planning, ABI export list, sharding + the 2-rank
gloo exchange of packed statistics.  No GPU compute is called here."""
import ctypes
import os
import pickle
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native, dist, synth, weights
from oracle import vggish_oracle as vo

ROOT = Path(__file__).resolve().parent.parent


def test_export_surface_matches_reference_init():
    # fadtk/__init__.py:1-4 star-exports fad, fad_batch, model_loader, utils
    for name in ["FrechetAudioDistance", "FADInfResults", "calc_embd_statistics", "calc_frechet_distance",
                 "cache_embedding_files", "ModelLoader", "VGGishModel", "get_all_models",
                 "calculate_embd_statistics_online", "get_cache_embedding_path", "find_sox_formats"]:
        assert hasattr(fk, name), name


def test_registry_names_match_reference():
    models = fk.get_all_models()
    names = [m.name for m in models]
    assert len(names) == len(set(names)) == 143                       # SURVEY.md section 3.1
    for must in ["vggish", "clap-laion-audio", "clap-laion-music", "clap-2023", "encodec-emb", "encodec-emb-48k",
                 "MERT-v1-95M", "MERT-v1-95M-1", "MERT-v1-95M-11", "w2v2-base", "w2v2-base-1", "w2v2-large",
                 "w2v2-large-23", "hubert-base", "hubert-large-5", "wavlm-base-plus", "wavlm-large",
                 "whisper-tiny", "whisper-small", "whisper-large"]:
        assert must in names, must
    vgg = dict(zip(names, models))["vggish"]
    assert (vgg.num_features, vgg.sr, vgg.min_len) == (128, 16000, 1)   # model_loader.py:94
    # instances travel to worker processes before load_model (fad_batch.py:48)
    clone = pickle.loads(pickle.dumps(vgg))
    assert clone.name == "vggish" and clone.model is None


def test_cache_path_scheme():
    p = fk.get_cache_embedding_path("vggish", "/data/set/clip 01.flac")
    assert p == Path("/data/set/embeddings/vggish/clip 01.npy")       # utils.py:60-68


def test_load_wav_and_min_len(tmp_path):
    pcm = synth.sine_clip(3, 0.4, 16000)
    synth.write_wav(tmp_path / "a.wav", pcm, 16000)
    ml = fk.VGGishModel()
    wav = ml.load_wav(tmp_path / "a.wav")
    assert wav.dtype == np.float64 and wav.shape[0] == 16000          # zero-padded to min_len = 1 s
    assert np.array_equal(wav[:pcm.shape[0]], pcm / 32768.0)
    assert np.all(wav[pcm.shape[0]:] == 0)
    assert np.array_equal(vo.load_wav_semantics(pcm), wav)            # oracle agrees


def test_synthetic_audio_is_deterministic_pcm16():
    a, b = synth.musiclike_clip(7, 1.0, 16000), synth.musiclike_clip(7, 1.0, 16000)
    assert a.dtype == np.int16 and np.array_equal(a, b)
    assert not np.array_equal(a, synth.musiclike_clip(7, 1.0, 16000, baseline=True))
    s = synth.sine_clip(12, 1.0, 16000)                               # 220 Hz, amplitude 0.5
    assert abs(int(s.max()) - 16384) <= 1


def test_library_exports_every_declared_symbol():
    header = (ROOT / "include" / "fadtk_b200.h").read_text()
    declared = set(re.findall(r"\b(fad_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_native.SIGNATURES), declared ^ set(_native.SIGNATURES)
    lib = ctypes.CDLL(str(_native.library_path()))
    for name in declared:
        assert hasattr(lib, name), name
    assert _native.lib().fad_version() == 1


def test_plan_counts_match_oracle_formula():
    lens = [0, 399, 400, 15599, 15600, 15759, 16000, 30960, 160000, 160001, 480000]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ex, rows = _native.Engine.vggish_plan(off)
    assert list(rows) == [vo.num_examples(n) for n in lens]
    assert ex.shape[0] == rows.sum()
    starts = np.concatenate([off[i] + 96 * 160 * np.arange(r) for i, r in enumerate(rows)])
    assert np.array_equal(ex, starts)


def test_weight_packing_layout():
    sd = weights.synthetic_vggish_state(3)
    pk = weights.pack_vggish(sd, split_mask=0)
    w = sd["features.3.weight"]                                        # [128, 64, 3, 3]
    assert pk["conv2.w"].shape == (128, 9 * 64) and pk["conv2.w"].dtype == torch.float16
    assert pk["conv2.w"][5, (1 * 3 + 2) * 64 + 7] == w[5, 7, 1, 2].to(torch.float16)
    assert pk["fc1.w"].shape == (4096, 12288) and pk["conv1.w"].shape == (64, 9)
    # default: every tensor-core layer carries hi/lo weights, 128 hi rows then 128 lo rows per tile
    ps = weights.pack_vggish(sd)
    assert ps["split_mask"] == 0xFF and ps["fc2.w"].shape == (2 * 4096, 4096)
    w2 = sd["embeddings.2.weight"]
    hi, lo = ps["fc2.w"][256 + 3].float(), ps["fc2.w"][256 + 128 + 3].float()   # row 131 of the layer
    assert torch.equal(hi, w2[131].to(torch.float16).float())
    assert (hi + lo - w2[131]).abs().max() <= 2.0 ** -21 * w2[131].abs().max()
    assert weights.state_fingerprint(sd) == weights.state_fingerprint(weights.synthetic_vggish_state(3))


def test_no_cpu_fallback_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_native.NativeError):
        _native.Engine()
    with pytest.raises(Exception):
        fk.calc_frechet_distance(np.zeros(4), np.eye(4), np.zeros(4), np.eye(4))


def test_shard_is_array_split():
    files = list(range(10))
    parts = [dist.shard(files, r, 4) for r in range(4)]
    assert parts == [list(x) for x in np.array_split(files, 4)]       # fad_batch.py:43


def test_cli_parsers_accept_reference_arguments():
    out = subprocess.run([sys.executable, "-m", "fadtk_b200", "--help"], cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0
    for flag in ["--inf", "--indiv", "--workers", "--sox-path", "baseline", "eval", "csv"]:
        assert flag in out.stdout
    out = subprocess.run([sys.executable, "-m", "fadtk_b200.embeds", "--help"], cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and "--models" in out.stdout and "--dirs" in out.stdout


_WORKER = r"""
import os, sys, numpy as np, torch
sys.path.insert(0, sys.argv[1])
from fadtk_b200 import dist
from fadtk_b200.utils import pack_statistics_numpy, finalize_packed_numpy
dist.init_from_env("gloo")
r, w = dist.rank(), dist.world_size()
rng = np.random.default_rng(0)
rows = (rng.normal(1.0, 2.0, (1001, 16))).astype(np.float16)
shift = rows[:64].astype(np.float32).mean(0).astype(np.float16)
mine = dist.shard(list(range(rows.shape[0])), r, w)
acc = torch.from_numpy(pack_statistics_numpy(rows[mine], shift))
dist.allreduce_sum_(acc)
mu, cov = finalize_packed_numpy(acc.numpy(), shift)
x = rows.astype(np.float64)
assert acc[0].item() == rows.shape[0]
assert np.allclose(mu, x.mean(0), rtol=0, atol=1e-12), np.abs(mu - x.mean(0)).max()
ref = np.cov(x, rowvar=False)
assert np.abs(cov - ref).max() < 1e-4 * np.abs(ref).max(), np.abs(cov - ref).max()   # y = fp16(x - shift)
assert dist.max_over_ranks(float(r)) == w - 1
sys.stdout.write(f"[rank{r}:ok]\n"); sys.stdout.flush()
"""


def test_two_rank_statistics_allreduce_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    env = dict(os.environ, OMP_NUM_THREADS="1")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", "29531", str(script), str(ROOT)],
                         capture_output=True, text=True, env=env, timeout=300)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert "rank0:ok" in out.stdout and "rank1:ok" in out.stdout, out.stdout


def test_registry_matches_the_reference(golden_dir):
    """get_all_models(): same names, order, dimensionality and sample rate as the reference's registry
    (fadtk/model_loader.py:676-701; golden list generated from the real package by oracle/make_golden.py)."""
    import json
    want = json.loads((golden_dir / "registry.json").read_text())
    got = [[m.name, int(m.num_features), int(m.sr)] for m in fk.get_all_models()]
    assert got == want
    unbuilt = [m.name for m in fk.get_all_models() if isinstance(m, fk.UnbuiltModel)]
    assert unbuilt == ["clap-2023"]                       # every other embedder has an sm_90a forward pass


def test_stats_cache_is_invalidated_when_embeddings_change(tmp_path, monkeypatch):
    """SURVEY.md section 8 (f)3: the reference reuses stats/<model>/{mu,cov}.npy forever (fad.py:279-283);
    caches written here are recomputed when the embedding files they came from change, while a cache
    without a fingerprint (written by the reference) is still loaded as is."""
    import numpy as np
    from fadtk_b200 import fad as fad_mod

    def cpu_stats(files):
        e = np.concatenate([np.load(f) for f in files]).astype(np.float64)
        return e.mean(0), np.cov(e, rowvar=False)

    monkeypatch.setattr(fad_mod, "calculate_embd_statistics_online", cpu_stats)

    class _ML:
        name = "vggish"

    f = fad_mod.FrechetAudioDistance.__new__(fad_mod.FrechetAudioDistance)
    f.ml = _ML()
    emb = tmp_path / "embeddings" / "vggish"
    emb.mkdir(parents=True)
    rng = np.random.default_rng(0)
    np.save(emb / "a.npy", rng.standard_normal((8, 4)).astype(np.float16))
    np.save(emb / "b.npy", rng.standard_normal((8, 4)).astype(np.float16))
    mu1, cov1 = f.load_stats(tmp_path)
    assert (tmp_path / "stats" / "vggish" / "source.json").exists()
    mu1b, _ = f.load_stats(tmp_path)                        # unchanged directory: served from the cache
    np.testing.assert_array_equal(mu1, mu1b)

    np.save(emb / "c.npy", (5 + rng.standard_normal((8, 4))).astype(np.float16))
    mu2, cov2 = f.load_stats(tmp_path)                      # a new file: recomputed
    assert not np.allclose(mu1, mu2)
    np.testing.assert_allclose(mu2, cpu_stats(sorted(emb.glob("*.npy")))[0])

    (tmp_path / "stats" / "vggish" / "source.json").unlink()   # a reference-written cache has no fingerprint
    np.save(emb / "d.npy", (9 + rng.standard_normal((8, 4))).astype(np.float16))
    mu3, _ = f.load_stats(tmp_path)
    np.testing.assert_array_equal(mu2, mu3)                 # trusted like the reference does


def test_bench_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (the CPU oracle timed on the host cores) needs no GPU: one JSON line with the
    driver's keys, cpu_baseline describing the run and e2e repeating the value."""
    import json
    import subprocess
    import sys
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
                "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert key in line, key
    assert line["impl"] == "reference" and line["value"] > 0 and line["unit"] == "audio-s/s"
    assert line["e2e"]["value"] == line["value"] and line["e2e"]["h2d_bytes_per_step"] == 0
    assert line["cpu_baseline"]["kind"] in ("port", "reference") and line["cpu_baseline"]["cores"] >= 1
    assert "workload" in line["config"]


def test_acceptance_harness_comparison_rule(tmp_path):
    """python -m fadtk_b200.test mirrors fadtk/test/__main__.py: per model, max |ours - published| must stay below
    5 % of the mean of our scores; song ids are 'samples/<stem>' whatever the path style."""
    sys.path.insert(0, str(ROOT))
    import importlib
    t = importlib.import_module("fadtk_b200.test.__main__")
    table = tmp_path / "scores.csv"
    table.write_text("song_id,dataset,FAD_vggish_fma_pop,FAD_clap_laion_audio_fma_pop\n"
                     "samples/all,all,5.0,0.4\nsamples/mg-1,mg,20.0,1.6\nsamples/mg-2,mg,10.0,\n")
    ref = t.reference_scores(table)
    assert ref["vggish"] == {"samples/all": 5.0, "samples/mg-1": 20.0, "samples/mg-2": 10.0}
    assert ref["clap_laion_audio"] == {"samples/all": 0.4, "samples/mg-1": 1.6}
    assert t.song_id(r"C:\data\samples\mg-1.opus") == "samples/mg-1" and t.song_id("/x/samples/all") == "samples/all"
    ok = t.compare({"samples/all": 5.1, "samples/mg-1": 20.4, "samples/mg-2": 9.9}, ref["vggish"])
    assert ok["pass"] and abs(ok["max_abs_diff"] - 0.4) < 1e-12 and abs(ok["mad%"] - 0.4 / (35.4 / 3) * 100) < 1e-9
    bad = t.compare({"samples/all": 5.0, "samples/mg-1": 21.0}, ref["vggish"])
    assert not bad["pass"]                                      # 1.0 / 13.0 = 7.7 %


def test_packaged_statistics_resolve_as_a_named_baseline(tmp_path, monkeypatch):
    """python -m fadtk_b200.package writes '<model>.mu' / '<model>.cov' keys (fadtk/package.py:33-42); the file is
    accepted by load_stats as a path and, from $FADTK_STATS_DIR, as a baseline name (fad.py:249-266)."""
    import numpy as np
    from fadtk_b200 import fad as fad_mod, package

    class _ML:
        def __init__(self, name):
            self.name, self.model = name, None

    rng = np.random.default_rng(3)
    data = tmp_path / "set"
    want = {}
    for name, d in (("vggish", 4), ("clap-laion-audio", 6)):   # statistics already cached: no embedding pass needed
        s = data / "stats" / name
        s.mkdir(parents=True)
        a = rng.standard_normal((d, d))
        want[name] = (rng.standard_normal(d), a @ a.T)
        np.save(s / "mu.npy", want[name][0])
        np.save(s / "cov.npy", want[name][1])
    out = package.pack_statistics(data, tmp_path / "stats_dir" / "my_set.npz", [_ML("vggish"), _ML("clap-laion-audio")])
    with np.load(out) as z:
        assert sorted(z.files) == ["clap-laion-audio.cov", "clap-laion-audio.mu", "vggish.cov", "vggish.mu"]
    f = fad_mod.FrechetAudioDistance.__new__(fad_mod.FrechetAudioDistance)
    f.ml = _ML("clap-laion-audio")
    mu, cov = f.load_stats(out)                                 # as a file
    np.testing.assert_array_equal(mu, want["clap-laion-audio"][0])
    monkeypatch.setenv("FADTK_STATS_DIR", str(out.parent))
    mu, cov = f.load_stats("My_Set")                            # as a (case-insensitive) name
    np.testing.assert_array_equal(cov, want["clap-laion-audio"][1])
    f.ml = _ML("encodec-emb")
    with pytest.raises(ValueError):
        f.load_stats(out)                                       # fad.py:265: the file lacks that model


def test_score_command_line_appends_the_reference_csv_row(tmp_path, monkeypatch, capsys):
    """cli.score_main with statistics files on both sides (no embedding, Frechet swapped for the CPU oracle):
    the result row and header are the reference's (fadtk/__main__.py:62-68), a second run appends."""
    import numpy as np
    from fadtk_b200 import cli, fad as fad_mod
    from oracle import fad_oracle as fo

    class _ML:
        name, model, sr = "vggish", None, 16000

    monkeypatch.setattr(cli, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(fad_mod, "calc_frechet_distance", fo.frechet_distance)
    rng = np.random.default_rng(0)
    for name in ("base", "eval"):
        x = rng.standard_normal((200, 8)) * (1.0 if name == "base" else 1.3)
        np.savez(tmp_path / f"{name}.npz", **{"vggish.mu": x.mean(0), "vggish.cov": np.cov(x, rowvar=False)})
    out = tmp_path / "results" / "scores.csv"
    argv = ["vggish", str(tmp_path / "base.npz"), str(tmp_path / "eval.npz"), str(out), "-w", "2"]
    assert cli.score_main(argv) == 0
    assert cli.score_main(argv) == 0
    lines = out.read_text().splitlines()
    assert lines[0] == "model,baseline,eval,score,inf_r2,time" and len(lines) == 3
    model, base, ev, score, r2, stamp = lines[1].split(",")
    with np.load(tmp_path / "base.npz") as b, np.load(tmp_path / "eval.npz") as e:
        want = fo.frechet_distance(b["vggish.mu"], b["vggish.cov"], e["vggish.mu"], e["vggish.cov"])
    assert (model, base, ev, r2) == ("vggish", str(tmp_path / "base.npz"), str(tmp_path / "eval.npz"), "None")
    assert abs(float(score) - want) < 1e-9 * abs(want) and float(stamp) > 1.6e9
    with pytest.raises(SystemExit):                             # unknown model: argparse rejects it like the reference's choices=
        cli.score_main(["no-such-model", "a", "b"])


def test_inf_wins_over_indiv_and_package_default_skips_unbuilt_models(tmp_path, monkeypatch, capsys):
    """Both flags given: the reference runs FAD-inf (fadtk/__main__.py:45-50, `if args.inf ... elif args.indiv`).
    `python -m fadtk_b200.package dir out.npz` with no -m walks the registry; entries without a forward pass
    (clap-2023) are skipped with a note instead of aborting the whole run."""
    import types
    from fadtk_b200 import cli, fad as fad_mod, package
    from fadtk_b200.model_loader import UnbuiltModel

    class _ML:
        name, model, sr = "vggish", None, 16000

    calls = []

    class _FAD:
        def __init__(self, ml, **kw): pass
        def score_inf(self, baseline, files):
            calls.append(("inf", baseline, len(files)))
            return types.SimpleNamespace(score=1.5, r2=0.9, slope=0.0, points=[])
        def score_individual(self, baseline, ev, csv):
            calls.append(("indiv", baseline))
        def score(self, baseline, ev):
            calls.append(("score", baseline))
            return 2.5

    monkeypatch.setattr(cli, "_registry", lambda: {"vggish": _ML()})
    monkeypatch.setattr(cli, "_embed_directories", lambda *a, **k: None)
    monkeypatch.setattr(fad_mod, "FrechetAudioDistance", _FAD)
    ev = tmp_path / "eval"
    ev.mkdir()
    (ev / "a.wav").write_bytes(b"")
    out = tmp_path / "scores.csv"
    assert cli.score_main(["vggish", "base", str(ev), str(out), "--inf", "--indiv"]) == 0
    assert [c[0] for c in calls] == ["inf"]
    assert out.read_text().splitlines()[1].split(",")[3:5] == ["1.5", "0.9"]
    calls.clear()
    assert cli.score_main(["vggish", "base", str(ev), "--indiv"]) == 0 and [c[0] for c in calls] == ["indiv"]

    packed = []
    monkeypatch.setattr(package, "pack_statistics", lambda d, o, chosen, workers=8: packed.append([m.name for m in chosen]) or o)
    assert package.main([str(ev), str(tmp_path / "s.npz")]) == 0
    assert packed and "clap-2023" not in packed[0] and "vggish" in packed[0]
    assert "skipping clap-2023" in capsys.readouterr().out
    packed.clear()
    with pytest.raises(NotImplementedError):                    # named explicitly: the loader says what is missing
        UnbuiltModel("clap-2023", 1024, 44100, "x").load_model()


def test_synthetic_weights_are_an_explicit_opt_in(tmp_path, monkeypatch):
    """The reference always loads pretrained weights; a FAD from random weights is meaningless and would be cached
    under the same embeddings/<model> paths.  Without a checkpoint the loaders refuse unless FADTK_SYNTHETIC=1, and
    a path that does not exist is an error in either case."""
    from fadtk_b200 import weights, weights_clap, weights_encodec, weights_w2v, weights_whisper
    for var in ("FADTK_SYNTHETIC", "FADTK_VGGISH_CKPT", "FADTK_CLAP_CKPT", "FADTK_ENCODEC_CKPT", "FADTK_WHISPER_CKPT", "FADTK_W2V2_CKPT"):
        monkeypatch.delenv(var, raising=False)
    for load in (lambda: weights.load_vggish_state(), lambda: weights_clap.load_clap_state(),
                 lambda: weights_encodec.load_encodec_state(), lambda: weights_whisper.load_whisper_state(),
                 lambda: weights_w2v.load_w2v_state(env="FADTK_W2V2_CKPT")):
        with pytest.raises(weights.MissingCheckpoint):
            load()
    monkeypatch.setenv("FADTK_SYNTHETIC", "1")
    assert "features.0.weight" in weights.load_vggish_state()
    with pytest.raises(weights.MissingCheckpoint):            # a mistyped path never silently becomes random weights
        weights.load_vggish_state(tmp_path / "no-such-vggish.pth")
    monkeypatch.setenv("FADTK_VGGISH_CKPT", str(tmp_path / "typo.pth"))
    with pytest.raises(weights.MissingCheckpoint):
        weights.load_vggish_state()
    import torch
    real = {k: v + 1.0 for k, v in weights.synthetic_vggish_state(3).items()}
    torch.save(real, tmp_path / "vggish.pth")
    got = weights.load_vggish_state(tmp_path / "vggish.pth")
    assert torch.equal(got["embeddings.4.bias"], real["embeddings.4.bias"])


def test_loaders_sharing_an_engine_slot_reload_instead_of_borrowing_weights():
    """hubert-base, then w2v2-base, then hubert-base again (a dirs-outer / models-inner loop, or two live
    FrechetAudioDistance objects): the engine holds ONE set of weights per family, so the third use must reload."""
    from fadtk_b200 import model_loader as mlmod

    class FakeEngine:
        torch_device = "cpu"

        def __init__(self):
            self.owners, self.loaded = {}, []

    eng = FakeEngine()

    class Probe(mlmod._DeviceBatch, mlmod.ModelLoader):
        _SLOT = "w2v"

        def __init__(self, family):
            super().__init__(family, 768, 16000)
            self.family, self.size, self.checkpoint, self.seed = family, "base", None, 0
            self._engine = None

        def load_model(self):
            self._engine = eng
            eng.owners.pop(self._SLOT, None)
            eng.loaded.append(self.family)
            self.model = eng
            self._claim()

        def _get_embedding(self, audio):
            self._ensure_loaded()
            return eng.loaded[-1]

    a, b = Probe("hubert"), Probe("w2v2")
    with pytest.raises(RuntimeError):
        a._ensure_loaded()
    a.load_model()
    assert a.owns_engine() and a._get_embedding(None) == "hubert" and eng.loaded == ["hubert"]
    b.load_model()
    assert b.owns_engine() and not a.owns_engine()
    assert a._get_embedding(None) == "hubert" and eng.loaded == ["hubert", "w2v2", "hubert"]   # reloaded, not borrowed
    assert not b.owns_engine() and b._get_embedding(None) == "w2v2"
    twin = Probe("w2v2")                                     # same configuration = same weights: no reload needed
    twin._engine = eng
    assert twin.owns_engine()


_SHARD_WORKER = r"""
import os, sys, json, numpy as np
sys.path.insert(0, sys.argv[1])
os.environ["FADTK_SYNTHETIC"] = "1"
from pathlib import Path
from fadtk_b200 import dist, fad as fad_mod, fad_batch, synth
from fadtk_b200.model_loader import ModelLoader
dist.init_from_env("gloo")
r = dist.rank()
root = Path(sys.argv[2])

class Tiny(ModelLoader):
    # a plain third-party plugin (no batched extension): 4 features per 0.1 s
    def __init__(self):
        super().__init__("tiny", 4, 16000)
    def load_model(self):
        self.model = object()
    def _get_embedding(self, audio):
        a = np.asarray(audio, dtype=np.float32)[: (len(audio) // 1600) * 1600].reshape(-1, 1600)
        return np.stack([a.mean(1), a.std(1), a.min(1), a.max(1)], 1).astype(np.float32)

def cpu_stats(files):
    e = np.concatenate([np.load(f) for f in files]).astype(np.float64)
    return e.mean(0), np.cov(e, rowvar=False)
fad_mod.calculate_embd_statistics_online = cpu_stats
fad_mod.FrechetAudioDistance.convert_audio = lambda self, f: synth.read_wav(f)[0]

ml = Tiny()
# one new file for two ranks: rank 1's shard is empty and must reach the barrier instead of raising
fad_batch.cache_embedding_files(root / "one", ml, workers=2)
assert sorted(p.name for p in (root / "one" / "embeddings" / "tiny").glob("*.npy")) == ["a.npy"]
fad_batch.cache_embedding_files(root / "many", ml, workers=2)
names = sorted(p.name for p in (root / "many" / "embeddings" / "tiny").glob("*.npy"))
assert names == [f"c{i}.npy" for i in range(5)], names
fad_batch.cache_embedding_files(root / "many", ml, workers=2)          # nothing left: every rank returns
# statistics of an uncached directory requested by every rank: rank 0 writes, the others read the finished cache
f = fad_mod.FrechetAudioDistance(ml, audio_load_worker=2, load_model=False)
mu, cov = f.load_stats(root / "many")
want = cpu_stats(sorted((root / "many" / "embeddings" / "tiny").glob("*.npy")))
assert np.array_equal(mu, want[0]) and np.array_equal(cov, want[1])
assert not list((root / "many" / "stats" / "tiny").glob("*.tmp*"))
sys.stdout.write(f"[rank{r}:ok]\n"); sys.stdout.flush()
"""


def test_two_rank_file_sharding_and_rank0_statistics_gloo(tmp_path):
    """ADVICE round 1: an empty shard must not hang the other ranks, the already-embedded filter must come from ONE
    listing, and directory statistics must have one writer."""
    from fadtk_b200 import synth
    (tmp_path / "one").mkdir()
    (tmp_path / "many").mkdir()
    synth.write_wav(tmp_path / "one" / "a.wav", synth.musiclike_clip(0, 1.0, 16000), 16000)
    for i in range(5):
        synth.write_wav(tmp_path / "many" / f"c{i}.wav", synth.musiclike_clip(i + 1, 1.0, 16000), 16000)
    script = tmp_path / "worker.py"
    script.write_text(_SHARD_WORKER)
    env = dict(os.environ, OMP_NUM_THREADS="1")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", "29533", str(script), str(ROOT), str(tmp_path)],
                         capture_output=True, text=True, env=env, timeout=300)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "rank0:ok" in out.stdout and "rank1:ok" in out.stdout, out.stdout


def test_named_baseline_resolves_from_an_installed_reference_package(tmp_path, monkeypatch):
    """VERDICT r1 #6: `fadtk vggish fma_pop <dir>` must keep working after the switch.  The reference ships its
    statistics as fadtk/stats/<name>.npz (fad.py:249-255); with that package importable its stats directory is searched
    after $FADTK_STATS_DIR and this package's own stats/ directory."""
    import importlib
    from fadtk_b200 import fad as fad_mod
    monkeypatch.delenv("FADTK_STATS_DIR", raising=False)
    assert fad_mod._named_statistics("fma_pop") is None or fad_mod._named_statistics("fma_pop").name == "fma_pop.npz"
    site = tmp_path / "site"
    (site / "fadtk" / "stats").mkdir(parents=True)
    (site / "fadtk" / "__init__.py").write_text("")
    np.savez(site / "fadtk" / "stats" / "toy_pop.npz", **{"vggish.mu": np.arange(3.0), "vggish.cov": np.eye(3)})
    monkeypatch.syspath_prepend(str(site))
    importlib.invalidate_caches()
    assert fad_mod._named_statistics("Toy_Pop") == site / "fadtk" / "stats" / "toy_pop.npz"

    class _ML:
        name = "vggish"
    f = fad_mod.FrechetAudioDistance.__new__(fad_mod.FrechetAudioDistance)
    f.ml = _ML()
    mu, cov = f.load_stats("toy_pop")
    np.testing.assert_array_equal(mu, np.arange(3.0))
    with pytest.raises(SystemExit):                            # an unknown name: the reference's exit(1) (fad.py:276-278)
        f.load_stats("no_such_set")


def test_checkpoint_files_safetensors_and_old_weight_norm_names(tmp_path, monkeypatch):
    """ADVICE r1: published wav2vec-family checkpoints spell the positional conv's weight norm ``weight_g`` /
    ``weight_v`` and ship as .safetensors; both must load into the names the packers read."""
    from safetensors.torch import save_file
    from fadtk_b200 import weights, weights_w2v
    sd = weights_w2v.synthetic_w2v_state(0)
    old = {}
    for k, v in sd.items():
        k = k.replace("parametrizations.weight.original0", "weight_g").replace("parametrizations.weight.original1", "weight_v")
        old["wav2vec2." + k] = v.contiguous()
    old["lm_head.weight"] = torch.zeros(4, 4)
    save_file(old, str(tmp_path / "model.safetensors"))
    torch.save({"state_dict": old}, tmp_path / "pytorch_model.bin")
    for name in ("model.safetensors", "pytorch_model.bin"):
        got = weights_w2v.load_w2v_state(tmp_path / name, env="FADTK_W2V2_CKPT")
        assert set(got) == set(sd), sorted(set(got) ^ set(sd))[:6]
        for k in sd:
            assert torch.equal(got[k], sd[k].float()), k
    packed = weights_w2v.pack_w2v(weights_w2v.load_w2v_state(tmp_path / "model.safetensors", env="FADTK_W2V2_CKPT"))
    ref = weights_w2v.pack_w2v(sd)
    assert len(packed) == len(ref) and all(torch.equal(a, b) for a, b in zip(packed, ref))
    raw = weights.load_checkpoint_file(tmp_path / "pytorch_model.bin")
    assert "wav2vec2.encoder.pos_conv_embed.conv.parametrizations.weight.original0" in raw


def test_device_memory_is_allocated_and_freed_only_by_device_buffer():
    """Every device allocation of the library has one owner: cudaMalloc and cudaFree are called inside DeviceBuffer
    (fadtk_b200.cu) and nowhere else, so a weight or workspace cannot be leaked or freed twice by hand."""
    csrc = ROOT / "fadtk_b200" / "csrc"
    calls = re.compile(r"\bcuda(Malloc|Free)\(")
    found = 0
    for path in sorted([*csrc.glob("*.cu"), *csrc.glob("*.inc"), *csrc.glob("*.cuh")]):
        src = path.read_text()
        lo = hi = -1
        m = re.search(r"\bclass DeviceBuffer\s*\{", src)
        if m:                                                  # the class body, by brace matching
            lo, depth = m.start(), 0
            for i in range(m.end() - 1, len(src)):
                depth += {"{": 1, "}": -1}.get(src[i], 0)
                if depth == 0:
                    hi = i
                    break
        for c in calls.finditer(src):
            assert lo <= c.start() <= hi, f"{path.name}:{src.count(chr(10), 0, c.start()) + 1}: {c.group(0)} outside DeviceBuffer"
            found += 1
    assert found >= 2, "DeviceBuffer no longer allocates and frees"
