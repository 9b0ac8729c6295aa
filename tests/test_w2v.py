"""wav2vec 2.0 / HuBERT / MERT embedders (fad_w2v_forward) against the reference's own dependency:
transformers' Wav2Vec2FeatureExtractor + Wav2Vec2Model / HubertModel with output_hidden_states, driven as
fadtk/model_loader.py:262-288, 540-560, 578-596 (oracle/w2v_oracle.py), shared seeded synthetic weights."""
import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import synth, weights_w2v as ww
from oracle import w2v_oracle as wo


def test_packing_and_registry():
    sd = ww.synthetic_w2v_state(0, layers=2)
    assert ww.config_of(sd) == (768, 12, 2, 3072, 0, 0, 0)
    pk = ww.pack_w2v(sd)
    assert len(pk) == 28 + 4 + 17 + 2 + 12 * 2
    assert pk[0].shape == (2 * 512, 64) and pk[4].shape == (2 * 512, 1536) and pk[24].shape == (2 * 512, 1024)
    w1 = sd["feature_extractor.conv_layers.1.conv.weight"]
    assert torch.equal(pk[4][9, 2 * 512 + 5].float(), w1[9, 5, 2].to(torch.float16).float())       # column = tap*Cin + c
    wp = ww.pos_conv_weight(sd)
    assert torch.allclose(wp.pow(2).sum(dim=(0, 1)).sqrt().flatten(), sd["encoder.pos_conv_embed.conv.parametrizations.weight.original0"].flatten(), rtol=1e-5)
    assert pk[32 + 3].shape == (2 * 128, 128 * 48)
    assert torch.equal(pk[32 + 3][7, 11 * 48 + 2].float(), wp[3 * 48 + 7, 2, 11].to(torch.float16).float())
    names = {m.name: m for m in fk.get_all_models()}
    for n, sr, layer in (("w2v2-base", 16000, 12), ("w2v2-base-3", 16000, 3), ("hubert-base-7", 16000, 7),
                         ("MERT-v1-95M", 24000, 12), ("MERT-v1-95M-1", 24000, 1)):
        m = names[n]
        assert isinstance(m, fk.Wav2VecFamilyModel) and m.sr == sr and m.layer == layer and m.num_features == 768
    assert names["w2v2-large"].num_features == 1024 and names["w2v2-large"].layer == 24 and names["hubert-large-3"].layer == 3
    lay = ww.synthetic_w2v_state(0, d=1024, layers=1, ffn=4096, variant="layer")
    assert ww.config_of(lay) == (1024, 16, 1, 4096, 1, 1, 0) and len(ww.pack_w2v(lay)) == 28 + 4 + 17 + 2 + 12
    wl = ww.synthetic_w2v_state(0, layers=2, wavlm=True)
    assert ww.config_of(wl)[6] == 1 and len(ww.pack_w2v(wl)) == 28 + 4 + 17 + 2 + 1 + 15 * 2
    assert names["wavlm-base-plus-4"].layer == 4 and names["wavlm-large"].num_features == 1024 and names["wavlm-large"].layer == 24
    assert isinstance(names["clap-2023"], fk.UnbuiltModel)
    from fadtk_b200 import _native
    assert _native.Engine.w2v_frames(160000) == 499 and _native.Engine.w2v_frames(240000) == 749


@pytest.mark.parametrize("heads", [12, 16])
@pytest.mark.parametrize("S", [49, 149, 499, 1499])
def test_wavlm_bias_table_matches_transformers(S, heads):
    """The position-bias table fad_w2v_forward uploads (fad_wavlm_bias_table) equals WavLMAttention.compute_bias
    (transformers' _relative_positions_bucket + rel_attn_embed gather) at every (head, query, key), bit for bit.
    S = 1499 (30-s clips) reaches distances far past the 800 buckets' max_distance."""
    from transformers.models.wavlm.modeling_wavlm import WavLMAttention
    from fadtk_b200 import _native
    torch.manual_seed(S + heads)
    att = WavLMAttention(heads * 64, heads, num_buckets=320, max_distance=800)
    with torch.no_grad():
        att.rel_attn_embed.weight.copy_(torch.randn(320, heads))
        want = att.compute_bias(S, S)                                        # [heads, S (query), S (key)]
    got = torch.from_numpy(_native.Engine.wavlm_bias_table(att.rel_attn_embed.weight.detach().numpy(), S))
    assert got.shape == (heads, 2 * S - 1)
    dist = torch.arange(S)[None, :] - torch.arange(S)[:, None]               # key - query
    assert torch.equal(got[:, dist + S - 1], want)


def test_oracle_is_the_reference_dependency():
    sd = ww.synthetic_w2v_state(0, layers=2)
    model, fe = wo.build(sd, "hubert")
    e = wo.embed(synth.musiclike_clip(1, 1.0, 16000) / 32768.0, model, fe, 2)
    assert e.shape == (49, 768) and e.dtype == np.float16


@pytest.mark.gpu
@pytest.mark.parametrize("family,sr,layer", [("w2v2", 16000, 12), ("hubert", 16000, 5), ("mert", 24000, 0)])
def test_hidden_states_match_transformers(engine, family, sr, layer):
    clips = [synth.musiclike_clip(4, 4.0, sr), synth.noise_clip(2, 4.0, sr), synth.musiclike_clip(9, 1.3, sr)]
    name = {"w2v2": "w2v2-base", "hubert": "hubert-base", "mert": "MERT-v1-95M"}[family]
    ml = fk.Wav2VecFamilyModel(family, name, layer, sr, max_clips=2, size='v1-95M' if family == 'mert' else 'base')
    ml.load_model()
    got = ml.embed_pcm_batch(clips)
    sd = ww.synthetic_w2v_state(0)
    model, fe = wo.build(sd, "w2v2" if family == "w2v2" else "hubert", sr)
    for g, c in zip(got, clips):
        want = wo.embed(c / 32768.0, model, fe, layer, sr).astype(np.float32)
        g = g.astype(np.float32)
        assert g.shape == want.shape == (ml._engine.w2v_frames(len(c)), 768)
        rel = np.sqrt(((g - want) ** 2).mean() / (want ** 2).mean())
        print(f"{name} layer {layer}, {len(c)} samples: rms rel err {rel:.2e}")
        assert rel < 5e-3, rel
    one = ml.get_embedding(clips[2] / 32768.0)
    assert one.dtype == np.float16 and np.array_equal(one, got[2])


@pytest.mark.gpu
@pytest.mark.parametrize("family,size,layer", [("hubert", "large", 24), ("hubert", "large", 2), ("w2v2", "large", 3)])
def test_large_variants_match_transformers(engine, family, size, layer):
    """hubert-large: layer-norm feature encoder + stable-LN (pre-LN) transformer, hidden_states[k < 24] = raw stream;
    w2v2-large: the base architecture at d = 1024.  Synthetic checkpoints with fewer layers keep the CPU oracle quick."""
    arch = dict(ww.ARCH[(family, size)])
    arch["layers"] = layer + 1 if layer < 24 else 3             # shortened synthetic stack; layer < 24 taps an inner (raw-stream) state
    sd = ww.synthetic_w2v_state(0, **arch)
    tap = layer if layer < 24 else arch["layers"]                # last layer of the shortened stack
    eng = engine
    eng.w2v_load(ww.config_of(sd), ww.pack_w2v(sd), 2, max_len=16000 * 5)
    clips = [synth.musiclike_clip(4, 3.0, 16000), synth.noise_clip(2, 3.0, 16000)]
    got = eng.w2v_forward(torch.from_numpy(np.stack(clips)).to(eng.torch_device), tap).cpu().numpy().astype(np.float32)
    model, fe = wo.build(sd, "w2v2" if family == "w2v2" else "hubert")
    for g, c in zip(got, clips):
        want = wo.embed(c / 32768.0, model, fe, tap).astype(np.float32)
        rel = np.sqrt(((g - want) ** 2).mean() / (want ** 2).mean())
        print(f"{family}-{size} hidden_states[{tap}] of {arch['layers']} layers: rms rel err {rel:.2e}")
        assert g.shape == want.shape and rel < 5e-3, rel


@pytest.mark.gpu
@pytest.mark.parametrize("size,layer", [("base", 3), ("large", 2)])
def test_wavlm_matches_transformers(engine, size, layer):
    """WavLM: the wav2vec2 skeleton + gated relative position bias (bucketed rel_attn_embed of layer 0, per-query gate)."""
    arch = dict(ww.ARCH[("wavlm", size)])
    arch["layers"] = layer + (1 if size == "large" else 0)
    sd = ww.synthetic_w2v_state(0, **arch)
    engine.w2v_load(ww.config_of(sd), ww.pack_w2v(sd), 2, max_len=16000 * 5)
    clips = [synth.musiclike_clip(4, 3.0, 16000), synth.noise_clip(2, 3.0, 16000)]
    got = engine.w2v_forward(torch.from_numpy(np.stack(clips)).to(engine.torch_device), layer).cpu().numpy().astype(np.float32)
    model, fe = wo.build(sd, "wavlm")
    for g, c in zip(got, clips):
        want = wo.embed(c / 32768.0, model, fe, layer).astype(np.float32)
        rel = np.sqrt(((g - want) ** 2).mean() / (want ** 2).mean())
        print(f"wavlm-{size} hidden_states[{layer}] of {arch['layers']} layers: rms rel err {rel:.2e}")
        assert g.shape == want.shape and rel < 5e-3, rel


@pytest.mark.gpu
def test_w2v_fad_parity_on_identical_audio(engine):
    """FAD against the reference CPU path (transformers fp32) on identical audio, 64 + 64 four-second clips (25 472 rows).
    Measured: -1.4e-4 ... -2.0e-4 relative - ABOVE the 1e-4 bar the BASELINE configurations meet (VGGish 7e-7 at
    1000 + 1000 clips, CLAP 8e-5 at 200 + 200: profiles/r2_parity_*.json).  What it is (DESIGN.md section 3, finding 6):
    under seeded random weights the hidden state of layer 12 is 99.2 % per-dimension mean (mean / rms = 0.996,
    profiles/r2_w2v_fad_terms_32clips.json), so the covariances the score is made of are those of a fluctuation 11x
    smaller than the values the fp16 GEMM operands round - not the attention kernel (the tensor-core and mma.sync kernels agree,
    profiles/r2_attention_accuracy.json) and, since the epilogue compensates the tensor core's accumulator truncation
    (gain error of a GEMM -8e-7 -> -9e-9, profiles/r2_gemm_bias_probe_*.json), not a gain error of the GEMMs either.
    The reference path itself with fp16-rounded Linear / Conv1d inputs moves the FAD of these sets by +6e-5 ... +1.1e-4 on the
    CPU (benchmarks/w2v_fp16_operand_emulation.py, profiles/r2_w2v_fp16_operand_emulation_cpu.jsonl): same order, either sign.
    Round 1's 8 + 8-clip version of this test passed at 5e-5 by chance (five independent 8 + 8 sets scatter over
    -2.2e-4 ... +2.6e-4, profiles/r2_w2v_fad_parity_sweep_*.json).  The bound below is the measured level with margin -
    a regression guard, not a claim of 1e-4 parity for this family (SURVEY.md section 8 (f) item 4, lowest priority)."""
    from oracle import fad_oracle as fo
    n = 64
    sets = {"base": [synth.noise_clip(i, 4.0, 16000) for i in range(n)],
            "eval": [synth.musiclike_clip(i, 4.0, 16000) for i in range(n)]}
    ml = fk.W2V2Model('base', 12, max_clips=8)
    ml.load_model()
    sd = ww.synthetic_w2v_state(0)
    model, fe = wo.build(sd, "w2v2")
    gpu = {k: np.concatenate([e for s in range(0, n, 8) for e in ml.embed_pcm_batch(v[s:s + 8])]) for k, v in sets.items()}
    cpu = {k: np.concatenate([wo.embed(c / 32768.0, model, fe, 12) for c in v]) for k, v in sets.items()}
    assert gpu["eval"].shape == cpu["eval"].shape == (n * 199, 768)
    fad_gpu = fk.calc_frechet_distance(*fk.calc_embd_statistics(gpu["base"]), *fk.calc_embd_statistics(gpu["eval"]))
    fad_cpu = fo.frechet_distance(*fo.embd_statistics(cpu["base"]), *fo.embd_statistics(cpu["eval"]))
    rel = abs(fad_gpu - fad_cpu) / abs(fad_cpu)
    print(f"w2v2-base FAD gpu {fad_gpu:.6f} cpu reference path {fad_cpu:.6f} rel {rel:.2e}")
    assert rel < 3.5e-4, (fad_gpu, fad_cpu, rel)
