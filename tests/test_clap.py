"""CLAP-LAION (HTSAT-tiny) path: host planning on CPU, CUDA parity against oracle/clap_oracle.py
(which tests/test_clap_oracle.py pins to transformers' independent port)."""
import numpy as np
import pytest
import torch

import fadtk_b200 as fk
from fadtk_b200 import _native, synth, weights_clap
from oracle import clap_oracle as co


def test_plan_follows_reference_windowing():
    # model_loader.py:396-404: one window per started second, each up to 10 s, zero padded
    lens = [480000, 1, 48000, 48001, 100000, 0]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    start, valid, rows = _native.Engine.clap_plan(off)
    assert list(rows) == [10, 1, 1, 2, 3, 0] == [len(co.chunks_of(np.zeros(n, np.float32))) if n else 0 for n in lens]
    assert list(start[:10]) == [48000 * i for i in range(10)]
    assert list(valid[:10]) == [480000 - 48000 * i for i in range(10)]
    assert (start[13], valid[13]) == (off[3] + 48000, 1)


def test_frame_pool_addresses_the_same_samples():
    """Every (window, frame) must map to a pool entry reading the same absolute samples with the same
    edge behaviour: interior frames (2..998) are shared between the windows of a clip, edge frames
    (reflect padding at 0/1/999/1000) stay per window."""
    lens = [480000, 1, 48000, 48001, 100000, 0, 600000]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    start, valid, rows = _native.Engine.clap_plan(off)
    plan = _native.Engine.clap_plan_frames(off)
    ps, pv, pf, fi = (plan[k] for k in ("pool_start", "pool_valid", "pool_frame", "frame_index"))
    assert fi.shape == (len(start), 1001) and np.array_equal(plan["rows_per_clip"], rows)
    assert fi.min() == 0 and fi.max() == len(ps) - 1 and len(np.unique(fi)) == len(ps)     # pool has no dead rows
    f = np.arange(1001)[None, :]
    pos_want = start[:, None] + 480 * f                      # centre sample of each frame
    assert np.array_equal(ps[fi] + 480 * pf[fi], np.broadcast_to(pos_want, fi.shape))
    clip_end_want = (start + valid)[:, None]                 # zero padding starts at the end of the clip
    inner = (f >= 2) & (f <= 998)
    # a shared frame never reaches the end of its source window unless that is the end of the clip
    src_end = ps[fi] + pv[fi]
    reach = pos_want + 512
    ok = np.where(inner, (src_end == clip_end_want) | ((reach <= src_end) & (reach <= clip_end_want)), True)
    assert ok.all()
    assert ((pf[fi] >= 2) & (pf[fi] <= 998))[np.broadcast_to(inner, fi.shape)].all()
    edge = ~np.broadcast_to(inner, fi.shape)
    assert np.array_equal(ps[fi][edge], np.broadcast_to(start[:, None], fi.shape)[edge])
    assert np.array_equal(pf[fi][edge], np.broadcast_to(f, fi.shape)[edge])
    n_win = len(start)
    assert len(ps) < 0.3 * n_win * 1001                      # ~5x fewer frames than windows x 1001 here


def test_packing_shapes_and_padding():
    sd = weights_clap.synthetic_clap_state(0)
    pk = weights_clap.pack_clap(sd)
    assert len(pk) == weights_clap.N_TENSORS == 180
    qkv = pk[6 + 2]                                   # stage 0: 3C = 288 -> 384 rows, K 96 -> 128, hi/lo tiles
    assert qkv.shape == (2 * 384, 128) and qkv.dtype == torch.float16
    wq = sd["layers.0.blocks.0.attention.self.query.weight"]
    assert torch.equal(qkv[5, :96].float(), wq[5].to(torch.float16).float()) and not qkv[5, 96:].any()
    assert not qkv[2 * 256 + 32:2 * 256 + 128].any()     # rows 288..383 of the padded N are zero
    rel = pk[6 + 4]
    assert rel.shape == (4, 64, 64)
    names = [m.name for m in fk.get_all_models()]
    assert "clap-laion-audio" in names


@pytest.mark.parametrize("variant", ["tiny", "base"])
def test_packed_relbias_is_the_oracle_gather(variant):
    """Every block's packed relbias [heads][64][64] is relative_position_bias_table[_rel_pos_index] of the oracle
    (pinned to transformers by test_clap_oracle.py), query row first, bit for bit."""
    sd = weights_clap.synthetic_clap_state(3, variant)
    pk = weights_clap.pack_clap(sd)
    _, depths = weights_clap.VARIANTS[variant]
    idx = co._rel_pos_index()
    blk = 0
    for i, (depth, heads) in enumerate(zip(depths, weights_clap.HEADS)):
        for j in range(depth):
            table = sd[f"layers.{i}.blocks.{j}.attention.self.relative_position_bias_table"]
            want = torch.stack([table[idx, hh] for hh in range(heads)])
            got = pk[6 + 13 * blk + 4]
            assert got.shape == (heads, 64, 64) and got.dtype == torch.float32
            assert torch.equal(got, want), f"stage {i} block {j}"
            blk += 1
    assert blk == sum(depths)


def _clips():
    return [synth.musiclike_clip(2, 10.0, 48000), synth.musiclike_clip(5, 2.5, 48000, baseline=True)]


@pytest.fixture(scope="module")
def clap_engine(engine):
    engine.clap_load(weights_clap.pack_clap(weights_clap.synthetic_clap_state(0)), max_chunks=8)
    return engine


@pytest.mark.gpu
def test_logmel_batchnorm_stage_matches_oracle(clap_engine):
    clips = _clips()
    off = np.concatenate([[0], np.cumsum([len(c) for c in clips])]).astype(np.int64)
    plan = clap_engine.clap_plan_frames(off)
    rows = plan["rows_per_clip"]
    # a 10-s clip has 1897 shared interior frames + 4 edge frames per window instead of 10 x 1001
    assert plan["pool_start"].shape[0] == (1897 + 40) + (200 + 997 + 12)
    dev = clap_engine.torch_device
    got = clap_engine.clap_logmel(torch.from_numpy(np.concatenate(clips)).to(dev),
                                  clap_engine.clap_plan_to_device(plan)).cpu()
    sd = co.synthetic_state(0)
    want = []
    for c in clips:
        ch = torch.from_numpy(co.chunks_of(co.quantize_like_reference(c / 32768.0)))
        lm = co.log_mel(ch)
        scale = sd["batch_norm.weight"] / torch.sqrt(sd["batch_norm.running_var"] + 1e-5)
        want.append(lm * scale + (sd["batch_norm.bias"] - sd["batch_norm.running_mean"] * scale))
    want = torch.cat(want)
    assert got.shape == want.shape == (int(rows.sum()), 1001, 64)
    loud = want > want.max() - 6.0                    # bins within ~90 dB of the peak (BN scale ~1/15)
    err = (got - want).abs()
    assert err[loud].max() < 5e-3, err[loud].max()
    assert err.mean() < 2e-3, err.mean()


@pytest.mark.gpu
def test_embeddings_match_oracle(clap_engine):
    clips = _clips()
    ml = fk.CLAPLaionModel('audio')
    ml.load_model()
    got = np.concatenate(ml.embed_pcm_batch(clips)).astype(np.float32)
    sd = co.synthetic_state(0)
    want = np.concatenate([co.embed(c / 32768.0, sd) for c in clips]).astype(np.float32)
    assert got.shape == want.shape == (13, 512)
    assert np.allclose(np.linalg.norm(got, axis=1), 1.0, atol=2e-3)
    cos = (got * want).sum(1)
    assert cos.min() > 0.9999, cos
    assert np.abs(got - want).max() < 3e-3, np.abs(got - want).max()
    # plugin contract: single clip through get_embedding
    one = ml.get_embedding(clips[1] / 32768.0)
    assert one.dtype == np.float16 and np.array_equal(one, got[10:].astype(np.float16))   # batch-invariant, deterministic


@pytest.mark.gpu
def test_clap_fad_parity_on_identical_audio(clap_engine):
    """FAD from CUDA CLAP embeddings vs the CPU oracle path on the same audio: 12 noise clips vs 12
    music-like clips (120 + 120 windows in 512-d: rank-deficient covariances, the hard case for the
    Frechet chain)."""
    from oracle import fad_oracle as fo
    n = 12
    sets = {"base": [synth.noise_clip(i, 10.0, 48000) for i in range(n)],
            "eval": [synth.musiclike_clip(i, 10.0, 48000) for i in range(n)]}
    ml = fk.CLAPLaionModel('audio')
    ml.load_model()
    sd = co.synthetic_state(0)
    gpu = {k: np.concatenate(ml.embed_pcm_batch(v)) for k, v in sets.items()}
    cpu = {k: np.concatenate([co.embed(c / 32768.0, sd) for c in v]) for k, v in sets.items()}
    fad_gpu = fk.calc_frechet_distance(*fk.calc_embd_statistics(gpu["base"]), *fk.calc_embd_statistics(gpu["eval"]))
    fad_same = fo.frechet_distance(*fo.embd_statistics(gpu["base"]), *fo.embd_statistics(gpu["eval"]))
    fad_cpu = fo.frechet_distance(*fo.embd_statistics(cpu["base"]), *fo.embd_statistics(cpu["eval"]))
    traces = sum(np.trace(np.cov(gpu[k].astype(np.float64), rowvar=False)) for k in gpu)
    print(f"CLAP FAD gpu {fad_gpu:.9f} oracle-on-gpu-emb {fad_same:.9f} cpu-path {fad_cpu:.9f} traces {traces:.6f}")
    assert abs(fad_gpu - fad_same) < 1e-4 * abs(fad_same) + 1e-6 * traces, (fad_gpu, fad_same)   # statistics + Frechet chain
    rel = abs(fad_gpu - fad_cpu) / abs(fad_cpu)
    assert rel < 1e-4, f"FAD gpu {fad_gpu} vs cpu reference path {fad_cpu}: rel {rel}"


@pytest.mark.gpu
def test_music_variant_htsat_base_matches_oracle(engine):
    """clap-laion-music = HTSAT-base (embed 128, depths 2-2-12-2, head dim 32, final width 1024,
    model_loader.py:385): same kernels, wider instantiations, checked against the HF-pinned oracle."""
    clips = [synth.musiclike_clip(3, 3.2, 48000), synth.noise_clip(1, 1.0, 48000)]
    ml = fk.CLAPLaionModel('music')
    ml.load_model()
    got = np.concatenate(ml.embed_pcm_batch(clips)).astype(np.float32)
    sd = co.synthetic_state(0, "base")
    want = np.concatenate([co.embed(c / 32768.0, sd) for c in clips]).astype(np.float32)
    assert got.shape == want.shape == (5, 512)
    cos = (got * want).sum(1)
    assert cos.min() > 0.9999, cos
    assert np.abs(got - want).max() < 3e-3, np.abs(got - want).max()
    fk.CLAPLaionModel('audio').load_model()           # leave the engine with the tiny variant for later tests
