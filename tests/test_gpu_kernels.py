"""Stage-by-stage parity of the sm_90a kernels (through the C ABI) against the CPU oracle.

Tolerances: the embedder computes with fp16 operands and fp32 accumulation (DESIGN.md
"precision budget"), so layer outputs are compared with a torch fp32 reference fed the SAME
fp16-rounded operands (tolerance = fp32 accumulation order noise), and whole-network embeddings
with the fp32 oracle at the fp16-operand noise level measured on CPU (8e-4 rms).  Statistics and
Frechet values are fp64 and compared at 1e-9 / 1e-7 relative.
"""
import numpy as np
import pytest
import torch

from fadtk_b200 import synth
from oracle import fad_oracle as fo
from oracle import vggish_oracle as vo

pytestmark = pytest.mark.gpu


def _clips():
    return [synth.musiclike_clip(3, 10.0, 16000), synth.sine_clip(5, 2.5, 16000),
            synth.noise_clip(7, 1.0, 16000), synth.musiclike_clip(11, 0.5, 16000)]


def _flat(clips):
    off = np.zeros(len(clips) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(c) for c in clips])
    return np.concatenate(clips), off


@pytest.mark.parametrize("use_double", [True, False])
def test_logmel_matches_float64_numpy(engine, use_double):
    clips = _clips()
    pcm, off = _flat(clips)
    ex, rows = engine.vggish_plan(off)
    assert list(rows) == [vo.num_examples(len(c)) for c in clips] == [10, 2, 1, 0]
    dev = engine.torch_device
    got = engine.vggish_logmel(torch.from_numpy(pcm).to(dev), torch.from_numpy(ex).to(dev), use_double)
    want = np.concatenate([vo.examples(vo.load_wav_semantics(c)) for c in clips if vo.num_examples(len(c))])
    err = np.abs(got.cpu().numpy() - want).max()
    assert err < (2e-6 if use_double else 2e-2), f"log-mel max abs err {err}"


def test_conv1_matches_torch(vgg_engine, vgg_state):
    """conv1 stage (CUDA-core fp32 stencil + bias + ReLU + 2x2 max-pool, fp16 NHWC out) vs torch fp32 on real
    log-mel examples: the only error is the final fp16 rounding of the output."""
    import torch.nn.functional as F
    clips = _clips()[:2]
    pcm, off = _flat(clips)
    ex, _ = vgg_engine.vggish_plan(off)
    dev = vgg_engine.torch_device
    logmel = vgg_engine.vggish_logmel(torch.from_numpy(pcm).to(dev), torch.from_numpy(ex).to(dev), use_double=False)
    got = vgg_engine.vggish_conv1(logmel.contiguous()).float().cpu()                 # [n, 48, 32, 64]
    x = logmel.cpu().unsqueeze(1)                                                  # [n, 1, 96, 64]
    want = F.max_pool2d(F.relu(F.conv2d(x, vgg_state["features.0.weight"], vgg_state["features.0.bias"], padding=1)), 2)
    want = want.permute(0, 2, 3, 1).contiguous()                                   # NHWC
    assert got.shape == want.shape
    err = (got - want).abs().max().item()
    assert err <= 2.0 ** -11 * want.abs().max().item() + 1e-6, f"conv1 max abs err {err}"


LAYERS = [
    # NB, H,  W,  Cin, Cout, taps, relu, pool
    (5, 48, 32, 64, 128, 9, True, True),
    (3, 24, 16, 128, 256, 9, True, False),
    (3, 24, 16, 256, 256, 9, True, True),
    (6, 12, 8, 256, 512, 9, True, False),
    (5, 12, 8, 512, 512, 9, True, True),
    (1, 12, 8, 256, 512, 9, False, False),
    (200, 1, 1, 12288, 4096, 1, True, False),
    (130, 1, 1, 4096, 128, 1, False, False),
    (1, 1, 1, 4096, 4096, 1, True, False),
]


# fp16 weights | fp16 hi/lo | hi/lo pair of weights exact in fp16 (all-zero lo parts, which the GEMM's truncation
# compensation does not count)
@pytest.mark.parametrize("split_w", [0, 1, "fp16-exact"])
@pytest.mark.parametrize("nb,hh,ww,cin,cout,taps,relu,pool", LAYERS)
def test_umma_layer_matches_fp32_reference(engine, nb, hh, ww, cin, cout, taps, relu, pool, split_w):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = engine.torch_device
    g = torch.Generator(device="cpu").manual_seed(nb * 1000 + cin + cout)
    x = (torch.randn((nb, hh, ww, cin), generator=g) * 1.0).to(torch.float16)
    w32 = torch.randn((cout, taps * cin), generator=g) * (2.0 / (taps * cin)) ** 0.5
    b = torch.randn((cout,), generator=g) * 0.1
    if split_w == "fp16-exact":
        split_w, w32 = 1, w32.half().float()
    if split_w:
        from fadtk_b200 import weights as wts
        w_dev = wts.split_hi_lo_tiles(w32).to(dev)          # [2*Cout, K] hi/lo tiles, 22-bit weights
        w = w32                                              # reference uses the fp32 weights
    else:
        w = w32.to(torch.float16)
        w_dev = w.to(dev)
    xd, wd, bd = x.to(dev), w.to(dev), b.to(dev)
    if pool:
        out = engine.umma_layer(xd, w_dev, bd, taps, relu, pool, split_w=split_w)
        out32 = None
    else:
        out, out32 = engine.umma_layer(xd, w_dev, bd, taps, relu, pool, want_f32=True, split_w=split_w)
    torch.cuda.synchronize()
    # fp32 reference on the same fp16-rounded operands
    if taps == 9:
        wt = wd.float().reshape(cout, 3, 3, cin).permute(0, 3, 1, 2).contiguous()
        ref = torch.nn.functional.conv2d(xd.float().permute(0, 3, 1, 2), wt, bd, padding=1)
        if relu:
            ref = torch.relu(ref)
        if pool:
            ref = torch.nn.functional.max_pool2d(ref, 2, 2)
        ref = ref.permute(0, 2, 3, 1)
    else:
        ref = xd.float().reshape(nb, cin) @ wd.float().t() + bd
        if relu:
            ref = torch.relu(ref)
        ref = ref.reshape(nb, 1, 1, cout)
    scale = ref.abs().max().item()
    if out32 is not None:
        e32 = (out32 - ref).abs().max().item()
        assert e32 < 2e-4 * scale + 1e-5, f"fp32 epilogue copy: max err {e32} (scale {scale})"
    e16 = (out.float() - ref).abs().max().item()
    assert e16 < 1.5e-3 * scale + 1e-4, f"fp16 output: max err {e16} (scale {scale})"


def test_vggish_embeddings_match_fp32_oracle(vgg_engine, vgg_state):
    clips = _clips()[:3] + [synth.musiclike_clip(21, 10.0, 16000, baseline=True)]
    pcm, off = _flat(clips)
    ex, rows = vgg_engine.vggish_plan(off)
    dev = vgg_engine.torch_device
    got = vgg_engine.vggish_forward(torch.from_numpy(pcm).to(dev), torch.from_numpy(ex).to(dev))
    torch.cuda.synchronize()
    got = got.cpu().numpy().astype(np.float64)
    want = np.concatenate([vo.embed(vo.load_wav_semantics(c), vgg_state) for c in clips]).astype(np.float64)
    assert got.shape == want.shape == (int(rows.sum()), 128)
    rel = np.sqrt(((got - want) ** 2).mean() / (want ** 2).mean())
    assert rel < 3e-3, f"embedding rms relative error {rel}"


@pytest.mark.parametrize("n,d", [(5000, 128), (3000, 512), (257, 128), (63, 128), (2, 128), (777, 384)])
@pytest.mark.parametrize("tensor_core", [0, 2, "gather"], ids=["dmma", "simt", "gather"])
def test_statistics_match_numpy_float64(engine, n, d, tensor_core):
    rng = np.random.default_rng(n + d)
    emb = (rng.normal(0.0, 1.0, (n, d)) * rng.uniform(0.2, 3.0, d) + rng.normal(0, 4.0, d)).astype(np.float16)
    dev = engine.torch_device
    e = torch.from_numpy(emb).to(dev)
    shift = e[: min(n, 64)].float().mean(0).to(torch.float16)
    acc = engine.stats_new(d)
    # "gather": fad_stats_accumulate_gather (DMMA) over the same rows, picked from the whole set in permuted order
    perm = torch.from_numpy(rng.permutation(n)).to(dev) if tensor_core == "gather" else None

    def accumulate(lo, hi):
        if perm is None:
            engine.stats_accumulate(e[lo:hi].contiguous(), shift, acc, tensor_core=tensor_core)
        else:
            engine.stats_accumulate_gather(e, perm[lo:hi].contiguous(), shift, acc)
    half = n // 2
    if half:
        accumulate(0, half)
    accumulate(half, n)
    mu, cov = engine.stats_finalize(acc, shift, d)
    torch.cuda.synchronize()
    x = emb.astype(np.float64)
    mu_ref, cov_ref = x.mean(0), np.cov(x, rowvar=False)
    assert acc[0].item() == n
    assert np.abs(mu.cpu().numpy() - mu_ref).max() < 1e-9 * (1 + np.abs(mu_ref).max())
    err = np.abs(cov.cpu().numpy() - cov_ref).max() / np.abs(cov_ref).max()
    # every path (DMMA on the fp64 tensor pipe, the default; CUDA-core fp64): Gram matrix of exact (x - shift) values
    assert err < 1e-12, f"cov rel err {err}"


def test_statistics_dmma_equals_simt_bitwise_inputs(engine):
    """Both kernels consume the identical exact y = x - shift; they differ only in the order of their fp64 sums."""
    rng = np.random.default_rng(1)
    emb = rng.normal(0.5, 2.0, (4096 + 33, 256)).astype(np.float16)
    dev = engine.torch_device
    e = torch.from_numpy(emb).to(dev)
    shift = e.float().mean(0).to(torch.float16)
    b = engine.stats_accumulate(e, shift, engine.stats_new(256), tensor_core=2)
    c = engine.stats_accumulate(e, shift, engine.stats_new(256), tensor_core=0)
    c2 = engine.stats_accumulate(e, shift, engine.stats_new(256), tensor_core=0)
    torch.cuda.synchronize()
    den = b.abs().max().item()
    # DMMA and CUDA-core fp64 sum the same exact products in different orders: 1e-16-level agreement;
    # the DMMA path has no atomics, so two runs are bit-identical
    assert (c - b).abs().max().item() / den < 1e-13
    assert torch.equal(c, c2)


def test_gather_statistics(engine):
    rng = np.random.default_rng(5)
    emb = rng.normal(0, 1, (1000, 128)).astype(np.float16)
    idx = rng.integers(0, 1000, 2500)
    dev = engine.torch_device
    e = torch.from_numpy(emb).to(dev)
    shift = torch.zeros(128, dtype=torch.float16, device=dev)
    acc = engine.stats_accumulate_gather(e, torch.from_numpy(idx).to(dev), shift, engine.stats_new(128))
    mu, cov = engine.stats_finalize(acc, shift, 128)
    x = emb[idx].astype(np.float64)
    assert np.abs(cov.cpu().numpy() - np.cov(x, rowvar=False)).max() < 1e-12


def _rand_cov(rng, d, n):
    x = rng.normal(0, 1, (n, d)) * rng.uniform(0.1, 2.0, d) @ rng.normal(0, 1, (d, d)) / np.sqrt(d)
    return x.mean(0), np.cov(x, rowvar=False)


@pytest.mark.parametrize("d,n1,n2", [(128, 2000, 3000), (256, 5000, 4000), (128, 40, 3000), (128, 3000, 32)])
def test_frechet_matches_reference_eig_route(engine, d, n1, n2):
    rng = np.random.default_rng(d + n1 + n2)
    mu1, c1 = _rand_cov(rng, d, n1)
    mu2, c2 = _rand_cov(rng, d, n2)
    mu2 = mu2 + 0.1
    want = fo.frechet_distance(mu1, c1, mu2, c2)
    dev = engine.torch_device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = engine.frechet(t(mu1), t(c1), t(mu2), t(c2)).cpu().numpy()
    rel = abs(out[0] - want) / abs(want)
    assert rel < 1e-6, f"FAD {out[0]} vs reference {want} (rel {rel}); residual {out[2]}"


def test_frechet_golden_fma_pop(engine, golden_dir):
    g = np.load(golden_dir / "frechet_fma_pop_128.npz")
    dev = engine.torch_device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = engine.frechet(t(g["mu1"]), t(g["cov1"]), t(g["mu2"]), t(g["cov2"])).cpu().numpy()
    rel = abs(out[0] - float(g["fad"])) / float(g["fad"])
    assert rel < 1e-6, f"FAD {out[0]} vs golden {float(g['fad'])} rel {rel}"


# "tcgen05" is the stable id of the default tensor-core attention kernel (legacy=False); on sm_90a that kernel is
# attention_wgmma_kernel.  The id is kept so the test keeps its identity across architectures.
@pytest.mark.parametrize("legacy", [False, True], ids=["tcgen05", "mma_sync"])
@pytest.mark.parametrize("n_clips,S,d", [(2, 1500, 768), (3, 499, 768), (1, 128, 128), (2, 77, 256), (1, 129, 64), (2, 640, 1024)])
def test_encoder_attention_matches_torch(engine, n_clips, S, d, legacy):
    """Encoder self-attention stage (Whisper / wav2vec family; heads of 64 dims, scores scaled by 1/8): wgmma kernel
    (S = Q K^T and P V as wgmma tiles, scores in registers) and the mma.sync kernel it replaced, against torch in fp32 on the
    same fp16 inputs.  Ragged sizes exercise the zero-filled key rows of the last 128-key block."""
    g = torch.Generator(device="cpu").manual_seed(S * 7 + d)
    qkv = (torch.randn((n_clips * S, 3 * d), generator=g) * 1.5).to(torch.float16)
    dev = engine.torch_device
    got = engine.attention(qkv.to(dev), n_clips, legacy=legacy).float().cpu()
    heads = d // 64
    x = qkv.float().view(n_clips, S, 3, heads, 64)
    q, k, v = (x[:, :, i].permute(0, 2, 1, 3) for i in range(3))                # [clips, heads, S, 64]
    p = torch.softmax(q @ k.transpose(-1, -2) / 8.0, dim=-1)
    want = (p @ v).permute(0, 2, 1, 3).reshape(n_clips * S, d)
    err = (got - want).abs().max().item()
    assert err < 4e-3 * want.abs().max().item() + 1e-3, f"attention max abs err {err} (max {want.abs().max().item()})"


@pytest.mark.parametrize("n_files,r,d", [(37, 10, 128), (5, 750, 128), (64, 2, 256), (9, 1, 64)])
def test_mirrored_directory_statistics_match_reference_merge(engine, n_files, r, d, monkeypatch):
    """fad_file_means + fad_stats_accumulate_f64 + fad_stats_finalize_mirrored == the reference's
    calculate_embd_statistics_online on the same files (fadtk/utils.py:13-46: np.mean of an fp16 file is fp16, per-file
    np.cov, Chan merge) - the oracle restatement is pinned to the real reference by tests/test_oracle_golden.py.
    r = 1: the reference's covariance is all NaN (utils.py:16)."""
    from oracle import fad_oracle as fo
    monkeypatch.delenv("FADTK_SINGLE_FRAME_FILES", raising=False)
    rng = np.random.default_rng(n_files * 100 + r)
    files = [(rng.normal(0.0, 1.0, (r, d)) * rng.uniform(0.3, 2.0, d) + rng.normal(0, 3.0, d) + 0.2 * f).astype(np.float16)
             for f in range(n_files)]
    emb = torch.from_numpy(np.concatenate(files)).to(engine.torch_device)
    shift = emb[: min(len(emb), 64)].float().mean(0).to(torch.float16)
    n_acc = engine.stats_acc_len(d)
    buf = torch.zeros(3 * n_acc, dtype=torch.float64, device=emb.device)
    engine.stats_accumulate(emb, shift, buf[:n_acc])
    m64, m16 = engine.file_means(emb, r)
    want16 = np.stack([np.mean(f, axis=0) for f in files])                        # fp16, as _process_file computes it
    assert np.array_equal(m16.cpu().numpy(), want16.astype(np.float64))
    assert np.abs(m64.cpu().numpy() - np.stack([f.astype(np.float64).mean(0) for f in files])).max() < 1e-12
    engine.stats_accumulate_f64(m64, buf[n_acc:2 * n_acc])
    engine.stats_accumulate_f64(m16, buf[2 * n_acc:])
    mu, cov = engine.stats_finalize_mirrored(buf[:n_acc], buf[n_acc:2 * n_acc], buf[2 * n_acc:], shift, r, d)
    with np.errstate(all="ignore"):
        mu_ref, cov_ref = fo.online_statistics(files)
    assert np.abs(mu.cpu().numpy() - mu_ref).max() < 1e-11
    if r == 1:
        assert np.isnan(cov.cpu().numpy()).all() and np.isnan(cov_ref).all()
    else:
        assert np.abs(cov.cpu().numpy() - cov_ref).max() < 1e-9 * np.abs(cov_ref).max()
