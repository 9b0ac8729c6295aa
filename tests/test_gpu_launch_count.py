"""The library's launch counter (fad_launch_count, bench.py's gpu_launches) is exact: every entry-point family, run once
under torch.profiler, launches as many of the library's kernels as the counter advances by.  The "a rejected call
launched nothing" assertions of the stage tests rely on it.  A second test runs one engine per device in one process
(the kernel setup is per handle) and checks that the devices agree bitwise."""
import re

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from fadtk_b200 import _native, synth, weights, weights_clap, weights_encodec as we, weights_w2v as w2w, \
    weights_whisper as wh

pytestmark = pytest.mark.gpu

# the fad:: kernels of the headers and the two the library defines in its own translation unit
LIBRARY_KERNEL = re.compile(r"\bfad::|\bwlo_absmax_kernel\b|\bdmma_peak_kernel\b")
W2V = {"w2v2-base": ("w2v2", "base"), "hubert-large": ("hubert", "large"), "wavlm-base": ("wavlm", "base")}
W2V_LEN = 16000
ENC_LEN = 24000                       # max_chunk_samples = one clip: two clips run as two conv chunks


@pytest.fixture(scope="module")
def eng():
    """A handle of this module's own: the models it loads do not replace the session engine's."""
    e = _native.Engine(torch.cuda.current_device(), max_examples=64)
    yield e
    e.close()


def counted(eng, fn):
    """(library kernels the profiler saw, launch-counter delta) of one call of fn"""
    torch.cuda.synchronize()
    before = eng.launches
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kernels = [e.name for e in prof.events()
               if e.device_type == torch.autograd.DeviceType.CUDA and LIBRARY_KERNEL.search(e.name)]
    return len(kernels), eng.launches - before


# ------------------------------------------------------------------------------------------------ loads
def load_vggish(eng):
    eng.vggish_load(weights.pack_vggish(weights.synthetic_vggish_state(0)))        # every layer split


def load_clap(eng):
    eng.clap_load(weights_clap.pack_clap(weights_clap.synthetic_clap_state(0)), max_chunks=8)


def load_whisper(eng):
    sd, start = wh.load_whisper_state(size="tiny")
    eng.whisper_load(wh.config_of(sd), wh.pack_whisper(sd, start), max_clips=2)


def load_encodec(variant):
    return lambda eng: eng.encodec_load(we.pack_encodec(we.synthetic_encodec_state(0, variant)), ENC_LEN, variant)


def load_w2v(name):
    def load(eng):
        arch = dict(w2w.ARCH[W2V[name]])
        arch["layers"] = 2
        sd = w2w.synthetic_w2v_state(0, **arch)
        eng.w2v_load(w2w.config_of(sd), w2w.pack_w2v(sd), 2, max_len=W2V_LEN)
    return load


LOADS = {"vggish": load_vggish, "clap": load_clap, "whisper": load_whisper, "encodec-24k": load_encodec("24k"),
         "encodec-48k": load_encodec("48k"), **{n: load_w2v(n) for n in W2V}}


def slot(name):
    return "w2v" if name in W2V else name.split("-")[0]


def ensure(eng, name):
    """the model `name` in its slot of the engine (loaded outside any profile)"""
    if eng.owners.get(slot(name)) != name:
        LOADS[name](eng)
        eng.owners[slot(name)] = name


# ------------------------------------------------------------------------------------------------ forwards
def pcm(clips, dev):
    return torch.from_numpy(np.concatenate(clips)).to(dev)


def vggish(eng):
    ensure(eng, "vggish")
    clips = [synth.musiclike_clip(i, 3.0, 16000) for i in range(2)]
    ex, _ = eng.vggish_plan(np.array([0, len(clips[0]), len(clips[0]) + len(clips[1])], dtype=np.int64))
    x, ex = pcm(clips, eng.torch_device), torch.from_numpy(ex).to(eng.torch_device)
    return lambda: eng.vggish_forward(x, ex)


def clap(eng):
    ensure(eng, "clap")
    clip = synth.musiclike_clip(7, 2.5, 48000)                                        # three windows
    plan = eng.clap_plan_to_device(eng.clap_plan_frames(np.array([0, len(clip)], dtype=np.int64)))
    x = pcm([clip], eng.torch_device)
    return lambda: eng.clap_forward(x, plan)


def whisper(eng):
    ensure(eng, "whisper")
    clip = synth.musiclike_clip(4, 2.0, 16000)
    dev = eng.torch_device
    x = pcm([clip], dev)
    start, n = torch.zeros(1, dtype=torch.int64, device=dev), torch.full((1,), len(clip), dtype=torch.int32, device=dev)
    return lambda: eng.whisper_forward(x, start, n)


def encodec(variant):
    def prepare(eng):
        ensure(eng, f"encodec-{variant}")
        x = pcm([synth.musiclike_clip(i, 1.0, ENC_LEN) for i in range(2)], eng.torch_device).view(2, ENC_LEN)
        return lambda: eng.encodec_forward(x)
    return prepare


def w2v(name):
    def prepare(eng):
        ensure(eng, name)
        x = pcm([synth.musiclike_clip(i, 1.0, W2V_LEN) for i in range(2)], eng.torch_device).view(2, W2V_LEN)
        return lambda: eng.w2v_forward(x, 2)
    return prepare


def statistics(eng):
    dev = eng.torch_device
    g = torch.Generator(device=dev).manual_seed(1)
    emb = torch.randn((300, 128), generator=g, device=dev).half()
    shift = emb[0].clone()
    idx = torch.arange(0, 300, 3, device=dev)
    acc, acc64, acc16 = eng.stats_new(128), eng.stats_new(128), eng.stats_new(128)

    def run():
        eng.stats_accumulate(emb, shift, acc)
        eng.stats_accumulate(emb, shift, acc, tensor_core=2)
        eng.stats_accumulate_gather(emb, idx, shift, acc)
        eng.stats_finalize(acc, shift, 128)
        m64, m16 = eng.file_means(emb, 3)
        eng.stats_accumulate_f64(m64, acc64)
        eng.stats_accumulate_f64(m16, acc16)
        eng.stats_finalize_mirrored(acc, acc64, acc16, shift, 3, 128)
    return run


def frechet(eng):
    dev = eng.torch_device
    g = torch.Generator(device=dev).manual_seed(2)
    x = torch.randn((200, 128), generator=g, device=dev, dtype=torch.float64)
    y = torch.randn((200, 128), generator=g, device=dev, dtype=torch.float64)
    mu1, cov1, mu2, cov2 = x.mean(0), torch.cov(x.T).contiguous(), y.mean(0), torch.cov(y.T).contiguous()
    emb = torch.randn((90, 128), generator=g, device=dev).half()
    emb100 = torch.randn((90, 100), generator=g, device=dev).half()
    off = torch.tensor([0, 30, 90], dtype=torch.int64, device=dev)
    base100 = _native.Baseline(eng, mu1[:100], cov1[:100, :100].contiguous())

    def run():
        eng.frechet(mu1, cov1, mu2, cov2)
        base = _native.Baseline(eng, mu1, cov1)
        base.frechet(mu2, cov2)
        base.frechet_batched(emb, off)                                                  # d % 64 == 0: DMMA statistics
        base100.frechet_batched(emb100, off)                                            # the CUDA-core ones
    return run


def kad(eng):
    dev = eng.torch_device
    g = torch.Generator(device=dev).manual_seed(3)
    z = torch.randn((400, 64), generator=g, device=dev).half()
    sigma = torch.tensor(2.0, dtype=torch.float64, device=dev)
    off = torch.tensor([0, 50, 120, 200], dtype=torch.int64, device=dev)

    def run():
        eng.kad_median_sq(z[:150].contiguous())
        eng.kad_sums(z, 150, sigma)
        eng.kad_song_sums(z, 200, off, sigma)
    return run


def resample(eng):
    dev = eng.torch_device
    x = torch.from_numpy(synth.musiclike_clip(5, 1.0, 44100)).to(dev)
    return lambda: (eng.resample(x, 44100, 16000), eng.resample(x, 16000, 16000))


def loads(eng):
    """every model's load: each notes its hi/lo weights with one launch per tensor"""
    def run():
        for name, load in LOADS.items():
            load(eng)
            eng.owners[slot(name)] = name
    return run


def split_linear(eng):
    """fad_linear and fad_umma_layer with caller-owned hi/lo weights, which they check on every call"""
    dev = eng.torch_device
    g = torch.Generator().manual_seed(4)
    a = torch.randn((200, 192), generator=g).half().to(dev)
    w = weights.split_hi_lo_tiles(torch.randn((256, 192), generator=g) * 0.1).to(dev)
    bias = torch.randn(256, generator=g).to(dev)
    out = torch.empty((200, 256), dtype=torch.float16, device=dev)
    x = torch.randn((4, 12, 8, 64), generator=g).half().to(dev)
    wc = weights.split_hi_lo_tiles(torch.randn((128, 9 * 64), generator=g) * 0.1).to(dev)
    bc = torch.randn(128, generator=g).to(dev)

    def run():
        eng.linear(a, 200, 192, w, bias, 256, split_w=1, out16=out)
        eng.umma_layer(x, wc, bc, 9, 1, 0, split_w=True)
    return run


FAMILIES = {"vggish": vggish, "clap": clap, "whisper": whisper, "encodec-24k": encodec("24k"),
            "encodec-48k": encodec("48k"), **{n: w2v(n) for n in W2V}, "statistics": statistics, "frechet": frechet,
            "kad": kad, "resample": resample, "loads": loads, "split-linear": split_linear}


@pytest.mark.parametrize("family", list(FAMILIES))
def test_launch_count_matches_profiler(eng, family):
    with torch.cuda.device(eng.device):
        run = FAMILIES[family](eng)
        seen, count = counted(eng, run)
    assert seen > 0, "the profiler saw none of the library's kernels"
    assert count == seen, f"{family}: the launch counter advanced by {count}, the profiler saw {seen} library kernels"


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible devices")
def test_engines_on_two_devices_agree():
    """One engine per device in one process: each device sets its own kernel attributes and GEMM cluster count, and
    the VGGish forward and a split-weight linear give bitwise the same results on both."""
    g = torch.Generator().manual_seed(5)
    a = torch.randn((200, 192), generator=g).half()
    w = weights.split_hi_lo_tiles(torch.randn((256, 192), generator=g) * 0.1)
    bias = torch.randn(256, generator=g)
    results = []
    for dev in (0, 1):
        with torch.cuda.device(dev):
            e = _native.Engine(dev, max_examples=64)
            emb = vggish(e)().cpu()
            out = torch.empty((200, 256), dtype=torch.float16, device=e.torch_device)
            e.linear(a.to(e.torch_device), 200, 192, w.to(e.torch_device), bias.to(e.torch_device), 256, split_w=1,
                     out16=out)
            results.append((emb, out.cpu()))
            e.close()
    for x, y in zip(*results):
        assert torch.equal(x, y)
