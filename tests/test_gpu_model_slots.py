"""Every model slot of a handle (VGGish, CLAP, Whisper, Encodec, the wav2vec family) is loaded all or nothing.  A load
the library rejects - a null tensor pointer right after the first hi/lo weight, or an argument out of range - launches
nothing and leaves the model that was loaded in place: its forward gives bitwise the output it gave before.  Handles
that load every slot and are destroyed, a few times over, leave nothing behind that a later handle would trip over.
The models are the seeded synthetic ones of test_gpu_launch_count.py."""
import ctypes as C
from functools import lru_cache

import numpy as np
import pytest
import torch

from fadtk_b200 import _native, synth, weights, weights_clap, weights_encodec as we, weights_w2v as w2w, \
    weights_whisper as wh

pytestmark = pytest.mark.gpu

W2V = {"w2v2-base": ("w2v2", "base"), "hubert-large": ("hubert", "large"), "wavlm-base": ("wavlm", "base")}
W2V_LEN = 16000
ENC_LEN = 24000                       # max_chunk_samples = one clip
NULL = "null tensor pointer"


@pytest.fixture(scope="module")
def eng():
    """A handle of this module's own: the models it loads do not replace the session engine's."""
    e = _native.Engine(torch.cuda.current_device(), max_examples=64)
    yield e
    e.close()


def pointers(tensors, null_at=None):
    """a c_void_p array of the tensors' data (None at null_at)"""
    ptrs = [t.data_ptr() for t in tensors]
    if null_at is not None:
        ptrs[null_at] = None
    return (C.c_void_p * len(ptrs))(*ptrs)


def pcm(clips, dev):
    return torch.from_numpy(np.concatenate(clips)).to(dev)


# ------------------------------------------------------------------------------------------------ the slots
@lru_cache(maxsize=None)
def vggish_packed():
    return weights.pack_vggish(weights.synthetic_vggish_state(0))                 # every layer split


class Vggish:
    def load(self, eng):
        eng.vggish_load(vggish_packed())

    def raw_load(self, eng, bad):
        """fad_vggish_load with conv2's bias (after conv2's hi/lo weight) null"""
        assert bad == NULL
        p = vggish_packed()
        w = _native.VggishWeights()
        w.conv1_w_host, w.conv1_b_host = p["conv1.w"].data_ptr(), p["conv1.b"].data_ptr()
        for i in range(5):
            w.conv_w_host[i], w.conv_b_host[i] = p[f"conv{i + 2}.w"].data_ptr(), p[f"conv{i + 2}.b"].data_ptr()
        for i in range(3):
            w.fc_w_host[i], w.fc_b_host[i] = p[f"fc{i + 1}.w"].data_ptr(), p[f"fc{i + 1}.b"].data_ptr()
        w.split_mask = int(p.get("split_mask", 0))
        w.conv_b_host[0] = None
        return _native.lib().fad_vggish_load(eng._h, C.byref(w))

    def forward(self, eng):
        clips = [synth.musiclike_clip(i, 3.0, 16000) for i in range(2)]
        ex, _ = eng.vggish_plan(np.array([0, len(clips[0]), len(clips[0]) + len(clips[1])], dtype=np.int64))
        x, ex = pcm(clips, eng.torch_device), torch.from_numpy(ex).to(eng.torch_device)
        return eng.vggish_forward(x, ex)


@lru_cache(maxsize=None)
def clap_packed():
    return weights_clap.pack_clap(weights_clap.synthetic_clap_state(0))


class Clap:
    def load(self, eng):
        eng.clap_load(clap_packed(), max_chunks=8)

    def raw_load(self, eng, bad):
        """tensor 8 is block 0's qkv weight, the first hi/lo one"""
        assert bad == NULL
        t = clap_packed()
        return _native.lib().fad_clap_load(eng._h, pointers(t, 9), len(t), 8)

    def forward(self, eng):
        clip = synth.musiclike_clip(7, 2.5, 48000)                                    # three windows
        plan = eng.clap_plan_to_device(eng.clap_plan_frames(np.array([0, len(clip)], dtype=np.int64)))
        return eng.clap_forward(pcm([clip], eng.torch_device), plan)


@lru_cache(maxsize=None)
def whisper_packed():
    sd, start = wh.load_whisper_state(size="tiny")
    return wh.config_of(sd), wh.pack_whisper(sd, start)


class Whisper:
    def load(self, eng):
        cfg, t = whisper_packed()
        eng.whisper_load(cfg, t, max_clips=2)

    def raw_load(self, eng, bad):
        assert bad == NULL
        cfg, t = whisper_packed()
        return _native.lib().fad_whisper_load(eng._h, (C.c_int * 5)(*cfg), pointers(t, 1), len(t), 2)

    def forward(self, eng):
        clip = synth.musiclike_clip(4, 2.0, 16000)
        dev = eng.torch_device
        start, n = torch.zeros(1, dtype=torch.int64, device=dev), torch.full((1,), len(clip), dtype=torch.int32, device=dev)
        return eng.whisper_forward(pcm([clip], dev), start, n)


@lru_cache(maxsize=None)
def encodec_packed(variant):
    return we.pack_encodec(we.synthetic_encodec_state(0, variant))


class Encodec:
    def __init__(self, variant):
        self.variant = variant

    def load(self, eng):
        eng.encodec_load(encodec_packed(self.variant), ENC_LEN, self.variant)

    def raw_load(self, eng, bad):
        t = encodec_packed(self.variant)
        variant = 0 if self.variant == "24k" else 1
        if bad == NULL:
            return _native.lib().fad_encodec_load(eng._h, pointers(t, 1), len(t), ENC_LEN, variant)
        return _native.lib().fad_encodec_load(eng._h, pointers(t), len(t), ENC_LEN, 2)

    def forward(self, eng):
        x = pcm([synth.musiclike_clip(i, 1.0, ENC_LEN) for i in range(2)], eng.torch_device).view(2, ENC_LEN)
        return eng.encodec_forward(x)


@lru_cache(maxsize=None)
def w2v_packed(name):
    arch = dict(w2w.ARCH[W2V[name]])
    arch["layers"] = 2
    sd = w2w.synthetic_w2v_state(0, **arch)
    return w2w.config_of(sd), w2w.pack_w2v(sd)


class W2v:
    def __init__(self, name):
        self.name = name

    def load(self, eng):
        cfg, t = w2v_packed(self.name)
        eng.w2v_load(cfg, t, 2, max_len=W2V_LEN)

    def raw_load(self, eng, bad):
        cfg, t = w2v_packed(self.name)
        c = (C.c_int * 7)(*cfg)
        if bad == NULL:
            return _native.lib().fad_w2v_load(eng._h, c, pointers(t, 1), len(t), 2, W2V_LEN)
        return _native.lib().fad_w2v_load(eng._h, c, pointers(t), len(t), 2, 399)

    def forward(self, eng):
        x = pcm([synth.musiclike_clip(i, 1.0, W2V_LEN) for i in range(2)], eng.torch_device).view(2, W2V_LEN)
        return eng.w2v_forward(x, 2)


MODELS = {"vggish": Vggish(), "clap": Clap(), "whisper": Whisper(), "encodec-24k": Encodec("24k"),
          "encodec-48k": Encodec("48k"), **{n: W2v(n) for n in W2V}}

REJECTED = [(n, NULL) for n in MODELS] + [(f"encodec-{v}", "variant must be 0") for v in ("24k", "48k")] + \
           [(n, "max_len too short") for n in W2V]


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("name,bad", REJECTED, ids=[f"{n}-{b.split()[0]}" for n, b in REJECTED])
def test_rejected_load_keeps_the_loaded_model(eng, name, bad):
    model = MODELS[name]
    with torch.cuda.device(eng.device):
        model.load(eng)
        first = model.forward(eng).cpu()
        torch.cuda.synchronize()
        before = eng.launches
        with pytest.raises(_native.NativeError, match=bad):
            _native._check(model.raw_load(eng, bad))
        assert eng.launches == before, "a rejected load launched a kernel"
        again = model.forward(eng).cpu()
    assert torch.equal(first, again), "the forward after a rejected load differs from the one before it"


def test_create_load_every_slot_destroy_cycles(eng):
    """Three handles in a row load every model into their slots (the Encodec and wav2vec slots several times over) and
    are destroyed; a fresh handle then runs the VGGish and CLAP forwards bitwise as this module's handle does."""
    with torch.cuda.device(eng.device):
        want = {}
        for name in ("vggish", "clap"):
            MODELS[name].load(eng)
            want[name] = MODELS[name].forward(eng).cpu()
        for _ in range(3):
            e = _native.Engine(eng.device, max_examples=64)
            for model in MODELS.values():
                model.load(e)
            e.close()
        e = _native.Engine(eng.device, max_examples=64)
        try:
            for name in want:
                MODELS[name].load(e)
                assert torch.equal(MODELS[name].forward(e).cpu(), want[name]), name
        finally:
            e.close()
