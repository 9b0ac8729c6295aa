"""Pin oracle/encodec_oracle.py to an independent implementation of the same architecture: transformers'
EncodecModel.encoder (default config == encodec_24khz), with shared random weights.  CPU only."""
import numpy as np
import pytest
import torch

from fadtk_b200 import weights_encodec as we
from oracle import encodec_oracle as eo


SHORT = [("24k", 1), ("24k", 100), ("24k", 1919), ("24k", 1920), ("48k", 5), ("48k", 960)]


@pytest.mark.parametrize("variant,length", [("24k", 24000), ("24k", 24000 * 3 + 137), ("24k", 500), ("48k", 48000), ("48k", 31337)]
                         + SHORT)
def test_encoder_matches_independent_hf_port(variant, length):
    """Lengths up to 1920 (24 kHz) and 960 (48 kHz) samples reach a conv whose input is no longer than its padding,
    where Encodec's pad1d extends the input with zeros before it reflects."""
    tr = pytest.importorskip("transformers")
    sd = we.synthetic_encodec_state(3, variant)
    if variant == "24k":
        cfg = tr.EncodecConfig()
        assert list(cfg.upsampling_ratios)[::-1] == list(we.RATIOS) and cfg.use_causal_conv and cfg.norm_type == "weight_norm"
    else:
        cfg = tr.EncodecConfig(sampling_rate=48000, audio_channels=2, normalize=True, chunk_length_s=1.0, overlap=0.01,
                               norm_type="time_group_norm", use_causal_conv=False)
    enc = tr.EncodecModel(cfg).eval().encoder
    hf = enc.state_dict()
    assert set(hf) == set(sd) and all(hf[k].shape == sd[k].shape for k in hf)
    enc.load_state_dict(sd)
    x = 0.3 * torch.randn((2, 1 if variant == "24k" else 2, length), generator=torch.Generator().manual_seed(length))
    with torch.no_grad():
        want = enc(x)
    got = eo.encoder(x, sd)
    assert got.shape == want.shape == (2, 128, -(-length // 320))
    assert torch.allclose(got, want, atol=2e-5 * want.abs().max().item() + 1e-6), (got - want).abs().max()
    got64 = eo.encoder(x, sd, torch.float64)                   # the float64 mode the GPU stage tests compare with
    assert got64.dtype == torch.float64
    assert torch.allclose(got64, want.double(), atol=2e-5 * want.abs().max().item() + 1e-6), (got64 - want).abs().max()


def test_embed_shape_and_packing():
    sd = we.synthetic_encodec_state(0)
    e = eo.embed(0.1 * np.random.default_rng(0).standard_normal(24000 * 2), sd)
    assert e.shape == (150, 128) and e.dtype == np.float16                     # 75 frames per second
    pk = we.pack_encodec(sd)
    n_convs = 1 + 4 * 4 + 1
    assert len(pk) == 6 * n_convs + 3 * 2
    assert pk[0].shape == (2 * 128, 64) and pk[0].dtype == torch.float16       # conv0: 32 x (7 taps x 1 ch) -> [128 pad, 64 pad]
    w = we.effective_weight(sd, "layers.3")                                     # first down conv [64, 32, 4]
    assert torch.allclose(w.flatten(1).norm(dim=1), sd["layers.3.conv.parametrizations.weight.original0"].flatten())
    g = pk[6 * 4]                                                               # its GEMM weight: column = tap * 32 + c
    assert g.shape == (2 * 128, 128) and torch.equal(g[5, 2 * 32 + 7].float(), w[5, 7, 2].to(torch.float16).float())
    gp = pk[6 * 4 + 4]                               # time-packed: 2 outputs per row from 4 + 2 = 6 input steps (stride 2)
    assert we.time_pack(64) == 2 and gp.shape == (2 * 128, 6 * 32)
    assert torch.equal(gp[64 + 5, (2 + 1) * 32 + 7].float(), w[5, 7, 1].to(torch.float16).float())     # output 1 is shifted by the stride
    assert not gp[:64, 4 * 32:].any() and not gp[64:128, :2 * 32].any()
