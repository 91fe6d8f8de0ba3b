"""CPU: the Oobleck strides whose block length is not what forward allocates are refused.  A block's conv has kernel
2s, stride s, padding ceil(s/2) (reference models/autoencoders.py:75,86): for an odd decoder stride the transposed
conv gives L * s - 1 positions, for encoder stride 1 the conv gives L + 1.  Both the Python constructors and
satb_oobleck_create refuse them; every accepted stride gives the oracle's length."""
import ctypes
import math

import pytest
import torch

from oracle import oobleck_oracle as oo

DEC_BAD, ENC_BAD = [1, 3, 5, 7], [1]
DEC_OK, ENC_OK = [2, 4, 6, 8], [2, 3, 4, 5, 8]
SHIPPED = [[2, 4, 8, 8], [2, 4, 4, 8, 8]]


def _dec(strides):
    from stable_audio_tools.models.autoencoders import OobleckDecoder
    return OobleckDecoder(out_channels=2, channels=32, latent_dim=8, c_mults=[1] * len(strides), strides=strides,
                          use_snake=True)


def _enc(strides):
    from stable_audio_tools.models.autoencoders import OobleckEncoder
    return OobleckEncoder(in_channels=2, channels=32, latent_dim=8, c_mults=[1] * len(strides), strides=strides,
                          use_snake=True)


def _create(strides, decoder):
    from stable_audio_tools import _native
    lib = _native.lib()
    cfg = _native.SatbOobleckConfig()
    cfg.in_channels, cfg.channels, cfg.latent_dim, cfg.n_stages = 2, 32, 8, len(strides)
    for i, s in enumerate(strides):
        cfg.c_mults[i], cfg.strides[i] = 1, s
    cfg.is_decoder = int(decoder)
    h = ctypes.c_void_p()
    rc = lib.satb_oobleck_create(ctypes.byref(cfg), ctypes.byref(h))
    if rc == 0:
        lib.satb_oobleck_destroy(h)
    return rc, lib.satb_last_error()


@pytest.mark.parametrize("s", DEC_BAD)
def test_decoder_refuses_odd_strides(s):
    with pytest.raises(NotImplementedError, match=f"stride {s} .*even"):
        _dec([2, s])
    rc, msg = _create([2, s], True)
    assert rc != 0 and f"stride {s}".encode() in msg and b"even" in msg


@pytest.mark.parametrize("s", ENC_BAD)
def test_encoder_refuses_stride_1(s):
    with pytest.raises(NotImplementedError, match=f"stride {s} .*>= 2"):
        _enc([s, 2])
    rc, msg = _create([s, 2], False)
    assert rc != 0 and f"stride {s}".encode() in msg and b">= 2" in msg


@pytest.mark.parametrize("strides", SHIPPED)
def test_shipped_strides_are_accepted(strides):
    _dec(strides)
    _enc(strides)
    assert _create(strides, True)[0] == 0
    assert _create(strides, False)[0] == 0


@pytest.mark.parametrize("s", sorted(set(DEC_OK + ENC_OK)))
def test_accepted_strides_give_the_oracles_length(s):
    """The oracle's one-block decoder / encoder output length equals what forward allocates."""
    L = 12
    if s in DEC_OK:
        cfg = dict(out_channels=2, channels=4, c_mults=[1], strides=[s], latent_dim=2, final_tanh=False)
        sd = oo.make_oobleck_weights(oo.decoder_param_shapes(cfg), transposed=oo.decoder_transposed_prefixes(cfg))
        y = oo.oobleck_decoder(torch.randn(1, 2, L), sd, cfg)
        assert y.shape[-1] == L * _dec([s]).upsampling_ratio
        assert _create([s], True)[0] == 0
    if s in ENC_OK:
        cfg = dict(in_channels=2, channels=4, c_mults=[1], strides=[s], latent_dim=2)
        sd = oo.make_oobleck_weights(oo.encoder_param_shapes(cfg))
        h = oo.oobleck_encoder(torch.randn(1, 2, L * s), sd, cfg)
        assert h.shape[-1] == (L * s) // _enc([s]).downsampling_ratio
        assert _create([s], False)[0] == 0


def test_refused_strides_would_give_another_length():
    """What the refusal protects: the reference's own modules give L * s - 1 (odd decoder stride) and L + 1
    (encoder stride 1)."""
    L = 12
    for s in (3, 5):
        y = torch.nn.functional.conv_transpose1d(torch.zeros(1, 1, L), torch.zeros(1, 1, 2 * s), stride=s,
                                                 padding=math.ceil(s / 2))
        assert y.shape[-1] == L * s - 1
    h = torch.nn.functional.conv1d(torch.zeros(1, 1, L), torch.zeros(1, 1, 2), stride=1, padding=1)
    assert h.shape[-1] == L + 1
