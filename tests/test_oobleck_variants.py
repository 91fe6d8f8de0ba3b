"""CPU: Oobleck VAEs with ELU activations (use_snake=False) and nearest-neighbour upsampling (use_nearest_upsample=True).

- the variants oracle reproduces the real reference's outputs stored in the goldens;
- the nearest-upsample fold equals F.interpolate + F.conv1d(padding='same') in float64;
- the drop-in modules build the reference's module tree and state-dict keys, also through create_model_from_config
  (as an autoencoder and as a diffusion_cond pretransform), and load a reference state dict strictly;
- satb_oobleck_create_variant refuses what it cannot run, with a message; antialias_activation stays refused.
"""
import ctypes
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import load_golden
from oracle import oobleck_variants_oracle as ov

GOLDENS = [("oobleck_elu_small.npz", "dec"), ("oobleck_elu_small.npz", "enc"), ("oobleck_nearest_small.npz", "dec"),
           ("oobleck_elu_nearest_small.npz", "dec")]


def _golden_weights(g, kind):
    cfg = json.loads(str(g[kind + "_cfg"]))
    make = ov.make_decoder_weights if kind == "dec" else ov.make_encoder_weights
    sd = make(cfg, seed=int(g[kind + "_seed"]))
    wsum = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(wsum - float(g[kind + "_wsum"])) <= 1e-6 * wsum, "synthetic weight RNG drifted from the golden run"
    return cfg, sd


@pytest.mark.parametrize("name,kind", GOLDENS)
def test_oracle_matches_reference_golden(name, kind):
    g = load_golden(name)
    cfg, sd = _golden_weights(g, kind)
    if kind == "dec":
        y, ref = ov.oobleck_decoder(torch.from_numpy(g["z"]), sd, cfg), torch.from_numpy(g["audio"])
    else:
        y, ref = ov.oobleck_encoder(torch.from_numpy(g["a"]), sd, cfg), torch.from_numpy(g["h"])
    assert y.shape == ref.shape
    assert float((y - ref).abs().max()) <= 1e-5


@pytest.mark.parametrize("s", [2, 3, 4, 5, 8])
@pytest.mark.parametrize("L", [1, 2, 7])
def test_nearest_fold_equals_upsample_then_same_conv(s, L):
    g = torch.Generator().manual_seed(100 * s + L)
    x = torch.randn(2, 3, L, generator=g, dtype=torch.float64)
    w = torch.randn(4, 3, 2 * s, generator=g, dtype=torch.float64)
    ref = F.conv1d(F.interpolate(x, scale_factor=s, mode="nearest"), w, padding="same")
    y = ov.nearest_conv_folded(x, ov.nearest_fold(w, s))
    assert y.shape == ref.shape == (2, 4, L * s)
    assert float((y - ref).abs().max()) <= 1e-12


def test_operand_rounding_includes_the_fold():
    """Under operand rounding the oracle's nearest conv runs the folded, rounded 3-tap weights: its fp16 floor is that
    of the native decoder, not that of fp16(W) in the upsample-then-conv form."""
    from oracle import oobleck_oracle as oo
    g = load_golden("oobleck_elu_nearest_small.npz")
    cfg, sd = _golden_weights(g, "dec")
    z = torch.from_numpy(g["z"])
    ref = ov.oobleck_decoder(z, sd, cfg)
    with oo.operand_rounding(torch.float16):
        y = ov.oobleck_decoder(z, sd, cfg)
        x = torch.randn(1, 64, 5, generator=torch.Generator().manual_seed(3))
        w = oo.fold_weight_norm(sd["layers.1.layers.1.1.weight_g"], sd["layers.1.layers.1.1.weight_v"])
        folded = ov._nearest_upsample_conv(x, sd, "layers.1.layers.1.1.", 4)
    want = ov.nearest_conv_folded(x.half().float(), ov.nearest_fold(w, 4).float().half().float())
    assert torch.equal(folded, want)
    err = float((y - ref).norm() / ref.norm())
    assert 1e-5 < err < 1e-2, err


def _ref_keys(g, kind):
    return {k: tuple(v) for k, v in json.loads(str(g[kind + "_keys"])).items()}


@pytest.mark.parametrize("name,kind", GOLDENS)
def test_modules_have_the_reference_state_dict(name, kind):
    from stable_audio_tools.models.autoencoders import OobleckDecoder, OobleckEncoder
    g = load_golden(name)
    cfg, sd = _golden_weights(g, kind)
    m = (OobleckDecoder if kind == "dec" else OobleckEncoder)(**cfg)
    mine = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert mine == _ref_keys(g, kind)
    assert {k: tuple(v.shape) for k, v in sd.items()} == mine
    res = m.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    if kind == "dec" and cfg.get("use_nearest_upsample"):
        up = m.layers[1].layers[1]
        assert isinstance(up[0], torch.nn.Upsample) and up[1].bias is None
    if not cfg.get("use_snake", False):
        assert isinstance(m.layers[1].layers[0].layers[0] if kind == "enc" else m.layers[1].layers[0], torch.nn.ELU)


def _ae_config():
    g = load_golden("oobleck_elu_small.npz")
    dcfg, ecfg = json.loads(str(g["dec_cfg"])), json.loads(str(g["enc_cfg"]))
    assert "use_snake" not in dcfg and "use_snake" not in ecfg      # the reference's default: ELU
    return g, {"encoder": {"type": "oobleck", "config": ecfg}, "decoder": {"type": "oobleck", "config": dcfg},
               "bottleneck": {"type": "vae"}, "latent_dim": 8, "downsampling_ratio": 8, "io_channels": 2}


def _load_reference_sd(ae, g):
    _, dsd = _golden_weights(g, "dec")
    _, esd = _golden_weights(g, "enc")
    sd = {**{"decoder." + k: v for k, v in dsd.items()}, **{"encoder." + k: v for k, v in esd.items()}}
    assert set(sd) == {"decoder." + k for k in _ref_keys(g, "dec")} | {"encoder." + k for k in _ref_keys(g, "enc")}
    res = ae.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert set(ae.state_dict()) == set(sd)


def test_autoencoder_config_without_use_snake_builds_an_elu_vae():
    from stable_audio_tools import create_model_from_config
    g, ae_cfg = _ae_config()
    ae = create_model_from_config(json.loads(json.dumps({"model_type": "autoencoder", "sample_rate": 16000,
                                                          "model": ae_cfg})))
    assert isinstance(ae.decoder.layers[1].layers[0], torch.nn.ELU)
    _load_reference_sd(ae, g)


def test_diffusion_cond_with_an_elu_vae_pretransform_loads_the_reference_keys():
    from stable_audio_tools import create_model_from_config
    g, ae_cfg = _ae_config()
    diff = dict(io_channels=8, embed_dim=128, depth=1, num_heads=2, cond_token_dim=0, global_cond_dim=0,
                project_cond_tokens=False, transformer_type="continuous_transformer")
    model_config = {"model_type": "diffusion_cond", "sample_rate": 16000,
                    "model": {"io_channels": 8, "diffusion": {"type": "dit", "config": diff},
                              "pretransform": {"type": "autoencoder", "config": ae_cfg}}}
    m = create_model_from_config(json.loads(json.dumps(model_config)))
    ae = m.pretransform.model
    assert isinstance(ae.encoder.layers[1].layers[0].layers[0], torch.nn.ELU)
    _load_reference_sd(ae, g)
    assert {k[len("pretransform.model."):] for k in m.state_dict() if k.startswith("pretransform.")} == set(ae.state_dict())


def test_nearest_decoder_accepts_odd_strides_and_transposed_still_refuses_them():
    from stable_audio_tools.models.autoencoders import OobleckDecoder
    dec = OobleckDecoder(out_channels=2, channels=32, latent_dim=8, c_mults=[1, 1, 1], strides=[3, 5, 7],
                         use_nearest_upsample=True)
    assert dec.upsampling_ratio == 105
    with pytest.raises(NotImplementedError, match="stride 3 .*even"):
        OobleckDecoder(out_channels=2, channels=32, latent_dim=8, c_mults=[1], strides=[3])
    with pytest.raises(NotImplementedError, match="stride 1 .*>= 2"):
        OobleckDecoder(out_channels=2, channels=32, latent_dim=8, c_mults=[1], strides=[1], use_nearest_upsample=True)


def test_antialias_activation_is_refused_with_the_reason():
    from stable_audio_tools.models.autoencoders import OobleckDecoder, OobleckEncoder
    for cls, kw in ((OobleckDecoder, dict(out_channels=2)), (OobleckEncoder, dict(in_channels=2))):
        for use_snake in (False, True):
            with pytest.raises(NotImplementedError, match="alias_free_torch"):
                cls(**kw, channels=32, latent_dim=8, c_mults=[1], strides=[2], use_snake=use_snake,
                    antialias_activation=True)


def _create(strides, decoder, act, nearest):
    from stable_audio_tools import _native
    lib = _native.lib()
    cfg = _native.SatbOobleckConfig()
    cfg.in_channels, cfg.channels, cfg.latent_dim, cfg.n_stages = 2, 32, 8, len(strides)
    for i, s in enumerate(strides):
        cfg.c_mults[i], cfg.strides[i] = 1, s
    cfg.is_decoder = int(decoder)
    h = ctypes.c_void_p()
    rc = lib.satb_oobleck_create_variant(ctypes.byref(cfg), act, nearest, ctypes.byref(h))
    if rc == 0:
        lib.satb_oobleck_destroy(h)
    return rc, lib.satb_last_error()


def test_create_variant_validates_its_options():
    bad = [(([2, 4], True, 2, 0), b"unknown activation 2"), (([2, 4], True, -1, 0), b"unknown activation -1"),
           (([2, 4], True, 0, 2), b"nearest_upsample must be 0 or 1"),
           (([2, 4], False, 0, 1), b"decoder only"), (([2, 4], False, 1, 1), b"decoder only"),
           (([3, 4], True, 1, 0), b"even"), (([1, 4], True, 0, 1), b"stride 1"), (([1, 2], False, 1, 0), b">= 2")]
    for args, msg in bad:
        rc, err = _create(*args)
        assert rc != 0 and msg in err, (args, rc, err)
    for args in (([2, 4], True, 1, 0), ([2, 4], False, 1, 0), ([3, 5, 7], True, 0, 1), ([3, 2], True, 1, 1),
                 ([2, 4], True, 0, 0)):
        rc, err = _create(*args)
        assert rc == 0, (args, err)
