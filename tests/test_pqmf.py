"""CPU: the PQMF pretransform and the Oobleck autoencoders built around it.

- the float64 oracle (oracle/pqmf_oracle.py) against the real reference's goldens (tests/golden/pqmf_small.npz,
  oobleck_pqmf_small.npz): rel-L2 <= 2e-6 (the reference runs in fp32; measured <= 6e-7);
- our host-side filter design against the reference's buffers: the prototype bit for bit, the bank within 5e-7
  max-abs (the reference modulates in fp32, we in fp64 rounded once; measured <= 2.3e-7, about 1e-5 of the peak tap);
- the reference config builds through create_model_from_config and loads the reference state dict key for key;
- the output-length rules the native kernels implement;
- the host refusals and the satb_pqmf_* argument checks, none of which reaches CUDA.
"""
import ctypes
import json

import numpy as np
import pytest
import torch

from helpers import load_golden, rel_l2

BANKS = [(100, 16), (100, 32), (80, 64)]


def _bank(att, n):
    g = load_golden("pqmf_small.npz")
    p = f"a{att}_n{n}_"
    return g, p, torch.from_numpy(g[p + "filter_bank"])


@pytest.mark.parametrize("att,n", BANKS)
def test_oracle_matches_reference_golden(att, n):
    from oracle import pqmf_oracle as po
    g, p, bank = _bank(att, n)
    for name in ("long", "short"):
        x, y = torch.from_numpy(g[p + "x_" + name]), torch.from_numpy(g[p + "y_" + name])
        T = x.shape[-1]
        assert T % n != 0
        assert y.shape == (2, 2 * n, -(-T // n))
        assert rel_l2(po.analysis(x, bank), y.double()) <= 2e-6
    assert g[p + "x_short"].shape[-1] < bank.shape[-1]
    z, s = torch.from_numpy(g[p + "z"]), torch.from_numpy(g[p + "s"])
    assert s.shape == (2, 2, z.shape[-1] * n)
    assert rel_l2(po.synthesis(z, bank), s.double()) <= 2e-6


@pytest.mark.parametrize("att,n", BANKS)
def test_filter_design_reproduces_reference_buffers(att, n):
    from stable_audio_tools.models.pretransforms import PQMF
    g, p, bank = _bank(att, n)
    ours = PQMF(att, n)
    assert torch.equal(ours.prototype, torch.from_numpy(g[p + "prototype"]))
    assert ours.filter_bank.shape == bank.shape and ours.filter_bank.dtype == torch.float32
    err = (ours.filter_bank - bank).abs().max().item()
    print(f"({att}, {n}): bank max-abs {err:.3g} (peak {bank.abs().max().item():.3g})")
    assert err <= 5e-7


def test_analysis_then_synthesis_reconstructs():
    """Near-perfect reconstruction of the designed bank (what makes the pretransform usable): away from the edges the
    round trip returns the signal, delayed by nothing, to within the bank's aliasing (measured rel-L2 1.7e-3 for
    32 bands)."""
    from oracle import pqmf_oracle as po
    _, _, bank = _bank(100, 32)
    x = torch.randn(1, 2, 32 * 200, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    y = po.synthesis(po.analysis(x, bank), bank)
    assert y.shape == x.shape
    inner = slice(2048, -2048)
    assert rel_l2(y[..., inner], x[..., inner]) < 5e-3


def _ae_golden():
    from oracle import pqmf_oracle as po
    g = load_golden("oobleck_pqmf_small.npz")
    cfg = json.loads(str(g["config"]))
    gb = load_golden("pqmf_small.npz")
    sd = po.autoencoder_state_dict(cfg, gb["a100_n16_filter_bank"], gb["a100_n16_prototype"], int(g["seed"]))
    return g, cfg, sd


def test_autoencoder_oracle_matches_reference_golden():
    from oracle import pqmf_oracle as po
    g, cfg, sd = _ae_golden()
    bank = sd["pretransform.pqmf.filter_bank"]
    a, z = torch.from_numpy(g["a"]), torch.from_numpy(g["z"])
    h = po.encode(a, sd, cfg, bank)
    y = po.decode(z, sd, cfg, bank)
    assert h.shape == g["h"].shape and y.shape == g["y"].shape
    assert y.shape == (2, 2, 13 * 4 * 16)
    assert rel_l2(h, torch.from_numpy(g["h"])) <= 1e-5
    assert rel_l2(y, torch.from_numpy(g["y"])) <= 1e-5


def test_reference_config_builds_and_loads_the_state_dict_key_for_key():
    from stable_audio_tools.models.factory import create_model_from_config
    from stable_audio_tools.models.pretransforms import PQMFPretransform
    g, cfg, sd = _ae_golden()
    model = create_model_from_config(cfg)
    assert isinstance(model.pretransform, PQMFPretransform)
    assert model.pretransform.downsampling_ratio is None and model.pretransform.io_channels == 1
    ref_keys = json.loads(str(g["keys"]))
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == ref_keys
    assert set(sd) == set(ref_keys)
    model.load_state_dict(sd, strict=True)
    assert torch.equal(model.pretransform.pqmf.filter_bank, sd["pretransform.pqmf.filter_bank"])


def test_diffusion_pretransform_wraps_a_pqmf_autoencoder():
    from stable_audio_tools.models.factory import create_pretransform_from_config
    _, cfg, _ = _ae_golden()
    pt = create_pretransform_from_config({"type": "autoencoder", "config": cfg["model"]}, cfg["sample_rate"])
    assert pt.model.pretransform.pqmf.num_bands == 16 and pt.downsampling_ratio == 64


def test_pqmf_pretransform_from_config():
    from stable_audio_tools.models.factory import create_pretransform_from_config
    pt = create_pretransform_from_config({"type": "pqmf", "config": {"attenuation": 100, "num_bands": 32}}, 44100)
    assert pt.pqmf.filter_bank.shape == (32, 1024) and not pt.enable_grad
    assert sorted(pt.state_dict()) == ["pqmf.filter_bank", "pqmf.prototype"]


@pytest.mark.parametrize("kind", ["wavelet", "dac_pretrained", "audiocraft_pretrained"])
def test_other_pretransform_kinds_stay_refused(kind):
    from stable_audio_tools.models.factory import create_pretransform_from_config
    with pytest.raises(NotImplementedError, match="outside the native hot path"):
        create_pretransform_from_config({"type": kind, "config": {}}, 44100)


def test_other_nested_pretransforms_keep_the_refusal():
    from stable_audio_tools.models.autoencoders import AudioAutoencoder
    from stable_audio_tools.models.pretransforms import Pretransform
    with pytest.raises(NotImplementedError, match="nested pretransforms are outside the native hot path"):
        AudioAutoencoder(None, None, 8, 64, 44100, pretransform=Pretransform(False, 2, False))


@pytest.mark.parametrize("n", [3, 12, 1, 512])
def test_bad_band_counts_are_refused(n):
    from stable_audio_tools.models.pretransforms import PQMFPretransform
    with pytest.raises(ValueError, match="power of 2"):
        PQMFPretransform(100, n)


def test_unsupported_subband_widths_are_refused():
    """io_channels x num_bands must be a width the native Oobleck takes (a multiple of 8 up to 128)."""
    from stable_audio_tools.models.autoencoders import AudioAutoencoder, OobleckEncoder
    from stable_audio_tools.models.pretransforms import PQMFPretransform
    with pytest.raises(NotImplementedError, match="multiple of 8 up to 128"):
        AudioAutoencoder(None, None, 8, 64, 44100, io_channels=2, pretransform=PQMFPretransform(100, 128))
    with pytest.raises(NotImplementedError, match="multiple of 8 up to 128"):
        AudioAutoencoder(None, None, 8, 64, 44100, io_channels=3, pretransform=PQMFPretransform(100, 2))
    for c in (3, 12, 136):
        with pytest.raises(NotImplementedError, match="in_channels = "):
            OobleckEncoder(in_channels=c, channels=32, c_mults=[1], strides=[2], latent_dim=8)
    for c in (8, 64, 128):
        OobleckEncoder(in_channels=c, channels=32, c_mults=[1], strides=[2], latent_dim=8)


def test_cpu_tensors_are_refused():
    from stable_audio_tools import _native
    from stable_audio_tools.models.pretransforms import PQMFPretransform
    pt = PQMFPretransform(100, 16)
    with pytest.raises(_native.NativeError):
        pt.encode(torch.zeros(1, 2, 256))
    with pytest.raises(_native.NativeError):
        pt.decode(torch.zeros(1, 32, 16))


def test_abi_argument_checks():
    """satb_pqmf_* refuse bad arguments before any CUDA call (fake pointers, never dereferenced)."""
    from stable_audio_tools import _native
    lib = _native.lib()
    h = ctypes.c_void_p()
    for n, taps, msg in [(12, 512, b"power of 2"), (1, 512, b"power of 2"), (512, 4096, b"power of 2"),
                         (16, 520, b"multiple of 2 * num_bands"), (16, 16, b"multiple of 2 * num_bands"),
                         (16, 32768, b"at most")]:
        assert lib.satb_pqmf_create(n, taps, ctypes.byref(h)) != 0
        assert msg in lib.satb_last_error(), (n, taps, lib.satb_last_error())
    assert lib.satb_pqmf_create(16, 512, None) != 0
    fake = ctypes.c_void_p(1 << 20)
    assert lib.satb_pqmf_load_filter(None, fake, None) != 0 and b"null" in lib.satb_last_error()
    assert lib.satb_pqmf_analysis(None, fake, fake, 1, 2, 100, None) != 0 and b"null" in lib.satb_last_error()
    assert lib.satb_pqmf_synthesis(None, fake, fake, 1, 2, 100, None) != 0 and b"null" in lib.satb_last_error()
    lib.satb_pqmf_destroy(None)


def test_oobleck_abi_accepts_wide_io_and_refuses_other_widths():
    from stable_audio_tools import _native
    lib = _native.lib()
    h = ctypes.c_void_p()
    for c in (3, 4, 12, 136, 0):
        oc = _native.SatbOobleckConfig()
        oc.in_channels, oc.channels, oc.latent_dim, oc.n_stages = c, 32, 8, 1
        oc.c_mults[0], oc.strides[0] = 1, 2
        assert lib.satb_oobleck_create(ctypes.byref(oc), ctypes.byref(h)) != 0
        assert b"multiple of 8 up to 128" in lib.satb_last_error()
    for c in (1, 2, 8, 32, 128):
        for dec in (0, 1):
            oc = _native.SatbOobleckConfig()
            oc.in_channels, oc.channels, oc.latent_dim, oc.n_stages, oc.is_decoder = c, 32, 8, 1, dec
            oc.c_mults[0], oc.strides[0] = 1, 2
            assert lib.satb_oobleck_create(ctypes.byref(oc), ctypes.byref(h)) == 0, lib.satb_last_error()
            lib.satb_oobleck_destroy(h)
