"""CPU: the time-sharded Oobleck decode / encode's host side (satb_oobleck_group_*, AudioAutoencoder.shard_time): the
split rule and its recompute margin against a brute-force receptive field, the refusals, shard_time's argument checks
and the ctypes signatures of the new entry points.  Nothing here touches a GPU."""
import ctypes

import pytest
import torch
from torch.nn import functional as F

from helpers import ROOT

SAO = dict(c_mults=[1, 2, 4, 8, 16], strides=[2, 4, 4, 8, 8])

# name -> (decoder?, strides, nearest upsampling); the margin depends on the layer list only, not on the widths
LAYER_LISTS = {
    "sao_dec": (True, SAO["strides"], False),
    "sao_dec_nearest": (True, SAO["strides"], True),
    "sao_enc": (False, SAO["strides"], False),
    "small_dec": (True, [2, 4, 8], False),
    "small_enc": (False, [2, 4, 8], False),
    "two_stage_dec": (True, [2, 4], False),
    "odd_nearest_dec": (True, [3, 5], True),
    "odd_enc": (False, [3, 2, 5], False),
}


def _module(name, **kw):
    from stable_audio_tools.models.autoencoders import OobleckDecoder, OobleckEncoder
    dec, strides, nearest = LAYER_LISTS[name]
    base = dict(dict(channels=32, c_mults=[1] * len(strides), strides=strides, latent_dim=8), **kw)
    if dec:
        return OobleckDecoder(out_channels=2, use_nearest_upsample=nearest, **base)
    return OobleckEncoder(in_channels=2, **base)


def _plan(name, world, L):
    from stable_audio_tools import _native
    m = _module(name)
    return _native.oobleck_group_plan(world, L, m.native_config(), LAYER_LISTS[name][2])


# ------------------------------------------------------------------------- brute-force receptive field
def _linear_walk(mod, x):
    """The module's layer list on one channel with all-ones kernels and identity activations: a linear map with no
    cancellation, whose input gradient is non-zero exactly where the output depends on the input."""
    from torch import nn
    from stable_audio_tools.models.autoencoders import ResidualUnit
    if isinstance(mod, ResidualUnit):
        return x + _linear_walk(mod.layers, x)
    if isinstance(mod, nn.Sequential):
        for sub in mod:
            x = _linear_walk(sub, x)
        return x
    if isinstance(mod, nn.Conv1d):
        w = torch.ones(1, 1, mod.kernel_size[0], dtype=x.dtype)
        return F.conv1d(x, w, stride=mod.stride, padding=mod.padding, dilation=mod.dilation)
    if isinstance(mod, nn.ConvTranspose1d):
        w = torch.ones(1, 1, mod.kernel_size[0], dtype=x.dtype)
        return F.conv_transpose1d(x, w, stride=mod.stride, padding=mod.padding, dilation=mod.dilation)
    if isinstance(mod, nn.Upsample):
        return F.interpolate(x, scale_factor=mod.scale_factor, mode="nearest")
    if hasattr(mod, "layers"):            # EncoderBlock / DecoderBlock
        return _linear_walk(mod.layers, x)
    return x                              # SnakeBeta, ELU, Tanh, Identity: elementwise, zero at zero


def _brute_force_margin(name):
    """Latents the outputs of one interior latent read, on either side (the encoder's in whole latents of samples)."""
    dec, strides, _ = LAYER_LISTS[name]
    m = _module(name)
    R = 1
    for s in strides:
        R *= s
    L = 160
    j = L // 2
    x = torch.zeros(1, 1, L * (1 if dec else R), dtype=torch.float64, requires_grad=True)
    y = _linear_walk(m.layers, x)
    assert y.shape[-1] == L * (R if dec else 1)
    (y[..., j * R:(j + 1) * R] if dec else y[..., j]).sum().backward()
    need = torch.nonzero(x.grad[0, 0] != 0).flatten()
    lo, hi = int(need.min()), int(need.max())
    if dec:
        return max(j - lo, hi - j)
    return max(-(-(j * R - lo) // R), -(-(hi - ((j + 1) * R - 1)) // R))


@pytest.mark.parametrize("name", sorted(LAYER_LISTS))
def test_margin_is_the_brute_force_receptive_field(name):
    assert _plan(name, 1, 400)[2] == _brute_force_margin(name)


def test_margin_values():
    assert _plan("sao_dec", 2, 1024)[2] == 10
    assert _plan("sao_dec_nearest", 2, 1024)[2] == 10
    assert _plan("sao_enc", 2, 1024)[2] == 8


# ------------------------------------------------------------------------- the split
@pytest.mark.parametrize("name", ["sao_dec", "sao_enc", "small_dec", "odd_nearest_dec"])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 7, 8])
@pytest.mark.parametrize("L", [1, 7, 33, 64, 101, 1024, 6144])
def test_plan_tiles_the_item_and_clips_the_margin_at_its_ends(name, world, L):
    from stable_audio_tools import _native
    m = _plan(name, 1, 400)[2]
    if world > L or (world > 1 and L // world < m):
        with pytest.raises(_native.NativeError, match="exceeds" if world > L else "recompute margin"):
            _plan(name, world, L)
        return
    begin, ext, margin = _plan(name, world, L)
    assert margin == m and len(begin) == world + 1 and len(ext) == world
    assert begin[0] == 0 and begin[-1] == L
    sizes = [b - a for a, b in zip(begin, begin[1:])]
    assert min(sizes) >= 1 and max(sizes) - min(sizes) <= 1          # an even split
    for r, (lo, hi) in enumerate(ext):
        assert lo == max(begin[r] - m, 0) and hi == min(begin[r + 1] + m, L)
        assert lo <= begin[r] and hi >= begin[r + 1]
        if world > 1:
            assert min(sizes) >= m
    assert ext[0][0] == 0 and ext[-1][1] == L


def test_plan_refusals_come_with_their_messages():
    from stable_audio_tools import _native
    with pytest.raises(_native.NativeError, match="world 8 exceeds the 7 latents"):
        _plan("sao_dec", 8, 7)
    with pytest.raises(_native.NativeError, match="fewer than the recompute margin of 10"):
        _plan("sao_dec", 2, 7)
    with pytest.raises(_native.NativeError, match="world must be 1 .. 8"):
        _plan("sao_dec", 9, 6144)
    with pytest.raises(_native.NativeError, match="L >= 1"):
        _plan("sao_dec", 1, 0)
    assert _plan("sao_dec", 1, 7) == ([0, 7], [(0, 7)], 10)           # one rank: no interior side, nothing refused
    enc = _module("sao_enc").native_config()
    with pytest.raises(_native.NativeError, match="nearest_upsample"):
        _native.oobleck_group_plan(2, 1024, enc, True)


# ------------------------------------------------------------------------- group create / call refusals
def _handles(n, **kw):
    from stable_audio_tools import _native
    hs = []
    for _ in range(n):
        h = ctypes.c_void_p()
        cfg = _module("small_dec", **kw).native_config()
        assert _native.lib().satb_oobleck_create_variant(ctypes.byref(cfg), 0, 0, ctypes.byref(h)) == 0
        hs.append(h)
    return hs


def _create(hs):
    from stable_audio_tools import _native
    lib = _native.lib()
    g = ctypes.c_void_p()
    arr = (ctypes.c_void_p * len(hs))(*[h.value for h in hs])
    ids = (ctypes.c_int * len(hs))(*([0] * len(hs)))
    rc = lib.satb_oobleck_group_create(arr, ids, len(hs), ctypes.byref(g))
    return rc, lib.satb_last_error().decode()


def _destroy(hs):
    from stable_audio_tools import _native
    for h in hs:
        _native.lib().satb_oobleck_destroy(h)


def test_group_create_refuses_mixed_models_shared_handles_and_unloaded_weights():
    hs = _handles(1) + _handles(1, operand_dtype="bf16")
    rc, err = _create(hs)
    _destroy(hs)
    assert rc != 0 and "config" in err
    hs = _handles(1)
    rc, err = _create(hs * 2)
    assert rc != 0 and "its own handle" in err
    rc, err = _create(hs)
    _destroy(hs)
    assert rc != 0 and "finalized" in err
    rc, err = _create(_handles(0))
    assert rc != 0 and "world" in err


def test_group_calls_refuse_null_arguments():
    from stable_audio_tools import _native
    lib = _native.lib()
    assert lib.satb_oobleck_group_decode(None, None, None, 1, 8, None) != 0
    assert b"bad argument" in lib.satb_last_error()
    assert lib.satb_oobleck_group_encode(None, None, None, 1, 8, None) != 0
    lib.satb_oobleck_group_destroy(None)


# ------------------------------------------------------------------------- shard_time's argument checks
def _dit():
    from stable_audio_tools.models.dit import DiffusionTransformer
    return DiffusionTransformer(io_channels=64, embed_dim=256, depth=1, num_heads=4,
                                transformer_type="continuous_transformer")


def _autoencoder():
    from stable_audio_tools.models.autoencoders import AudioAutoencoder
    return AudioAutoencoder(_module("small_enc", latent_dim=8), _module("small_dec"), latent_dim=8,
                            downsampling_ratio=64, sample_rate=16000, io_channels=2)


@pytest.mark.parametrize("devices,exc", [
    (["cuda:0"] * 9, ValueError),                     # 1 to 8 devices
    ([], ValueError),
    (["cuda:0", "cpu"], "NativeError"),                # CUDA devices only
])
def test_shard_time_refuses_what_shard_tokens_refuses_in_a_flat_list(devices, exc):
    from stable_audio_tools import _native
    from stable_audio_tools.models.pretransforms import AutoencoderPretransform
    exc = _native.NativeError if exc == "NativeError" else exc
    with pytest.raises(exc) as dit_err:
        _dit().shard_tokens(devices)
    ae = _autoencoder()
    for target in (ae, ae.decoder, ae.encoder, AutoencoderPretransform(ae)):
        with pytest.raises(exc) as err:
            target.shard_time(devices)
        assert str(err.value).replace("shard_time", "shard_tokens") == str(dit_err.value)
    assert ae.decoder.__dict__["_shard"] is None and ae.encoder.__dict__["_shard"] is None


def test_shard_time_takes_a_flat_list_only_and_none_returns_to_one_device():
    from stable_audio_tools.models.pretransforms import AutoencoderPretransform
    ae = _autoencoder()
    with pytest.raises(ValueError, match="flat list"):
        ae.shard_time([["cuda:0"], ["cuda:0"]])
    assert AutoencoderPretransform(ae).shard_time(["cuda:0", "cuda:0", "cuda:1"]).model is ae
    for m in (ae.encoder, ae.decoder):
        sh = m.__dict__["_shard"]
        assert [str(d) for d in sh["devices"]] == ["cuda:0", "cuda:0", "cuda:1"] and sh["handles"] is None
    ae.shard_time(None)
    assert ae.decoder.__dict__["_shard"] is None and ae.encoder.__dict__["_shard"] is None
    assert ae.shard_time(("cuda:0",)) is ae                            # a tuple, and one rank, are fine


def test_ctypes_signatures_of_the_group_entry_points():
    from stable_audio_tools import _native
    VP, I, LL = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    S = _native.SIGNATURES
    assert S["satb_oobleck_group_plan"] == (I, [I, I, ctypes.POINTER(_native.SatbOobleckConfig), I, VP, VP, VP])
    assert S["satb_oobleck_group_create"] == (I, [VP, VP, I, ctypes.POINTER(VP)])
    assert S["satb_oobleck_group_destroy"] == (None, [VP])
    assert S["satb_oobleck_group_decode"] == (I, [VP, VP, VP, I, I, VP])
    assert S["satb_oobleck_group_encode"] == (I, [VP, VP, VP, I, LL, VP])
    header = open(f"{ROOT}/include/satb200.h").read()
    for decl in ("int satb_oobleck_group_create(SatbOobleck* const* handles, const int* devices, int world, "
                 "SatbOobleckGroup** out);",
                 "void satb_oobleck_group_destroy(SatbOobleckGroup* g);",
                 "int satb_oobleck_group_decode(SatbOobleckGroup* g, const float* z, float* audio, int B, int L, "
                 "void* stream);"):
        assert decl in header
    lib = _native.lib()
    for name in S:
        if name.startswith("satb_oobleck_group_"):
            assert getattr(lib, name).argtypes == S[name][1]
