"""CPU: the token-sharded DiT forward's host side (satb_dit_group_*, DiffusionTransformer.shard_tokens): the split rule,
the refusals, and the ctypes signatures of the new entry points.  Nothing here touches a GPU."""
import ctypes

import pytest

from helpers import ROOT


def _plan(world, P, L):
    from stable_audio_tools import _native
    return _native.group_plan(world, P, L)


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("P,L", [(1, 6144), (1, 1024), (0, 4096), (4, 2000), (1, 1100), (1, 300), (0, 9), (3, 5), (1, 7)])
def test_plan_covers_every_token_once_with_prepended_tokens_on_rank_0(world, P, L):
    N = P + L
    if world > N or (P > 0 and N - P < world - 1):
        pytest.skip("refused; see test_plan_refuses_more_ranks_than_tokens")
    tb = _plan(world, P, L)
    assert len(tb) == world + 1 and tb[0] == 0 and tb[-1] == N
    sizes = [b - a for a, b in zip(tb, tb[1:])]
    assert min(sizes) >= 1                       # no empty shard
    assert tb[1] >= P                            # the prepended tokens on rank 0
    if N >= 128 * world:
        assert all(b % 128 == 0 for b in tb[1:-1])                       # 128-token boundaries
        whole = sizes[:-1]                                                  # the last shard may end in a partial tile
        assert not whole or max(whole) - min(whole) <= 128                 # as even as whole tiles allow
    else:                                         # even, or rank 0 holds the prepended tokens and the rest is even
        rest = sizes if sizes[0] > P or world == 1 else sizes[1:]
        assert max(rest) - min(rest) <= 1


def test_plan_values():
    assert _plan(1, 1, 6144) == [0, 6145]
    assert _plan(2, 1, 6144) == [0, 3072, 6145]                 # 49 tiles of 128: 24 | 25
    assert _plan(8, 1, 6144) == [0, 768, 1536, 2304, 3072, 3840, 4608, 5376, 6145]
    assert _plan(4, 1, 1024) == [0, 256, 512, 768, 1025]
    assert _plan(3, 1, 300) == [0, 100, 200, 301]               # 301 < 3 * 128: even split of the tokens
    assert _plan(8, 0, 9) == [0, 1, 2, 3, 4, 5, 6, 7, 9]
    assert _plan(2, 3, 2) == [0, 3, 5]                          # rank 0 keeps all prepended tokens
    assert _plan(4, 200, 400) == [0, 256, 384, 512, 600]        # rank 0 takes the two tiles the prepend spans


def test_plan_refuses_more_ranks_than_tokens():
    from stable_audio_tools import _native
    with pytest.raises(_native.NativeError, match="exceeds"):
        _plan(8, 1, 6)
    with pytest.raises(_native.NativeError, match="world"):
        _plan(9, 1, 6144)
    with pytest.raises(_native.NativeError, match="fewer than one token"):
        _plan(4, 6, 2)                                          # 8 tokens, but 6 of them must stay on rank 0


def _cfg(**kw):
    from stable_audio_tools import _native
    base = dict(io_channels=64, embed_dim=256, depth=1, num_heads=4, cond_token_dim=128, global_cond_dim=256,
                project_cond_tokens=0, project_global_cond=1, global_cond_type=0, patch_size=1, operand_dtype=0)
    base.update(kw)
    return _native.SatbDitConfig(**base)


def _handles(n, setup=None, **cfg_kw):
    from stable_audio_tools import _native
    lib = _native.lib()
    hs = []
    for i in range(n):
        h = ctypes.c_void_p()
        assert lib.satb_dit_create(ctypes.byref(_cfg(**cfg_kw)), ctypes.byref(h)) == 0
        if setup is not None:
            assert setup(lib, h, i) == 0
        hs.append(h)
    return hs


def _create(hs, devices=None):
    from stable_audio_tools import _native
    lib = _native.lib()
    g = ctypes.c_void_p()
    arr = (ctypes.c_void_p * len(hs))(*[h.value for h in hs])
    ids = (ctypes.c_int * len(hs))(*(devices or [0] * len(hs)))
    rc = lib.satb_dit_group_create(arr, ids, len(hs), ctypes.byref(g))
    return rc, lib.satb_last_error().decode()


def _destroy(hs):
    from stable_audio_tools import _native
    for h in hs:
        _native.lib().satb_dit_destroy(h)


@pytest.mark.parametrize("option,msg", [
    (lambda lib, h, i: lib.satb_dit_set_conformer(h, 1), "conformer"),
    (lambda lib, h, i: lib.satb_dit_set_feedforward(h, 1024, 0, 3, 1), "use_conv"),
    (lambda lib, h, i: lib.satb_dit_set_attention_fp8(h, 1), "fp8"),
])
def test_group_create_refuses_the_token_convolutions_and_fp8_attention(option, msg):
    """Refused before any CUDA call, with its own error code (-5)."""
    hs = _handles(2, option)
    rc, err = _create(hs)
    _destroy(hs)
    assert rc == -5 and msg in err


def test_group_create_refuses_mixed_models_shared_handles_and_unloaded_weights():
    hs = _handles(1) + _handles(1, embed_dim=384, num_heads=6)
    rc, err = _create(hs)
    _destroy(hs)
    assert rc != 0 and "config" in err
    hs = _handles(1) + _handles(1, lambda lib, h, i: lib.satb_dit_set_positions(h, 0, 0, 0))
    rc, err = _create(hs)
    _destroy(hs)
    assert rc != 0 and "option" in err
    hs = _handles(1)
    rc, err = _create(hs * 2)
    assert rc != 0 and "its own handle" in err
    rc, err = _create(hs)
    _destroy(hs)
    assert rc != 0 and "finalized" in err


def test_group_forward_refuses_null_arguments():
    from stable_audio_tools import _native
    lib = _native.lib()
    assert lib.satb_dit_group_forward(None, None, None, None, 1, 8, 1.0, 0.0, None) != 0
    assert b"null" in lib.satb_last_error()


SHARD_REFUSALS = [
    (dict(conformer=True), "conformer"),
    (dict(ff_kwargs=dict(glu=False, use_conv=True, conv_kernel_size=3)), "use_conv"),
    (dict(attention_dtype="fp8"), "fp8"),
]


@pytest.mark.parametrize("kw,msg", SHARD_REFUSALS)
def test_shard_tokens_refuses_before_any_cuda_call(kw, msg):
    from stable_audio_tools.models.dit import DiffusionTransformer
    m = DiffusionTransformer(io_channels=64, embed_dim=256, depth=1, num_heads=4, cond_token_dim=128,
                             project_cond_tokens=False, transformer_type="continuous_transformer", **kw)
    with pytest.raises(NotImplementedError, match=msg):
        m.shard_tokens(["cuda:0", "cuda:0"])
    m.shard_tokens(None)                      # returning to one device is always fine


def test_sharded_forward_refuses_return_info_and_cpu_devices():
    import torch
    from stable_audio_tools import _native
    from stable_audio_tools.models.dit import DiffusionTransformer
    m = DiffusionTransformer(io_channels=64, embed_dim=256, depth=1, num_heads=4, transformer_type="continuous_transformer")
    with pytest.raises(_native.NativeError, match="not a CUDA device"):
        m.shard_tokens(["cuda:0", "cpu"])
    with pytest.raises(ValueError, match="1 to 8"):
        m.shard_tokens(["cuda:0"] * 9)
    m.shard_tokens(["cuda:0", "cuda:0"])
    with pytest.raises(NotImplementedError, match="return_info"):
        m(torch.zeros(1, 64, 16), torch.zeros(1), return_info=True)
    m.shard_tokens(None)


def test_ctypes_signatures_of_the_group_entry_points():
    from stable_audio_tools import _native
    VP, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    S = _native.SIGNATURES
    assert S["satb_dit_group_plan"] == (I, [I, I, I, VP])
    assert S["satb_dit_group_create"] == (I, [VP, VP, I, ctypes.POINTER(VP)])
    assert S["satb_dit_group_destroy"] == (None, [VP])
    assert S["satb_dit_group_forward"] == (I, [VP, VP, VP, VP, I, I, F, F, VP])
    header = open(f"{ROOT}/include/satb200.h").read()
    for decl in ("int satb_dit_group_plan(int world, int n_prepend, int L, int* token_begin);",
                 "int satb_dit_group_create(SatbDit* const* handles, const int* devices, int world, SatbDitGroup** out);",
                 "void satb_dit_group_destroy(SatbDitGroup* g);"):
        assert decl in header
    lib = _native.lib()
    for name in S:
        if name.startswith("satb_dit_group_"):
            assert getattr(lib, name).argtypes == S[name][1]
