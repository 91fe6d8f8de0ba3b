"""CPU: the host side of the token-sharded forward's CUDA graph (satb_dit_group_graph_*): argument checks that return an
error code and a message before any CUDA call, and the ctypes signatures.  Nothing here touches a GPU."""
import ctypes

import pytest

from helpers import ROOT


def _lib():
    from stable_audio_tools import _native
    return _native.lib()


def test_graph_forward_refuses_null_arguments_without_a_device():
    lib = _lib()
    fake = ctypes.c_void_p(1 << 20)            # never dereferenced: every call below fails its checks first
    streams = (ctypes.c_void_p * 2)(1 << 21, 1 << 22)
    for args in [(None, fake, fake, fake, streams), (fake, None, fake, fake, streams), (fake, fake, None, fake, streams),
                 (fake, fake, fake, None, streams), (fake, fake, fake, fake, None)]:
        g, x, t, out, st = args
        rc = lib.satb_dit_group_graph_forward(g, x, t, out, 1, 8, 1.0, 0.0, st, None)
        assert rc != 0 and b"null" in lib.satb_last_error()


def test_graph_reset_and_stats_refuse_null_arguments():
    lib = _lib()
    assert lib.satb_dit_group_graph_reset(None) != 0
    assert b"null" in lib.satb_last_error()
    c, r, n = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_ulonglong()
    assert lib.satb_dit_group_graph_stats(None, ctypes.byref(c), ctypes.byref(r), ctypes.byref(n)) != 0
    assert b"null" in lib.satb_last_error()


def test_unsharded_model_has_no_graph_stats():
    from stable_audio_tools.models.dit import DiffusionTransformer
    m = DiffusionTransformer(io_channels=64, embed_dim=256, depth=1, num_heads=4, transformer_type="continuous_transformer")
    assert m.shard_graph_stats() is None
    m.shard_tokens(["cuda:0", "cuda:0"])
    assert m.shard_graph_stats() is None      # the group is made by the first call
    m.refresh_native_weights()                # dropping a graph that does not exist yet is fine
    m.shard_tokens(None)


def test_ctypes_signatures_of_the_graph_entry_points():
    from stable_audio_tools import _native
    VP, I, F, LL, ULL = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_longlong, ctypes.c_ulonglong
    S = _native.SIGNATURES
    assert S["satb_dit_group_graph_forward"] == (I, [VP, VP, VP, VP, I, I, F, F, VP, VP])
    assert S["satb_dit_group_graph_reset"] == (I, [VP])
    assert S["satb_dit_group_graph_stats"] == (I, [VP, ctypes.POINTER(LL), ctypes.POINTER(LL), ctypes.POINTER(ULL)])
    header = " ".join(open(f"{ROOT}/include/satb200.h").read().split())
    for decl in ("int satb_dit_group_graph_forward(SatbDitGroup* g, const float* x, const float* t, float* out, int B, "
                 "int L, float cfg_scale, float scale_phi, void* const* rank_streams, void* home_stream);",
                 "int satb_dit_group_graph_reset(SatbDitGroup* g);",
                 "int satb_dit_group_graph_stats(const SatbDitGroup* g, long long* captures, long long* replays, "
                 "unsigned long long* launches);"):
        assert decl in header
    lib = _native.lib()
    assert lib.satb_abi_version() == 3
    for name in ("satb_dit_group_graph_forward", "satb_dit_group_graph_reset", "satb_dit_group_graph_stats"):
        assert getattr(lib, name).argtypes == S[name][1]
