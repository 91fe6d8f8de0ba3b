"""CPU: the host side of the CFG-split DiT forward (DiffusionTransformer.shard_tokens with two rows,
satb_dit_group_create_cfg): every refusal, raised before any CUDA call, and the ctypes signature of the new entry
point.  Nothing here touches a GPU."""
import ctypes

import pytest

from helpers import ROOT
from test_dit_group import SHARD_REFUSALS, _destroy, _handles


def _model(**kw):
    from stable_audio_tools.models.dit import DiffusionTransformer
    return DiffusionTransformer(io_channels=64, embed_dim=256, depth=1, num_heads=4, cond_token_dim=128,
                                project_cond_tokens=False, transformer_type="continuous_transformer", **kw)


def _create_cfg(hs, world, devices=None):
    from stable_audio_tools import _native
    lib = _native.lib()
    g = ctypes.c_void_p()
    arr = (ctypes.c_void_p * len(hs))(*[h.value for h in hs])
    ids = (ctypes.c_int * len(hs))(*(devices or [0] * len(hs)))
    rc = lib.satb_dit_group_create_cfg(arr, ids, world, ctypes.byref(g))
    return rc, lib.satb_last_error().decode()


@pytest.mark.parametrize("kw,msg", SHARD_REFUSALS)
@pytest.mark.parametrize("rows", [[["cuda:0"] * 2] * 2, [["cuda:0"] * 4] * 2])
def test_cfg_split_refuses_the_token_convolutions_and_fp8_attention_with_several_devices_per_row(kw, msg, rows):
    m = _model(**kw)
    with pytest.raises(NotImplementedError, match=msg):
        m.shard_tokens(rows)
    assert m.__dict__["_shard"] is None
    m.shard_tokens(None)


@pytest.mark.parametrize("kw,msg", SHARD_REFUSALS)
def test_cfg_split_with_one_device_per_row_accepts_every_model_option(kw, msg):
    m = _model(**kw)
    m.shard_tokens([["cuda:0"], ["cuda:0"]])   # no CUDA call: the group is made by the first forward
    sh = m.__dict__["_shard"]
    assert sh["cfg_split"] and sh["world"] == 1 and len(sh["devices"]) == 2
    with pytest.raises(NotImplementedError, match=msg):   # the flat list keeps its refusal
        m.shard_tokens(["cuda:0"])
    m.shard_tokens(None)


def test_flat_list_with_conformer_keeps_the_existing_message():
    m = _model(conformer=True)
    with pytest.raises(NotImplementedError, match=r"shard_tokens: conformer blocks are not supported \(their depthwise "
                                                  r"convolution needs the neighbouring ranks' tokens\)"):
        m.shard_tokens(["cuda:0", "cuda:0"])


@pytest.mark.parametrize("rows,msg", [
    ([["cuda:0", "cuda:0"], ["cuda:0"]], "same length"),
    ([[], []], "1 to 8 devices per row"),
    ([["cuda:0"] * 9] * 2, "1 to 8 devices per row"),
    ([["cuda:0"]] * 3, "two rows"),
    ([["cuda:0"]], "two rows"),
    ([[["cuda:0"]], [["cuda:0"]]], "deeper nesting"),
    ([["cuda:0"], "cuda:0"], "not a mix"),
])
def test_cfg_split_refuses_bad_layouts(rows, msg):
    m = _model()
    with pytest.raises(ValueError, match=msg):
        m.shard_tokens(rows)
    assert m.__dict__["_shard"] is None


def test_cfg_split_layout_home_device_and_cpu_refusal():
    import torch
    from stable_audio_tools import _native
    m = _model()
    m.shard_tokens([["cuda:0", "cuda:1"], ["cuda:2", "cuda:3"]])
    sh = m.__dict__["_shard"]
    assert sh["world"] == 2 and sh["cfg_split"]
    assert sh["devices"] == [torch.device("cuda", i) for i in range(4)]   # row 0, then row 1; home = devices[0][0]
    with pytest.raises(_native.NativeError, match="not a CUDA device"):
        m.shard_tokens([["cuda:0"], ["cpu"]])
    m.shard_tokens([["cuda:0"], ["cuda:0"]])
    with pytest.raises(NotImplementedError, match="return_info"):
        m(torch.zeros(1, 64, 16), torch.zeros(1), return_info=True)
    m.shard_tokens(None)
    assert m.__dict__["_shard"] is None and m.shard_graph_stats() is None


def test_group_create_cfg_refusals_without_a_device():
    """The -5 refusals at world > 1, mixed models, shared handles and unloaded weights: all before any CUDA call."""
    from stable_audio_tools import _native
    lib = _native.lib()
    for option, msg in [(lambda lib, h, i: lib.satb_dit_set_conformer(h, 1), "conformer"),
                        (lambda lib, h, i: lib.satb_dit_set_feedforward(h, 1024, 0, 3, 1), "use_conv"),
                        (lambda lib, h, i: lib.satb_dit_set_attention_fp8(h, 1), "fp8")]:
        hs = _handles(4, option)
        rc, err = _create_cfg(hs, 2)
        assert rc == -5 and msg in err, (rc, err)
        rc, err = _create_cfg(hs[:2], 1)      # one rank per row: accepted options, refused later for the weights
        _destroy(hs)
        assert rc != -5 and "finalized" in err, (rc, err)
    hs = _handles(1) + _handles(1, embed_dim=384, num_heads=6)
    rc, err = _create_cfg(hs, 1)
    _destroy(hs)
    assert rc != 0 and "config" in err
    hs = _handles(1)
    rc, err = _create_cfg(hs * 2, 1)
    assert rc != 0 and "its own handle" in err
    _destroy(hs)
    hs = _handles(2)
    rc, err = _create_cfg(hs, 9)
    _destroy(hs)
    assert rc != 0 and "world" in err
    assert lib.satb_dit_group_create_cfg(None, None, 1, None) != 0
    assert b"null" in lib.satb_last_error()


def test_ctypes_signature_of_the_cfg_entry_point():
    from stable_audio_tools import _native
    VP, I = ctypes.c_void_p, ctypes.c_int
    assert _native.SIGNATURES["satb_dit_group_create_cfg"] == (I, [VP, VP, I, ctypes.POINTER(VP)])
    header = " ".join(open(f"{ROOT}/include/satb200.h").read().split())
    assert ("int satb_dit_group_create_cfg(SatbDit* const* handles, const int* devices, int world, "
            "SatbDitGroup** out);") in header
    lib = _native.lib()
    assert lib.satb_dit_group_create_cfg.argtypes == [VP, VP, I, ctypes.POINTER(VP)]
    assert lib.satb_dit_group_create_cfg.restype == I
    assert lib.satb_abi_version() == 3
