"""CPU: the C-ABI library loads without a GPU and exports every symbol include/satb200.h declares;
the ctypes table covers the header; argument validation returns error codes (no compute here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    text = open(os.path.join(ROOT, "include", "satb200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(satb_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_the_expected_entry_points():
    syms = _header_symbols()
    for must in ("satb_dit_create", "satb_dit_load_weight", "satb_dit_prepare_cond", "satb_dit_forward",
                 "satb_oobleck_decode", "satb_oobleck_encode", "satb_snake_beta", "satb_last_error"):
        assert must in syms


def test_library_loads_and_exports_every_declared_symbol():
    from stable_audio_tools import _native
    lib = _native.lib()
    for s in _header_symbols():
        assert hasattr(lib, s), f"{s} declared in include/satb200.h but not exported"
    assert set(_native.SIGNATURES) == set(_header_symbols()), "ctypes signature table out of sync with the header"
    assert lib.satb_abi_version() == 3


def test_create_validates_config_and_reports_errors():
    from stable_audio_tools import _native
    lib = _native.lib()
    h = ctypes.c_void_p()
    bad = _native.SatbDitConfig(io_channels=64, embed_dim=100, depth=1, num_heads=2, cond_token_dim=0, global_cond_dim=0,
                                project_cond_tokens=0, project_global_cond=1, global_cond_type=0, patch_size=1, operand_dtype=0)
    rc = lib.satb_dit_create(ctypes.byref(bad), ctypes.byref(h))
    assert rc != 0 and b"embed_dim" in lib.satb_last_error()
    good = _native.SatbDitConfig(io_channels=64, embed_dim=128, depth=1, num_heads=2, cond_token_dim=64, global_cond_dim=128,
                                 project_cond_tokens=0, project_global_cond=1, global_cond_type=0, patch_size=1, operand_dtype=0)
    assert lib.satb_dit_create(ctypes.byref(good), ctypes.byref(h)) == 0
    # forward before weights are loaded must fail loudly, not compute
    rc = lib.satb_dit_forward(h, None, None, None, 1, 8, 1.0, 0.0, None)
    assert rc != 0 and b"finalized" in lib.satb_last_error()
    lib.satb_dit_destroy(h)
    oc = _native.SatbOobleckConfig()
    oc.in_channels, oc.channels, oc.latent_dim, oc.n_stages = 2, 33, 8, 2
    rc = lib.satb_oobleck_create(ctypes.byref(oc), ctypes.byref(h))
    assert rc != 0 and b"channels" in lib.satb_last_error()


def test_attention_probe_refuses_bad_layouts():
    """satb_attention_probe validates before any CUDA call: fake 16-byte-aligned addresses, never dereferenced."""
    from stable_audio_tools import _native
    lib = _native.lib()
    fake = 1 << 20

    def probe(**kw):
        # the fused QKV layout of the forward: 2 items x 33 rows x 3 x 4 heads of 64
        p = dict(B=2, H=4, Hkv=4, Nq=33, Nk=33, head_dim=64, bf16=0, q=fake, k=fake, v=fake, o=fake + 4096,
                 ldq=768, ldk=768, ldv=768, ldo=256, q_bs=33 * 768, k_bs=33 * 768, v_bs=33 * 768, o_bs=33 * 256,
                 q_cols=768, k_cols=768, v_cols=768, q_col=0, k_col=256, v_col=512)
        p.update(kw)
        return lib.satb_attention_probe(ctypes.byref(_native.SatbAttentionProbe(**p)), None)

    bad = [(dict(head_dim=48), b"head dim"), (dict(Hkv=3), b"multiple of kv heads"),
           (dict(Nq=0), b"empty"), (dict(Nk=0), b"empty"),
           (dict(k_col=260), b"16B aligned"), (dict(v_col=516), b"16B aligned"), (dict(q_col=4), b"16B aligned"),
           (dict(ldk=772, ldq=772, ldv=772), b"16B aligned"), (dict(k_bs=33 * 768 + 4), b"16B aligned"),
           (dict(ldo=260), b"16B aligned"), (dict(v_col=520), b"exceed"), (dict(q_cols=248), b"exceed"),
           (dict(k_cols=500), b"exceed"), (dict(q=fake + 8), b"16B aligned"),
           (dict(q_cols=800), b"row pitch"), (dict(B=0), b"batch item"), (dict(o=None), b"null"),
           (dict(q_col=-8), b"negative"), (dict(k_col=-256), b"negative"), (dict(ldv=-768), b"negative"),
           (dict(o_bs=-33 * 256), b"negative")]
    for kw, msg in bad:
        rc = probe(**kw)
        err = lib.satb_last_error()
        assert rc != 0 and msg in err, f"{kw}: rc {rc}, {err}"


def test_no_cpu_fallback_in_the_product_path():
    """CPU tensors are rejected by the drop-in modules; nothing under the package imports oracle/."""
    import torch
    from stable_audio_tools import _native
    from stable_audio_tools.models.autoencoders import OobleckDecoder
    from stable_audio_tools.models.blocks import SnakeBeta
    from stable_audio_tools.models.dit import DiffusionTransformer
    m = DiffusionTransformer(io_channels=64, embed_dim=128, depth=1, num_heads=2, transformer_type="continuous_transformer")
    with pytest.raises(_native.NativeError):
        m(torch.zeros(1, 64, 8), torch.zeros(1))
    with pytest.raises(_native.NativeError):
        SnakeBeta(4)(torch.zeros(1, 4, 8))
    dec = OobleckDecoder(out_channels=2, channels=32, c_mults=[1, 2], strides=[2, 2], latent_dim=8, use_snake=True)
    with pytest.raises(_native.NativeError):
        dec(torch.zeros(1, 8, 4))
    pkg = os.path.join(ROOT, "friendly-stable-audio-tools_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f"{f} imports the oracle"


def test_library_reads_no_environment_variables():
    """Every launch route is chosen from the model config and the shape, never from a process-global switch."""
    for d in (os.path.join(ROOT, "friendly-stable-audio-tools_b200", "csrc"), os.path.join(ROOT, "include")):
        for f in sorted(os.listdir(d)):
            if f.endswith((".cu", ".cuh", ".h")):
                assert "getenv" not in open(os.path.join(d, f)).read(), f"{f} reads an environment variable"
