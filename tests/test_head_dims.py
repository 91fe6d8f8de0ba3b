"""CPU: DiTs whose attention head dim is 32, 96 or 128.  The oracle against golden outputs of the real reference
(tests/golden/dit_hd*.npz, made by oracle/make_golden_head_dims.py), and the refusal of unsupported head dims
by the Python constructors and by satb_dit_create."""
import ctypes
import json

import pytest
import torch

from helpers import load_golden, max_abs
from oracle import dit_oracle as do

HEAD_DIM_GOLDENS = ["dit_hd128_small.npz", "dit_hd96_small.npz", "dit_hd32_small.npz", "dit_hd128_adaln_small.npz"]


@pytest.mark.parametrize("name", HEAD_DIM_GOLDENS)
def test_dit_oracle_matches_reference_golden_at_other_head_dims(name):
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    assert cfg["embed_dim"] // cfg["num_heads"] in (32, 96, 128)
    sd = do.make_dit_weights(cfg, seed=int(g["seed"]))
    wsum = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(wsum - float(g["wsum"])) <= 1e-9 * wsum
    T = lambda k: torch.from_numpy(g[k])
    x, t, c, ge, neg = T("x"), T("t"), T("cross"), T("glob"), T("neg")
    # same gates as test_oracle_golden.py: fp32 restatement vs fp32 reference, identical op order
    assert max_abs(do.dit_forward(sd, cfg, x, t, c, ge, cfg_scale=1.0), T("y_nocfg")) <= 1e-6
    assert max_abs(do.dit_forward(sd, cfg, x, t, c, ge, cfg_scale=7.0), T("y_cfg7")) <= 1e-5
    assert max_abs(do.dit_forward(sd, cfg, x, t, c, ge, cfg_scale=4.0, scale_phi=0.7), T("y_cfg4_phi")) <= 1e-5
    assert max_abs(do.dit_forward(sd, cfg, x, t, c, ge, negative_cross_attn_cond=neg, cfg_scale=3.0), T("y_neg3")) <= 1e-5
    hs = []
    do.dit_inner_forward(sd, cfg, x, t, c, ge, hidden_states=hs)
    assert max_abs(hs[-1], T("hidden_last")) <= 1e-5


BASE = dict(io_channels=64, depth=1, global_cond_dim=0, project_cond_tokens=False,
            transformer_type="continuous_transformer")
# (embed_dim, num_heads, cond_token_dim, qk_norm) -> head dim 48, 256, 128 with qk_norm
UNSUPPORTED = [(384, 8, 0, False), (512, 2, 0, False), (256, 2, 0, True)]
SUPPORTED = [(256, 8, 128), (256, 4, 128), (384, 4, 192), (256, 2, 128)]   # head dim 32, 64, 96, 128


@pytest.mark.parametrize("embed_dim,num_heads,cond,qk_norm", UNSUPPORTED)
def test_constructors_refuse_unsupported_head_dims(embed_dim, num_heads, cond, qk_norm):
    from stable_audio_tools.models.dit import DiffusionTransformer
    from stable_audio_tools.models.transformer import Attention
    kw = dict(attn_kwargs={"qk_norm": True}) if qk_norm else {}
    with pytest.raises(NotImplementedError, match="head dim" if not qk_norm else "qk_norm"):
        DiffusionTransformer(**dict(BASE, embed_dim=embed_dim, num_heads=num_heads, cond_token_dim=cond), **kw)
    with pytest.raises(NotImplementedError):
        Attention(embed_dim, dim_heads=embed_dim // num_heads, qk_norm=qk_norm)


def test_unsupported_head_dim_message_lists_the_supported_dims():
    from stable_audio_tools.models.dit import DiffusionTransformer
    with pytest.raises(NotImplementedError) as e:
        DiffusionTransformer(**dict(BASE, embed_dim=384, num_heads=8))
    assert "32, 64, 96, 128" in str(e.value)
    with pytest.raises(NotImplementedError):
        DiffusionTransformer(**dict(BASE, embed_dim=384, num_heads=5))    # not a whole head dim


@pytest.mark.parametrize("embed_dim,num_heads,cond", SUPPORTED)
def test_constructor_accepts_supported_head_dims(embed_dim, num_heads, cond):
    from stable_audio_tools.models.dit import DiffusionTransformer
    m = DiffusionTransformer(**dict(BASE, embed_dim=embed_dim, num_heads=num_heads, cond_token_dim=cond))
    dh = embed_dim // num_heads
    assert m.transformer.rotary_pos_emb.inv_freq.shape == (max(dh // 2, 32) // 2,)
    assert m.transformer.layers[0].cross_attn.kv_heads == cond // dh


def _create(embed_dim, num_heads, cond=0, qk_norm=0):
    from stable_audio_tools import _native
    lib = _native.lib()
    cfg = _native.SatbDitConfig(io_channels=64, embed_dim=embed_dim, depth=1, num_heads=num_heads, cond_token_dim=cond,
                                global_cond_dim=0, project_cond_tokens=0, project_global_cond=1, global_cond_type=0,
                                patch_size=1, operand_dtype=0, qk_norm=qk_norm)
    h = ctypes.c_void_p()
    rc = lib.satb_dit_create(ctypes.byref(cfg), ctypes.byref(h))
    if rc == 0:
        lib.satb_dit_destroy(h)
    return rc, lib.satb_last_error()


@pytest.mark.parametrize("embed_dim,num_heads,cond,qk_norm", UNSUPPORTED)
def test_native_create_refuses_unsupported_head_dims(embed_dim, num_heads, cond, qk_norm):
    rc, msg = _create(embed_dim, num_heads, cond, int(qk_norm))
    assert rc != 0
    assert (b"qk_norm" if qk_norm else b"32, 64, 96 or 128") in msg


@pytest.mark.parametrize("embed_dim,num_heads,cond", SUPPORTED)
def test_native_create_accepts_supported_head_dims(embed_dim, num_heads, cond):
    assert _create(embed_dim, num_heads, cond)[0] == 0


def test_native_create_checks_cross_attention_kv_heads_against_the_head_dim():
    # head dim 128: a 192-wide context is 1.5 heads; 384 = 3 kv heads does not divide 4 heads
    for cond in (192, 384):
        rc, msg = _create(512, 4, cond)
        assert rc != 0 and b"head dim (128)" in msg
    assert _create(512, 4, 256)[0] == 0                               # 2 kv heads
