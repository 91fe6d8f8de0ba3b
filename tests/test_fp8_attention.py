"""CPU: the FP8 self-attention option (attention_dtype "fp8") - the emulation's quantisers, that the emulation touches
self-attention only, the constructor's validation and the native setter's refusals (no GPU needed)."""
import ctypes
import json

import pytest
import torch

from fp8_attn_ref import (dequant, fp8_attention, fp8_attention_core, key_of, quantize_heads, quantize_v,
                          stored_key_order)
from helpers import load_golden


def _pow2(e):
    return torch.ldexp(torch.ones_like(e, dtype=torch.float32), e)


# ------------------------------------------------------------------------------------------------ quantisers
def test_head_scale_at_and_just_above_a_power_of_two_boundary():
    x = torch.zeros(4, 64)
    x[0, 5] = 448.0                                    # exactly 448 * 2^0: scale 1
    x[1, 5] = torch.nextafter(torch.tensor(448.0), torch.tensor(1e9))   # just above: scale 2
    x[2, 9] = -448.0 * 2.0 ** -20                      # negative, exactly on a boundary
    x[3, 0] = 224.0                                    # 448 * 2^-1
    q, s = quantize_heads(x)
    assert s.flatten().tolist() == [1.0, 2.0, 2.0 ** -20, 0.5]
    d = dequant(q, s)
    assert d[0, 5] == 448.0 and d[1, 5] == 448.0 and d[2, 9] == -448.0 * 2.0 ** -20 and d[3, 0] == 224.0


def test_zero_heads_get_scale_one_and_zero_values():
    x = torch.zeros(3, 64)
    q, s = quantize_heads(x)
    assert s.flatten().tolist() == [1.0] * 3
    assert torch.equal(q.to(torch.float32), x)
    v = torch.zeros(1, 7, 64)
    v[0, :, 3] = 1.0                                   # one live channel; the others are all zero over the tokens
    qv, sv = quantize_v(v)
    assert sv.shape == (1, 1, 64)
    assert sv[0, 0, 3] == 2.0 ** -8 and bool((sv[0, 0, torch.arange(64) != 3] == 1.0).all())


def test_values_in_the_e4m3_subnormals_round_to_the_2_pow_minus_9_grid():
    x = torch.zeros(1, 64)
    x[0, 0] = 448.0
    x[0, 1:8] = torch.tensor([2.0 ** -9, 1.4 * 2.0 ** -9, 1.6 * 2.0 ** -9, 2.0 ** -7 + 2.0 ** -10, 2.0 ** -10,
                              0.49 * 2.0 ** -9, 3 * 2.0 ** -9])
    q, s = quantize_heads(x)
    assert s.item() == 1.0
    got = q.to(torch.float32)[0, 1:8].tolist()
    assert got == [2.0 ** -9, 2.0 ** -9, 2 * 2.0 ** -9, 2.0 ** -7, 0.0, 0.0, 3 * 2.0 ** -9]


def test_no_scaled_value_exceeds_448_and_the_scale_is_the_smallest():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 3, 50, 64, generator=g) * torch.logspace(-30, 30, 50).view(1, 1, 50, 1)
    for q, s, dim in (quantize_heads(x) + (-1,), quantize_v(x) + (-2,)):
        qf = q.to(torch.float32)
        assert bool(torch.isfinite(qf).all()) and float(qf.abs().max()) <= 448.0
        amax = x.abs().amax(dim=dim, keepdim=True)
        assert bool((amax <= 448.0 * s).all()) and bool((amax > 448.0 * s / 2).all())


def test_stored_key_order_is_a_permutation_of_each_32_key_group():
    assert sorted(key_of(j) for j in range(32)) == list(range(32))
    # thread t % 4 = q of a quad holds k indices 4q .. 4q + 3 and 16 + 4q .. 16 + 4q + 3; its S columns are
    # 8g + 2q + {0, 1} for the 8-column groups g of the group
    for q in range(4):
        held = [key_of(j) for j in list(range(4 * q, 4 * q + 4)) + list(range(16 + 4 * q, 16 + 4 * q + 4))]
        assert sorted(held) == sorted(8 * g + 2 * q + e for g in range(4) for e in range(2))
    order = stored_key_order(256)
    assert sorted(order.tolist()) == list(range(256))


def test_emulated_core_is_close_to_the_exact_softmax():
    g = torch.Generator().manual_seed(1)
    q, k, v = (torch.randn(1, 2, 65, 64, generator=g) for _ in range(3))
    ref = torch.softmax(q.double() @ k.double().transpose(-1, -2) / 8, -1) @ v.double()
    emu = fp8_attention_core(q, k, v).double()
    rel = float((emu - ref).norm() / ref.norm())
    assert 1e-4 < rel < 0.1, rel


# ------------------------------------------------------------------------------------------------ self-attention only
def test_emulation_changes_self_attention_and_leaves_cross_attention_bit_equal():
    from oracle import dit_oracle as do
    g = torch.Generator().manual_seed(2)
    D, heads = 128, 2
    sd = {"a.to_qkv.weight": torch.randn(3 * D, D, generator=g) * 0.1, "a.to_out.weight": torch.randn(D, D, generator=g) * 0.1,
          "c.to_q.weight": torch.randn(D, D, generator=g) * 0.1, "c.to_kv.weight": torch.randn(2 * D, 96, generator=g) * 0.1,
          "c.to_out.weight": torch.randn(D, D, generator=g) * 0.1}
    x, ctx = torch.randn(2, 33, D, generator=g), torch.randn(2, 9, 96, generator=g)
    freqs = do.rotary_freqs(33, 1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32)))
    cross_off = do.cross_attention(x, ctx, sd, "c.", 64)
    self_off = do.self_attention(x, sd, "a.", 64, freqs)
    with fp8_attention():
        cross_on = do.cross_attention(x, ctx, sd, "c.", 64)
        self_on = do.self_attention(x, sd, "a.", 64, freqs)
    assert torch.equal(cross_on, cross_off)
    assert not torch.equal(self_on, self_off)
    assert do.self_attention(x, sd, "a.", 64, freqs).equal(self_off), "the context did not restore the oracle"


# ------------------------------------------------------------------------------------------------ the constructor
def _cfg(**kw):
    g = load_golden("dit_prepend_small.npz")
    return dict(json.loads(str(g["cfg"])), **kw)


@pytest.mark.parametrize("operand_dtype", ["fp16", "bf16", "fp8"])
def test_attention_dtype_fp8_is_accepted_with_every_operand_dtype(operand_dtype):
    from stable_audio_tools.models.dit import DiffusionTransformer
    m = DiffusionTransformer(**_cfg(), operand_dtype=operand_dtype, attention_dtype="fp8")
    assert m.attention_dtype == "fp8"
    assert DiffusionTransformer(**_cfg(), operand_dtype=operand_dtype).attention_dtype is None


@pytest.mark.parametrize("bad", ["fp16", "FP8", "e4m3", 8, torch.float8_e4m3fn])
def test_other_attention_dtypes_raise_value_error(bad):
    from stable_audio_tools.models.dit import DiffusionTransformer
    with pytest.raises(ValueError, match="attention_dtype"):
        DiffusionTransformer(**_cfg(), attention_dtype=bad)


@pytest.mark.parametrize("num_heads", [8, 2, 1])   # head dims 32, 128, 256
def test_attention_dtype_fp8_needs_head_dim_64(num_heads):
    from stable_audio_tools.models.dit import DiffusionTransformer
    with pytest.raises(NotImplementedError, match="64"):
        DiffusionTransformer(**_cfg(num_heads=num_heads), attention_dtype="fp8")


def test_attention_dtype_reaches_the_model_as_a_config_kwarg():
    from stable_audio_tools.models.factory import create_model_from_config
    cfg = _cfg()
    model_config = {"model_type": "diffusion_cond", "sample_size": 4096, "sample_rate": 44100, "audio_channels": 2,
                    "model": {"diffusion": {"type": "dit", "config": dict(cfg, attention_dtype="fp8")},
                              "io_channels": cfg["io_channels"]}}
    model = create_model_from_config(model_config)
    dits = [m for m in model.modules() if type(m).__name__ == "DiffusionTransformer"]
    assert dits and all(m.attention_dtype == "fp8" for m in dits)


# ------------------------------------------------------------------------------------------------ the setter
def _handle(num_heads=4):
    from stable_audio_tools import _native
    lib = _native.lib()
    cfg = _native.SatbDitConfig(io_channels=64, embed_dim=256, depth=1, num_heads=num_heads, cond_token_dim=0,
                                global_cond_dim=0, project_cond_tokens=0, project_global_cond=1, global_cond_type=0,
                                patch_size=1, operand_dtype=0, qk_norm=0, input_concat_dim=0, prepend_cond_dim=0)
    h = ctypes.c_void_p()
    assert lib.satb_dit_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    return lib, h


def test_setter_accepts_0_and_1_at_head_dim_64():
    lib, h = _handle()
    try:
        assert lib.satb_dit_set_attention_fp8(h, 1) == 0
        assert lib.satb_dit_set_attention_fp8(h, 0) == 0
    finally:
        lib.satb_dit_destroy(h)


@pytest.mark.parametrize("enable", [2, -1])
def test_setter_refuses_an_enable_other_than_0_or_1(enable):
    lib, h = _handle()
    try:
        assert lib.satb_dit_set_attention_fp8(h, enable) != 0
        assert b"enable" in lib.satb_last_error()
    finally:
        lib.satb_dit_destroy(h)


@pytest.mark.parametrize("num_heads", [8, 2])   # head dims 32, 128
def test_setter_refuses_other_head_dims(num_heads):
    lib, h = _handle(num_heads)
    try:
        assert lib.satb_dit_set_attention_fp8(h, 1) != 0
        assert b"head dim 64" in lib.satb_last_error()
    finally:
        lib.satb_dit_destroy(h)


def test_setter_refuses_a_null_handle():
    from stable_audio_tools import _native
    lib = _native.lib()
    assert lib.satb_dit_set_attention_fp8(None, 1) != 0


def test_core_and_quantiser_entry_points_refuse_bad_arguments_before_any_cuda_call():
    from stable_audio_tools import _native
    lib = _native.lib()
    p = ctypes.c_void_p(16)
    assert lib.satb_attention_fp8_vt(None, p, p, 1, 1, 1, 0, None) != 0
    assert lib.satb_attention_fp8_vt(p, p, p, 0, 1, 1, 0, None) != 0
    pr, o = _native.SatbGemmProbe(), _native.SatbQkE4m3(q8=16, k8=16, sq=16, sk=16, heads=1, scale_ld=1)
    pr.epi, pr.bn, pr.seq_len = _native.EPI_QKV_ROPE_E4M3, 256, 1
    assert lib.satb_gemm_probe_qk8(p, p, None, None, 1, 96, 64, ctypes.byref(pr), ctypes.byref(o), None) != 0
    assert b"multiple of 64" in lib.satb_last_error()
    assert lib.satb_attention_fp8_core(p, p, p, p, p, p, None, 1, 1, 1, 1, 0, None) != 0
    assert lib.satb_attention_fp8_core(p, p, p, p, p, p, p, 1, 1, 0, 1, 0, None) != 0
    assert b"Nq" in lib.satb_last_error()
