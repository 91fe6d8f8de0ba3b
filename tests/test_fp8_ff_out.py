"""CPU: the FP8 FF-out option (ff_out_dtype "fp8") - the block quantiser, that the emulation touches exactly the FF-out
Linears, the constructor's validation and the native setter's refusals (no GPU needed)."""
import ctypes

import pytest
import torch

from fp8_ff_out_ref import fp8_block_roundtrip, fp8_ff_out_operands, ff_out_weight_keys, quantize_fp8_blocks
from fp8_ref import fp8_operands, fp8_row_exponent

KW = dict(io_channels=64, embed_dim=128, depth=2, num_heads=2, cond_token_dim=64, global_cond_dim=128,
          project_cond_tokens=False, transformer_type="continuous_transformer")


# ------------------------------------------------------------------------------------------------ quantiser
def test_block_scales_follow_the_row_rule_per_128_columns():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(5, 384, generator=g) * torch.logspace(-20, 20, 3, base=2.0).repeat_interleave(128)
    x[2, 128:256] = 0.0                                            # an all-zero block: scale 1
    x[3, 0] = 448.0 * 2.0 ** 5                                     # exactly on a boundary
    q, s = quantize_fp8_blocks(x)
    assert q.shape == x.shape and s.shape == (5, 3)
    amax = x.reshape(5, 3, 128).abs().amax(-1)
    assert torch.equal(s, torch.ldexp(torch.ones_like(amax), fp8_row_exponent(amax)))
    assert s[2, 1] == 1.0 and s[3, 0] == 2.0 ** 5
    assert float(q.float().abs().max()) <= 448.0
    dq = fp8_block_roundtrip(x)
    err = (dq - x).abs()
    assert torch.all(err <= torch.maximum(x.abs() * 2.0 ** -4, s.repeat_interleave(128, -1) * 2.0 ** -10))


def test_a_short_last_block_equals_the_zero_padded_one():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(3, 200, generator=g)
    xp = torch.nn.functional.pad(x, (0, 56))
    q, s = quantize_fp8_blocks(x)
    qp, sp = quantize_fp8_blocks(xp)
    assert torch.equal(s, sp) and torch.equal(q.float(), qp.float()[:, :200])
    assert torch.equal(fp8_block_roundtrip(x), fp8_block_roundtrip(xp)[:, :200])


def test_blocks_of_one_row_are_scaled_independently():
    x = torch.ones(1, 256)
    x[0, 128:] = 2.0 ** -20
    q, s = quantize_fp8_blocks(x)
    assert s.tolist() == [[2.0 ** -8, 2.0 ** -28]]
    assert torch.equal(fp8_block_roundtrip(x), x)                  # both blocks exact at their own scale


# ------------------------------------------------------------------------------------------------ emulation
def _inputs():
    g = torch.Generator().manual_seed(1)
    return (torch.randn(2, 64, 24, generator=g), torch.rand(2, generator=g), torch.randn(2, 5, 64, generator=g),
            torch.randn(2, 128, generator=g))


@pytest.mark.parametrize("gtype", ["prepend", "adaLN"])
def test_emulation_routes_exactly_ff_out_through_the_block_quantiser(gtype):
    """With both quantisers replaced by recording fp16 roundings, the emulation must route exactly ff.ff.2 of every
    layer through them - the activation by block, the weight by row, once each per call and layer - and otherwise
    reproduce fp8_operands bit for bit."""
    from oracle import dit_oracle as do
    cfg = dict(KW, global_cond_type=gtype)
    sd = do.make_dit_weights(cfg, seed=3)
    x, t, c, ge = _inputs()
    names = {id(v): k for k, v in sd.items()}
    acts, weights = [], []

    def rec_act(v):
        acts.append(tuple(v.shape))
        return v.to(torch.float16).to(v.dtype)

    def rec_w(v):
        weights.append(names.get(id(v)))
        return v.to(torch.float16).to(v.dtype)

    run = lambda: do.dit_forward(sd, cfg, x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=3.0)
    with fp8_operands(sd), fp8_ff_out_operands(sd, act_roundtrip=rec_act, weight_roundtrip=rec_w):
        y_emu = run()
    with fp8_operands(sd):
        y8 = run()
    assert torch.equal(y_emu, y8)
    assert sorted(weights) == ff_out_weight_keys(sd) and len(weights) == cfg["depth"]
    assert len(acts) == cfg["depth"] and all(a[-1] == 4 * cfg["embed_dim"] for a in acts)
    # the real quantisers change the output, by about the e4m3 rounding, and the contexts restore the oracle
    with fp8_operands(sd), fp8_ff_out_operands(sd):
        y88 = run()
    rel = float((y88 - y8).norm() / y8.norm())
    assert 1e-4 < rel < 0.2, rel
    assert do._lin16.__name__ == "_lin16"


def test_emulation_refuses_a_convolutional_ff_out():
    from oracle import feedforward_oracle as fo
    cfg = dict(KW, ff_kwargs=dict(use_conv=True, conv_kernel_size=3))
    sd = fo.make_dit_weights(cfg, seed=4)
    with pytest.raises(NotImplementedError):
        fp8_ff_out_operands(sd)


# ------------------------------------------------------------------------------------------------ interface
def test_operand_dtypes_are_unchanged():
    from stable_audio_tools.models.dit import OPERAND_DTYPES
    assert OPERAND_DTYPES == {"fp16": 0, "bf16": 1, "fp8": 2}


def test_constructor_validation():
    from stable_audio_tools.models.diffusion import DiTWrapper
    from stable_audio_tools.models.dit import DiffusionTransformer
    m = DiffusionTransformer(**KW, operand_dtype="fp8", ff_out_dtype="fp8")
    assert m.ff_out_dtype == "fp8" and m.native_config().operand_dtype == 2
    assert DiffusionTransformer(**KW).ff_out_dtype is None
    assert DiTWrapper(**KW, operand_dtype="fp8", ff_out_dtype="fp8").model.ff_out_dtype == "fp8"
    for bad in ("fp16", "FP8", "e4m3", "", 8):
        with pytest.raises(ValueError):
            DiffusionTransformer(**KW, operand_dtype="fp8", ff_out_dtype=bad)
    for od in ("fp16", "bf16"):
        with pytest.raises(ValueError):
            DiffusionTransformer(**KW, operand_dtype=od, ff_out_dtype="fp8")
    with pytest.raises(NotImplementedError):
        DiffusionTransformer(**KW, operand_dtype="fp8", ff_out_dtype="fp8",
                             ff_kwargs=dict(use_conv=True, conv_kernel_size=3))
    with pytest.raises(NotImplementedError):                      # inner 320: a multiple of 64, not of 128
        DiffusionTransformer(**KW, operand_dtype="fp8", ff_out_dtype="fp8", ff_kwargs=dict(mult=2.5))
    # inner 330 pads to 384 natively; plain SiLU, bias-free, conformer and FP8 attention are accepted
    for extra in (dict(ff_kwargs=dict(mult=330 / 128)), dict(ff_kwargs=dict(glu=False, no_bias=True)),
                  dict(conformer=True), dict(attention_dtype="fp8", num_heads=2)):
        DiffusionTransformer(**dict(KW, **extra), operand_dtype="fp8", ff_out_dtype="fp8")


def _handle(lib, nat, operand_dtype=2):
    cfg = nat.SatbDitConfig(io_channels=64, embed_dim=128, depth=1, num_heads=2, cond_token_dim=64,
                            global_cond_dim=128, project_cond_tokens=0, project_global_cond=1, global_cond_type=0,
                            patch_size=1, operand_dtype=operand_dtype)
    h = ctypes.c_void_p()
    assert lib.satb_dit_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    return h


def test_setter_refusals_before_any_cuda_call():
    from stable_audio_tools import _native as nat
    lib = nat.lib()
    assert lib.satb_dit_set_ff_out_fp8(None, 1) != 0 and b"null" in lib.satb_last_error()
    h = _handle(lib, nat)
    try:
        for bad in (2, -1):
            assert lib.satb_dit_set_ff_out_fp8(h, bad) != 0 and b"enable" in lib.satb_last_error()
        assert lib.satb_dit_set_ff_out_fp8(h, 1) == 0
        assert lib.satb_dit_set_ff_out_fp8(h, 0) == 0
    finally:
        lib.satb_dit_destroy(h)
    for od in (0, 1):
        h = _handle(lib, nat, od)
        try:
            assert lib.satb_dit_set_ff_out_fp8(h, 1) != 0 and b"fp8" in lib.satb_last_error()
            assert lib.satb_dit_set_ff_out_fp8(h, 0) == 0
        finally:
            lib.satb_dit_destroy(h)
    for spec, what in (((512, 1, 3, 1), b"use_conv"), ((320, 1, 0, 1), b"128"), ((300, 0, 0, 0), b"128")):
        h = _handle(lib, nat)
        try:
            assert lib.satb_dit_set_feedforward(h, *spec) == 0
            assert lib.satb_dit_set_ff_out_fp8(h, 1) != 0 and what in lib.satb_last_error(), spec
        finally:
            lib.satb_dit_destroy(h)
    h = _handle(lib, nat)                                          # inner 330 pads to 384: accepted
    try:
        assert lib.satb_dit_set_feedforward(h, 330, 0, 0, 1) == 0
        assert lib.satb_dit_set_ff_out_fp8(h, 1) == 0
    finally:
        lib.satb_dit_destroy(h)


def test_other_probes_refuse_the_new_epilogue_codes():
    """satb_gemm_probe, satb_gemm_probe_fp8 and satb_gemm_probe_qk8 refuse the new codes before any launch (the
    argument checks and the instance switch come first; no CUDA call is made)."""
    from stable_audio_tools import _native as nat
    lib = nat.lib()
    buf = ctypes.create_string_buffer(1 << 16)
    a = ctypes.c_void_p((ctypes.addressof(buf) + 15) // 16 * 16)
    for epi in (nat.EPI_SWIGLU_E4M3, nat.EPI_SILU_E4M3, nat.EPI_RESIDUAL_A8):
        for bn in (128, 256):
            p = nat.SatbGemmProbe()
            p.epi, p.bn, p.out, p.h, p.ld = epi, bn, a, a, 256
            assert lib.satb_gemm_probe(a, a, 128, 256, 256, ctypes.byref(p), None) != 0
            assert lib.satb_gemm_probe_fp8(a, a, a, a, 128, 256, 256, ctypes.byref(p), None) != 0
            assert b"no such instance" in lib.satb_last_error()
    p = nat.SatbGemmProbe()
    p.epi, p.bn = nat.EPI_SWIGLU, 256
    assert lib.satb_gemm_probe_ff8(a, a, a, a, 128, 512, 256, ctypes.byref(p), a, a, None) != 0
    assert b"no such instance" in lib.satb_last_error()
