"""CPU: the FP8 operand mode's quantiser rule, its oracle emulation, the operand_dtype mapping and the C ABI's config
check (no GPU needed)."""
import ctypes

import pytest
import torch

from fp8_ref import fp8_operands, fp8_row_exponent, fp8_weight_keys, quantize_fp8_rows


def _row_scale(row):
    q, s = quantize_fp8_rows(torch.tensor([row], dtype=torch.float32))
    return q[0], float(s[0, 0])


@pytest.mark.parametrize("k", [-20, -3, 0, 1, 7, 30])
def test_scale_rule_at_and_just_above_a_boundary(k):
    top = 448.0 * 2.0 ** k
    q, s = _row_scale([top, -top / 3, 1.0 * 2.0 ** k])
    assert s == 2.0 ** k                                    # amax == 448 * 2^k: e = k, the row maximum maps to 448
    assert [float(v) for v in q.float()] == [448.0, -144.0, 1.0]   # -149.33 -> -144 (e4m3 step 16 in [128, 256))
    assert float(q[0].float()) * s == top                    # exact round trip of the maximum
    above = float(torch.nextafter(torch.tensor(top), torch.tensor(float("inf"))))
    q, s = _row_scale([above, 2.0 ** k])
    assert s == 2.0 ** (k + 1)                              # just above: the next power of two
    assert float(q[0].float()) == 224.0                      # 448.000x / 2 rounds to 224
    below = float(torch.nextafter(torch.tensor(top), torch.tensor(0.0)))
    assert _row_scale([below])[1] == 2.0 ** k


def test_scale_rule_zero_row_and_clamp():
    q, s = _row_scale([0.0, -0.0, 0.0, 0.0])
    assert s == 1.0 and torch.all(q.float() == 0)
    # amax far below 448 * 2^-126: e is kept at -126, values then land in the e4m3 subnormals or flush to 0
    assert int(fp8_row_exponent(torch.tensor([2.0 ** -140]))[0]) == -126
    assert int(fp8_row_exponent(torch.tensor([1e-45]))[0]) == -126          # fp32 subnormal amax
    assert int(fp8_row_exponent(torch.tensor([448.0 * 2.0 ** -126]))[0]) == -126
    assert int(fp8_row_exponent(torch.tensor([float.fromhex("0x1.c00002p-118")]))[0]) == -125


def test_small_elements_fall_into_e4m3_subnormals():
    # scale 1 (amax 448): e4m3 subnormals are multiples of 2^-9 below 2^-6
    row = [448.0, 2.0 ** -9, 3 * 2.0 ** -10, 5 * 2.0 ** -10, 2.0 ** -11, 2.0 ** -10, 3 * 2.0 ** -11, 7 * 2.0 ** -9]
    q, s = _row_scale(row)
    assert s == 1.0
    got = [float(v) for v in q.float()]
    # 1.5 * 2^-9 ties to the even 2 * 2^-9; 2.5 * 2^-9 ties to 2 * 2^-9; 2^-11 = 0.25 ulp -> 0; 2^-10 = half an ulp, tie
    # to the even 0; 0.75 ulp -> 1 ulp; 7 * 2^-9 is exact
    assert got == [448.0, 2.0 ** -9, 2.0 ** -8, 2.0 ** -8, 0.0, 0.0, 2.0 ** -9, 7 * 2.0 ** -9]


def test_quantiser_never_overflows_and_is_within_half_an_ulp():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(64, 256, generator=g) * torch.logspace(-30, 30, 64, base=2.0)[:, None]
    q, s = quantize_fp8_rows(x)
    dq = q.float() * s
    assert torch.isfinite(dq).all() and float(q.float().abs().max()) <= 448.0
    amax = x.abs().amax(-1, keepdim=True)
    assert torch.all(amax <= 448.0 * s) and torch.all(amax > 224.0 * s)    # the smallest such power of two
    # e4m3 normals: 3 mantissa bits -> half an ulp is 2^-4 relative; subnormals: 2^-10 absolute (times s)
    err = (dq - x).abs()
    assert torch.all(err <= torch.maximum(x.abs() * 2.0 ** -4, s * 2.0 ** -10))


CFG = dict(io_channels=64, embed_dim=128, depth=2, num_heads=2, cond_token_dim=64, global_cond_dim=128,
           project_cond_tokens=False, transformer_type="continuous_transformer")


def _inputs():
    g = torch.Generator().manual_seed(1)
    return (torch.randn(2, 64, 24, generator=g), torch.rand(2, generator=g), torch.randn(2, 5, 64, generator=g),
            torch.randn(2, 128, generator=g))


@pytest.mark.parametrize("gtype", ["prepend", "adaLN"])
def test_emulation_quantises_exactly_the_three_layernorm_fed_linears(gtype):
    """With the quantiser replaced by a recording fp16 rounding, the FP8 emulation must route exactly to_qkv, cross to_q and
    ff.0 of every layer through it - activation and weight each once per call - and otherwise compute the bits of
    operand_rounding(torch.float16)."""
    from oracle import dit_oracle as do
    cfg = dict(CFG, global_cond_type=gtype)
    sd = do.make_dit_weights(cfg, seed=3)
    x, t, c, ge = _inputs()
    names = {id(v): k for k, v in sd.items()}
    seen = []

    def record(v):   # records the operand and rounds it to fp16, as operand_rounding does
        seen.append(names.get(id(v), "activation"))
        return v.to(torch.float16).to(v.dtype)

    with fp8_operands(sd, roundtrip=record):
        y8 = do.dit_forward(sd, cfg, x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=3.0)
    with do.operand_rounding(torch.float16):
        y16 = do.dit_forward(sd, cfg, x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=3.0)
    assert torch.equal(y8, y16)
    weights = [s for s in seen if s != "activation"]
    assert sorted(weights) == fp8_weight_keys(sd) and len(fp8_weight_keys(sd)) == 3 * cfg["depth"]
    assert seen.count("activation") == len(weights)
    # and the real quantiser changes the output, by about the e4m3 rounding
    with fp8_operands(sd):
        y8 = do.dit_forward(sd, cfg, x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=3.0)
    rel = float((y8 - y16).norm() / y16.norm())
    assert 1e-3 < rel < 0.2, rel
    assert do._lin16.__name__ == "_lin16"                   # the oracle is restored on exit


def test_operand_dtype_strings_map_to_the_abi_values():
    from stable_audio_tools.models.dit import OPERAND_DTYPES, DiffusionTransformer
    assert OPERAND_DTYPES == {"fp16": 0, "bf16": 1, "fp8": 2}
    kw = dict(io_channels=64, embed_dim=128, depth=1, num_heads=2, transformer_type="continuous_transformer")
    for name, code in OPERAND_DTYPES.items():
        assert DiffusionTransformer(**kw, operand_dtype=name).native_config().operand_dtype == code
    assert DiffusionTransformer(**kw).native_config().operand_dtype == 0
    for bad in ("fp32", "FP8", "e4m3", "fp16x3", ""):
        with pytest.raises(ValueError):
            DiffusionTransformer(**kw, operand_dtype=bad)
    from stable_audio_tools.models.diffusion import DiTWrapper
    assert DiTWrapper(**kw, operand_dtype="fp8").model.native_config().operand_dtype == 2
    with pytest.raises(ValueError):
        DiTWrapper(**kw, operand_dtype="int8")


def test_dit_create_accepts_fp8_and_refuses_unknown_operand_types():
    from stable_audio_tools import _native
    lib = _native.lib()
    base = dict(io_channels=64, embed_dim=128, depth=1, num_heads=2, cond_token_dim=64, global_cond_dim=128,
                project_cond_tokens=0, project_global_cond=1, global_cond_type=0, patch_size=1)
    for code in (0, 1, 2):
        h = ctypes.c_void_p()
        assert lib.satb_dit_create(ctypes.byref(_native.SatbDitConfig(**base, operand_dtype=code)), ctypes.byref(h)) == 0
        lib.satb_dit_destroy(h)
    for code in (3, -1):
        h = ctypes.c_void_p()
        rc = lib.satb_dit_create(ctypes.byref(_native.SatbDitConfig(**base, operand_dtype=code)), ctypes.byref(h))
        assert rc != 0 and b"operand_dtype" in lib.satb_last_error()
