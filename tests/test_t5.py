"""CPU: the T5 oracle against the goldens (transformers' T5EncoderModel in fp32, and the reference's own
T5Conditioner), the host bucket table against transformers' _relative_position_bucket, the native encoder's refusals
and ABI entry points (no CUDA call), and the sharpness of the per-element checkers of tests/t5_ref.py."""
import ctypes
import json

import pytest
import torch

import gemm_epilogue_ref as R
import t5_ref
from helpers import load_golden, max_abs, rel_l2
from oracle import t5_oracle as to

GOLDENS = ["t5_relu_hd64.npz", "t5_gelu_hd64_inner.npz", "t5_relu_hd128_inner.npz"]


@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_matches_transformers_golden(name):
    g = load_golden(name)
    cfg = json.loads(str(g["config"]))
    sd = to.make_t5_weights(cfg, int(g["seed"]))
    ids, mask = torch.from_numpy(g["input_ids"]), torch.from_numpy(g["attention_mask"])
    out = to.t5_encoder(sd, cfg, ids, mask)
    assert max_abs(out, torch.from_numpy(g["last_hidden_state"])) <= 1e-5


def test_golden_configs_cover_the_encoder_options():
    cfgs = [json.loads(str(load_golden(n)["config"])) for n in GOLDENS]
    assert {c["feed_forward_proj"] for c in cfgs} == {"relu", "gated-gelu"}
    assert {c["d_kv"] for c in cfgs} == {64, 128}
    assert any(c["num_heads"] * c["d_kv"] != c["d_model"] for c in cfgs if c["d_kv"] == 64)
    assert any(c["num_heads"] * c["d_kv"] != c["d_model"] for c in cfgs if c["d_kv"] == 128)
    assert {(c["relative_attention_num_buckets"], c["relative_attention_max_distance"]) for c in cfgs} >= {(16, 40), (8, 20)}
    for n in GOLDENS:
        m = load_golden(n)["attention_mask"]
        lengths = set(m.sum(1).tolist())
        assert 1 in lengths and m.shape[1] in lengths and len(lengths) >= 3


def test_oracle_matches_the_reference_conditioner_golden():
    """The reference's T5Conditioner (its fp16 model on the CPU, proj_out, mask multiply): padded rows exactly zero,
    the mask as tokenised, and the oracle (fp64 on the fp16-cast weights) within the fp16 stream's own error."""
    g = load_golden("t5_conditioner.npz")
    cfg = json.loads(str(g["config"]))
    sd = {k: v.half().float() for k, v in to.make_t5_weights(cfg, int(g["seed"])).items()}
    w, b = to.make_proj_out(cfg["d_model"], int(g["output_dim"]), int(g["proj_seed"]))
    ids, mask = torch.from_numpy(g["input_ids"]), torch.from_numpy(g["attention_mask"])
    emb = torch.from_numpy(g["embeddings"])
    assert torch.equal(torch.from_numpy(g["mask"]), mask.bool())
    valid = mask.bool()
    assert torch.all(emb[~valid] == 0)
    assert mask.sum(1).tolist()[2] == 0 and mask.sum(1).tolist()[3] == int(g["max_length"])   # an empty and a full prompt
    ref = to.t5_conditioner(sd, cfg, ids, mask, w, b)
    assert rel_l2(emb[valid], ref[valid]) < 1e-2


@pytest.mark.parametrize("nb,md", [(32, 128), (16, 40), (8, 20), (64, 256)])
@pytest.mark.parametrize("L", [1, 16, 128, 512])
def test_bucket_table_is_bit_identical_to_transformers(nb, md, L):
    from transformers.models.t5.modeling_t5 import T5Attention
    from stable_audio_tools.models import t5
    pos = torch.arange(L, dtype=torch.long)
    rel = pos[None, :] - pos[:, None]
    hf = T5Attention._relative_position_bucket(rel, bidirectional=True, num_buckets=nb, max_distance=md)
    assert torch.equal(t5.relative_position_buckets(rel, nb, md), hf)
    assert torch.equal(to.relative_position_bucket(rel, nb, md), hf)
    tab = t5.bucket_table(nb, md)   # what the native encoder indexes with j - i + 511
    assert tab.dtype == torch.int32 and tab.numel() == 1023
    assert torch.equal(tab[(rel + 511).flatten()].view(L, L).long(), hf)


def test_encoder_refuses_unsupported_configs_before_any_cuda_call():
    from stable_audio_tools.models.t5 import T5Encoder
    ok = dict(vocab_size=100, d_model=256, d_kv=64, num_heads=4, d_ff=512, num_layers=1)
    T5Encoder(**ok)
    T5Encoder(**dict(ok, d_kv=128, num_heads=8, d_model=1024, feed_forward_proj="gated-gelu"))
    for bad in (dict(d_kv=32), dict(d_kv=96), dict(feed_forward_proj="gelu"), dict(feed_forward_proj="gated-relu"),
                dict(d_model=200), dict(d_model=4224), dict(d_ff=48)):
        with pytest.raises(NotImplementedError):
            T5Encoder(**dict(ok, **bad))
    with pytest.raises(ValueError):
        T5Encoder(**ok, operand_dtype="fp8")


def test_every_named_t5_model_is_within_the_supported_shapes():
    """d_kv, d_model and d_ff of the ten names of T5_MODEL_DIMS (t5-3b / t5-11b: d_kv 128, inner != d_model)."""
    from stable_audio_tools.models.t5 import check_config
    shapes = {"t5-small": (512, 64, 2048, "relu"), "t5-base": (768, 64, 3072, "relu"), "t5-large": (1024, 64, 4096, "relu"),
              "t5-3b": (1024, 128, 16384, "relu"), "t5-11b": (1024, 128, 65536, "relu"),
              "google/flan-t5-small": (512, 64, 1024, "gated-gelu"), "google/flan-t5-base": (768, 64, 2048, "gated-gelu"),
              "google/flan-t5-large": (1024, 64, 2816, "gated-gelu"), "google/flan-t5-xl": (2048, 64, 5120, "gated-gelu"),
              "google/flan-t5-xxl": (4096, 64, 10240, "gated-gelu")}
    from stable_audio_tools.models.conditioners import T5Conditioner
    assert set(shapes) == set(T5Conditioner.T5_MODEL_DIMS)
    for d_model, d_kv, d_ff, ff in shapes.values():
        check_config(d_model, d_kv, d_ff, ff, "fp16")


def test_prompt_checks():
    from stable_audio_tools.models.t5 import prompt_lengths
    ids = torch.tensor([[5, 6, 7, 0], [9, 0, 0, 0], [0, 0, 0, 0]])
    mask = torch.tensor([[1, 1, 1, 0], [1, 0, 0, 0], [0, 0, 0, 0]])
    assert prompt_lengths(ids, mask, 10).tolist() == [3, 1, 0]
    with pytest.raises(NotImplementedError):
        prompt_lengths(torch.zeros(1, 513, dtype=torch.long), torch.ones(1, 513, dtype=torch.long), 10)
    with pytest.raises(NotImplementedError):   # left padding
        prompt_lengths(ids, torch.tensor([[0, 1, 1, 1], [1, 0, 0, 0], [0, 0, 0, 0]]), 10)
    with pytest.raises(NotImplementedError):   # a hole
        prompt_lengths(ids, torch.tensor([[1, 0, 1, 0], [1, 0, 0, 0], [0, 0, 0, 0]]), 10)
    for bad in (-1, 10):
        b = ids.clone()
        b[0, 0] = bad
        with pytest.raises(ValueError):
            prompt_lengths(b, mask, 10)


def test_cpu_tensors_raise_native_error():
    from stable_audio_tools._native import NativeError
    from stable_audio_tools.models.t5 import T5Encoder
    enc = T5Encoder(vocab_size=100, d_model=256, d_kv=64, num_heads=4, d_ff=512, num_layers=1)
    with pytest.raises(NativeError):
        enc(torch.zeros(1, 4, dtype=torch.long), torch.ones(1, 4, dtype=torch.long))
    with pytest.raises(NativeError):
        enc.load_state_dict({}, device="cpu")


def test_conditioner_refuses_native_with_grad_or_long_prompts():
    from stable_audio_tools.models.conditioners import T5Conditioner
    with pytest.raises(NotImplementedError):
        T5Conditioner(768, native=True, enable_grad=True)
    with pytest.raises(NotImplementedError):
        T5Conditioner(768, native=True, max_length=513)


def test_c_abi_refuses_bad_configs_and_foreign_probe_ids():
    from stable_audio_tools import _native
    lib = _native.lib()
    h = ctypes.c_void_p()
    good = dict(vocab_size=100, d_model=256, d_kv=64, num_heads=4, d_ff=512, num_layers=1,
                relative_attention_num_buckets=32, relative_attention_max_distance=128, feed_forward_proj=0,
                layer_norm_epsilon=1e-6, operand_dtype=0)
    for bad, msg in ((dict(d_kv=96), b"d_kv"), (dict(feed_forward_proj=2), b"feed_forward_proj"),
                     (dict(d_model=200), b"d_model"), (dict(d_model=4224), b"d_model"), (dict(d_ff=40), b"d_ff"),
                     (dict(operand_dtype=2), b"operand_dtype")):
        rc = lib.satb_t5_create(ctypes.byref(_native.SatbT5Config(**dict(good, **bad))), ctypes.byref(h))
        assert rc != 0 and msg in lib.satb_last_error()
    assert lib.satb_t5_create(ctypes.byref(_native.SatbT5Config(**good)), ctypes.byref(h)) == 0
    rc = lib.satb_t5_encode(h, ctypes.c_void_p(1 << 20), (ctypes.c_int * 1)(3), 1, 4, ctypes.c_void_p(1 << 21), None)
    assert rc != 0 and b"finalize" in lib.satb_last_error()
    rc = lib.satb_t5_finalize(h, None)
    assert rc != 0 and b"missing" in lib.satb_last_error()
    bad_buckets = (ctypes.c_int * 1023)(*([0] * 1022 + [32]))
    assert lib.satb_t5_set_buckets(h, bad_buckets, 1023) != 0
    lib.satb_t5_destroy(h)
    fake = ctypes.c_void_p(1 << 20)
    p = _native.SatbGemmProbe(epi=_native.EPI_RELU16, bn=256, out=1 << 22, ld=256)
    rc = lib.satb_gemm_probe(fake, fake, 64, 256, 64, ctypes.byref(p), None)
    assert rc != 0 and b"no such instance" in lib.satb_last_error()
    p.epi = _native.EPI_GEGLU16
    rc = lib.satb_gemm_probe_fp8(fake, fake, fake, fake, 64, 256, 128, ctypes.byref(p), None)
    assert rc != 0 and b"no such instance" in lib.satb_last_error()
    p.epi = _native.EPI_STORE16
    rc = lib.satb_t5_gemm_probe(fake, fake, 64, 256, 64, ctypes.byref(p), None)
    assert rc != 0 and b"no such instance" in lib.satb_last_error()


# ------------------------------------------------------------------------------------------- checker sharpness
def test_rmsnorm_checker_is_sharp():
    g = torch.Generator().manual_seed(0)
    x, w = torch.randn(9, 256, generator=g) * 3, 1 + 0.1 * torch.randn(256, generator=g)
    y = t5_ref.rmsnorm(x, w, 1e-6)
    for out in ("fp16", "bf16", "fp32"):
        good = y.to(R.TORCH_DT[out])
        assert t5_ref.check_rmsnorm(good, y, out)[0] <= 1.0
        assert t5_ref.check_rmsnorm(good.double() * (1 + 4 * (R.E_OUT[out] + 2.0 ** -20)), y, out)[0] > 1.0
        centred = t5_ref.rmsnorm(x - x.mean(-1, keepdim=True), w, 1e-6).to(R.TORCH_DT[out])   # a LayerNorm
        assert t5_ref.check_rmsnorm(centred, y, out)[0] > 1.0
    big = t5_ref.rmsnorm(x, w * 1e5, 1e-6)
    assert t5_ref.check_rmsnorm(big.clamp(-65504, 65504).half(), big, "fp16")[0] <= 1.0
    assert t5_ref.check_rmsnorm(big.half(), big, "fp16")[1] > 0   # inf instead of saturation


@pytest.mark.parametrize("dk", [64, 128])
def test_attention_checker_is_sharp(dk):
    g = torch.Generator().manual_seed(1)
    H, lengths = 2, [1, 17, 40]
    M = sum(lengths)
    for out in ("fp16", "bf16"):
        qkv = (torch.randn(M, 3 * H * dk, generator=g) * 0.3).to(R.TORCH_DT[out])
        bias = torch.randn(H, 1023, generator=g) * 2
        ref = t5_ref.attention(qkv, bias, lengths, H, dk)
        assert t5_ref.check_attention(ref[0].to(R.TORCH_DT[out]), ref, out)[0] <= 1.0
        for wrong in (dict(scale=dk ** -0.5), dict(bias_sign=-1)):
            bad = t5_ref.attention(qkv, bias, lengths, H, dk, **wrong)[0].to(R.TORCH_DT[out])
            assert t5_ref.check_attention(bad, ref, out)[0] > 1.0, wrong
        # keys of the wrong item: one item of all M rows
        bad = t5_ref.attention(qkv, bias, [M], H, dk)[0].to(R.TORCH_DT[out])
        assert t5_ref.check_attention(bad, ref, out)[0] > 1.0


def _attention_dense(qkv16, bias_tab, lengths, H, dk):
    """t5_ref.attention's earlier formulation, all heads at once with the [H, n, n, dk] difference tensor."""
    x = qkv16.double()
    inner = H * dk
    o = torch.zeros(x.shape[0], inner, dtype=torch.float64)
    t1, t2 = torch.zeros_like(o), torch.zeros_like(o)
    r0 = 0
    for n in lengths:
        if n == 0:
            continue
        rows = x[r0:r0 + n]
        q = rows[:, :inner].view(n, H, dk).transpose(0, 1)
        k = rows[:, inner:2 * inner].view(n, H, dk).transpose(0, 1)
        v = rows[:, 2 * inner:].view(n, H, dk).transpose(0, 1)
        i = torch.arange(n)
        b = bias_tab.double()[:, (i[None, :] - i[:, None]) + 511]
        s = q @ k.transpose(1, 2) + b
        p = torch.softmax(s, dim=-1)
        oh = p @ v
        ds = (dk / 16 + 1) * 2.0 ** -22 * (q.abs() @ k.abs().transpose(1, 2)) + 2.0 ** -22 * s.abs()
        dv = (v[:, None, :, :] - oh[:, :, None, :]).abs()
        o[r0:r0 + n] = oh.transpose(0, 1).reshape(n, inner)
        t1[r0:r0 + n] = (p @ v.abs()).transpose(0, 1).reshape(n, inner)
        t2[r0:r0 + n] = ((p * ds)[..., None] * dv).sum(2).transpose(0, 1).reshape(n, inner)
        r0 += n
    return o, t1, t2


@pytest.mark.parametrize("dk", [64, 128])
def test_attention_reference_equals_the_dense_formulation(dk):
    """The head-by-head, query-block-by-block evaluation computes the same three terms to float64 rounding."""
    g = torch.Generator().manual_seed(3)
    H, lengths = 3, [1, 0, 17, 64, 65, 150]
    qkv = (torch.randn(sum(lengths), 3 * H * dk, generator=g) * 0.3).half()
    bias = torch.randn(H, 1023, generator=g) * 2
    new = t5_ref.attention(qkv, bias, lengths, H, dk)
    for a, b in zip(new, _attention_dense(qkv, bias, lengths, H, dk)):
        assert torch.allclose(a, b, rtol=1e-12, atol=0), float(((a - b).abs() / b.abs().clamp_min(1e-300)).max())


@pytest.mark.parametrize("dk", [64, 128])
def test_attention_checker_is_sharp_at_128_heads(dk):
    """t5-11b's head count: a head that reads its neighbour's q columns, a mirrored bias and keys of the wrong item
    are each rejected."""
    g = torch.Generator().manual_seed(4)
    H, lengths = 128, [1, 17, 40]
    M, inner = sum(lengths), H * dk
    qkv = (torch.randn(M, 3 * inner, generator=g) * 0.25).half()
    rel = torch.randn(32, H, generator=g)
    pos = torch.arange(-511, 512)
    bias = rel[to.relative_position_bucket(pos, 32, 128)].T.contiguous()
    ref = t5_ref.attention(qkv, bias, lengths, H, dk)
    assert t5_ref.check_attention(ref[0].half(), ref, "fp16")[0] <= 1.0
    neighbour = qkv.clone()
    neighbour[:, :inner] = qkv[:, :inner].roll(-dk, dims=1)            # head h reads head h + 1's q
    bad = t5_ref.attention(neighbour, bias, lengths, H, dk)[0].half()
    assert t5_ref.check_attention(bad, ref, "fp16")[0] > 1.0
    bad = t5_ref.attention(qkv, bias, lengths, H, dk, bias_sign=-1)[0].half()
    assert t5_ref.check_attention(bad, ref, "fp16")[0] > 1.0
    bad = t5_ref.attention(qkv, bias, [M], H, dk)[0].half()              # keys of the wrong item
    assert t5_ref.check_attention(bad, ref, "fp16")[0] > 1.0


def test_gemm_bound_rejects_a_dropped_k_block_at_k65536():
    """t5-11b's FF-out (K = 65536, residual into the fp32 stream) on t5_ref.gemm_operand's rows: an accumulator that
    loses any one 64-wide k-block fails the bound, the float64 sum rounded to fp32 passes."""
    K, N = 65536, 32
    M = K // 64                        # every k-block is heavy in one row
    g = torch.Generator().manual_seed(5)
    a = t5_ref.both_16bit(t5_ref.gemm_operand(M, K, g))
    w = t5_ref.both_16bit(torch.randn(N, K, generator=g) * K ** -0.5)
    h0 = torch.randn(M, N, generator=g)
    acc, S = R.accumulate(a, w)
    exp = R.epi_residual(acc, S, h0)
    assert R.check((h0.double() + acc).float(), exp, K, "fp32").ok
    for blk in (0, 1, 511, 1023):
        c = slice(64 * blk, 64 * blk + 64)
        dropped = acc - a[:, c].double() @ w[:, c].double().T
        assert not R.check((h0.double() + dropped).float(), exp, K, "fp32").ok, blk


def test_operands_shared_by_fp16_and_bf16_are_exact_in_both():
    g = torch.Generator().manual_seed(6)
    x = t5_ref.both_16bit(torch.cat([torch.randn(4096, generator=g) * s for s in (1e-6, 1e-3, 1, 300)]))
    assert torch.equal(x.half().float(), x) and torch.equal(x.bfloat16().float(), x)
    a = t5_ref.gemm_operand(40, 4096, g)
    heavy = a.abs().view(40, 64, 64).mean(-1).argmax(-1)
    assert torch.equal(heavy, torch.arange(40) % 64)


@pytest.mark.parametrize("out", ["fp16", "bf16"])
def test_ff_in_epilogue_checkers_are_sharp(out):
    g = torch.Generator().manual_seed(2)
    dt = R.TORCH_DT[out]
    a = torch.randn(300, 128, generator=g).to(dt)
    w = (torch.randn(256, 128, generator=g) * 128 ** -0.5).to(dt)
    acc, S = R.accumulate(a, w)
    e = t5_ref.epi_relu(acc, S, out)
    assert R.check(e.ref.to(dt), e, 128, out).ok
    assert not R.check(acc.to(dt), e, 128, out).ok                          # no ReLU
    # an exact accumulator a hair below zero whose fp32 one, off by half the rounding bound, lands above it
    tiny = acc.clone()
    tiny[0, 0] = -0.25 * R.e_acc(128) * S[0, 0]
    e = t5_ref.epi_relu(tiny, S, out)
    kernel = tiny.clone()
    kernel[0, 0] = 0.25 * R.e_acc(128) * S[0, 0]
    assert R.check(kernel.clamp_min(0).to(dt), e, 128, out).ok
    e = t5_ref.epi_geglu(acc, S, out)
    assert R.check(e.ref.to(dt), e, 128, out, col_scale=2).ok
    n = 128
    erf = acc[:, :n] * torch.nn.functional.gelu(acc[:, n:])                # the erf GELU
    assert not R.check(erf.to(dt), e, 128, out, col_scale=2).ok
    swapped = acc[:, n:] * t5_ref.gelu_new(acc[:, :n])                     # gate and value exchanged
    assert not R.check(swapped.to(dt), e, 128, out, col_scale=2).ok
    if out == "fp16":
        big = acc * 1e5
        e = t5_ref.epi_relu(big, S * 1e5, out)
        assert R.check(e.ref.to(dt), e, 128, out).ok
        assert not R.check(big.clamp_min(0).to(dt), e, 128, out).ok         # inf instead of saturation
