"""GPU: the native T5 encoder (csrc/t5.cu, models/t5.py).  Each new kernel against float64 element by element with
the bounds of tests/t5_ref.py (RMSNorm, the attention core on ragged items, the FF-in epilogues through
gemm_epilogue_ref's bound); the whole encoder against the oracle (oracle/t5_oracle.py) at the goldens' configs and
the t5-base / flan-t5-base shapes, gated at 1.25 x the oracle's own 16-bit-operand floor; exactness properties bit for
bit; and T5Conditioner(native=True) end to end."""
import ctypes
import json

import pytest
import torch

import gemm_epilogue_ref as R
import t5_ref
from helpers import load_golden, rel_l2
from oracle import t5_oracle as to

pytestmark = pytest.mark.gpu
DEV = "cuda"
DT = {"fp16": torch.float16, "bf16": torch.bfloat16}


def _lib():
    from stable_audio_tools import _native
    return _native, _native.lib()


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("D", [512, 768, 4096])
@pytest.mark.parametrize("out", ["fp16", "bf16", "fp32"])
def test_rmsnorm_kernel(D, out):
    N, lib = _lib()
    g = torch.Generator().manual_seed(D)
    x = (torch.randn(37, D, generator=g) * 4).to(DEV)
    w = (1 + 0.1 * torch.randn(D, generator=g)).to(DEV)
    kind = {"fp16": 0, "bf16": 1, "fp32": 2}[out]
    y = torch.empty(37, D, device=DEV, dtype=R.TORCH_DT[out])
    N.check(lib.satb_t5_rmsnorm_probe(_p(x), _p(w), _p(y), 37, D, ctypes.c_float(1e-6), kind, None))
    torch.cuda.synchronize()
    ratio, nonfinite = t5_ref.check_rmsnorm(y, t5_ref.rmsnorm(x, w, 1e-6), out)
    assert nonfinite == 0 and ratio <= 1.0, ratio


def test_rmsnorm_kernel_saturates_in_fp16():
    N, lib = _lib()
    x = torch.randn(4, 256, device=DEV)
    w = torch.full((256,), 3e4, device=DEV)
    y = torch.empty(4, 256, device=DEV, dtype=torch.float16)
    N.check(lib.satb_t5_rmsnorm_probe(_p(x), _p(w), _p(y), 4, 256, ctypes.c_float(1e-6), 0, None))
    torch.cuda.synchronize()
    ref = t5_ref.rmsnorm(x, w, 1e-6)
    assert (ref.abs() > 65504).any() and torch.isfinite(y).all()
    ratio, nonfinite = t5_ref.check_rmsnorm(y, ref, "fp16")
    assert nonfinite == 0 and ratio <= 1.0, ratio


@pytest.mark.parametrize("dk", [64, 128])
@pytest.mark.parametrize("out", ["fp16", "bf16"])
def test_attention_core_ragged_items(dk, out):
    N, lib = _lib()
    H, lengths = 2, [1, 17, 64, 65, 127, 128, 512]
    M = sum(lengths)
    g = torch.Generator().manual_seed(dk)
    qkv = (torch.randn(M, 3 * H * dk, generator=g) * 0.25).to(DT[out]).to(DEV)
    bias = (torch.randn(H, 1023, generator=g) * 2).to(DEV)
    o = torch.full((M, H * dk), float("nan"), device=DEV, dtype=DT[out])
    ln = (ctypes.c_int * len(lengths))(*lengths)
    N.check(lib.satb_t5_attention_probe(_p(qkv), _p(bias), ln, len(lengths), H, dk, int(out == "bf16"), _p(o), None))
    torch.cuda.synchronize()
    ratio, nonfinite = t5_ref.check_attention(o, t5_ref.attention(qkv, bias, lengths, H, dk), out)
    assert nonfinite == 0 and ratio <= 1.0, ratio


def _ff_probe(epi, a, w, bn, out):
    N, lib = _lib()
    M, K = a.shape
    n = w.shape[0]
    cols = n // 2 if epi == "geglu" else n
    y = torch.full((M, cols), float("nan"), device=DEV, dtype=DT[out])
    p = N.SatbGemmProbe(epi=N.EPI_GEGLU16 if epi == "geglu" else N.EPI_RELU16, bn=bn, bf16=int(out == "bf16"),
                        out=y.data_ptr(), ld=cols)
    N.check(lib.satb_t5_gemm_probe(_p(a), _p(w), M, n, K, ctypes.byref(p), None))
    torch.cuda.synchronize()
    return y


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("out", ["fp16", "bf16"])
@pytest.mark.parametrize("epi", ["relu", "geglu"])
def test_ff_in_epilogues(epi, out, bn):
    g = torch.Generator().manual_seed(bn)
    M, K, n = 300, 200, 512
    a = torch.randn(M, K, generator=g).to(DT[out])
    w = (torch.randn(n, K, generator=g) * K ** -0.5).to(DT[out])
    acc, S = R.accumulate(a, w)          # reference column order
    if epi == "geglu":
        stored = w[R.ff_perm(n // 2)]      # every 64 rows: 32 of wi_1 (value), then the same 32 of wi_0 (gate)
        exp = t5_ref.epi_geglu(acc, S, out)
    else:
        stored = w
        exp = t5_ref.epi_relu(acc, S, out)
    y = _ff_probe(epi, a.to(DEV).contiguous(), stored.to(DEV).contiguous(), bn, out)
    rep = R.check(y.cpu(), exp, K, out, bn, col_scale=2 if epi == "geglu" else 1)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("epi", ["relu", "geglu"])
def test_ff_in_epilogues_saturate_in_fp16(epi):
    g = torch.Generator().manual_seed(5)
    M, K, n = 130, 64, 256
    a = (torch.randn(M, K, generator=g) * 80).half()    # |acc| up to ~ 4 x 80 x 80 x 8: past 65504
    w = (torch.randn(n, K, generator=g) * 80).half()
    acc, S = R.accumulate(a, w)
    exp = t5_ref.epi_geglu(acc, S, "fp16") if epi == "geglu" else t5_ref.epi_relu(acc, S, "fp16")
    assert (exp.ref.abs() == 65504).any()
    stored = w[R.ff_perm(n // 2)] if epi == "geglu" else w
    y = _ff_probe(epi, a.to(DEV), stored.to(DEV).contiguous(), 256, "fp16")
    assert torch.isfinite(y).all()
    rep = R.check(y.cpu(), exp, K, "fp16", 256, col_scale=2 if epi == "geglu" else 1)
    assert rep.ok, str(rep)


# ------------------------------------------------------------------------------------------------ encoder
def _native(cfg, sd, dtype="fp16"):
    from stable_audio_tools.models.t5 import T5Encoder
    return T5Encoder.from_config(cfg, operand_dtype=dtype).load_state_dict(sd, device=DEV)


def _gate(cfg, sd, ids, mask, got, dtype):
    """rel-L2 over valid rows against the fp64 oracle, and the oracle's own floor with the kernels' roundings."""
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    ids, mask = ids.to(DEV), mask.to(DEV)
    exact = to.t5_encoder(sdd, cfg, ids, mask)
    rounded = to.t5_encoder(sdd, cfg, ids, mask, rounding=to.operand_rounding(DT[dtype]))
    v = mask.bool()
    return rel_l2(got[v], exact[v]), rel_l2(rounded[v], exact[v])


def _prompts(B, L, lengths, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(B, L, dtype=torch.long)
    mask = torch.zeros(B, L, dtype=torch.long)
    for b, n in enumerate(lengths):
        ids[b, :n] = torch.randint(1, vocab, (n,), generator=g)
        mask[b, :n] = 1
    return ids, mask


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("name", ["t5_relu_hd64.npz", "t5_gelu_hd64_inner.npz", "t5_relu_hd128_inner.npz"])
def test_encoder_matches_oracle_on_golden_configs(name, dtype):
    gold = load_golden(name)
    cfg = json.loads(str(gold["config"]))
    sd = to.make_t5_weights(cfg, int(gold["seed"]))
    ids, mask = torch.from_numpy(gold["input_ids"]), torch.from_numpy(gold["attention_mask"])
    out = _native(cfg, sd, dtype)(ids.to(DEV), mask.to(DEV))
    assert torch.all(out[~mask.bool().to(DEV)] == 0)
    err, floor = _gate(cfg, sd, ids, mask, out, dtype)
    assert err <= 1.25 * floor, (err, floor)


T5_BASE = dict(vocab_size=32128, d_model=768, d_kv=64, num_heads=12, d_ff=3072, num_layers=12,
               relative_attention_num_buckets=32, relative_attention_max_distance=128, feed_forward_proj="relu",
               layer_norm_epsilon=1e-6)
FLAN_T5_BASE = dict(T5_BASE, d_ff=2048, feed_forward_proj="gated-gelu")


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", ["t5-base", "flan-t5-base"])
def test_encoder_matches_oracle_at_full_shapes(shape, dtype):
    cfg = T5_BASE if shape == "t5-base" else FLAN_T5_BASE
    sd = to.make_t5_weights(cfg, 21)
    enc = _native(cfg, sd, dtype)
    g = torch.Generator().manual_seed(22)
    lengths = torch.randint(8, 41, (16,), generator=g).tolist()
    lengths[0], lengths[1] = 1, 128
    for B, L, lens in ((16, 128, lengths), (2, 512, [512, 300])):
        ids, mask = _prompts(B, L, lens, cfg["vocab_size"], 23)
        out = enc(ids.to(DEV), mask.to(DEV))
        assert torch.all(out[~mask.bool().to(DEV)] == 0)
        err, floor = _gate(cfg, sd, ids, mask, out, dtype)
        assert err <= 1.25 * floor, (L, err, floor)


def test_encoder_exactness_properties():
    cfg = dict(T5_BASE, num_layers=3)
    sd = to.make_t5_weights(cfg, 31)
    enc = _native(cfg, sd)
    ids, mask = _prompts(5, 128, [23, 1, 40, 0, 128], cfg["vocab_size"], 32)
    ids, mask = ids.to(DEV), mask.to(DEV)
    out = enc(ids, mask)
    assert torch.all(out[~mask.bool()] == 0)
    assert torch.all(out[3] == 0)                                   # an empty prompt
    alone = enc(ids[:1, :], mask[:1, :])
    assert torch.equal(alone[0], out[0])                            # alone == inside a batch of 5 other lengths
    ids256 = torch.zeros(5, 256, dtype=ids.dtype, device=DEV)
    mask256 = torch.zeros(5, 256, dtype=mask.dtype, device=DEV)
    ids256[:, :128], mask256[:, :128] = ids, mask
    out256 = enc(ids256, mask256)
    assert torch.equal(out256[:, :128], out) and torch.all(out256[:, 128:] == 0)   # max_length 128 == 256
    none = enc(torch.zeros(2, 16, dtype=torch.long, device=DEV), torch.zeros(2, 16, dtype=torch.long, device=DEV))
    assert none.shape == (2, 16, 768) and torch.all(none == 0)


# ------------------------------------------------------------------------------------------------ conditioner
def _patched_t5(monkeypatch, cfg, sd):
    import transformers
    from oracle import make_golden as mg
    from oracle.make_golden_t5 import hf_model
    model = hf_model(cfg, sd)
    monkeypatch.setattr(transformers.AutoTokenizer, "from_pretrained", classmethod(lambda cls, *a, **k: mg.FakeTokenizer()))
    monkeypatch.setattr(transformers.T5EncoderModel, "from_pretrained", classmethod(lambda cls, *a, **k: model))
    return mg


def test_native_conditioner_matches_transformers_fp32(monkeypatch):
    from stable_audio_tools.models.conditioners import T5Conditioner
    cfg = dict(T5_BASE, vocab_size=1001, num_layers=4)
    sd = to.make_t5_weights(cfg, 41)
    mg = _patched_t5(monkeypatch, cfg, sd)
    cond = T5Conditioner(512, t5_model_name="t5-base", max_length=64, native=True)
    w, b = to.make_proj_out(768, 512, 42)
    with torch.no_grad():
        cond.proj_out.weight.copy_(w)
        cond.proj_out.bias.copy_(b)
    cond.set_device(DEV)
    texts = ["warm analog pad with slow attack", "kick", "", " ".join(f"w{i}" for i in range(70))]
    emb, mask = cond(texts)
    assert emb.device.type == "cuda" and next(cond.model.parameters()).device.type == "cpu"   # HF module not moved
    enc = mg.FakeTokenizer()(texts, max_length=64)
    assert torch.equal(mask.cpu(), enc["attention_mask"].bool())
    # the same (fp16-cast) weights through HF's module in fp32 on the GPU, masked and projected as the conditioner does
    from oracle.make_golden_t5 import hf_model
    sd16 = {k: v.half().float() for k, v in sd.items()}
    hf = hf_model(cfg, sd16).to(DEV)
    ids, m = enc["input_ids"].to(DEV), enc["attention_mask"].to(DEV)
    with torch.no_grad():
        ref = hf(input_ids=ids, attention_mask=m)["last_hidden_state"]
        ref = (ref @ w.to(DEV).T + b.to(DEV)) * m[..., None].float()
    v = m.bool()
    assert torch.all(emb[~v] == 0)
    sdd = {k: t.to(DEV) for k, t in sd16.items()}
    exact = to.t5_conditioner(sdd, cfg, ids, m, w.to(DEV), b.to(DEV))
    rounded = to.t5_conditioner(sdd, cfg, ids, m, w.to(DEV), b.to(DEV), rounding=to.operand_rounding(torch.float16))
    floor = rel_l2(rounded[v], exact[v])
    assert rel_l2(ref[v], exact[v]) < 1e-5        # HF fp32 == the oracle
    err = rel_l2(emb[v], ref[v])
    assert err <= 1.25 * floor, (err, floor)


def test_generate_txt2audio_with_native_t5(monkeypatch):
    from oracle import make_golden as mg
    from stable_audio_tools import create_model_from_config
    from stable_audio_tools.inference.generation import generate_diffusion_cond
    gold = load_golden("reference_checks.npz")
    cfg = mg.small_txt2audio(json.loads(str(gold["stable_audio_open_1_0_cfg"])))
    for c in cfg["model"]["conditioning"]["configs"]:
        if c["type"] == "t5":
            c["config"]["native"] = True
    t5cfg = dict(T5_BASE, vocab_size=1001, num_layers=2)
    _patched_t5(monkeypatch, t5cfg, to.make_t5_weights(t5cfg, 51))
    torch.manual_seed(0)
    model = create_model_from_config(cfg).eval()
    model.load_state_dict(mg.seeded_conditioner_params(model.state_dict()), strict=False)
    model = model.to(DEV)
    audio = generate_diffusion_cond(model, steps=3, cfg_scale=6, conditioning=mg.CHECK_META[:1], sample_size=8192,
                                    seed=3, device=DEV, disable_tqdm=True)
    assert audio.shape[0] == 1 and audio.shape[-1] == 8192
    assert torch.isfinite(audio).all() and audio.abs().max() > 0
