"""GPU: the native RoBERTa encoder behind CLAPTextConditioner (csrc/roberta.cu, models/roberta.py).  Each launch against
float64 element by element (embedding + LayerNorm with the id-derived positions, the attention core with key prefixes
1 - 512 and every query row, the GELU-bias FF-in epilogue, the residual GEMM followed by the post-LayerNorm); the whole
encoder at the roberta-base shape against the oracle (oracle/clap_oracle.py), gated at 1.25 x the oracle's own
16-bit-operand floor; the conditioner against the reference-side golden; batch invariance bit for bit; and a
text-to-audio generation through the Stable Audio 2.0 conditioning block."""
import ctypes
import json
import os

import pytest
import torch

import gemm_epilogue_ref as R
import t5_ref
from helpers import load_golden, rel_l2
from oracle import clap_oracle as co
from oracle import make_golden as mg
from oracle.make_golden import GOLDEN_DIR
from oracle.make_golden_clap import ids_and_mask
from oracle.t5_oracle import operand_rounding

pytestmark = pytest.mark.gpu
DEV = "cuda"
DT = {"fp16": torch.float16, "bf16": torch.bfloat16}
GELU_SLOPE_MAX = 1.13     # max |gelu'(x)| of the erf GELU (at x ~ 1.5)


def _lib():
    from stable_audio_tools import _native
    return _native, _native.lib()


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


# ------------------------------------------------------------------------------------------------ float64 checkers
def _ln_bound(x, g, b, eps, out):
    """LayerNorm of x [rows, D] in float64 and the per-element bound of an fp32 LayerNorm stored in `out`: half an ulp
    of the output plus the fp32 statistics (mean, centred variance, rsqrtf) relative to |g| (|x| + |mean|) rstd."""
    x, g, b = x.double(), g.double(), b.double()
    mu = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt((x - mu).pow(2).mean(-1, keepdim=True) + eps)
    y = (x - mu) * rstd * g + b
    ref = y.clamp(-65504.0, 65504.0) if out == "fp16" else y
    scale = g.abs() * ((x.abs() + mu.abs()) * rstd + 1.0) + b.abs()
    return ref, R.E_OUT[out] * ref.abs() + 2.0 ** -19 * scale + R.TAU[out]


def _ratio(got, ref, bound):
    got = got.double()
    r = (got - ref).abs() / bound
    return float(torch.where(torch.isfinite(got), r, torch.full_like(r, float("inf"))).max())


def attention_ref(qkv16, lengths, L, H, dk=64):
    """float64 attention of every one of the L query rows of each item over its first lengths[b] keys, scale 1/8, and
    the two bound terms of t5_ref.check_attention."""
    x = qkv16.double()
    inner = H * dk
    o = torch.zeros(x.shape[0], inner, dtype=torch.float64, device=x.device)
    t1, t2 = torch.zeros_like(o), torch.zeros_like(o)
    for b, n in enumerate(lengths):
        rows = x[b * L:(b + 1) * L]
        for h in range(H):
            c = slice(h * dk, (h + 1) * dk)
            q = rows[:, c]
            k = rows[:n, inner + h * dk:inner + (h + 1) * dk]
            v = rows[:n, 2 * inner + h * dk:2 * inner + (h + 1) * dk]
            s = (q @ k.T) * dk ** -0.5
            p = torch.softmax(s, dim=-1)
            oh = p @ v
            ds = (dk / 16 + 1) * 2.0 ** -22 * dk ** -0.5 * (q.abs() @ k.abs().T) + 2.0 ** -22 * s.abs()
            w = p * ds
            o[b * L:(b + 1) * L, c] = oh
            t1[b * L:(b + 1) * L, c] = p @ v.abs()
            for i0 in range(0, L, 64):
                blk = slice(i0, min(i0 + 64, L))
                t2[b * L + i0:b * L + blk.stop, c] = (w[blk, :, None] * (v[None] - oh[blk, None, :]).abs()).sum(1)
    return o, t1, t2


def epi_bias_gelu(acc, S, bias, out):
    x = acc + bias.double()
    y = 0.5 * x * (1 + torch.erf(x / 2 ** 0.5))
    ref = y.clamp(-65504.0, 65504.0) if out == "fp16" else y
    return R.Expect(ref, GELU_SLOPE_MAX * S, y.abs() * (x.abs() + 4) + acc.abs() + bias.double().abs())


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("D", [128, 768, 1024])
@pytest.mark.parametrize("out", ["fp16", "bf16"])
def test_embedding_layernorm_kernel(D, out):
    N, lib = _lib()
    g = torch.Generator().manual_seed(D)
    vocab, max_pos, L = 1001, 514, 77
    ids, mask = ids_and_mask([77, 1, 40, 77, 9], L, vocab, D)   # pad ids inside prompts 0 and 3
    ids[4, 3] = 0
    word, pos = torch.randn(vocab, D, generator=g), torch.randn(max_pos, D, generator=g)
    tok, gam, bet = torch.randn(1, D, generator=g), 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    B = ids.shape[0]
    y32 = torch.full((B * L, D), float("nan"), device=DEV)
    y16 = torch.full((B * L, D), float("nan"), device=DEV, dtype=DT[out])
    d = {k: v.to(DEV).contiguous() for k, v in dict(ids=ids, word=word, pos=pos, tok=tok, g=gam, b=bet).items()}
    N.check(lib.satb_roberta_embed_probe(_p(d["ids"]), B, L, _p(d["word"]), vocab, _p(d["pos"]), max_pos, _p(d["tok"]),
                                         _p(d["g"]), _p(d["b"]), D, 1, ctypes.c_float(1e-5), _p(y32), _p(y16),
                                         int(out == "bf16"), None))
    torch.cuda.synchronize()
    p = co.position_ids(ids, 1)
    x = (word.double()[ids] + tok.double()[0]) + pos.double()[p]
    ref32, b32 = _ln_bound(x.view(B * L, D).to(DEV), d["g"], d["b"], 1e-5, "fp32")
    ref16, b16 = _ln_bound(x.view(B * L, D).to(DEV), d["g"], d["b"], 1e-5, out)
    assert _ratio(y32, ref32, b32) <= 1.0
    assert _ratio(y16, ref16, b16) <= 1.0
    # a position off by one is far outside the bound
    wrong = (word.double()[ids] + tok.double()[0]) + pos.double()[(p + 1).clamp_max(max_pos - 1)]
    refw, _ = _ln_bound(wrong.view(B * L, D).to(DEV), d["g"], d["b"], 1e-5, "fp32")
    assert _ratio(refw.float(), ref32, b32) > 1.0


@pytest.mark.parametrize("D", [768, 1024])
@pytest.mark.parametrize("out", ["fp16", "bf16"])
def test_residual_then_post_layernorm(D, out):
    """The out-proj / FF-out GEMM with bias into the fp32 stream (EpiResidual), then the LayerNorm kernel in place."""
    N, lib = _lib()
    g = torch.Generator().manual_seed(D + 1)
    M, K = 300, 3072 if D == 768 else 1024
    a = torch.randn(M, K, generator=g).to(DT[out])
    w = (torch.randn(D, K, generator=g) * K ** -0.5).to(DT[out])
    bias = 0.1 * torch.randn(D, generator=g)
    h0 = torch.randn(M, D, generator=g)
    gam, bet = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    h = h0.to(DEV).contiguous()
    ad, wd, bd, gd, btd = a.to(DEV), w.to(DEV), bias.to(DEV), gam.to(DEV), bet.to(DEV)   # alive across the launch
    p = N.SatbGemmProbe(epi=N.EPI_RESIDUAL, bf16=int(out == "bf16"), h=h.data_ptr(), ld=D, bias=bd.data_ptr())
    N.check(lib.satb_roberta_linear_probe(_p(ad), _p(wd), M, D, K, ctypes.byref(p), None))
    torch.cuda.synchronize()
    acc, S = R.accumulate(a, w)
    rep = R.check(h.cpu(), R.epi_residual(acc, S, h0, bias), K, "fp32")
    assert rep.ok, str(rep)
    x = h.clone()
    y16 = torch.full((M, D), float("nan"), device=DEV, dtype=DT[out])
    N.check(lib.satb_roberta_layernorm_probe(_p(h), _p(gd), _p(btd), M, D, ctypes.c_float(1e-5), _p(h), _p(y16),
                                             int(out == "bf16"), None))
    torch.cuda.synchronize()
    ref32, b32 = _ln_bound(x, gd, btd, 1e-5, "fp32")
    ref16, b16 = _ln_bound(x, gd, btd, 1e-5, out)
    assert _ratio(h, ref32, b32) <= 1.0 and _ratio(y16, ref16, b16) <= 1.0


@pytest.mark.parametrize("out", ["fp16", "bf16"])
@pytest.mark.parametrize("L,lengths", [(77, [1, 2, 33, 77]), (512, [512, 1, 2, 33, 77, 300])])
def test_attention_core_key_prefixes(L, lengths, out):
    N, lib = _lib()
    H = 12
    B = len(lengths)
    g = torch.Generator().manual_seed(L + len(lengths))
    qkv = (torch.randn(B * L, 3 * H * 64, generator=g) * 0.5).to(DT[out]).to(DEV)
    o = torch.full((B * L, H * 64), float("nan"), device=DEV, dtype=DT[out])
    ln = (ctypes.c_int * B)(*lengths)
    N.check(lib.satb_roberta_attention_probe(_p(qkv), ln, B, L, H, int(out == "bf16"), _p(o), None))
    torch.cuda.synchronize()
    ref = attention_ref(qkv, lengths, L, H)
    ratio, nonfinite = t5_ref.check_attention(o, ref, out)
    assert nonfinite == 0 and ratio <= 1.0, ratio
    # sharpness: keys past the prefix, or no 1/8 scale, are rejected
    wrong = attention_ref(qkv, [L] * B, L, H)[0]
    assert t5_ref.check_attention(wrong.to(DT[out]), ref, out)[0] > 1.0


@pytest.mark.parametrize("out", ["fp16", "bf16"])
@pytest.mark.parametrize("M,N_", [(300, 3072), (77, 512), (1232, 3072)])
def test_ff_in_bias_gelu_epilogue(M, N_, out):
    N, lib = _lib()
    g = torch.Generator().manual_seed(M)
    K = 768
    a = torch.randn(M, K, generator=g).to(DT[out])
    w = (torch.randn(N_, K, generator=g) * K ** -0.5 * 2).to(DT[out])
    bias = 0.5 * torch.randn(N_, generator=g)
    y = torch.full((M, N_), float("nan"), device=DEV, dtype=DT[out])
    ad, wd, bd = a.to(DEV), w.to(DEV), bias.to(DEV)   # alive across the launch
    p = N.SatbGemmProbe(epi=N.EPI_BIAS_GELU16, bf16=int(out == "bf16"), out=y.data_ptr(), ld=N_, bias=bd.data_ptr())
    N.check(lib.satb_roberta_linear_probe(_p(ad), _p(wd), M, N_, K, ctypes.byref(p), None))
    torch.cuda.synchronize()
    acc, S = R.accumulate(a, w)
    exp = epi_bias_gelu(acc, S, bias, out)
    rep = R.check(y.cpu(), exp, K, out)
    assert rep.ok, str(rep)
    tanh = acc + bias.double()
    tanh = t5_ref.gelu_new(tanh)                                  # T5's gelu_new is not this epilogue
    assert not R.check(tanh.to(DT[out]), exp, K, out).ok


# ------------------------------------------------------------------------------------------------ encoder
@pytest.fixture(scope="module")
def roberta_base():
    return co.make_roberta_weights(co.ROBERTA_BASE, 91)


def _encoder(cfg, sd, feature_layer_ix, dtype, proj=None):
    from stable_audio_tools.models.roberta import RobertaEncoder
    enc = RobertaEncoder.from_config(cfg, feature_layer_ix=feature_layer_ix, operand_dtype=dtype)
    enc.load_state_dict(sd, device=DEV)
    if proj is not None:
        enc.set_proj_out(*proj)
    return enc


def _gate(cfg, sd, ids, mask, ix, got, dtype, proj=(None, None)):
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    ids, mask = ids.to(DEV), mask.to(DEV)
    pw, pb = (t.to(DEV) if t is not None else None for t in proj)
    exact = co.clap_features(sdd, cfg, ids, mask, ix, pw, pb)
    rounded = co.clap_features(sdd, cfg, ids, mask, ix, pw, pb, rounding=operand_rounding(DT[dtype]))
    return rel_l2(got, exact), rel_l2(rounded, exact)


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("B", [1, 2, 5, 16])
def test_encoder_matches_oracle_at_roberta_base(roberta_base, B, dtype):
    cfg = co.ROBERTA_BASE
    g = torch.Generator().manual_seed(B)
    lengths = torch.randint(2, 78, (B,), generator=g).tolist()
    lengths[0] = 77
    if B > 1:
        lengths[1] = 1
    ids, mask = ids_and_mask(lengths, 77, cfg["vocab_size"], 92 + B)
    w, b = torch.randn(768, 768, generator=g) * 768 ** -0.5, 0.1 * torch.randn(768, generator=g)
    for ix, proj in ((-2, None), (-1, (w, b))):
        enc = _encoder(cfg, roberta_base, ix, dtype, proj)
        out = enc(ids.to(DEV), mask.to(DEV))
        assert out.shape == (B, 77, 768) and torch.isfinite(out).all()
        err, floor = _gate(cfg, roberta_base, ids, mask, ix, out, dtype, proj or (None, None))
        assert err <= 1.25 * floor, (ix, err, floor)
        enc.close()


@pytest.mark.parametrize("name", ["clap_d128_l2.npz", "clap_d256_l3.npz"])
def test_encoder_matches_oracle_at_every_depth_of_the_goldens(name):
    gold = load_golden(name)
    cfg = json.loads(str(gold["config"]))
    sd = co.make_roberta_weights(cfg, int(gold["seed"]))
    ids, mask = torch.from_numpy(gold["input_ids"]), torch.from_numpy(gold["attention_mask"])
    for ix in range(cfg["num_hidden_layers"] + 1):   # 0 is the embedding output
        out = _encoder(cfg, sd, ix, "fp16")(ids.to(DEV), mask.to(DEV))
        err, floor = _gate(cfg, sd, ids, mask, ix, out, "fp16")
        assert err <= 1.25 * floor + 1e-6, (ix, err, floor)


def test_one_item_alone_equals_the_item_inside_a_batch(roberta_base):
    cfg = co.ROBERTA_BASE
    enc = _encoder(cfg, roberta_base, -2, "fp16")
    ids, mask = ids_and_mask([23, 1, 77, 40, 5, 77, 12], 77, cfg["vocab_size"], 95)
    ids, mask = ids.to(DEV), mask.to(DEV)
    out = enc(ids, mask)
    for b in (0, 1, 3):
        assert torch.equal(enc(ids[b:b + 1], mask[b:b + 1])[0], out[b]), b


# ------------------------------------------------------------------------------------------------ conditioner
@pytest.fixture
def stub_tokenizer(monkeypatch):
    import transformers
    monkeypatch.setattr(transformers.RobertaTokenizer, "from_pretrained",
                        classmethod(lambda cls, *a, **k: mg.FakeTokenizer()))


def _checkpoint(tmp_path, sd):
    path = str(tmp_path / "clap.pt")
    torch.save({"state_dict": {"module.text_branch." + k: v for k, v in sd.items()}}, path)
    return path


def test_conditioner_matches_the_reference_golden(tmp_path, stub_tokenizer):
    from stable_audio_tools.models.conditioners import CLAPTextConditioner
    gold = load_golden("clap_conditioner.npz")
    cfg = json.loads(str(gold["config"]))
    sd = co.make_roberta_weights(cfg, int(gold["seed"]))
    cond = CLAPTextConditioner(int(gold["output_dim"]), clap_ckpt_path=_checkpoint(tmp_path, sd),
                               use_text_features=True, feature_layer_ix=int(gold["feature_layer_ix"]))
    cond.set_device(DEV)
    texts = [str(t) for t in gold["texts"]]
    feats, mask = cond(texts)
    assert torch.equal(mask.cpu(), torch.from_numpy(gold["mask"]))
    ref = torch.from_numpy(gold["features"]).to(DEV)
    ids, m = torch.from_numpy(gold["input_ids"]), torch.from_numpy(gold["attention_mask"])
    _, floor = _gate(cfg, sd, ids, m, -2, feats, "fp16")
    err = rel_l2(feats, ref)   # every position, padded ones included
    assert err <= 1.25 * floor, (err, floor)
    single, m1 = cond(texts[:1])
    assert single.shape == (1, 77, 768) and torch.equal(m1.cpu(), torch.from_numpy(gold["single_mask"]))
    assert torch.equal(single[0], feats[0])


def test_generate_txt2audio_through_the_sa20_conditioning(tmp_path, stub_tokenizer):
    from stable_audio_tools import create_model_from_config
    from stable_audio_tools.inference.generation import generate_diffusion_cond
    gold = load_golden("reference_checks.npz")
    cfg = mg.small_txt2audio(json.loads(str(gold["stable_audio_2_0_cfg"])))
    cfg["model"]["conditioning"] = json.load(open(os.path.join(GOLDEN_DIR, "clap_sa20_conditioning.json")))
    small = dict(co.ROBERTA_BASE, vocab_size=1001, num_hidden_layers=2, intermediate_size=256)
    path = _checkpoint(tmp_path, co.make_roberta_weights(small, 97))
    for c in cfg["model"]["conditioning"]["configs"]:
        if c["type"] == "clap_text":
            c["config"]["clap_ckpt_path"] = path
    torch.manual_seed(0)
    model = create_model_from_config(cfg).eval()
    model.load_state_dict(mg.seeded_conditioner_params(model.state_dict()), strict=False)
    model = model.to(DEV)
    meta = [{"prompt": "warm analog pad", "seconds_start": 0, "seconds_total": 4}]
    audio = generate_diffusion_cond(model, steps=3, cfg_scale=6, conditioning=meta, sample_size=8192, seed=3,
                                    device=DEV, disable_tqdm=True)
    assert audio.shape[0] == 1 and audio.shape[-1] == 8192
    assert torch.isfinite(audio).all() and audio.abs().max() > 0
