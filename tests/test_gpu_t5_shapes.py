"""GPU: the native T5 encoder (csrc/t5.cu) at the shapes of all ten named T5 models of T5Conditioner.T5_MODEL_DIMS,
launch by launch against float64 and end to end against the oracle.

  a. the attention core element by element at every (heads, d_kv) of the ten, on ragged items, with the bias table
     of the real buckets (32 / 128);
  b. every GEMM of an encode (QKV, o-projection, FF-in, FF-out, proj_out) at each model's (N, K) through
     satb_t5_linear_probe, the encoder's own launch: M 1, 37 and 2048 (and 8192 at the largest N), BN 128, 256 and the
     one auto_bn picks; rows of A past M (inside the tensor map, as in the encoder's workspace) hold NaN and must not
     change a bit of the output;
  c. the finalized bias table bit for bit against rel[bucket(j - i), h];
  d. RMSNorm at the widths only these models reach;
  e. the whole encoder, two blocks at full width, against the oracle at 1.25 x its own 16-bit-operand floor;
  f. T5Conditioner(native=True) for each name against HF's module in fp32.
Every check prints its worst err / bound (or err / floor) into a table at the end of the module (pytest -s).
Two blocks are enough in (e) and one in (f): every launch shape is independent of depth."""
import ctypes
import time

import pytest
import torch

import gemm_epilogue_ref as R
import t5_ref
from helpers import rel_l2
from oracle import t5_oracle as to

pytestmark = pytest.mark.gpu
DEV = "cuda"
DT = {"fp16": torch.float16, "bf16": torch.bfloat16}

# The published T5Config values of the ten names (the table of tests/test_t5.py, with heads and depth).
COMMON = dict(vocab_size=32128, relative_attention_num_buckets=32, relative_attention_max_distance=128,
              layer_norm_epsilon=1e-6)
MODELS = {
    "t5-small": dict(COMMON, d_model=512, d_kv=64, num_heads=8, d_ff=2048, feed_forward_proj="relu", num_layers=6),
    "t5-base": dict(COMMON, d_model=768, d_kv=64, num_heads=12, d_ff=3072, feed_forward_proj="relu", num_layers=12),
    "t5-large": dict(COMMON, d_model=1024, d_kv=64, num_heads=16, d_ff=4096, feed_forward_proj="relu", num_layers=24),
    "t5-3b": dict(COMMON, d_model=1024, d_kv=128, num_heads=32, d_ff=16384, feed_forward_proj="relu", num_layers=24),
    "t5-11b": dict(COMMON, d_model=1024, d_kv=128, num_heads=128, d_ff=65536, feed_forward_proj="relu", num_layers=24),
    "google/flan-t5-small": dict(COMMON, d_model=512, d_kv=64, num_heads=6, d_ff=1024, feed_forward_proj="gated-gelu",
                                 num_layers=8),
    "google/flan-t5-base": dict(COMMON, d_model=768, d_kv=64, num_heads=12, d_ff=2048, feed_forward_proj="gated-gelu",
                                num_layers=12),
    "google/flan-t5-large": dict(COMMON, d_model=1024, d_kv=64, num_heads=16, d_ff=2816, feed_forward_proj="gated-gelu",
                                 num_layers=24),
    "google/flan-t5-xl": dict(COMMON, d_model=2048, d_kv=64, num_heads=32, d_ff=5120, feed_forward_proj="gated-gelu",
                              num_layers=24),
    "google/flan-t5-xxl": dict(COMMON, d_model=4096, d_kv=64, num_heads=64, d_ff=10240, feed_forward_proj="gated-gelu",
                               num_layers=24),
}
SHORT = {n: n.split("/")[-1] for n in MODELS}
PROJ_OUT = (768, 1536, 40)     # conditioner output widths: SA-Open's 768, 1536, and one that is not a multiple of 32


def _lib():
    from stable_audio_tools import _native
    return _native, _native.lib()


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.fixture(scope="module")
def report():
    """Rows (check, shape, kernel, dtype, worst ratio) printed as one table when the module ends."""
    rows = []
    t0 = time.perf_counter()
    yield rows
    print(f"\n{'check':<10} {'shape':<44} {'kernel / GEMM role, BN':<42} {'dtype':<5} worst")
    for check, shape, kernel, dtype, ratio in rows:
        print(f"{check:<10} {shape:<44} {kernel:<42} {dtype:<5} {ratio:.3f}")
    print(f"test_gpu_t5_shapes: {time.perf_counter() - t0:.0f} s")


# ------------------------------------------------------------------------------------------------ a. attention core
HEAD_SHAPES = sorted({(c["num_heads"], c["d_kv"]) for c in MODELS.values()})


def _bias_table(H, seed):
    """[H, 1023]: rel[bucket(k - 511), h] with the real buckets (32 / 128) and a seeded rel [32, H]."""
    rel = torch.randn(32, H, generator=torch.Generator().manual_seed(seed))
    pos = torch.arange(-(t5_ref.BIAS_SPAN // 2), t5_ref.BIAS_SPAN // 2 + 1)
    return rel, rel[to.relative_position_bucket(pos, 32, 128)].T.contiguous()


@pytest.mark.parametrize("out", ["fp16", "bf16"])
@pytest.mark.parametrize("H,dk", HEAD_SHAPES, ids=[f"H{h}_dk{d}" for h, d in HEAD_SHAPES])
def test_attention_core_at_named_head_shapes(H, dk, out, report):
    N, lib = _lib()
    lengths = [1, 65, 512] if H == 128 else [1, 63, 64, 65, 129, 511, 512]
    M = sum(lengths)
    g = torch.Generator().manual_seed(H * dk)
    qkv = (torch.randn(M, 3 * H * dk, generator=g) * 0.25).to(DT[out]).to(DEV)
    bias = _bias_table(H, H)[1].to(DEV)
    o = torch.full((M, H * dk), float("nan"), device=DEV, dtype=DT[out])
    ln = (ctypes.c_int * len(lengths))(*lengths)
    N.check(lib.satb_t5_attention_probe(_p(qkv), _p(bias), ln, len(lengths), H, dk, int(out == "bf16"), _p(o), None))
    torch.cuda.synchronize()
    ratio, nonfinite = t5_ref.check_attention(o, t5_ref.attention(qkv, bias, lengths, H, dk), out)
    names = ", ".join(SHORT[n] for n, c in MODELS.items() if (c["num_heads"], c["d_kv"]) == (H, dk))
    report.append(("attention", names, f"t5_attn_kernel<{dk}> H {H}", out, ratio))
    assert nonfinite == 0 and ratio <= 1.0, ratio


# ------------------------------------------------------------------------------------------------ b. GEMMs
def _gemm_cases():
    """(role, N, K) -> the names that run it; one case per distinct GEMM."""
    cases = {}
    for name, c in MODELS.items():
        D, inner, F = c["d_model"], c["num_heads"] * c["d_kv"], c["d_ff"]
        gated = c["feed_forward_proj"] == "gated-gelu"
        roles = [("qkv", 3 * inner, D), ("o_proj", D, inner), ("ff_in_geglu" if gated else "ff_in_relu", 2 * F if gated else F, D),
                 ("ff_out", D, F)] + [("proj_out", n, D) for n in PROJ_OUT]
        for r in roles:
            cases.setdefault(r, []).append(SHORT[name])
    return cases


GEMM_CASES = _gemm_cases()
LARGEST_N = max(n for (_, n, _) in GEMM_CASES)
EPI = {"qkv": "EPI_STORE16", "o_proj": "EPI_RESIDUAL", "ff_out": "EPI_RESIDUAL", "ff_in_relu": "EPI_RELU16",
       "ff_in_geglu": "EPI_GEGLU16", "proj_out": "EPI_STORE32"}
INSTANCE = {"qkv": "EpiStore16", "o_proj": "EpiResidual", "ff_out": "EpiResidual", "ff_in_relu": "EpiRelu16",
            "ff_in_geglu": "EpiGeglu16", "proj_out": "EpiStore32"}
ROW_CHUNK = 2048          # rows of the float64 reference at a time


def _out_cols(role, N):
    return N // 2 if role == "ff_in_geglu" else N


def _run_probe(role, a16, a_rows, M, w16, N, K, bn, dtype, bias, h0):
    """One satb_t5_linear_probe call: the output [M, cols] (16-bit, fp32, or the updated residual stream)."""
    nat, lib = _lib()
    cols = _out_cols(role, N)
    p = nat.SatbGemmProbe(epi=getattr(nat, EPI[role]), bn=bn, bf16=int(dtype == "bf16"))
    if role in ("o_proj", "ff_out"):
        y = h0[:M].clone()
        p.h, p.ld = y.data_ptr(), N
    else:
        y = torch.full((M, cols), float("nan"), device=DEV, dtype=torch.float32 if role == "proj_out" else DT[dtype])
        p.out, p.ld = y.data_ptr(), cols
        if role == "proj_out":
            p.bias = bias.data_ptr()
    nat.check(lib.satb_t5_linear_probe(_p(a16), a_rows, _p(w16), M, N, K, ctypes.byref(p), None))
    return y


def _expect(role, acc, S, dtype, bias, h0):
    if role == "qkv":
        return R.epi_store(acc, S)
    if role in ("o_proj", "ff_out"):
        return R.epi_residual(acc, S, h0)
    if role == "proj_out":
        return R.epi_store(acc, S, bias)
    if role == "ff_in_relu":
        return t5_ref.epi_relu(acc, S, dtype)
    return t5_ref.epi_geglu(acc, S, dtype)


def _gemm_params():
    out = []
    for (role, N, K), names in sorted(GEMM_CASES.items(), key=lambda kv: (kv[0][0], kv[0][1] * kv[0][2])):
        out.append(pytest.param(role, N, K, ",".join(names), id=f"{role}-N{N}-K{K}"))
    return out


@pytest.mark.parametrize("role,N,K,names", _gemm_params())
def test_every_gemm_of_an_encode(role, N, K, names, report):
    """One set of operands (bf16 values fp16 holds exactly, t5_ref.gemm_operand's heavy k-blocks) and so one float64
    reference for both operand types; M = 1 and 37 are the first rows of the M = 2048 (8192) operand."""
    Ms = [1, 37, 2048] + ([8192] if N == LARGEST_N else [])
    M_max = max(Ms)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator().manual_seed(N * 7 + K)
    a32 = t5_ref.both_16bit(t5_ref.gemm_operand(M_max, K, g)).to(DEV)
    w_ref = t5_ref.both_16bit(torch.randn(N, K, generator=g) * K ** -0.5).to(DEV)    # reference row order
    w_stored = w_ref[R.ff_perm(N // 2).to(DEV)].contiguous() if role == "ff_in_geglu" else w_ref
    bias = (0.1 * torch.randn(N, generator=g)).to(DEV) if role == "proj_out" else None
    h0 = torch.randn(M_max, N, generator=g).to(DEV) if role in ("o_proj", "ff_out") else None
    outs = {}
    for dtype in ("fp16", "bf16"):
        a16, w16 = a32.to(DT[dtype]), w_stored.to(DT[dtype])
        for M in Ms:
            pad = torch.full((M + 256, K), float("nan"), device=DEV, dtype=DT[dtype])   # rows M.. of A: NaN
            pad[:M] = a16[:M]
            for bn in (128, 256, 0):
                y = _run_probe(role, a16, M, M, w16, N, K, bn, dtype, bias, h0)
                y_pad = _run_probe(role, pad, M + 256, M, w16, N, K, bn, dtype, bias, h0)
                torch.cuda.synchronize()
                assert torch.equal(y.view(torch.int16 if y.element_size() == 2 else torch.int32),
                                   y_pad.view(torch.int16 if y.element_size() == 2 else torch.int32)), \
                    (dtype, M, bn, "rows past M changed the output")
                outs[(dtype, M, bn)] = y
        del pad, y_pad
    worst = {}
    for r0 in range(0, M_max, ROW_CHUNK):
        r1 = min(r0 + ROW_CHUNK, M_max)
        acc, S = R.accumulate(a32[r0:r1], w_ref)
        for dtype in ("fp16", "bf16"):
            exp = _expect(role, acc, S, dtype, bias, h0[r0:r1] if h0 is not None else None)
            for (dt, M, bn), y in outs.items():
                if dt != dtype or M <= r0:
                    continue
                m1 = min(r1, M) - r0
                sub = R.Expect(exp.ref[:m1], exp.sens[:m1], exp.mag[:m1])
                out_kind = "fp32" if role in ("o_proj", "ff_out", "proj_out") else dtype
                rep = R.check(y[r0:r0 + m1], sub, K, out_kind, bn or 256, col_scale=2 if role == "ff_in_geglu" else 1)
                key = (dtype, bn)
                if key not in worst or rep.ratio > worst[key][0].ratio or not rep.ok:
                    worst[key] = (rep, M)
                assert rep.ok, (dtype, M, bn, str(rep))
            del exp
        del acc, S
    for (dtype, bn), (rep, M) in sorted(worst.items(), key=lambda kv: (kv[0][0], kv[0][1] or 999)):
        picks = {}
        for m in Ms:
            picks.setdefault(t5_ref.auto_bn(m, N, sms), []).append(str(m))
        label = f"BN {bn}" if bn else "BN 0 -> " + ", ".join(f"{b} (M {','.join(ms)})" for b, ms in sorted(picks.items()))
        report.append(("gemm", f"{names} N {N} K {K}", f"{role} {INSTANCE[role]} {label}", dtype, rep.ratio))


def test_proj_out_auto_tile_at_conditioner_shapes_is_bn128():
    """auto_bn at a conditioner's rows (one m-tile) and widths 768 / 1536 picks BN 128: the EpiStore32 BN 128 instance
    test_every_gemm_of_an_encode runs with bn 0 is the one every native conditioner output comes from."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for n in (768, 1536):
        assert t5_ref.auto_bn(37, n, sms) == 128
        assert t5_ref.auto_bn(1, n, sms) == 128


# ------------------------------------------------------------------------------------------------ c. bias table
@pytest.mark.parametrize("H", [6, 12, 64, 128])
def test_bias_table_is_bit_exact(H, report):
    """The finalized table of a one-block encoder equals rel[bucket(k - 511), h]; 32 buckets != H, so a transposed
    index into rel [num_buckets, H] cannot pass."""
    nat, lib = _lib()
    from stable_audio_tools.models.t5 import T5Encoder
    cfg = dict(COMMON, vocab_size=8, d_model=128, d_kv=64, num_heads=H, d_ff=32, num_layers=1, feed_forward_proj="relu")
    sd = to.make_t5_weights(cfg, 60 + H)
    enc = T5Encoder.from_config(cfg).load_state_dict(sd, device=DEV)
    got = torch.full((H, t5_ref.BIAS_SPAN), float("nan"), device=DEV)
    nat.check(lib.satb_t5_bias_table(enc._h, _p(got), None))
    rel = sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"]
    pos = torch.arange(-(t5_ref.BIAS_SPAN // 2), t5_ref.BIAS_SPAN // 2 + 1)
    exp = rel[to.relative_position_bucket(pos, 32, 128)].T
    enc.close()
    report.append(("bias", f"H {H}", "t5_bias_table_kernel (bit-exact)", "fp32", 0.0 if torch.equal(got.cpu(), exp) else 1e9))
    assert torch.equal(got.cpu(), exp)


# ------------------------------------------------------------------------------------------------ d. RMSNorm
@pytest.mark.parametrize("D", [1024, 2048])
@pytest.mark.parametrize("out", ["fp16", "bf16", "fp32"])
def test_rmsnorm_at_named_widths(D, out, report):
    nat, lib = _lib()
    g = torch.Generator().manual_seed(D + 1)
    x = (torch.randn(37, D, generator=g) * 4).to(DEV)
    w = (1 + 0.1 * torch.randn(D, generator=g)).to(DEV)
    y = torch.full((37, D), float("nan"), device=DEV, dtype=R.TORCH_DT[out])
    nat.check(lib.satb_t5_rmsnorm_probe(_p(x), _p(w), _p(y), 37, D, ctypes.c_float(1e-6), {"fp16": 0, "bf16": 1, "fp32": 2}[out], None))
    torch.cuda.synchronize()
    ratio, nonfinite = t5_ref.check_rmsnorm(y, t5_ref.rmsnorm(x, w, 1e-6), out)
    report.append(("rmsnorm", f"D {D}", "t5_rmsnorm_kernel", out, ratio))
    assert nonfinite == 0 and ratio <= 1.0, ratio


# ------------------------------------------------------------------------------------------------ e. whole encoder
def _prompts(B, L, lengths, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(B, L, dtype=torch.long)
    mask = torch.zeros(B, L, dtype=torch.long)
    for b, n in enumerate(lengths):
        ids[b, :n] = torch.randint(1, vocab, (n,), generator=g)
        mask[b, :n] = 1
    return ids.to(DEV), mask.to(DEV)


@pytest.mark.parametrize("name", list(MODELS), ids=list(SHORT.values()))
def test_encoder_at_named_shapes(name, report):
    """Two blocks at the model's full width; 16 ragged prompts at max_length 128 and two at 512; fp16 and bf16, with
    and without proj_out (768 wide); gated at 1.25 x the oracle's floor with the kernels' roundings."""
    from stable_audio_tools.models.t5 import T5Encoder
    cfg = dict(MODELS[name], num_layers=2)
    sd = {k: v.to(DEV) for k, v in to.make_t5_weights(cfg, 70).items()}
    pw, pb = (t.to(DEV) for t in to.make_proj_out(cfg["d_model"], 768, 71))
    lengths = torch.randint(8, 41, (16,), generator=torch.Generator().manual_seed(72)).tolist()
    lengths[0], lengths[1] = 1, 128
    prompts = [_prompts(16, 128, lengths, cfg["vocab_size"], 73), _prompts(2, 512, [512, 300], cfg["vocab_size"], 74)]
    got = {}
    for dtype in ("fp16", "bf16"):
        enc = T5Encoder.from_config(cfg, operand_dtype=dtype).load_state_dict(sd, device=DEV)
        for i, (ids, mask) in enumerate(prompts):
            got[(dtype, False, i)] = enc(ids, mask)
        enc.set_proj_out(pw, pb)
        for i, (ids, mask) in enumerate(prompts):
            got[(dtype, True, i)] = enc(ids, mask)
        enc.close()
        del enc
    for i, (ids, mask) in enumerate(prompts):
        v = mask.bool()
        exact = to.t5_encoder(sd, cfg, ids, mask)
        exact_p = exact @ pw.double().T + pb.double()
        for dtype in ("fp16", "bf16"):
            r = to.operand_rounding(DT[dtype])
            rounded = to.t5_encoder(sd, cfg, ids, mask, rounding=r)
            rounded_p = r(rounded) @ r(pw.double()).T + pb.double()
            for proj, ex, ro in ((False, exact, rounded), (True, exact_p, rounded_p)):
                out = got[(dtype, proj, i)]
                assert torch.all(out[~v] == 0)
                err, floor = rel_l2(out[v], ex[v]), rel_l2(ro[v], ex[v])
                L = ids.shape[1]
                report.append(("encoder", f"{SHORT[name]} L {L}", "2 blocks" + (" + proj_out 768" if proj else ""),
                               dtype, err / floor))
                assert err <= 1.25 * floor, (dtype, proj, L, err, floor)
            del rounded, rounded_p
        del exact, exact_p
    del sd, got
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ f. conditioner
@pytest.mark.parametrize("name", list(MODELS), ids=list(SHORT.values()))
def test_native_conditioner_for_every_name(name, monkeypatch, report):
    import transformers
    from oracle import make_golden as mg
    from oracle.make_golden_t5 import hf_model
    from stable_audio_tools.models.conditioners import T5Conditioner
    cfg = dict(MODELS[name], vocab_size=1001, num_layers=1)
    assert T5Conditioner.T5_MODEL_DIMS[name] == cfg["d_model"]
    sd = to.make_t5_weights(cfg, 80)
    model = hf_model(cfg, sd)
    monkeypatch.setattr(transformers.AutoTokenizer, "from_pretrained", classmethod(lambda cls, *a, **k: mg.FakeTokenizer()))
    monkeypatch.setattr(transformers.T5EncoderModel, "from_pretrained", classmethod(lambda cls, *a, **k: model))
    cond = T5Conditioner(768, t5_model_name=name, max_length=64, project_out=True, native=True)
    assert isinstance(cond.proj_out, torch.nn.Linear)
    assert (cond.proj_out.in_features, cond.proj_out.out_features) == (cfg["d_model"], 768)
    w, b = to.make_proj_out(cfg["d_model"], 768, 81)
    with torch.no_grad():
        cond.proj_out.weight.copy_(w)
        cond.proj_out.bias.copy_(b)
    cond.set_device(DEV)
    texts = ["warm analog pad with slow attack", "kick", "", " ".join(f"w{i}" for i in range(70))]
    emb, mask = cond(texts)
    enc = mg.FakeTokenizer()(texts, max_length=64)
    assert torch.equal(mask.cpu(), enc["attention_mask"].bool())
    sd16 = {k: v.half().float() for k, v in sd.items()}
    hf = hf_model(cfg, sd16).to(DEV)
    ids, m = enc["input_ids"].to(DEV), enc["attention_mask"].to(DEV)
    with torch.no_grad():
        ref = hf(input_ids=ids, attention_mask=m)["last_hidden_state"]
        ref = (ref @ w.to(DEV).T + b.to(DEV)) * m[..., None].float()
    v = m.bool()
    assert emb.shape[-1] == 768 and torch.all(emb[~v] == 0)
    sdd = {k: t.to(DEV) for k, t in sd16.items()}
    exact = to.t5_conditioner(sdd, cfg, ids, m, w.to(DEV), b.to(DEV))
    rounded = to.t5_conditioner(sdd, cfg, ids, m, w.to(DEV), b.to(DEV), rounding=to.operand_rounding(torch.float16))
    floor = rel_l2(rounded[v], exact[v])
    assert rel_l2(ref[v], exact[v]) < 1e-5        # HF fp32 == the oracle
    err = rel_l2(emb[v], ref[v])
    report.append(("condition", SHORT[name], "T5Conditioner(native) + proj_out 768", "fp16", err / floor))
    assert err <= 1.25 * floor, (err, floor)
    del hf, sdd, cond
    torch.cuda.empty_cache()
